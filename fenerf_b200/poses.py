"""The gradient of a camera render w.r.t. its pose inputs: the chain from cam2world, pitch and yaw to h_mean, v_mean,
h_stddev and v_stddev (sample_camera_positions + create_cam2world_matrix, generators/volumetric_rendering.py:179-248).

The forward is camera_kernel (ops.camera_poses_launch), unchanged.  The backward re-evaluates the reference's
expressions in float64 from the same draws -- angles, the clamps, the origin on the unit sphere, the look-at with both
normalisations, hybrid's doubled stddev, spherical_uniform's arccos -- and takes their vector-Jacobian product with
torch.autograd.  It is B scalars per input, not a hot path.  The clamps pass the gradient where the reference's float32
clamp does: their masks come from the float32 values camera_kernel clamped, recomputed with its operations.  An input the
mode never reads gets no gradient (its .grad stays None), and the draws carry none (truncated_normal_ writes through
.data in the reference).
"""
import math

import torch

from . import ops

PHI_LO, PHI_HI = 1e-5, math.pi - 1e-5          # torch.clamp(phi, 1e-5, math.pi - 1e-5)
V_LO, V_HI = 1e-5, 1 - 1e-5                    # spherical_uniform's torch.clamp(v, 1e-5, 1 - 1e-5)


def _truncated_pick(d):
    """truncated_normal_'s choice among four normal draws (n, 1, 4) -> (n, 1): the first inside (-2, 2), else the first."""
    valid = (d < 2) & (d > -2)
    return d.gather(-1, valid.max(-1, keepdim=True)[1]).squeeze(-1)


def _angles(code, doubled, values, d_theta, d_phi, clamp_v):
    """theta, phi before phi's final clamp: the reference's expressions on `values` (POSE_ARGS order), in their dtype.
    clamp_v(v) is spherical_uniform's clamp of v."""
    h_std, v_std, h_mean, v_mean = values
    if code == 1:
        if doubled:
            theta = (d_theta - 0.5) * 2 * h_std * 2 + h_mean
            phi = (d_phi - 0.5) * 2 * v_std * 2 + v_mean
        else:
            theta = (d_theta - 0.5) * 2 * h_std + h_mean
            phi = (d_phi - 0.5) * 2 * v_std + v_mean
    elif code == 2:
        theta = d_theta * h_std + h_mean
        phi = d_phi * v_std + v_mean
    elif code == 3:
        theta = _truncated_pick(d_theta) * h_std + h_mean
        phi = _truncated_pick(d_phi) * v_std + v_mean
    elif code == 4:
        theta = (d_theta - .5) * 2 * h_std + h_mean
        v = (d_phi - .5) * 2 * (v_std / math.pi) + v_mean / math.pi
        phi = torch.arccos(1 - 2 * clamp_v(v))
    else:
        n = d_theta.shape[0]
        theta = torch.ones((n, 1), dtype=d_theta.dtype, device=d_theta.device) * h_mean
        phi = torch.ones((n, 1), dtype=d_theta.dtype, device=d_theta.device) * v_mean
    return theta, phi


def _normalize(v):
    return v / torch.norm(v, dim=-1, keepdim=True)


def pose_chain(code, doubled, values, d_theta, d_phi, phi_mask=None, v_mask=None):
    """(cam2world rows 0..2 (n, 3, 4), pitch (n, 1), yaw (n, 1)) by the reference's expressions in the dtype of
    d_theta.  phi_mask / v_mask (bool, (n, 1)): where the final clamp of phi / spherical_uniform's clamp of v passes the
    gradient; None: torch.clamp's own rule on these values."""
    def clamp(x, lo, hi, mask):
        if mask is None:
            return torch.clamp(x, lo, hi)
        return torch.where(mask, x, x.detach().clamp(lo, hi))

    theta, phi = _angles(code, doubled, values, d_theta, d_phi, lambda v: clamp(v, V_LO, V_HI, v_mask))
    phi = clamp(phi, PHI_LO, PHI_HI, phi_mask)
    origin = torch.cat([torch.sin(phi) * torch.cos(theta), torch.cos(phi), torch.sin(phi) * torch.sin(theta)], dim=-1)
    forward = _normalize(_normalize(-origin))
    up = torch.zeros_like(forward)
    up[:, 1] = 1
    left = _normalize(torch.cross(up, forward, dim=-1))
    up = _normalize(torch.cross(forward, left, dim=-1))
    rot = torch.stack((-left, up, -forward), dim=-1)
    return torch.cat([rot, origin.unsqueeze(-1)], dim=-1), phi, theta


def _clamp_masks(n, code, doubled, values, d_theta, d_phi, device):
    """Where camera_kernel's clamps of phi (and spherical_uniform's v) pass the gradient, (n, 1) bool each: its float32
    values before the clamps, recomputed with its own operations on the values it read."""
    vals, _ = ops.camera_kernel_values(code, doubled, values, device)
    _, v_std, _, v_mean = (t.reshape(-1, 1) for t in vals)
    dp = None if d_phi is None else d_phi.to(device=device, dtype=torch.float32)
    if code == 4:     # phi = arccos(1 - 2 v) of v inside [1e-5, 1 - 1e-5] lies well inside phi's clamp
        v = (dp - 0.5) * 2 * v_std + v_mean
        return torch.ones((n, 1), dtype=torch.bool, device=device), (v >= V_LO) & (v <= V_HI)
    if code == 1:
        phi = (dp - 0.5) * 2 * v_std + v_mean
    elif code in (2, 3):
        phi = (_truncated_pick(dp) if code == 3 else dp) * v_std + v_mean
    else:
        phi = v_mean.expand(n, 1)
    return (phi >= PHI_LO) & (phi <= PHI_HI), None


def pose_vjp(n, code, doubled, values, d_theta, d_phi, need, d_c2w, d_pitch, d_yaw):
    """The gradients of the pose inputs `values` (POSE_ARGS order) from d cam2world (n, 4, 4), d pitch and d yaw (n, 1):
    for each value with need[k] (a tensor), a tensor of its shape, dtype and device, or None where the mode never reads
    it."""
    dev = d_c2w.device
    phi_mask, v_mask = _clamp_masks(n, code, doubled, values, d_theta, d_phi, dev)
    with torch.enable_grad():
        leaves, vals = [], []
        for v, want in zip(values, need):
            if isinstance(v, torch.Tensor):
                t = v.detach().to(device=dev, dtype=torch.float64).reshape(-1, 1).requires_grad_(bool(want))
                if want:
                    leaves.append(t)
                vals.append(t)
            else:
                vals.append(v)
        dt = torch.zeros((n, 1), dtype=torch.float64, device=dev) if d_theta is None else d_theta.to(dev, torch.float64)
        dp = None if d_phi is None else d_phi.to(dev, torch.float64)
        m34, pitch, yaw = pose_chain(code, doubled, vals, dt, dp, phi_mask, v_mask)
        outs = [o for o in (m34, pitch, yaw) if o.requires_grad]
        grads = torch.autograd.grad(outs, leaves, grad_outputs=[
            g.to(torch.float64) for o, g in zip((m34, pitch, yaw), (d_c2w[:, :3, :], d_pitch, d_yaw)) if o.requires_grad],
            allow_unused=True) if outs and leaves else [None] * len(leaves)
    it = iter(grads)
    out = []
    for v, want in zip(values, need):
        g = next(it) if isinstance(v, torch.Tensor) and want else None
        out.append(None if g is None else g.to(dtype=v.dtype, device=v.device).reshape(v.shape))
    return out


class CameraPoses(torch.autograd.Function):
    """(cam2world (n,4,4), pitch (n,1), yaw (n,1)) = camera_kernel(pose values, draws); differentiable w.r.t. the pose
    values that are tensors.  call: n, code, doubled, d_theta, d_phi, device (ops.camera_draws)."""

    @staticmethod
    def forward(ctx, call, h_stddev, v_stddev, h_mean, v_mean):
        values = (h_stddev, v_stddev, h_mean, v_mean)
        ctx.call, ctx.values = call, tuple(v.detach() if isinstance(v, torch.Tensor) else v for v in values)
        return ops.camera_poses_launch(call['n'], call['code'], call['doubled'], values, call['d_theta'], call['d_phi'],
                                       call['device'])

    @staticmethod
    def backward(ctx, d_c2w, d_pitch, d_yaw):
        c = ctx.call
        return (None,) + tuple(pose_vjp(c['n'], c['code'], c['doubled'], ctx.values, c['d_theta'], c['d_phi'],
                                        ctx.needs_input_grad[1:], d_c2w, d_pitch, d_yaw))
