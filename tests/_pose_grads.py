"""Helpers of tests/test_pose_grads.py: the reference's camera expressions transcribed, the render inputs of
forward_with_frequencies, and the float64 chain from a rays-in backward's point and direction gradients to d cam2world.
"""
import math
import os
import random

import numpy as np
import torch

import _cases

KW = dict(fov=12, ray_start=0.88, ray_end=1.12, clamp_mode='relu', nerf_noise=0.0, sample_dist='gaussian',
          hierarchical_sample=True, h_stddev=0.3, v_stddev=0.155, h_mean=math.pi * 0.5, v_mean=math.pi * 0.5)

#: sample_dist of every camera mode; None is the mean pose
MODES = ("uniform", "gaussian", "hybrid", "truncated_gaussian", "spherical_uniform", None)


def kwargs(img_size, num_steps, **kw):
    d = dict(KW, img_size=img_size, num_steps=num_steps)
    d.update(kw)
    return d


def seed(s):
    torch.manual_seed(s)
    random.seed(s)


def reference_camera(n, mode, h_stddev, v_stddev, h_mean, v_mean, d_theta, d_phi, coin=None):
    """sample_camera_positions + create_cam2world_matrix (volumetric_rendering.py:179-248) written out as the reference
    writes them, on the given draws (rand / randn (n, 1), truncated_gaussian's randn (n, 1, 4)) and hybrid's coin ->
    (cam2world (n, 4, 4), pitch, yaw)."""
    if mode == 'uniform':
        theta = (d_theta - 0.5) * 2 * h_stddev + h_mean
        phi = (d_phi - 0.5) * 2 * v_stddev + v_mean
    elif mode in ('normal', 'gaussian'):
        theta = d_theta * h_stddev + h_mean
        phi = d_phi * v_stddev + v_mean
    elif mode == 'hybrid':
        if coin < 0.5:
            theta = (d_theta - 0.5) * 2 * h_stddev * 2 + h_mean
            phi = (d_phi - 0.5) * 2 * v_stddev * 2 + v_mean
        else:
            theta = d_theta * h_stddev + h_mean
            phi = d_phi * v_stddev + v_mean
    elif mode == 'truncated_gaussian':
        def trunc(tmp):
            valid = (tmp < 2) & (tmp > -2)
            ind = valid.max(-1, keepdim=True)[1]
            return tmp.gather(-1, ind).squeeze(-1)
        theta = trunc(d_theta) * h_stddev + h_mean
        phi = trunc(d_phi) * v_stddev + v_mean
    elif mode == 'spherical_uniform':
        theta = (d_theta - .5) * 2 * h_stddev + h_mean
        vs, vm = v_stddev / math.pi, v_mean / math.pi
        v = ((d_phi - .5) * 2 * vs + vm)
        v = torch.clamp(v, 1e-5, 1 - 1e-5)
        phi = torch.arccos(1 - 2 * v)
    else:
        theta = torch.ones((n, 1), dtype=torch.float64) * h_mean
        phi = torch.ones((n, 1), dtype=torch.float64) * v_mean
    phi = torch.clamp(phi, 1e-5, math.pi - 1e-5)
    origin = torch.cat([torch.sin(phi) * torch.cos(theta), torch.cos(phi), torch.sin(phi) * torch.sin(theta)], -1)

    def normalize_vecs(v):
        return v / (torch.norm(v, dim=-1, keepdim=True))

    forward = normalize_vecs(normalize_vecs(-origin))
    up = torch.tensor([0, 1, 0], dtype=origin.dtype).expand_as(forward)
    left = normalize_vecs(torch.cross(up, forward, dim=-1))
    up = normalize_vecs(torch.cross(forward, left, dim=-1))
    rot = torch.eye(4, dtype=origin.dtype).unsqueeze(0).repeat(n, 1, 1)
    rot[:, :3, :3] = torch.stack((-left, up, -forward), axis=-1)
    trans = torch.eye(4, dtype=origin.dtype).unsqueeze(0).repeat(n, 1, 1)
    trans[:, :3, 3] = origin
    return trans @ rot, phi, theta


def film_inputs(gen, zs):
    """forward_with_frequencies' FiLM inputs for latents zs: (frequencies, phase_shifts), or the double-latent
    generators' (frequencies geo, app, phase shifts geo, app)."""
    with torch.no_grad():
        if len(zs) == 1:
            return list(gen.siren.mapping_network(zs[0]))
        fg, pg = gen.siren.geo_mapping_network(zs[0])
        fa, pa = gen.siren.app_mapping_network(zs[1])
    return [fg, fa, pg, pa]


def latents(model, batch, device, s=1000):
    g = torch.Generator().manual_seed(s)
    return [torch.randn(batch, 256, generator=g).to(device) for _ in range(_cases.n_latents(model))]


def camera_samples(img_size, num_steps, ray_start, ray_end, fov, perturb):
    """The camera-space sample points (B, N, S, 3) and ray directions (N, 3) of get_initial_rays_trig + perturb_points,
    in float64 from the float32 tables and draw #1."""
    from fenerf_b200 import ops
    x_lin, y_lin, z_lin = (t.double() for t in ops.ray_tables(img_size, num_steps, ray_start, ray_end, perturb.device))
    zc = -1.0 / math.tan((2 * math.pi * fov / 360) / 2)
    y, x = torch.meshgrid(y_lin, x_lin, indexing='ij')
    d = torch.stack([x.reshape(-1), y.reshape(-1), torch.full_like(x.reshape(-1), zc)], -1)
    d = d / d.norm(dim=-1, keepdim=True)
    off = (perturb.double()[..., 0] - 0.5) * (z_lin[1] - z_lin[0])
    p = d[None, :, None, :] * (z_lin[None, None, :, None] + off[..., None])
    return p, d


def chain_cam2world(dx, ddir, p_cam, d_cam):
    """d cam2world (B, 4, 4) in float64 from d world points (B, N, S, 3) and d world directions per ray (B, N, 3) or None:
    dR = sum dx p_cam^T + sum ddir d_cam^T, dT = sum dx."""
    dx = dx.double()
    out = torch.zeros((dx.shape[0], 4, 4), dtype=torch.float64, device=dx.device)
    out[:, :3, :3] = torch.einsum('bnsi,bnsj->bij', dx, p_cam)
    if ddir is not None:
        out[:, :3, :3] += torch.einsum('bni,nj->bij', ddir.double(), d_cam)
    out[:, :3, 3] = dx.sum((1, 2))
    return out


def rel(got, want):
    """max |got - want| / max |want|."""
    got, want = got.double(), want.double()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


# ---------------------------------------------------------------------------------------------------------------------
# goldens of the reference (tests/golden/make_pose_grad_goldens.py)
# ---------------------------------------------------------------------------------------------------------------------
_H_PER_IMAGE, _V_PER_IMAGE = (math.pi / 2 + 0.1, math.pi / 2 - 0.15), (math.pi / 2 + 0.05, math.pi / 2 - 0.1)


def _golden(model, seed, mode, grad, per_image=(), hier=True, lock=False, pose_loss=False, batch=2):
    return dict(model=model, seed=seed, sample_dist=mode, grad=grad, per_image=per_image, hier=hier, lock=lock,
                pose_loss=pose_loss, batch=batch)


_MEANS = ("h_mean", "v_mean")
_ALL = ("h_stddev", "v_stddev", "h_mean", "v_mean")
#: name -> the case: model, seed (torch and random), camera mode, the pose arguments that are tensors requiring grad,
#: those of them given per image (B, 1), hierarchical sampling, lock_view_dependence, a loss term on the poses
GOLDEN_CASES = {
    "a_gauss_hier": _golden("A", 100, "gaussian", _MEANS),
    "a_uniform_perimage_nohier": _golden("A", 102, "uniform", _ALL, per_image=_MEANS, hier=False),
    # random.seed(100): coin < 0.5; per-image stddevs, whose gradient is each image's own (a shared stddev's sums
    # terms of both signs over the images, and the fp16 streams' error on each term does not cancel with them)
    "a_hybrid_uniform": _golden("A", 100, "hybrid", _ALL, per_image=_ALL, pose_loss=True),
    "a_hybrid_gaussian": _golden("A", 101, "hybrid", _ALL),                     # random.seed(101): coin >= 0.5
    "a_truncgauss": _golden("A", 103, "truncated_gaussian", _ALL, per_image=("v_mean",), pose_loss=True),
    "a_spherical": _golden("A", 104, "spherical_uniform", ("v_stddev", "h_mean", "v_mean"), per_image=_MEANS),
    "a_mean_pose": _golden("A", 105, None, _ALL, pose_loss=True),
    "b_gauss_hier_perimage": _golden("B", 106, "gaussian", ("v_stddev",) + _MEANS, per_image=_MEANS, pose_loss=True),
    "b_lockview_nohier": _golden("B", 107, "gaussian", _MEANS, hier=False, lock=True),
    "d_gauss_hier": _golden("D", 108, "gaussian", ("h_stddev",) + _MEANS),
    "d_uniform_perimage_nohier": _golden("D", 109, "uniform", _MEANS, per_image=_MEANS, hier=False, batch=3),
}


def golden_kwargs(c):
    kw = kwargs(12, 8, sample_dist=c["sample_dist"], hierarchical_sample=c["hier"], lock_view_dependence=c["lock"])
    for k in ("h_stddev", "v_stddev", "h_mean", "v_mean"):
        del kw[k]
    return kw


def golden_pose(c, device, values=None):
    """The case's pose arguments: numbers, or float32 tensors requiring grad (per image: (B, 1)).  values: the stored
    values (a golden's pose_<name> arrays) instead of the case's own."""
    b = c["batch"]
    base = dict(h_stddev=(0.3, 0.25), v_stddev=(0.155, 0.12), h_mean=_H_PER_IMAGE, v_mean=_V_PER_IMAGE)
    out = {}
    for k, v in base.items():
        if values is not None:
            t = torch.as_tensor(values[k], dtype=torch.float32)
            out[k] = t.to(device).requires_grad_(True) if k in c["grad"] else float(t)
            continue
        if k not in c["grad"]:
            out[k] = v[0] if isinstance(v, tuple) else v
            continue
        if k in c["per_image"]:
            t = torch.tensor([[v[i % len(v)]] for i in range(b)], dtype=torch.float32)
        else:
            t = torch.tensor(v[0] if isinstance(v, tuple) else v, dtype=torch.float32)
        out[k] = t.to(device).requires_grad_(True)
    return out


def pose_loss_weights(shape):
    g = torch.Generator().manual_seed(98)
    return torch.randn(shape, generator=g)


def golden_path(name):
    return os.path.join(_cases.GOLDEN_DIR, "grad_pose_%s.npz" % name)


def load_golden(name):
    """-> (npz dict, draws [(kind, tensor)] for ReplayRng)."""
    z = dict(np.load(golden_path(name)))
    draws = []
    for i in range(int(z["n_draws"])):
        key = next(k for k in z if k.startswith("draw%d_" % i))
        draws.append((key.split("_", 1)[1], torch.from_numpy(z[key])))
    return z, draws
