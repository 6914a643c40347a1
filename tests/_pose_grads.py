"""Helpers of tests/test_pose_grads.py and tests/test_gpu_fp64_pose_grads.py: the reference's camera expressions
transcribed, the render inputs of forward_with_frequencies, the float64 chain from a rays-in backward's point and
direction gradients to d cam2world, and the float64 pose chain of a camera render on its own intermediates
(pose_chain_fp64), which uses no backward code of the library.
"""
import copy
import math
import os
import random

import numpy as np
import torch

import _cases
from _fp64 import pass_dirs

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


# ---------------------------------------------------------------------------------------------------------------------
# the float64 pose chain of a camera render (tests/test_gpu_fp64_pose_grads.py)
# ---------------------------------------------------------------------------------------------------------------------
#: float64 rows per field VJP chunk: the float64 autograd of one chunk stays a few GB at any batch
CHAIN_ROWS = 1 << 17
#: faults of the chain, for the fault checks: the fine points given the pose gradient, the fine pass's direction term
#: dropped, the direction term dropped entirely, the camera-space directions (and so the points) left unnormalised,
#: d T summed over the merged 2S samples (the fine points' d points added to the translation alone)
CHAIN_FAULTS = ("fine_points_get_the_gradient", "fine_directions_dropped", "directions_dropped", "d_cam_unnormalised",
                "dT_over_merged_samples")
#: how far a face row's coordinate is moved onto the kernel's side, in grid cells
_NUDGE_CELLS = 1e-8


def kernel_side_points(siren, points):
    """float64 copy of the fp32 points (B, P, 3), each coordinate whose fp32 grid index (as the kernels form it) lies
    within FACE_CELLS of a cell face moved _NUDGE_CELLS onto the side of the kernel's fp32 cell -> (points, face rows
    (B, P) bool).  A trilinear lookup's derivative along an axis is constant inside a cell and its derivatives along the
    other axes are continuous across the face, so the float64 VJP at the moved point is the one-sided derivative the
    kernel takes; the point moves by ~1e-10, far below any bound."""
    from test_gpu_fp64_ray_grads import FACE_CELLS
    from test_ray_grads import fp32_cell_index
    pts = points.double()
    spec = siren.field_spec()
    if not spec.grid_channels:
        return pts, torch.zeros(pts.shape[:-1], dtype=torch.bool, device=pts.device)
    R, s = spec.grid_res, spec.input_scale
    i32 = torch.from_numpy(fp32_cell_index(points.cpu().numpy(), s, R)).double().to(pts.device)
    k = i32.round()
    on = (i32 - k).abs() < FACE_CELLS
    side = torch.where(torch.floor(i32) >= k, 1.0, -1.0)          # the kernel's cell: k (above the face) or k - 1
    moved = (((k + side * _NUDGE_CELLS) / (R - 1)) * 2 - 1) / s
    return torch.where(on, moved, pts), on.any(-1)


def _pose_leaves(pose):
    """pose values (numbers or tensors) -> ({name: float64 CPU value}, {name: leaf} of those that require grad)."""
    vals, leaves = {}, {}
    for k in ("h_stddev", "v_stddev", "h_mean", "v_mean"):
        v = pose[k]
        if isinstance(v, torch.Tensor):
            t = v.detach().to("cpu", torch.float64)
            if v.requires_grad:
                t.requires_grad_(True)
                leaves[k] = t
            vals[k] = t
        else:
            vals[k] = float(v)
    return vals, leaves


def _draw64(t):
    return None if t is None else t.detach().to("cpu", torch.float64)


def pose_camera(n, mode, vals, draws):
    """pg.reference_camera on the float64 values and the draws {'d_theta', 'd_phi', 'coin'} -> (cam2world, pitch, yaw)."""
    return reference_camera(n, mode, vals["h_stddev"], vals["v_stddev"], vals["h_mean"], vals["v_mean"],
                            _draw64(draws.get("d_theta")), _draw64(draws.get("d_phi")), coin=draws.get("coin"))


def _jacobians(n, mode, vals, leaves, draws):
    """{name: (d cam2world rows 0..2 (n, 3, 4), d pitch (n, 1), d yaw (n, 1))} of each image w.r.t. the leaf (its own
    entry for a (B, 1) leaf)."""
    names = list(leaves)

    def f(*xs):
        v = dict(vals, **dict(zip(names, xs)))
        c2w, pitch, yaw = pose_camera(n, mode, v, draws)
        return c2w[:, :3, :], pitch, yaw

    jac = torch.autograd.functional.jacobian(f, tuple(leaves[k].detach() for k in names))
    out = {}
    for i, k in enumerate(names):
        parts = []
        for o in range(3):
            j = jac[o][i]
            lead = j.shape[:j.dim() - leaves[k].dim()]
            j = j.reshape(tuple(lead) + (-1,))
            j = j[..., 0] if j.shape[-1] == 1 else torch.stack([j[b, ..., b] for b in range(n)])
            parts.append(j)
        out[k] = tuple(parts)
    return out


def pose_chain_fp64(*args, **kwargs):
    with torch.enable_grad():
        return _pose_chain_fp64(*args, **kwargs)


def _pose_chain_fp64(siren, film, st, draws, pose, mode, lock, opt, noise, d_pixels, d_poses, fault=None,
                     ray_start=0.88, ray_end=1.12, fov=12):
    """The float64 gradient of sum(pixels * d_pixels) + sum(poses * d_poses) of a camera render w.r.t. its pose inputs
    and its cam2world, on the render's own intermediates st (ops.render_forward_stages: points_c, z_c, dirs, raw_c and,
    hierarchical, points_f, z_f, raw_f), so that relu switches, refined densities and fine depths are the kernel's.

    1. composite_vjp of the NCHW pixels (`* 2 - 1` included) -> d raw_c, d raw_f.
    2. _field_vjp on a float64 copy of the field: d points of the coarse pass; d directions of both passes summed per
       ray (the fine points carry none: the reference builds them under no_grad).  No direction term under
       lock_view_dependence or for the direction-free field.  Grid fields: face rows evaluated on the kernel's side
       (kernel_side_points).
    3. torch.autograd from float64 leaves (the pose tensors that require grad) through reference_camera on the same
       draws (draws: 'perturb' (B, N, S, 1), 'd_theta', 'd_phi', 'coin'), points = p_cam R^T + T and dirs = d_cam R^T
       (camera_samples), and the surrogate sum(points d points) + sum(dirs d dirs) + sum(pitch d pitch) + sum(yaw d yaw).

    No backward code of the library takes part.  fault: one of CHAIN_FAULTS.  -> dict: grads {name: float64 gradient
    of the input's shape, or None where the mode never reads it}, d_c2w (B, 4, 4), A {name: sum of the absolute
    per-sample (and per-ray, pitch and yaw) contributions: per image for a (B, 1) input, else over the batch},
    A_c2w (B, 4, 4) likewise per entry, face (face rows, their share of A at most)."""
    from test_gpu_fp64_ray_grads import _field_vjp
    from test_gpu_fp64_reference import composite_vjp
    b, n, s, c = st["raw_c"].shape
    img = math.isqrt(n)
    dev = st["raw_c"].device
    hier = st["points_f"] is not None
    chunk = max(1, CHAIN_ROWS // b)
    siren64 = copy.deepcopy(siren).double()
    for p in siren64.parameters():
        p.requires_grad_(False)
    film64 = film.detach().double()
    d_c, d_f = composite_vjp(st["raw_c"], st["z_c"], st["raw_f"], st["z_f"], noise, opt, d_pixels)
    wo_dir = bool(siren.field_spec().wo_dir)
    dir_term = not lock and not wo_dir and fault != "directions_dropped"
    dirs_pp = pass_dirs(st["dirs"].double(), s, lock)
    pts_c, face_c = kernel_side_points(siren, st["points_c"].reshape(b, -1, 3))
    d_pts, d_dirs_c = _field_vjp(siren64, film64, pts_c, dirs_pp, d_c.reshape(b, -1, c), chunk)
    d_pts = d_pts.reshape(b, n, s, 3)
    d_dirs = d_dirs_c.reshape(b, n, s, 3).sum(2) if dir_term else None
    d_pts_f, n_face_f = None, 0
    if hier and (dir_term or fault in ("fine_points_get_the_gradient", "dT_over_merged_samples")):
        pts_f, face_f = kernel_side_points(siren, st["points_f"].reshape(b, -1, 3))
        n_face_f = int(face_f.sum())
        d_pts_f, d_dirs_f = _field_vjp(siren64, film64, pts_f, dirs_pp, d_f.reshape(b, -1, c), chunk)
        d_pts_f = d_pts_f.reshape(b, n, s, 3)
        if dir_term and fault != "fine_directions_dropped":
            d_dirs = d_dirs + d_dirs_f.reshape(b, n, s, 3).sum(2)
    del siren64

    p_cam, d_cam = camera_samples(img, s, ray_start, ray_end, fov, draws["perturb"].to(dev))
    if fault == "d_cam_unnormalised":
        x_lin, y_lin, _ = (t.double() for t in _tables(img, s, ray_start, ray_end, dev))
        zc = -1.0 / math.tan((2 * math.pi * fov / 360) / 2)
        y, x = torch.meshgrid(y_lin, x_lin, indexing='ij')
        norm = torch.sqrt(x.reshape(-1) ** 2 + y.reshape(-1) ** 2 + zc ** 2)
        p_cam, d_cam = p_cam * norm[None, :, None, None], d_cam * norm[:, None]
    vals, leaves = _pose_leaves(pose)
    with torch.enable_grad():
        c2w_cpu, pitch, yaw = pose_camera(b, mode, vals, draws)
        c2w = c2w_cpu.to(dev)
        R, T = c2w[:, :3, :3], c2w[:, :3, 3]
        points = torch.einsum('bnsj,bij->bnsi', p_cam, R) + T[:, None, None, :]
        sur = (points * d_pts).sum()
        if d_dirs is not None:
            sur = sur + (torch.einsum('nj,bij->bni', d_cam, R) * d_dirs).sum()
        if fault == "fine_points_get_the_gradient":
            p_f = d_cam[None, :, None, :] * st["z_f"].double()[..., None]
            sur = sur + ((torch.einsum('bnsj,bij->bnsi', p_f, R) + T[:, None, None, :]) * d_pts_f).sum()
        elif fault == "dT_over_merged_samples":
            sur = sur + (T * d_pts_f.sum((1, 2))).sum()
        if d_poses is not None:
            d_poses = d_poses.detach().to("cpu", torch.float64)
            sur = sur + (pitch * d_poses[:, :1]).sum().to(dev) + (yaw * d_poses[:, 1:]).sum().to(dev)
        names = list(leaves)
        got = torch.autograd.grad(sur, [leaves[k] for k in names] + [c2w], allow_unused=True)
    grads = {k: None for k in ("h_stddev", "v_stddev", "h_mean", "v_mean") if k in leaves}
    grads.update({k: (None if g is None else g.reshape(leaves[k].shape)) for k, g in zip(names, got[:-1])})
    d_c2w = got[-1]

    # the absolute contributions: per sample d x . (dR p + dT), per ray d dir . dR d_cam, pitch and yaw
    A, share = {}, 0.0
    jac = _jacobians(b, mode, vals, leaves, draws)
    dp = d_poses if d_poses is not None else torch.zeros((b, 2), dtype=torch.float64)
    for k in names:
        if grads[k] is None:
            continue
        J, JP, JY = (t.to(dev) for t in jac[k])
        c_pts = torch.einsum('bnsi,bij,bnsj->bns', d_pts, J[:, :, :3], p_cam) + torch.einsum('bnsi,bi->bns', d_pts, J[:, :, 3])
        a = c_pts.abs().sum((1, 2))
        if d_dirs is not None:
            a = a + torch.einsum('bni,bij,nj->bn', d_dirs, J[:, :, :3], d_cam).abs().sum(1)
        a = a + (JP[:, 0] * dp[:, 0].to(dev)).abs() + (JY[:, 0] * dp[:, 1].to(dev)).abs()
        face = (c_pts.reshape(b, -1).abs() * face_c).sum(1)
        share = max(share, (face / a.clamp_min(1e-300)).max().item())
        per_image = tuple(leaves[k].shape) == (b, 1)
        A[k] = (a.reshape(b, 1) if per_image else a.sum()).reshape(grads[k].shape).to(grads[k].device)
    A_c2w = torch.zeros((b, 4, 4), dtype=torch.float64, device=dev)
    A_c2w[:, :3, :3] = torch.einsum('bnsi,bnsj->bij', d_pts.abs(), p_cam.abs())
    if d_dirs is not None:
        A_c2w[:, :3, :3] += torch.einsum('bni,nj->bij', d_dirs.abs(), d_cam.abs())
    A_c2w[:, :3, 3] = d_pts.abs().sum((1, 2))
    return dict(grads=grads, d_c2w=d_c2w, A=A, A_c2w=A_c2w, face=(int(face_c.sum()) + n_face_f, share))


def _tables(img, s, ray_start, ray_end, dev):
    from fenerf_b200 import ops
    return ops.ray_tables(img, s, ray_start, ray_end, dev)


def pose_errors(got, want, A):
    """Per entry: rel |got - want| / |want|, abs_rel |got - want| / A and A / |want| (float64 tensors of want's shape)."""
    got, want, A = got.double().to(want.device), want.double(), A.double().to(want.device)
    err = (got - want).abs()
    tiny = torch.full_like(want, 1e-300)
    mag = torch.maximum(want.abs(), tiny)
    return err / mag, err / torch.maximum(A, tiny), A / mag
