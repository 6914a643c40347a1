"""The camera-pose gradient of forward_with_frequencies against float64, at the shapes users run.

The pose gradient is a sum over every coarse sample (1.6 M at the inversion step) and every ray, whose terms cancel; its
accuracy does not follow from the per-sample accuracy of the point and direction gradients.  Here it is held to a
float64 chain that uses no backward code of the library (_pose_grads.pose_chain_fp64: composite_vjp, the float64
field's VJP, then torch.autograd from the pose leaves through the reference's camera, points = p_cam R^T + T and
dirs = d_cam R^T).

  1. CPU: the chain is the reference's derivative: forward_with_frequencies written as one float64 function of the pose
     leaves (camera, rays, field, a fine pass under no_grad from the stages' fine depths, compositor) and torch.autograd
     of it, to 1e-10, in every camera mode (both hybrid branches), hierarchical and flat, lock_view_dependence, per-image
     and shared means, a loss on the returned poses.  Faults of the chain move it by >= 10 x FIELD_BOUND['exact'].
  2. GPU: fenerf_cam2world_grad called directly, against a float64 einsum on the kernel's own fp32 camera-space samples
     (ops.ray_setup with an identity cam2world), from 45 samples per image to 512² x 48 (3,072 chunks), 64 images,
     ray-sharded windows, with and without d dirs, and on inputs whose sum survives only in fp64.
  3. GPU: forward_with_frequencies end to end (vr.ReplayRng on draws made here; render_forward_stages reproduces its frame
     bit for bit) against the chain: the pose inputs' gradients, and d cam2world of backward.render_with_grad with a
     cam2world leaf (the network backward plus the kernel, without the pose chain).

Error measures, per pose input (per image for a (B, 1) input) and per d cam2world entry: rel = |got - want| / |want| and
abs_rel = |got - want| / A, A the float64 sum of the absolute per-sample, per-ray, pitch and yaw contributions; A / |want|
shows how much the sum cancels.  Bounds: measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), see each constant.
"""
import copy
import ctypes
import dataclasses
import functools
import gc
import math

import numpy as np
import pytest
import torch

import _cases
import _pose_grads as pg
from _fp64 import _film, _opt, _siren, composite_ref, pass_dirs
from fenerf_b200 import _lib, backward, ops
from fenerf_b200 import dist as fdist
from fenerf_b200.generators import volumetric_rendering as vr
from oracle import render_oracle as oracle
from test_gpu_fp64_ray_grads import L_BOUND, RAY_BOUND
from test_gpu_fp64_reference import FIELD_BOUND
from test_split_backward import P_BOUND

DEV = "cuda:0"
gpu = pytest.mark.gpu
POSE_ARGS = ops.POSE_ARGS

#: the direct call of fenerf_cam2world_grad: |got - fp32(want)| <= 1 ulp + CAM2WORLD_A * A per entry (fp64 sums)
CAM2WORLD_A = 1e-12
GIB = 1 << 30
#: peak torch.cuda.max_memory_allocated() of any GPU test here (measured: 15.5 GB, the inversion step's float64 chain)
MEM_CAP = 24 * GIB


@pytest.fixture(autouse=True)
def _memory(request):
    """GPU tests: the peak allocation printed and kept under MEM_CAP, and the allocator's cached blocks handed back after
    each test.  The float64 chains allocate many large blocks of many sizes; kept in this process's cache they would
    leave later tests, and the child processes some of them start, a card with little free memory."""
    if request.node.get_closest_marker("gpu") is None:
        yield
        return
    torch.empty(1, device=DEV)                      # the caching allocator exists before its statistics are reset
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    peak, reserved = torch.cuda.max_memory_allocated(DEV), torch.cuda.max_memory_reserved(DEV)
    _gen.cache_clear()
    gc.collect()
    torch.cuda.empty_cache()
    print("%s: max_memory_allocated %.2f GB, max_memory_reserved %.2f GB, %.2f GB reserved after the test" % (
        request.node.name, peak / 1e9, reserved / 1e9, torch.cuda.memory_reserved(DEV) / 1e9))
    assert peak <= MEM_CAP, "peak allocation %.2f GB above MEM_CAP" % (peak / 1e9)


# ---------------------------------------------------------------------------------------------------------------------
# draws and pose values
# ---------------------------------------------------------------------------------------------------------------------
def camera_draws(mode, b, g, coin=None, d_phi=None):
    """[(kind, tensor)] of the camera draws of `mode` in the reference's order (hybrid: its coin first), and
    {'d_theta', 'd_phi', 'coin'} for the chain.  d_phi: fixed phi draws instead of random ones."""
    draws, out = [], dict(d_theta=None, d_phi=None, coin=coin)
    code = {"uniform": 1, "spherical_uniform": 1, "gaussian": 2, "truncated_gaussian": 3}.get(mode, 0)
    if mode == "hybrid":
        draws.append(("coin", torch.tensor(coin)))
        code = 1 if coin < 0.5 else 2
    if code == 1:
        t = [torch.rand((b, 1), generator=g) for _ in range(2)]
        kind = "rand"
    elif code == 2:
        t = [torch.randn((b, 1), generator=g) for _ in range(2)]
        kind = "randn"
    elif code == 3:
        t = [torch.randn((b, 1, 4), generator=g) * 1.5 for _ in range(2)]    # some draws outside (-2, 2)
        kind = "randn"
    else:
        return draws, out
    if d_phi is not None:
        t[1] = torch.tensor(d_phi, dtype=torch.float32).reshape(b, 1)
    draws += [(kind, t[0]), (kind, t[1])]
    out.update(d_theta=t[0], d_phi=t[1])
    return draws, out


#: the pose values of the cases: stddevs and, per image, the means' offsets from pi / 2
_STD = dict(h_stddev=0.3, v_stddev=0.155)


def pose_values(b, grad, per_image, g, device, v_mean=None, h_mean=None, std=None):
    """{name: number or float32 tensor}: the names in `grad` are tensors requiring grad, (B, 1) for those in
    `per_image`, 0-dim otherwise."""
    out = {}
    base = dict(_STD, **(std or {}))
    for k in POSE_ARGS:
        if k in base:
            v = torch.full((b, 1), base[k])
        else:
            mean = v_mean if k == "v_mean" else h_mean
            v = (math.pi / 2 + (0.1 if k == "h_mean" else 0.05) * torch.randn((b, 1), generator=g)) if mean is None \
                else torch.full((b, 1), mean)
        if k not in grad:
            out[k] = float(v[0, 0])
            continue
        t = v if k in per_image else v[0, 0].clone()
        out[k] = t.float().to(device).requires_grad_(True)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the chain is the derivative of the render written as one float64 function of the pose leaves
# ---------------------------------------------------------------------------------------------------------------------
def direct_forward(siren64, film64, vals, mode, cam, perturb, z_c, z_f, lock, opt, noise, img, s):
    """forward_with_frequencies in float64 as a function of the pose values `vals` (leaves among them): the reference's
    camera, points = p_cam R^T + T, dirs = d_cam R^T, the field on the coarse points, the fine points built under
    no_grad from the fine depths z_f (origin + dir z_f; None: flat) with the directions carrying their gradient, the
    compositor.  -> (NCHW pixels, poses (B, 2), stages for the chain)."""
    b = perturb.shape[0]
    c2w, pitch, yaw = pg.pose_camera(b, mode, vals, cam)
    p_cam, d_cam = pg.camera_samples(img, s, 0.88, 1.12, 12, perturb)
    R, T = c2w[:, :3, :3], c2w[:, :3, 3]
    pts = torch.einsum('bnsj,bij->bnsi', p_cam, R) + T[:, None, None, :]
    dirs = torch.einsum('nj,bij->bni', d_cam, R)
    n = img * img
    dpp = pass_dirs(dirs, s, lock)
    raw_c = oracle.field_eval(siren64, pts.reshape(b, -1, 3), film64, dpp).reshape(b, n, s, -1)
    raw_f = pts_f = None
    if z_f is not None:
        with torch.no_grad():
            pts_f = T[:, None, None, :] + dirs[:, :, None, :] * z_f.double()[..., None]
        raw_f = oracle.field_eval(siren64, pts_f.reshape(b, -1, 3), film64, dpp).reshape(b, n, s, -1)
    px = composite_ref(raw_c, z_c, raw_f, z_f, noise, opt)
    st = dict(points_c=pts.detach(), z_c=z_c, dirs=dirs.detach(), raw_c=raw_c.detach(), points_f=pts_f, z_f=z_f,
              raw_f=None if raw_f is None else raw_f.detach())
    return px, torch.cat([pitch, yaw], -1), st


_ALL = POSE_ARGS
_MEANS = ("h_mean", "v_mean")
#: variant -> (model, camera mode, hybrid coin, hierarchical, lock_view_dependence, per-image inputs, pose loss)
_CPU_VARIANTS = {
    "uniform": ("A", "uniform", None, True, False, _MEANS, True),
    "gaussian": ("A", "gaussian", None, True, False, _MEANS, True),
    "hybrid_uniform": ("A", "hybrid", 0.25, True, False, _ALL, True),
    "hybrid_gaussian": ("A", "hybrid", 0.75, True, False, _ALL, True),
    "truncated_gaussian": ("A", "truncated_gaussian", None, True, False, ("v_mean",), True),
    "spherical_uniform": ("A", "spherical_uniform", None, True, False, _MEANS, True),
    "mean_pose": ("A", None, None, True, False, (), True),
    "flat": ("D", "gaussian", None, False, False, _MEANS, False),
    "lock_view_dependence": ("D", "gaussian", None, True, True, _MEANS, True),
    "shared_means": ("D", "gaussian", None, True, False, (), False),
    "gaussian_D": ("D", "gaussian", None, True, False, _MEANS, True),       # the fault checks' render
}


@functools.lru_cache(maxsize=None)
def _cpu_field(model):
    siren = _siren(model, "cpu")
    siren64 = copy.deepcopy(siren).double()
    for p in siren64.parameters():
        p.requires_grad_(False)
    return siren, siren64


def _cpu_run(variant, fault=None):
    """The direct float64 forward of a variant on 2 images of 8² rays x 6 samples, torch.autograd of it, and the chain
    on its stages -> (want {name: grad}, chain result)."""
    model, mode, coin, hier, lock, per_image, pose_loss = _CPU_VARIANTS[variant]
    b, img, s = 2, 8, 6
    n = img * img
    siren, siren64 = _cpu_field(model)
    film = _film(siren, b, 7)
    g = torch.Generator().manual_seed(sum(map(ord, variant)))
    _, cam = camera_draws(mode, b, g, coin)
    std = dict(v_stddev=1.2) if mode == "spherical_uniform" else None
    pose = pose_values(b, _ALL, per_image, g, "cpu", std=std)
    perturb = torch.rand((b, n, s, 1), generator=g)
    x_lin, y_lin, z_lin = vr.ray_tables(img, s, 0.88, 1.12, "cpu")
    z_c = z_lin + (perturb[..., 0] - 0.5) * (z_lin[1] - z_lin[0])
    z_f = torch.sort(0.88 + 0.24 * torch.rand((b, n, s), generator=g), -1)[0] if hier else None
    opt = _opt("relu")
    d_pixels = torch.randn((b, siren.field_spec().out_dim - 1, img, img), generator=g, dtype=torch.float64)
    d_poses = torch.randn((b, 2), generator=g, dtype=torch.float64) if pose_loss else None
    vals, leaves = pg._pose_leaves(pose)
    px, poses, st = direct_forward(siren64, film.double(), vals, mode, cam, perturb, z_c, z_f, lock, opt, None, img, s)
    loss = (px * d_pixels).sum() + ((poses * d_poses).sum() if d_poses is not None else 0)
    got = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    want = dict(zip(leaves, got))
    cam = dict(cam, perturb=perturb)
    chain = pg.pose_chain_fp64(siren, film, st, cam, pose, mode, lock, opt, None, d_pixels, d_poses, fault=fault)
    return want, chain


@pytest.mark.parametrize("variant", list(_CPU_VARIANTS))
def test_pose_chain_matches_autograd_of_the_direct_forward(variant):
    """pose_chain_fp64 (the composite VJP, the coarse points' and both passes' direction terms, the fine points left out,
    the pose leaves through the reference camera) equals float64 autograd of the render written as one function of the
    pose leaves, to 1e-10 of each gradient; an input the mode never reads gets None on both sides; the chain's A is the
    sum of |contributions| (at least |want|)."""
    want, chain = _cpu_run(variant)
    assert set(want) == set(chain["grads"])
    for k, w in want.items():
        got = chain["grads"][k]
        assert (w is None) == (got is None), (k, w, got)
        if w is None:
            continue
        err = (got - w).abs().max().item() / w.abs().max().item()
        print("pose chain %s %s: %.2e of the largest entry (A / |want| %s)" % (
            variant, k, err, ["%.3g" % v for v in (chain["A"][k] / w.abs()).flatten().tolist()]))
        assert err <= 1e-10, (variant, k, err)
        assert (chain["A"][k] >= w.abs() * (1 - 1e-12)).all()


@pytest.mark.parametrize("fault", pg.CHAIN_FAULTS)
def test_pose_chain_faults_exceed_the_bound(fault):
    """Each fault of the chain (model D, 2 x 8² x 6 + 6, gaussian, per-image means, a pose loss) moves a pose-input
    gradient or d cam2world, relative to the tensor's largest entry, by more than 10 x FIELD_BOUND['exact']; the factor
    against the guard bound (RAY_BOUND['guard']) is printed beside it."""
    _, good = _cpu_run("gaussian_D")
    _, bad = _cpu_run("gaussian_D", fault=fault)
    moved = {k: pg.rel(bad["grads"][k], good["grads"][k]) for k in good["grads"] if good["grads"][k] is not None}
    moved["cam2world"] = pg.rel(bad["d_c2w"], good["d_c2w"])
    worst = max(moved, key=moved.get)
    print("pose chain fault %s: %s moved %.3g (FIELD_BOUND exact x %.3g, guard bound x %.3g)" % (
        fault, worst, moved[worst], moved[worst] / FIELD_BOUND["exact"], moved[worst] / RAY_BOUND["guard"]))
    assert moved[worst] > 10 * FIELD_BOUND["exact"], moved



# ---------------------------------------------------------------------------------------------------------------------
# GPU: fenerf_cam2world_grad called directly
# ---------------------------------------------------------------------------------------------------------------------
def _desc(b, r, s, rows=None):
    rd = ops.make_render_desc(batch=b, img_size=r, num_steps=s, hierarchical=False, clamp_mode='relu', nerf_noise=0.0,
                              fov=12)
    if rows is not None:
        rd.img_h = rows[1] - rows[0]
    return rd


def cam2world_grad(rd, x_lin, y_lin, z_lin, perturb, d_points, d_dirs, inv_scale, input_scale):
    """One fenerf_cam2world_grad call as backward._cam2world_grad makes it, into a NaN-prefilled (B, 4, 4)."""
    lib = _lib.lib()
    ws = torch.empty(lib.fenerf_cam2world_grad_workspace_bytes(ctypes.byref(rd)), dtype=torch.uint8, device=DEV)
    out = torch.full((rd.batch, 4, 4), float("nan"), device=DEV)
    inv = torch.tensor([inv_scale], dtype=torch.float32, device=DEV)
    _lib.check(lib.fenerf_cam2world_grad(
        ctypes.byref(rd), x_lin.data_ptr(), y_lin.data_ptr(), z_lin.data_ptr(), perturb.data_ptr(), d_points.data_ptr(),
        d_dirs.data_ptr() if d_dirs is not None else 0, inv.data_ptr(), input_scale, ws.data_ptr(), ws.numel(),
        out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return out


def camera_space(rd, x_lin, y_lin, z_lin, perturb):
    """The kernel's fp32 camera-space samples (B, N S, 3) and ray directions (B N, 3): ops.ray_setup with cam2world = I."""
    eye = torch.eye(4, device=DEV).expand(rd.batch, 4, 4).contiguous()
    pts, _, dirs, _ = ops.ray_setup(rd, x_lin, y_lin, z_lin, eye, perturb)
    return pts.reshape(rd.batch, -1, 3), dirs.reshape(-1, 3)


def _tables_for(r, s, rows=None):
    x_lin, y_lin, z_lin = ops.ray_tables(r, s, 0.88, 1.12, DEV)
    if rows is not None:
        y_lin = y_lin[rows[0]:rows[1]].contiguous()
    return x_lin, y_lin, z_lin


@gpu
def test_identity_ray_setup_is_the_kernels_camera_space():
    """The reference below reads p_cam and d_cam from ops.ray_setup with an identity cam2world.  One-hot d points (one
    sample of each of 8 images, inv_scale = input_scale = 1) and one-hot d dirs make fenerf_cam2world_grad return that
    sample's camera-space point and direction exactly: the two kernels' camera-space values agree bit for bit."""
    b, r, s = 8, 37, 23
    rd = _desc(b, r, s)
    x_lin, y_lin, z_lin = _tables_for(r, s)
    g = torch.Generator(device=DEV).manual_seed(3)
    perturb = torch.rand((b, r * r, s, 1), generator=g, device=DEV)
    p_cam, d_cam = camera_space(rd, x_lin, y_lin, z_lin, perturb)
    ns = r * r * s
    pick = torch.randint(0, ns, (b,), generator=g, device=DEV)
    img = torch.arange(b, device=DEV)
    ray = img * r * r + pick // s
    for a in range(3):
        dx = torch.zeros((b, ns, 3), device=DEV)
        dx[img, pick, a] = 1
        dd = torch.zeros((b * r * r, 3), device=DEV)
        out = cam2world_grad(rd, x_lin, y_lin, z_lin, perturb, dx, None, 1.0, 1.0)
        assert torch.equal(out[:, a, :3], p_cam[img, pick]) and torch.equal(out[:, a, 3], torch.ones(b, device=DEV))
        dd[ray, a] = 1
        out = cam2world_grad(rd, x_lin, y_lin, z_lin, perturb, torch.zeros_like(dx), dd, 1.0, 1.0)
        assert torch.equal(out[:, a, :3], d_cam[ray])
    # and they are the float64 camera space to fp32 rounding
    p64, d64 = pg.camera_samples(r, s, 0.88, 1.12, 12, perturb)
    assert (p_cam.double() - p64.reshape(b, -1, 3)).abs().max().item() <= 1e-6
    assert (d_cam.reshape(b, -1, 3)[0].double() - d64).abs().max().item() <= 1e-6


#: name -> (B, R, S, window rows or None): NS < 256; NS = 31,487 (not a multiple of the 4,096-sample chunk, odd S);
#: exactly 64 chunks; 256² x 24 (384 chunks, past the final pass's 256 threads); 512² x 48 (3,072 chunks, the scripts'
#: render size); 64 images; a one-row window and a ragged 22-of-64-row window of a ray-sharded render
_C2W_SHAPES = {
    "ns45": (2, 3, 5, None),
    "ns31487-odd-s": (2, 37, 23, None),
    "64-chunks": (2, 128, 16, None),
    "256x256x24": (1, 256, 24, None),
    "512x512x48": (1, 512, 48, None),
    "b64": (64, 16, 12, None),
    "one-row": (2, 64, 24, (17, 18)),
    "22-of-64-rows": (2, 64, 24, (30, 52)),
}
#: inputs: d points alone, d points and d dirs (both inv_scale = 2^-13 and an input_scale != 1), and cancelling ones
_C2W_INPUTS = ("points", "points+dirs", "cancelling")
_C2W_RUNS = [(k, i) for k in _C2W_SHAPES for i in _C2W_INPUTS[:2]] + [("256x256x24", "cancelling"),
                                                                      ("512x512x48", "cancelling")]


def _c2w_inputs(kind, b, ns, n, g):
    """d points (B, NS, 3), d dirs (B N, 3) or None.  cancelling: sample i of the first half carries +L_i (L in
    1e3 [0.5, 1.5]) and sample i of the second half -L_i, each on a randn 1e-3 signal, so the sums are a remainder of
    ~1 of partial sums that reach 1e3 NS / 2; the directions likewise."""
    if kind != "cancelling":
        dx = torch.randn((b, ns, 3), generator=g, device=DEV)
        return dx, (torch.randn((b * n, 3), generator=g, device=DEV) if kind == "points+dirs" else None)

    def pairs(m):
        big = (0.5 + torch.rand((b, m, 3), generator=g, device=DEV)) * 1e3
        h = m // 2
        big[:, h:2 * h] = -big[:, :h]
        big[:, 2 * h:] = 0
        return big + 1e-3 * torch.randn((b, m, 3), generator=g, device=DEV)
    return pairs(ns), pairs(n).reshape(b * n, 3)


@gpu
@pytest.mark.parametrize("shape,inputs", _C2W_RUNS, ids=["%s-%s" % r for r in _C2W_RUNS])
def test_cam2world_grad_vs_fp64(shape, inputs):
    """fenerf_cam2world_grad against dR = sum dx p_cam^T inv_scale input_scale + sum ddir d_cam^T, dT = sum dx inv_scale
    input_scale in float64 on the kernel's own camera-space samples: every entry within 1 ulp of fp32(want) + 1e-12 A
    (A the sum of the absolute terms), the last row exactly 0, nothing left NaN, and two calls the same bits.  On the
    cancelling inputs an fp32 sequential sum of the same terms misses dT by far more than that tolerance."""
    b, r, s, rows = _C2W_SHAPES[shape]
    rd = _desc(b, r, s, rows)
    x_lin, y_lin, z_lin = _tables_for(r, s, rows)
    n = rd.img_h * r
    ns = n * s
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, shape + inputs)))
    perturb = torch.rand((b, n, s, 1), generator=g, device=DEV)
    dx, dd = _c2w_inputs(inputs, b, ns, n, g)
    inv_scale, input_scale = 2.0 ** -13, float(torch.tensor(1 / 0.24).float())
    got = cam2world_grad(rd, x_lin, y_lin, z_lin, perturb, dx, dd, inv_scale, input_scale)
    again = cam2world_grad(rd, x_lin, y_lin, z_lin, perturb, dx, dd, inv_scale, input_scale)
    p_cam, d_cam = camera_space(rd, x_lin, y_lin, z_lin, perturb)
    sc = inv_scale * input_scale
    want = torch.zeros((b, 4, 4), dtype=torch.float64, device=DEV)
    A = torch.zeros_like(want)
    want[:, :3, :3] = torch.einsum('bpi,bpj->bij', dx.double(), p_cam.double()) * sc
    A[:, :3, :3] = torch.einsum('bpi,bpj->bij', dx.double().abs(), p_cam.double().abs()) * sc
    want[:, :3, 3] = dx.double().sum(1) * sc
    A[:, :3, 3] = dx.double().abs().sum(1) * sc
    if dd is not None:
        dd3, dc3 = dd.double().reshape(b, n, 3), d_cam.double().reshape(b, n, 3)
        want[:, :3, :3] += torch.einsum('bni,bnj->bij', dd3, dc3)
        A[:, :3, :3] += torch.einsum('bni,bnj->bij', dd3.abs(), dc3.abs())
    del p_cam
    assert not torch.isnan(got).any(), "an entry was not written"
    assert torch.equal(got, again), "two calls differ"
    assert torch.equal(got[:, 3], torch.zeros_like(got[:, 3]))
    w32 = want.float()
    ulp = torch.nextafter(w32.abs(), torch.full_like(w32, float("inf"))) - w32.abs()
    err = (got.double() - w32.double()).abs()[:, :3]
    tol = (ulp.double() + CAM2WORLD_A * A)[:, :3]
    ratio = (A / want.abs().clamp_min(1e-300))[:, :3]
    print("cam2world grad %s %s (NS = %d, %d chunks): max err / tolerance %.3g, max err / A %.2e, A / |want| up to %.3g"
          % (shape, inputs, ns, -(-ns // 4096), (err / tol).max().item(), (err / A[:, :3]).max().item(),
             ratio.max().item()))
    assert (err <= tol).all(), (err - tol).max().item()
    if inputs == "cancelling":
        seq = float(np.add.accumulate(dx[0, :, 0].cpu().numpy(), dtype=np.float32)[-1]) * sc     # fp32, in sample order
        miss = abs(seq - want[0, 0, 3].item())
        print("  fp32 sequential sum of d T_x: off by %.3g, %.3g x the tolerance" % (miss, miss / tol[0, 0, 3].item()))
        assert miss > 10 * tol[0, 0, 3].item()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: forward_with_frequencies end to end against the chain
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class PoseCase:
    model: str
    b: int
    r: int
    s: int
    hier: bool
    mode: object = "gaussian"               # sample_dist; None: the mean pose
    grad: tuple = ("v_stddev",) + _MEANS    # the pose inputs that are tensors requiring grad
    per_image: tuple = _MEANS               # of those, the (B, 1) ones (the others 0-dim)
    lock: bool = False
    opt: tuple = (("clamp", "relu"),)
    upstream: str = "weights"               # 'weights' (_cases.loss_weights), 'mse' (the inversion's), 'gan'
    pose_loss: bool = False
    coin: float = None                      # hybrid's coin
    frozen: bool = False                    # generator parameters requires_grad_(False), FiLM constant
    film_grad: bool = False
    opaque: bool = False                    # density bias + 0.5
    v_mean: float = None
    std: tuple = ()
    d_phi: tuple = None                     # fixed phi draws
    world: int = 0                          # ray-sharded over `world` virtual ranks


_INV = dict(model="B", b=1, r=256, s=24, hier=False, mode=None, grad=_MEANS, per_image=(), upstream="mse")
_MODE = dict(model="B", b=3, r=64, s=24, hier=True, grad=_ALL, per_image=_ALL)
POSE_CASES = {
    "inversion": PoseCase(**_INV, film_grad=True),
    "inversion-pose-only": PoseCase(**_INV, frozen=True),
    "cfg2": PoseCase("A", 4, 128, 24, True, upstream="gan", pose_loss=True),
    "label-lock": PoseCase("D", 2, 64, 24, True, lock=True),
    "grid-trunk": PoseCase("L", 2, 64, 24, True, opaque=True),
    "feature-head": PoseCase("K", 1, 48, 24, True),
    "bridge": PoseCase("N", 2, 64, 24, False, opt=(("clamp", "softplus"), ("noise", 0.5))),
    "direction-free": PoseCase("P", 2, 64, 24, True),
    "uniform": PoseCase(**_MODE, mode="uniform"),
    "hybrid-uniform": PoseCase(**_MODE, mode="hybrid", coin=0.25),
    "hybrid-gaussian": PoseCase(**_MODE, mode="hybrid", coin=0.75),
    "truncated-gaussian": PoseCase(**_MODE, mode="truncated_gaussian"),
    "spherical-uniform": PoseCase(**_MODE, mode="spherical_uniform", std=(("v_stddev", 1.2),)),
    # phi = (d - 0.5) 2 v_stddev + v_mean: -0.073 (clamped), 0.113, 0.0355 -- each >= 1e-6 from the edge
    "clamp": PoseCase("A", 3, 64, 24, True, mode="uniform", grad=_ALL, per_image=_ALL, v_mean=0.02,
                      d_phi=(0.2, 0.8, 0.55)),
    "sharded": PoseCase("B", 2, 64, 24, True, world=3),
}
_G, _F, _E, _S, _SS = ("guard", None), ("fast", None), ("exact", None), ("split", None), ("split", "split")
_PRECISIONS = {"inversion": [_G, _F, _E, _S, _SS], "inversion-pose-only": [_G, _E], "cfg2": [_G, _E, _S],
               "direction-free": [_E, _SS], "clamp": [_E]}
_RUNS_E2E = [(k, p, gp) for k in POSE_CASES for p, gp in _PRECISIONS.get(k, [_G, _E])]

#: guard / fast (the fp16 gradient streams): the largest abs_rel of the pose inputs and d cam2world, measured x 1.5 and
#: rounded up; every one far below RAY_BOUND['guard'].  Measured on an H100 80GB HBM3 (700 W): inversion 1.43e-4 (fast
#: 1.42e-4), pose-only inversion 1.27e-4, cfg2 2.57e-4, label-lock 9.52e-4, grid-trunk 2.60e-4, feature-head 2.49e-4,
#: bridge 3.32e-4, uniform 4.54e-4, hybrid-uniform 4.82e-4, hybrid-gaussian 5.39e-4, truncated-gaussian 3.25e-4,
#: spherical-uniform 4.93e-4, sharded 3.50e-4.  rel, printed: at the inversion shape 1.2e-3 (h_mean) and 4.3e-4 (v_mean)
#: in guard, 9.7e-4 / 7.1e-4 in fast; up to 0.87 on other cases' inputs whose sum cancels (A / |want| 1.6e4).
GUARD_BOUND = {
    ("inversion", "guard"): 3e-4, ("inversion", "fast"): 3e-4, ("inversion-pose-only", "guard"): 2e-4,
    ("cfg2", "guard"): 4e-4, ("label-lock", "guard"): 1.5e-3, ("grid-trunk", "guard"): 4e-4,
    ("feature-head", "guard"): 4e-4, ("bridge", "guard"): 5e-4, ("uniform", "guard"): 7e-4,
    ("hybrid-uniform", "guard"): 8e-4, ("hybrid-gaussian", "guard"): 9e-4, ("truncated-gaussian", "guard"): 5e-4,
    ("spherical-uniform", "guard"): 8e-4, ("sharded", "guard"): 6e-4,
}
assert max(GUARD_BOUND.values()) <= RAY_BOUND["guard"]
#: exact / split / split + grad split: FIELD_BOUND['exact'] on abs_rel everywhere and on rel wherever A / |want| <= 1e2
#: (measured: abs_rel <= 3.5e-6, L; rel <= 7.0e-5 where A / |want| <= 1e2).  L: L_BOUND (measured rel 1.9e-4).  P:
#: P_BOUND on abs_rel (measured 3.9e-4).  P's rel is held to P_REL_BOUND instead: measured where A / |want| <= 1e2
#: 1.2e-2 in exact and 1.8e-2 with grad_precision='split' (d cam2world), 8.5e-3 on the pose inputs.  P's per-sample point gradients carry fp32 error up to 2.6e-3 of their largest entry (its first
#: colour layer amplifies the rounding; test_gpu_fp64_ray_grads.py), systematic from sample to sample, so it adds up in
#: the pose sum instead of cancelling.
P_REL_BOUND = 3e-2


def bound_of(case, precision):
    if precision in ("guard", "fast"):
        return GUARD_BOUND[(case, precision)]
    return {"P": P_BOUND, "L": L_BOUND}.get(POSE_CASES[case].model, FIELD_BOUND["exact"])


def rel_bound_of(case, precision):
    return P_REL_BOUND if POSE_CASES[case].model == "P" else bound_of(case, precision)


@functools.lru_cache(maxsize=1)
def _gen(model, opaque):
    return _cases.build_mirror(_cases.Case("fp64_pose_" + model, model, 1, 0, sigma_bias_shift=0.5 if opaque else 0.0),
                               DEV)


def _gan_factors(b):
    spread = 10.0 ** (-3.0 * torch.arange(b, dtype=torch.float64) / max(1, b - 1))
    return spread[torch.randperm(b, generator=torch.Generator().manual_seed(b))]


def run_pose_case(name, precision, grad_precision):
    """forward_with_frequencies on draws made here (vr.ReplayRng), its pose-input gradients, d cam2world of
    render_with_grad with a cam2world leaf on the same inputs, and the chain on render_forward_stages' intermediates."""
    from test_gpu_fp64_train_grads import gan_d_pixels
    c = POSE_CASES[name]
    gen = _gen(c.model, c.opaque)
    params = list(gen.parameters())
    for p in params:
        p.grad = None
    b, r, s = c.b, c.r, c.s
    n = r * r
    seed = sum(map(ord, name))
    g = torch.Generator().manual_seed(seed)
    film_in = pg.film_inputs(gen, pg.latents(c.model, b, DEV, seed))
    if c.film_grad:
        film_in = [f.clone().requires_grad_(True) for f in film_in]
    cam_draws, cam = camera_draws(c.mode, b, g, c.coin, c.d_phi)
    pose = pose_values(b, c.grad, c.per_image, g, DEV, v_mean=c.v_mean, std=dict(c.std))
    perturb = torch.rand((b, n, s, 1), generator=g)
    noise_c = torch.randn((b, n, s, 1), generator=g) if c.hier else None
    u = torch.rand((b * n, s), generator=g) if c.hier else None
    noise_f = torch.randn((b, n, 2 * s if c.hier else s, 1), generator=g)
    draws = [("rand", perturb)] + cam_draws + ([("randn", noise_c), ("rand", u)] if c.hier else []) + [("randn", noise_f)]
    o = _opt(**dict(c.opt))
    kw = pg.kwargs(r, s, sample_dist=c.mode, hierarchical_sample=c.hier, lock_view_dependence=c.lock,
                   clamp_mode=o["clamp"], nerf_noise=o["noise"], precision=precision, grad_precision=grad_precision)
    kw = {k: v for k, v in kw.items() if k not in POSE_ARGS}
    c_img = gen.siren.field_spec().out_dim - 1

    def render(pose_kw, shard=None):
        extra = dict(_ray_shard=shard) if shard is not None else {}
        return gen.forward_with_frequencies(*film_in, **kw, **pose_kw, _rng=vr.ReplayRng(draws, DEV), **extra)

    d_poses = pg.pose_loss_weights((b, 2)).to(DEV) if c.pose_loss else None
    if c.upstream == "gan":
        d_pixels = gan_d_pixels(b, c_img, r, torch.Generator(device=DEV).manual_seed(seed))
    elif c.upstream == "weights":
        d_pixels = _cases.loss_weights((b, c_img, r, r)).to(DEV)
    else:
        # the inversion's MSE to a target rendered at (h, v) + (0.06, -0.04)
        off = dict(h_mean=0.06, v_mean=-0.04)
        with torch.no_grad():
            target, _ = render({k: (v.detach() + off.get(k, 0.0)) if isinstance(v, torch.Tensor) else v + off.get(k, 0.0)
                                for k, v in pose.items()})
        d_pixels = None
    frozen = [p for p in params if p.requires_grad] if c.frozen else []
    for p in frozen:
        p.requires_grad_(False)
    try:
        shards = [fdist.RayShard(k, c.world, collective=False) for k in range(c.world)] if c.world else [None]
        px = 0
        for shard in shards:
            win, po = render(pose, shard)
            if d_pixels is None:
                d_pixels = (2 * (win.detach() - target) / win.numel())
            loss = (win * d_pixels).sum() + ((po * d_poses).sum() if d_poses is not None else 0)
            loss.backward()
            px = px + win.detach()
        if c.frozen:
            assert all(p.grad is None for p in params), "a frozen generator's parameter got a gradient"
    finally:
        for p in frozen:
            p.requires_grad_(True)
    got = {k: v.grad for k, v in pose.items() if isinstance(v, torch.Tensor)}

    # the same render's stages, the kernel's cam2world from the same draws
    code, doubled, d_theta, d_phi = ops.camera_draws(b, c.mode, vr.ReplayRng(cam_draws, DEV))
    values = tuple(pose[k].detach() if isinstance(pose[k], torch.Tensor) else pose[k] for k in POSE_ARGS)
    c2w, _, _ = ops.camera_poses_launch(b, code, doubled, values, d_theta, d_phi, torch.device(DEV))
    rd = ops.make_render_desc(batch=b, img_size=r, num_steps=s, hierarchical=c.hier, clamp_mode=o["clamp"],
                              nerf_noise=o["noise"], fov=12, softmax_label=gen.softmax_label, lock_view_dependence=c.lock,
                              precision=precision, guard_tau=getattr(gen.siren, '_guard_tau', 0.0))
    table = gen.siren.film_table(*[f.detach() for f in film_in])
    args = (*ops.ray_tables(r, s, 0.88, 1.12, DEV), c2w, perturb.to(DEV).contiguous(),
            *(None if t is None else t.to(DEV) for t in (noise_c, u, noise_f)))
    with torch.no_grad():
        st = ops.render_forward_stages(gen.siren, rd, table, *args)
    assert torch.equal(st["pixels"], px), "render_forward_stages differs from forward_with_frequencies"
    got_c2w = None
    if not c.world:
        leaf = c2w.clone().requires_grad_(True)
        frame = backward.render_with_grad(gen.siren, rd, table, *args[:3], leaf, *args[4:], grad_precision=grad_precision)
        (frame * d_pixels).sum().backward()
        got_c2w = leaf.grad
        for p in params:
            p.grad = None
    noise = args[-1][..., 0] if o["noise"] else None
    chain = pg.pose_chain_fp64(gen.siren, table, st, dict(cam, perturb=perturb), pose, c.mode, c.lock, o, noise,
                               d_pixels, d_poses)
    return c, got, got_c2w, chain


def _fmt(t):
    return "[%s]" % " ".join("%.2e" % v for v in t.flatten().tolist())


@gpu
@pytest.mark.parametrize("name,precision,grad_precision", _RUNS_E2E,
                         ids=["%s-%s%s" % (k, p, "-gs" if gp else "") for k, p, gp in _RUNS_E2E])
def test_pose_grads_vs_fp64(monkeypatch, name, precision, grad_precision):
    """The pose inputs' gradients of forward_with_frequencies and d cam2world of the same render against the float64
    chain: exact / split within the field's bound on abs_rel everywhere and on rel wherever A / |want| <= 1e2; guard /
    fast on abs_rel within GUARD_BOUND (rel printed)."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    c, got, got_c2w, chain = run_pose_case(name, precision, grad_precision)
    tag = "%s %s%s" % (name, precision, "+gs" if grad_precision else "")
    bound = bound_of(name, precision)
    exact_like = precision not in ("guard", "fast")
    n_face, share = chain["face"]
    print("pose grads %s: %d face rows carrying at most %.2e of A" % (tag, n_face, share))
    worst = 0.0
    for k, want in chain["grads"].items():
        assert (got[k] is None) == (want is None), (k, got[k], want)
        if want is None:
            continue
        rel, abs_rel, ratio = pg.pose_errors(got[k], want, chain["A"][k])
        print("  %-8s rel %s abs_rel %s A/|want| %s" % (k, _fmt(rel), _fmt(abs_rel), _fmt(ratio)))
        worst = max(worst, abs_rel.max().item())
        assert abs_rel.max().item() <= bound, (k, abs_rel)
        if exact_like and (ratio <= 1e2).any():
            assert rel[ratio <= 1e2].max().item() <= rel_bound_of(name, precision), (k, rel)
    if got_c2w is not None:
        rel, abs_rel, ratio = pg.pose_errors(got_c2w[:, :3], chain["d_c2w"][:, :3], chain["A_c2w"][:, :3])
        print("  cam2world: rel %.2e where A/|want| <= 1e2 (%.2e over all), abs_rel %.2e, A/|want| up to %.3g" % (
            rel[ratio <= 1e2].max().item() if (ratio <= 1e2).any() else 0.0, rel.max().item(), abs_rel.max().item(),
            ratio.max().item()))
        worst = max(worst, abs_rel.max().item())
        assert abs_rel.max().item() <= bound, abs_rel.max().item()
        if exact_like and (ratio <= 1e2).any():
            assert rel[ratio <= 1e2].max().item() <= rel_bound_of(name, precision)
    print("  worst abs_rel %.3g (bound %g)" % (worst, bound))
    if c.upstream == "gan":
        f = _gan_factors(c.b)
        for k in c.per_image:
            rel = pg.pose_errors(got[k], chain["grads"][k], chain["A"][k])[0]
            print("  %s per image under the GAN spread: %s" % (
                k, " ".join("%.0e: %.2e" % (a, e) for a, e in zip(f.tolist(), rel.flatten().tolist()))))
    if name == "clamp":
        phi = (cam_phi(c) - 0.5) * 2 * 0.155 + c.v_mean
        clamped = phi < 1e-5
        assert clamped.any() and (phi - 1e-5).abs().min() >= 1e-6
        for k in ("v_stddev", "v_mean"):
            assert (got[k][clamped] == 0).all() and (chain["grads"][k][clamped.to(chain["grads"][k].device)] == 0).all()
            assert (got[k][~clamped] != 0).all() and (chain["grads"][k][~clamped.cpu()] != 0).all()


def cam_phi(c):
    return torch.tensor(c.d_phi, dtype=torch.float64, device=DEV).reshape(-1, 1)
