"""point_forward(..., ray_grad=True)'s kernels against float64, at production shapes.

  1. The depth gradient (fenerf_composite_backward_rays_dz) on exact duplicate coarse depths: zero-width intervals,
     one at the far end.  Its other cases are the '-rays_dz' entries of test_gpu_fp64_reference.py,
     test_many_samples.py and test_hd_fields.py.
  2. fenerf_grid_coord_grad on model B's 32 x 96³ grid at B = 4 x 128² x 24 points, d feat fp32 and fp16, with points
     planted on interior cell faces, exactly on x s = +-1, straddling the box and fully outside (gradient exactly 0),
     against a float64 reference that takes each point's cell from the kernel's fp32 index (the side of a one-sided
     derivative); fenerf_ray_dir_grad bit for bit against an fp32 restatement of its stated order (coarse then fine, in
     index order, times a power of two), on NaN-prefilled outputs, at S = 3, 255, 256.
  3. render_rays_with_grad(..., ray_grad=True) end to end: every ray gradient against a float64 VJP on the render's own
     intermediates (render_rays_stages), the fine directions gathered by slots derived here from the stand-alone
     resampler (the stable argsort of its draw-order depths), in every precision each field serves; the cfg2 cases
     again under point chunks.
  4. The cfg2 cases of 3 and test_gpu_fp64_train_grads.py's cfg2 camera render in a child process under
     torch.use_deterministic_algorithms(True) (tests/_fp64_det_child.py): the same float64 bounds as without the flag.

CPU: the float64 ray chain of 3 against autograd of the render written as one float64 function of the ray leaves
(per-sample and per-ray directions, lock_view_dependence, flat).  The depth gradient's semantics under every compositing
option are anchored in the reference itself by test_ray_grads.py's flat goldens (white_back, black_back, the label
softmax, softplus + noise, duplicate depths).

Bounds: measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), see each constant.  The GPU part of this module and
the '-rays_dz' entries elsewhere ran in 43 s there.
"""
import copy
import ctypes
import dataclasses
import functools
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _fp64 import _film, _opt, _rel, _siren, composite_ref
from fenerf_b200 import _lib, backward, ops
from oracle import render_oracle as oracle
from test_gpu_fp64_rays import camera_rays, edit_rays
from test_gpu_fp64_reference import (COMPOSITE_BOUND, DEPTH_BOUND, FIELD_BOUND, LAYOUT_BOUND, _composite_backward,
                                     _composite_inputs, composite_vjp)
from test_ray_grads import _precisions, fp32_cell_index, grid_coord_grad_ref, plant_face_points
from test_split_backward import P_BOUND

DEV = "cuda:0"
gpu = pytest.mark.gpu

#: the grid coordinate gradient, max |kernel - fp64| / max |fp64| (fp32 corner products and dot products of 32 terms).
#: Measured: 9.4e-6 on face, boundary and straddling points, 7.8e-6 inside, exactly 0 outside (fp32 and fp16 d feat)
GRID_BOUND = 2e-5
#: ray gradients end to end, max |gpu - fp64| / max |fp64| per ray tensor: exact / split / split + grad_precision='split'
#: at FIELD_BOUND['exact'] (measured <= 3.5e-5, d z <= 4.6e-5), guard (fp16 gradient streams) at test_ray_grads.py's 5e-2
#: (measured <= 1.4e-2, M).  P: P_BOUND (its first colour layer amplifies fp32 rounding; measured 2.6e-3, 4.2e-3 with
#: grad_precision='split'); L, the grid in the trunk: L_BOUND (measured: points 3.1e-4, directions 8.1e-5 -- the directions
#: reach only the colour branch and carry no grid term, so the excess over 1e-4 is the opaque L field's fp32 conditioning
#: at 49,152 points, where test_ray_grads.py's restatement test sees the worst of 1,440).  Rows whose fp32 grid index lies
#: within 1e-5 cells of a face are
#: left out: the kernel takes the derivative on the side of its fp32 cell, the float64 chain on its own
#: (test_grid_coord_grad_vs_fp64 checks those rows against the kernel's side).
RAY_BOUND = {"exact": FIELD_BOUND["exact"], "split": FIELD_BOUND["exact"], "guard": 5e-2}
L_BOUND = 5e-4
FACE_CELLS = 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# 1. zero-width intervals
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("c,steps,opt", [(4, 24, _opt("relu")), (22, 64, _opt("softplus", noise=0.5)),
                                         (22, 256, _opt("relu", white_back=True))], ids=["C4-S24", "C22-S64", "C22-S256"])
def test_depth_gradient_with_zero_width_intervals(c, steps, opt):
    """Coarse depths with exact duplicates (every 5th sample repeats its predecessor on every 3rd ray; the last two
    samples equal on every 4th ray): d raw is the ray-major entry's bit for bit and d z is float64's, every entry written."""
    x = dict(_composite_inputs(c, steps, False, False))
    z = x["z_c"].clone()
    z[:, ::3, 5::5] = z[:, ::3, 4:-1:5][..., :z[:, ::3, 5::5].shape[-1]]
    z[:, ::4, -1] = z[:, ::4, -2]
    x["z_c"] = z.contiguous()
    assert (z[..., 1:] == z[..., :-1]).any() and (z[..., 1:] >= z[..., :-1]).all()
    g = torch.Generator().manual_seed(steps)
    b, n = z.shape[:2]
    noise = torch.randn(b, n, steps, generator=g).to(DEV) if opt["noise"] else None
    d_pixels = torch.randn(b, n, c - 1, generator=g).to(DEV)
    img = math.isqrt(n)
    d_c, d_z = _composite_backward(opt, steps, False, x, noise, d_pixels, "rays_dz", b, img)
    e_c = _composite_backward(opt, steps, False, x, noise, d_pixels, "rays", b, img)[0]
    assert torch.equal(d_c, e_c)
    w_c, w_z = composite_vjp(x["raw_c"], x["z_c"], None, None, noise, opt, d_pixels, ray_major=True, want_z=True)
    errs = dict(d_raw_c=_rel(d_c, w_c), d_z=_rel(d_z, w_z))
    print("zero-width intervals C=%d S=%d: %s" % (c, steps, errs))
    assert all(v == v for v in errs.values()), errs
    assert errs["d_raw_c"] <= COMPOSITE_BOUND and errs["d_z"] <= DEPTH_BOUND, errs


# ---------------------------------------------------------------------------------------------------------------------
# 2. the two ray-gradient kernels, called directly
# ---------------------------------------------------------------------------------------------------------------------
_GRID_P = 4 * 128 * 128 * 24          # cfg2's coarse pass: B = 4, 128² rays, 24 samples


@functools.lru_cache(maxsize=1)
def _grid_inputs():
    siren = _siren("B", DEV)
    spec = siren.field_spec()
    R = spec.grid_res
    pts, cls, axis = plant_face_points(torch.Generator().manual_seed(31), _GRID_P, spec.input_scale, R)
    return siren, pts, cls, axis


@gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_grid_coord_grad_vs_fp64(dtype):
    siren, pts, cls, axis = _grid_inputs()
    spec = siren.field_spec()
    R, s = spec.grid_res, spec.input_scale
    P = pts.shape[0]
    g = torch.Generator().manual_seed(32)
    d_feat = torch.randn((P, 32), generator=g).to(DEV).to(torch.float32 if dtype == "fp32" else torch.float16).contiguous()
    points = pts.to(DEV).contiguous()
    out = torch.full((P, 3), float("nan"), device=DEV)
    packed = siren.packed()
    _lib.check(_lib.lib().fenerf_grid_coord_grad(ctypes.byref(packed.desc), packed.ptr, points.data_ptr(), d_feat.data_ptr(),
                                                 32, P, out.data_ptr(), 1 if dtype == "fp32" else 0,
                                                 torch.cuda.current_stream().cuda_stream))
    cells = torch.from_numpy(np.floor(fp32_cell_index(pts.numpy(), s, R))).long().to(DEV)
    grid = siren.spatial_embeddings.detach().double()
    want = torch.empty((P, 3), dtype=torch.float64, device=DEV)
    for p0 in range(0, P, 1 << 18):
        sl = slice(p0, p0 + (1 << 18))
        want[sl] = grid_coord_grad_ref(grid, points[sl].double() * s, d_feat[sl].double(), cell=cells[sl])
    assert torch.isfinite(out).all(), "an entry was not written"
    assert torch.count_nonzero(out[cls.to(DEV) == 3]).item() == 0, "points fully outside the box got a gradient"
    errs = {}
    scale = want.abs().max().item()
    for c, name in enumerate(("face", "boundary", "straddle", "outside", "inside")):
        m = cls.to(DEV) == c
        errs[name] = (out[m].double() - want[m]).abs().max().item() / scale
    print("grid coord grad %s (P = %d): %s" % (dtype, P, {k: "%.2e" % v for k, v in errs.items()}))
    assert max(errs.values()) <= GRID_BOUND, errs


def _ray_dir_grad(n_rays, S, dir_group, dc, df, slots, inv):
    out = torch.full(((n_rays * S) // dir_group, 3), float("nan"), device=DEV)
    p = lambda t: t.data_ptr() if t is not None else 0                  # noqa: E731
    _lib.check(_lib.lib().fenerf_ray_dir_grad(n_rays, S, dir_group, p(dc), p(df), p(slots), p(inv), out.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
    return out


def ray_dir_grad_ref(n_rays, S, dir_group, dc, df, slots, inv):
    """The kernel's stated order in fp32: dir_group 1, slot k of a ray = (coarse k + the fine sample j that drew slot k)
    x inv; dir_group S, per ray (the coarse samples summed in index order + the fine ones summed likewise) x inv."""
    dc, inv = dc.reshape(n_rays, S, 3), inv.cpu()
    df = df.reshape(n_rays, S, 3) if df is not None else None
    if dir_group == 1:
        v = torch.zeros_like(dc)
        if df is not None:
            v.scatter_(1, slots.long().unsqueeze(-1).expand(-1, -1, 3), df)
        return ((dc + v) * inv).reshape(-1, 3)
    sc = torch.zeros((n_rays, 3))
    sf = torch.zeros((n_rays, 3))
    for k in range(S):
        sc = sc + dc[:, k]
        if df is not None:
            sf = sf + df[:, k]
    return (sc + sf) * inv


#: (n_rays, S, dir_group, fine): ray counts that are not multiples of the 256-thread block where one thread is a ray
_DIR_CASES = [(100003, 3, 1, True), (4099, 255, 1, True), (4097, 256, 1, True), (65536, 24, 1, False),
              (65539, 24, "S", True), (4097, 256, "S", True), (65539, 24, "S", False)]


@gpu
@pytest.mark.parametrize("n_rays,S,group,fine", _DIR_CASES,
                         ids=["n%d-S%d-g%s%s" % (n, s, g, "" if f else "-no_fine") for n, s, g, f in _DIR_CASES])
def test_ray_dir_grad_is_its_stated_order(n_rays, S, group, fine):
    """Random per-ray slot permutations (slot 255 at S = 256); d dirs bit for bit the fp32 restatement, every slot
    written (NaN-prefilled output)."""
    dir_group = S if group == "S" else 1
    g = torch.Generator().manual_seed(n_rays + S)
    dc = torch.randn((n_rays * S, 3), generator=g)
    df = torch.randn((n_rays * S, 3), generator=g) if fine else None
    slots = torch.argsort(torch.rand((n_rays, S), generator=g), -1).to(torch.uint8) if fine and dir_group == 1 else None
    if slots is not None and S == 256:
        assert (slots == 255).any()
    inv = torch.tensor([2.0 ** -7])
    got = _ray_dir_grad(n_rays, S, dir_group, dc.to(DEV), df.to(DEV) if fine else None,
                        slots.to(DEV).contiguous() if slots is not None else None, inv.to(DEV))
    want = ray_dir_grad_ref(n_rays, S, dir_group, dc, df, slots, inv)
    assert not torch.isnan(got).any(), "a slot was not written"
    assert torch.equal(got.cpu(), want)


# ---------------------------------------------------------------------------------------------------------------------
# 3. end to end on the render's own intermediates
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class RayCase:
    model: str
    batch: int
    r: int               # r² rays per image
    s: int
    hier: bool
    opt: tuple           # _opt keyword items
    dirs: str = "sample"   # 'sample': one per sample (dir_group 1); 'ray': one per ray (dir_group S)
    lock: bool = False
    tie_u: bool = False  # duplicated u draws on every 7th ray: exact ties between fine depths


_RELU, _RELU_NOISE = (("clamp", "relu"),), (("clamp", "relu"), ("noise", 0.5))
RAY_CASES = {
    "B-cfg2-hier": RayCase("B", 4, 128, 24, True, _RELU),
    "B-cfg2-flat": RayCase("B", 4, 128, 24, False, _RELU_NOISE),
    "B-flat-white-softmax": RayCase("B", 2, 32, 24, False, (("clamp", "relu"), ("white_back", True), ("softmax", True))),
    "D-flat-black-softplus": RayCase("D", 2, 32, 24, False, (("clamp", "softplus"), ("black_back", True))),
    "B-s256-hier": RayCase("B", 1, 24, 256, True, _RELU),
    "B-s256-flat": RayCase("B", 1, 24, 256, False, _RELU_NOISE),
    "K-s160-flat": RayCase("K", 1, 20, 160, False, (("clamp", "relu"), ("softmax", True))),
    "L-hier": RayCase("L", 2, 32, 24, True, _RELU),
    "M-hier": RayCase("M", 2, 32, 24, True, _RELU),
    "N-flat": RayCase("N", 2, 32, 24, False, _RELU_NOISE),
    "P-hier": RayCase("P", 2, 32, 24, True, _RELU),
    "B-expand-lock": RayCase("B", 2, 32, 24, True, _RELU, dirs="ray", lock=True),
    "B-tie-u": RayCase("B", 2, 32, 24, True, _RELU, tie_u=True),
}
#: the split forward is not built for label FiLM, feature-head or grid-trunk fields (K, L): exact and guard, as M / N
_RUNS = [(name, p, e) for name, c in RAY_CASES.items() for p, e in _precisions("M" if c.model in "KL" else c.model)]


@functools.lru_cache(maxsize=2)
def _field(model, device=DEV):
    return _siren(model, device, sigma_bias_shift=0.5 if model == "L" else 0.0)


def _case_inputs(case, seed):
    b, r, s = case.batch, case.r, case.s
    n = r * r
    g = torch.Generator(device=DEV).manual_seed(seed)
    rays = edit_rays(*camera_rays(b, r, s, g), g, case.dirs == "sample")
    draws = [torch.randn(b, n, s, generator=g, device=DEV), torch.rand(b * n, s, generator=g, device=DEV),
             torch.randn(b, n, 2 * s if case.hier else s, generator=g, device=DEV)]
    if case.tie_u:
        draws[1][::7, 1] = draws[1][::7, 0]
        draws[1][::7, -1] = draws[1][::7, 2]
    return rays, draws, g


def _field_vjp(siren64, film64, pts, dirs, d_raw, chunk=1 << 15):
    """float64 (d points, d dirs) (B, P, 3) of sum(field(points, dirs) * d_raw), per point, in chunks."""
    d_p, d_d = torch.empty_like(pts), torch.empty_like(dirs)
    for p0 in range(0, pts.shape[1], chunk):
        sl = slice(p0, p0 + chunk)
        x = pts[:, sl].detach().requires_grad_(True)
        d = dirs[:, sl].detach().requires_grad_(True)
        out = oracle.field_eval(siren64, x, film64, d)
        gx, gd = torch.autograd.grad((out * d_raw[:, sl]).sum(), [x, d], allow_unused=True)
        d_p[:, sl] = gx
        d_d[:, sl] = gd if gd is not None else 0
    return d_p, d_d


def ray_chain_vjp(siren, film, st, rays, slots, case, opt, noise, d_pixels):
    """float64 ray gradients of sum(pixels * d_pixels) on the render's intermediates st: ray-major composite_vjp (with the
    coarse depths a leaf on flat renders), then each field pass's VJP w.r.t. its points and directions.  The fine pass
    reads the caller's directions at `slots` (B, N, S) (per sample), the per-ray ones, or (0, 0, -1) under
    lock_view_dependence; its points are built from the per-ray origins and directions under no_grad.
    -> {'points', 'dirs', 'z_vals'} (None where the reference gives none)."""
    b, n, s, c = st["raw_c"].shape
    siren64 = copy.deepcopy(siren).double()
    for p in siren64.parameters():
        p.requires_grad_(False)
    film64 = film.double()
    d_c, second = composite_vjp(st["raw_c"], rays["z_vals"], st["raw_f"], st["z_f"], noise, opt, d_pixels, ray_major=True,
                                want_z=not case.hier)
    per_sample = rays["dirs"].dim() == 4
    dirs64 = rays["dirs"].double()
    dirs_c = dirs64.reshape(b, n * s, 3) if per_sample else dirs64.repeat_interleave(s, dim=1)
    d_pts, d_dc = _field_vjp(siren64, film64, rays["points"].double().reshape(b, n * s, 3), dirs_c, d_c.reshape(b, -1, c))
    d_dirs = d_dc.reshape(b, n, s, 3)
    if case.hier and not case.lock:
        gathered = torch.gather(dirs64, 2, slots.unsqueeze(-1).expand(-1, -1, -1, 3)) if per_sample else \
            dirs64.unsqueeze(2).expand(b, n, s, 3)
        _, d_df = _field_vjp(siren64, film64, st["points_f"].double().reshape(b, n * s, 3), gathered.reshape(b, n * s, 3),
                             second.reshape(b, -1, c))
        d_df = d_df.reshape(b, n, s, 3)
        if per_sample:
            d_dirs = d_dirs.scatter_add(2, slots.unsqueeze(-1).expand(-1, -1, -1, 3), d_df)
        else:
            d_dirs = d_dirs + d_df
    if siren.field_spec().wo_dir:
        d_dirs = None
    elif not per_sample:
        d_dirs = d_dirs.sum(2)
    return dict(points=d_pts.reshape(b, n, s, 3), dirs=d_dirs, z_vals=None if case.hier else second)


def _gpu_ray_grads(siren, rd, film, rays, draws, weights, grad_precision):
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in rays.items()}
    px = backward.render_rays_with_grad(siren, rd, film, leaves["points"], leaves["dirs"], leaves["origins"],
                                        leaves["ray_dirs"], leaves["z_vals"], *draws, grad_precision=grad_precision,
                                        ray_grad=True)
    (px * weights).sum().backward()
    return px.detach(), {k: v.grad for k, v in leaves.items()}


def face_rows(siren, points):
    """(B, N, S) samples whose fp32 grid index (as the kernels form it) lies within FACE_CELLS of a cell face."""
    spec = siren.field_spec()
    if not spec.grid_channels:
        return torch.zeros(points.shape[:3], dtype=torch.bool, device=points.device)
    i = torch.from_numpy(fp32_cell_index(points.cpu().numpy(), spec.input_scale, spec.grid_res)).double()
    return ((i - i.round()).abs() < FACE_CELLS).any(-1).to(points.device)


def _errors(got, want, skip=None):
    errs = {}
    for k in ("points", "dirs", "z_vals"):
        if want[k] is None:
            continue
        g, w = got[k], want[k]
        if skip is not None and k != "dirs":
            g, w = g[~skip], w[~skip]
        errs[k] = _rel(g, w)
    return errs


@dataclasses.dataclass
class Run:
    """One case's render set-up, its intermediates (render_rays_stages) and the float64 ray gradients on them."""
    name: str
    case: RayCase
    precision: str
    grad_precision: str
    siren: object
    rd: object
    film: torch.Tensor
    rays: dict
    draws: list
    weights: torch.Tensor
    st: dict
    want: dict


def run_case(name, precision, extra, case=None):
    case = case or RAY_CASES[name]
    o = _opt(**dict(case.opt))
    siren = _field(case.model)
    seed = 5000 + sum(map(ord, name))
    rays, draws, g = _case_inputs(case, seed)
    b, n, s = case.batch, case.r * case.r, case.s
    rd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=s, hierarchical=case.hier, clamp_mode=o["clamp"],
                            nerf_noise=o["noise"], last_back=o["last_back"], white_back=o["white_back"],
                            black_back=o["black_back"], softmax_label=o["softmax"], lock_view_dependence=case.lock,
                            precision=precision)
    film = _film(siren, b, seed)
    c = siren.field_spec().out_dim
    weights = torch.randn(b, n, c - 1, generator=g, device=DEV)
    with torch.no_grad():
        st = ops.render_rays_stages(siren, rd, film, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                                    rays["z_vals"], *draws, slots=True)
    slots = None
    if case.hier and case.dirs == "sample" and not case.lock:
        z_sa = ops.resample(rd, st["raw_c"], rays["z_vals"], rays["ray_dirs"], rays["origins"][:, 0].contiguous(),
                            draws[0], draws[1])[0].reshape(b, n, s)
        slots = torch.sort(z_sa, dim=-1, stable=True)[1]
        assert torch.equal(st["slots_f"].long(), slots), "the render's draw slots differ from the stable argsort"
        if case.tie_u:
            ties = (z_sa[..., 1:] == z_sa[..., :1]).any(-1)
            assert ties.any(), "no exact tie between fine depths"
    else:
        assert st["slots_f"] is None
    noise = draws[2] if o["noise"] else None
    want = ray_chain_vjp(siren, film, st, rays, slots, case, o, noise, weights)
    return Run(name, case, precision, extra.get("grad_precision"), siren, rd, film, rays, draws, weights, st, want)


def gpu_ray_grads(run):
    return _gpu_ray_grads(run.siren, run.rd, run.film, run.rays, run.draws, run.weights, run.grad_precision)


def bound_of(run):
    if run.precision == "guard":
        return RAY_BOUND["guard"]
    return {"P": P_BOUND, "L": L_BOUND}.get(run.case.model, RAY_BOUND[run.precision])


def check(run, got, px, label=""):
    assert torch.equal(px, run.st["pixels"]), "render_rays_stages differs from the differentiable render"
    assert got["origins"] is None and got["ray_dirs"] is None
    for k in ("points", "dirs", "z_vals"):
        assert (got[k] is None) == (run.want[k] is None), (k, got[k] is None)
    skip = face_rows(run.siren, run.rays["points"])
    assert skip.float().mean().item() <= 1e-3
    errs = _errors(got, run.want, skip)
    print("ray grads %s %s%s%s: %s (%d face rows left out; with them %s)" % (
        run.name, run.precision, "+gs" if run.grad_precision else "", label, {k: "%.2e" % v for k, v in errs.items()},
        skip.sum().item(), {k: "%.2e" % v for k, v in _errors(got, run.want).items()}))
    assert all(v == v for v in errs.values()), errs
    assert max(errs.values()) <= bound_of(run), errs
    return errs


@gpu
@pytest.mark.parametrize("name,precision,extra", _RUNS, ids=["%s-%s%s" % (n, p, "-gs" if e else "") for n, p, e in _RUNS])
def test_ray_grads_vs_fp64(monkeypatch, name, precision, extra):
    """Every ray gradient of render_rays_with_grad(..., ray_grad=True) against the float64 VJP on its own intermediates;
    the None pattern (origins and per-ray directions always, z_vals with hierarchical sampling, directions for P)."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    run = run_case(name, precision, extra)
    px, got = gpu_ray_grads(run)
    check(run, got, px)


#: CHUNK_POINTS for the cfg2 cases' chunked runs: not a multiple of S = 24 (each image of 393,216 points per pass in
#: point chunks), and three images per chunk (chunks of 3 and 1 images)
_CHUNKS = {"points_not_multiple_of_s": 100001, "ragged_images": 3 * 128 * 128 * 24}


@gpu
@pytest.mark.parametrize("chunk", list(_CHUNKS))
@pytest.mark.parametrize("name", ["B-cfg2-hier", "B-cfg2-flat"])
def test_ray_grads_under_point_chunks(monkeypatch, name, chunk):
    """The cfg2 cases (exact) with _add_points' point chunks: within the float64 bound, and within LAYOUT_BOUND of the
    one-chunk run."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    run = run_case(name, "exact", {})
    monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
    _, one = gpu_ray_grads(run)
    monkeypatch.setattr(backward, "CHUNK_POINTS", _CHUNKS[chunk])
    px, got = gpu_ray_grads(run)
    check(run, got, px, label=" chunks of %d" % _CHUNKS[chunk])
    inv = _errors(got, one)
    print("  against one chunk: %s" % {k: "%.2e" % v for k, v in inv.items()})
    assert max(inv.values()) <= LAYOUT_BOUND, inv


@gpu
def test_ray_grads_past_one_chunk_per_image(monkeypatch):
    """B = 1, 160² rays x 24 flat: 614,400 points in the pass, more than CHUNK_POINTS = 2^19, so _add_points splits the
    image into point chunks with the library's own constant."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    assert 160 * 160 * 24 > backward.CHUNK_POINTS
    run = run_case("B-160-flat", "exact", {}, case=RayCase("B", 1, 160, 24, False, _RELU_NOISE))
    px, got = gpu_ray_grads(run)
    check(run, got, px)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the deterministic flag
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_deterministic_gradients_meet_the_fp64_bounds(tmp_path):
    """One child process in which torch.use_deterministic_algorithms(True) is on while the library renders and
    differentiates (tests/_fp64_det_child.py) runs the cfg2 B cases
    of part 3 (hierarchical and flat, exact) and test_gpu_fp64_train_grads.py's cfg2 camera render (B, fast): the ray
    gradients, d film and every parameter gradient (the grid included) meet the bounds they meet with the flag off."""
    from test_gpu_fp64_reference import _grad_errors
    from test_gpu_fp64_train_grads import bound_of as train_bound
    child = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_fp64_det_child.py")
    path = str(tmp_path / "det.pt")
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [child, path]
    subprocess.run(cmd, check=True, env=env, timeout=900)
    out = torch.load(path)
    assert out["deterministic"]
    for name in ("B-cfg2-hier", "B-cfg2-flat"):
        r = out["rays/" + name]
        errs = _errors(r["got"], r["want"], r["skip"])
        print("deterministic ray grads %s: %s" % (name, {k: "%.2e" % v for k, v in errs.items()}))
        assert set(errs) == ({"points", "dirs"} if name.endswith("hier") else {"points", "dirs", "z_vals"})
        assert max(errs.values()) <= RAY_BOUND["exact"], errs
    t = out["train"]
    assert "spatial_embeddings" in t["want"], sorted(t["want"])
    errs = _grad_errors(t["d_film"], {k: t["grads"][k] for k in t["want"]}, t["want_film"], t["want"])
    worst = max(errs, key=errs.get)
    print("deterministic train grads cfg2-B-fast: worst %s %.3g" % (worst, errs[worst]))
    assert errs[worst] <= train_bound("fast"), {k: "%.2e" % v for k, v in errs.items() if v > train_bound("fast")}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the float64 ray chain against autograd of a direct float64 forward
# ---------------------------------------------------------------------------------------------------------------------
def _direct_pixels(siren64, film64, leaves, st, slots, case, opt, noise):
    """The render as one float64 function of the ray leaves: the coarse field on the points and directions, the fine
    field on the fine points with the directions gathered at `slots` (or the per-ray ones, or (0, 0, -1)), composited
    ray-major on the coarse depths (a leaf when flat).  -> (pixels, raw_c, raw_f)."""
    b, n, s = leaves["points"].shape[:3]
    dirs = leaves["dirs"] if leaves["dirs"].dim() == 4 else leaves["dirs"].unsqueeze(2).expand(b, n, s, 3)
    raw_c = oracle.field_eval(siren64, leaves["points"].reshape(b, -1, 3), film64, dirs.reshape(b, -1, 3)).reshape(b, n, s, -1)
    raw_f = None
    if case.hier:
        if case.lock:
            dirs_f = torch.zeros_like(dirs.detach())
            dirs_f[..., 2] = -1
        elif leaves["dirs"].dim() == 4:
            dirs_f = torch.gather(dirs, 2, slots.unsqueeze(-1).expand(-1, -1, -1, 3))
        else:
            dirs_f = dirs
        raw_f = oracle.field_eval(siren64, st["points_f"].reshape(b, -1, 3), film64, dirs_f.reshape(b, -1, 3)).reshape(b, n, s, -1)
    z = leaves["z_vals"] if not case.hier else leaves["z_vals"].detach().float()
    return composite_ref(raw_c, z, raw_f, st["z_f"], noise, opt, ray_major=True), raw_c, raw_f


@pytest.mark.parametrize("variant", ["per_sample", "per_ray", "lock", "flat"])
def test_ray_chain_matches_autograd_of_the_direct_forward(variant):
    """ray_chain_vjp (the composite VJP, the fine directions' slot gather and its scatter-add adjoint, the per-ray sum,
    the fine pass dropped under lock, the depth leaf of a flat render) equals float64 autograd of the render written as
    one function of the ray leaves, on 2 images x 3 rays x 5 samples of model B with random slot permutations."""
    hier = variant != "flat"
    case = RayCase("B", 2, 1, 5, hier, _RELU_NOISE, dirs="ray" if variant in ("per_ray", "lock") else "sample",
                   lock=variant == "lock")
    opt = _opt(**dict(case.opt))
    siren = _field("B", "cpu")
    siren64 = copy.deepcopy(siren).double()
    for p in siren64.parameters():
        p.requires_grad_(False)
    film = _film(siren, 2, 7)
    g = torch.Generator().manual_seed(8)
    b, n, s = 2, 3, 5
    org = torch.randn(b, n, 3, generator=g, dtype=torch.float64) * 0.01
    ray_dirs = F.normalize(torch.randn(b, n, 3, generator=g, dtype=torch.float64) * 0.1 + torch.tensor([0., 0., -1.]), dim=-1)
    z = torch.sort(0.88 + 0.24 * torch.rand(b, n, s, generator=g), -1)[0]
    pts = (org.unsqueeze(2) + ray_dirs.unsqueeze(2) * z.double().unsqueeze(-1)) * 0.2
    dirs = F.normalize(ray_dirs.unsqueeze(2) + 0.3 * torch.randn(b, n, s, 3, generator=g, dtype=torch.float64), dim=-1) \
        if case.dirs == "sample" else ray_dirs
    z_f = torch.sort(0.88 + 0.24 * torch.rand(b, n, s, generator=g), -1)[0] if hier else None
    st = dict(z_f=z_f, points_f=(org.unsqueeze(2) + ray_dirs.unsqueeze(2) * z_f.double().unsqueeze(-1)) * 0.2 if hier else None)
    slots = torch.argsort(torch.rand(b, n, s, generator=g), -1) if case.dirs == "sample" and hier else None
    noise = torch.randn(b, n, 2 * s if hier else s, generator=g)
    d_pixels = torch.randn(b, n, siren.field_spec().out_dim - 1, generator=g, dtype=torch.float64)
    leaves = dict(points=pts.requires_grad_(True), dirs=dirs.requires_grad_(True), z_vals=z.double().requires_grad_(True))
    px, raw_c, raw_f = _direct_pixels(siren64, film.double(), leaves, st, slots, case, opt, noise)
    keys = ["points", "dirs"] + ([] if hier else ["z_vals"])
    want = dict(zip(keys, torch.autograd.grad((px * d_pixels).sum(), [leaves[k] for k in keys])))
    st.update(raw_c=raw_c.detach(), raw_f=raw_f.detach() if hier else None)
    rays = dict(points=pts.detach(), dirs=dirs.detach(), z_vals=z)
    got = ray_chain_vjp(siren, film, st, rays, slots, case, opt, noise, d_pixels)
    assert (got["z_vals"] is None) == hier
    for k in keys:
        err = _rel(got[k], want[k])
        assert err <= 1e-10, (k, err)
