"""point_forward(..., ray_grad=True): gradients w.r.t. the caller's sample points, directions and depths.

What the reference differentiates (generators/generators.py:800-856): the coarse points (the fine ones are built under
no_grad from the per-ray origins and directions, which therefore get none), the per-sample directions of both passes
(fine sample k of sample_pdf's order reads direction slot k; the fine pass adds nothing under lock_view_dependence), and
z_vals only without hierarchical sampling.

CPU: the grid coordinate gradient restated (the formula of csrc/ray_grads.cu) against grid_sample's float64 autograd;
the float64 restatement of the chain (tests/_ray_grads.py) against the reference's goldens
(tests/golden/make_ray_grad_goldens.py), values and which tensors get None; the fault rows both comparisons catch; the
keyword's refusals.  GPU: the goldens in every precision each field's rays-in backward serves; the single-latent fields
(grid in the trunk, 129 channels) against the restatement; a production shape on a ray subset; a learnable camera yaw;
the keyword adds outputs only (the other gradients bit for bit under the deterministic flag), reproducibly across
processes; per-ray directions given as an expand() get the per-sample gradients' per-ray sum.
"""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
import _point_forward as pf
import _ray_grads as rg
from fenerf_b200 import _lib, backward, ops
from fenerf_b200.generators import volumetric_rendering as vr
from oracle import render_oracle as oracle

gpu = pytest.mark.gpu
DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the grid coordinate gradient
# ---------------------------------------------------------------------------------------------------------------------
def grid_coord_grad_ref(grid, x, d_feat, fault=None):
    """d feat . d feat / d x of grid_sample(align_corners=True, zeros) at x (P, 3), grid (1, G, D, H, W), d_feat (P, G):
    the 8 corners' features dotted with d feat, the other two axes' weights, the per-axis sign and (R - 1) / 2 (what
    grid_coord_grad_kernel computes).  fault: 'swap_axes' reads x -> D and z -> W, 'no_half' drops (R - 1) / 2,
    'align_false' takes align_corners=False's coordinate map and factor R / 2."""
    g = grid[0].permute(1, 2, 3, 0)                                   # (D, H, W, G)
    R = g.shape[0]
    xs = x.flip(-1) if fault == "swap_axes" else x
    if fault == "align_false":
        i = ((xs + 1) * R - 1) / 2
        half = R / 2
    else:
        i = (xs + 1) / 2 * (R - 1)
        half = 1.0 if fault == "no_half" else (R - 1) / 2
    i0 = torch.floor(i)
    w1 = i - i0
    w = torch.stack([1 - w1, w1], -1)                                  # (P, 3, 2)
    out = torch.zeros_like(x)
    for k in range(8):
        e = [k & 1, (k >> 1) & 1, k >> 2]
        idx = i0.long() + torch.tensor(e)
        inside = ((idx >= 0) & (idx < R)).all(-1)
        ic = idx.clamp(0, R - 1)
        feat = g[ic[:, 2], ic[:, 1], ic[:, 0]] * inside.unsqueeze(-1)
        dot = (feat * d_feat).sum(-1)
        wa = [w[:, a, e[a]] for a in range(3)]
        for a in range(3):
            others = [wa[b] for b in range(3) if b != a]
            out[:, a] += (1.0 if e[a] else -1.0) * others[0] * others[1] * dot
    out = out * half
    return out.flip(-1) if fault == "swap_axes" else out


def _grid_case(seed=0, R=9, G=32, P=4000):
    g = torch.Generator().manual_seed(seed)
    grid = torch.randn((1, G, R, R, R), generator=g, dtype=torch.float64)
    x = (torch.rand((P, 3), generator=g, dtype=torch.float64) * 2.4 - 1.2)     # some points outside the grid
    d_feat = torch.randn((P, G), generator=g, dtype=torch.float64)
    return grid, x, d_feat


def _grid_sample_grad(grid, x, d_feat, align_corners=True):
    x = x.clone().requires_grad_(True)
    feat = F.grid_sample(grid, x.reshape(1, 1, 1, -1, 3), mode='bilinear', padding_mode='zeros',
                         align_corners=align_corners).reshape(grid.shape[1], -1).t()
    (feat * d_feat).sum().backward()
    return x.grad


GRID_BOUND = 1e-12


def test_grid_coord_grad_restatement_matches_grid_sample_autograd():
    grid, x, d_feat = _grid_case()
    want = _grid_sample_grad(grid, x, d_feat)
    err = (grid_coord_grad_ref(grid, x, d_feat) - want).abs().max().item() / want.abs().max().item()
    assert err <= GRID_BOUND, err


@pytest.mark.parametrize("fault", ["swap_axes", "no_half", "align_false"])
def test_the_grid_comparison_catches(fault):
    grid, x, d_feat = _grid_case()
    want = _grid_sample_grad(grid, x, d_feat)
    err = (grid_coord_grad_ref(grid, x, d_feat, fault=fault) - want).abs().max().item() / want.abs().max().item()
    assert err > 5 * GRID_BOUND, err


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the keyword's refusals
# ---------------------------------------------------------------------------------------------------------------------
def _cpu_args(name="pf_b_hier", which=0):
    case = pf.CASE_BY_NAME[name]
    rays = pf.load_rays(case)
    args = [rays[k].clone() for k in ("points", "dirs", "origins", "ray_dirs", "z_vals")]
    args[which].requires_grad_(True)
    return case, args, _cases.make_latents(pf.base_case(case))


def test_ray_grad_on_a_cpu_generator_is_cuda_only():
    case, args, z = _cpu_args()
    gen = _cases.build_mirror(pf.base_case(case), "cpu")
    with pytest.raises(RuntimeError, match="CUDA only"):
        gen.point_forward(*args, *z, ray_grad=True, **pf.call_kwargs(case))


def test_the_refusal_names_the_keyword():
    case, args, z = _cpu_args(which=4)
    gen = _cases.build_mirror(pf.base_case(case), "cpu")
    with pytest.raises(RuntimeError, match="not built.*ray_grad=True"):
        gen.point_forward(*args, *z, **pf.call_kwargs(case))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the reference's goldens
# ---------------------------------------------------------------------------------------------------------------------
#: max |restatement - reference| / max |reference| per ray tensor.  The reference runs in fp32; P's first colour layer
#: (U(+-1/3) weights at f ~ 30) amplifies its rounding (measured: 1.7e-3 for P, at most 3.8e-5 for the others)
CHAIN_BOUND = 5e-5
CHAIN_BOUND_P = 3e-3


def _chain_bound(name):
    return CHAIN_BOUND_P if rg.CASES[name][0].model == "P" else CHAIN_BOUND


@pytest.mark.parametrize("name", sorted(rg.CASES))
def test_restatement_matches_the_reference_golden(name):
    rays, gold, g = rg.load_golden(name)
    got = rg.chain_grads(name, "cpu", rays=rays)
    for k in rg.RAY_KEYS:
        assert (got[k] is None) == bool(g.get("none_" + k, False)) == (gold[k] is None), k
        if gold[k] is not None:
            err = rg.rel(got[k], gold[k])
            assert err <= _chain_bound(name), (k, err)


@pytest.mark.parametrize("fault,key", [("sorted_dirs", "dirs"), ("no_grid_term", "points"), ("no_box_warp", "points")])
def test_the_golden_comparison_catches(fault, key):
    """Fine directions in depth order instead of the draw order, the grid lookup's coordinate term dropped, the box-warp
    scale left out of the points' gradient: each moves the restatement past 5x its bound (model B's random-init grid
    carries 7 % of the points' gradient, no scaling needed)."""
    rays, gold, _ = rg.load_golden("pf_b_vardirs")
    got = rg.chain_grads("pf_b_vardirs", "cpu", rays=rays, fault=fault)
    assert rg.rel(got[key], gold[key]) > 5 * CHAIN_BOUND


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _gpu_call(name, call, latents, run, precision, ray_grad=True, **extra):
    """point_forward on the GPU (backward.render_rays_with_grad with point_forward's set-up for the single-latent
    generators, which have no point_forward)."""
    case, _ = {**rg.CASES, **rg.EXTRA_CASES}[name]
    gen = _cases.build_mirror(rg.base_case(case), DEV)
    rng = vr.ReplayRng(run["draws"], DEV)
    kw = dict(pf.call_kwargs(case), precision=precision, **extra)
    if hasattr(gen, "point_forward"):
        return gen.point_forward(call["points"], call["dirs"], call["origins"], call["ray_dirs"], call["z_vals"], *latents,
                                 _rng=rng, **({"ray_grad": True} if ray_grad else {}), **kw)
    b, n, s = call["points"].shape[:3]
    hier = kw["hierarchical_sample"]
    noise_c = rng.randn(b, n, s, 1) if hier else None
    u = rng.rand(b * n, s) if hier else None
    noise_f = rng.randn(b, n, 2 * s if hier else s, 1)
    rd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=s, hierarchical=hier, clamp_mode=kw["clamp_mode"],
                            nerf_noise=kw["nerf_noise"], precision=precision)
    film = gen.siren.film_from_latents(*latents)
    return backward.render_rays_with_grad(gen.siren, rd, film, call["points"], call["dirs"], call["origins"],
                                          call["ray_dirs"], call["z_vals"], noise_c, u, noise_f,
                                          grad_precision=extra.get("grad_precision"), ray_grad=ray_grad)


def _gpu_grads(name, rays, precision, weights=None, **extra):
    case, _ = {**rg.CASES, **rg.EXTRA_CASES}[name]
    run = rg.oracle_run(case, {k: v.contiguous() for k, v in rays.items()})
    leaves, call = rg.leaf_rays(rays, device=DEV)
    latents = [z.to(DEV) for z in run["latents"]]
    px = _gpu_call(name, call, latents, run, precision, **extra)
    w = _cases.loss_weights(px.shape) if weights is None else weights
    (px * w.to(DEV)).sum().backward()
    return {k: leaves[k].grad for k in rg.RAY_KEYS}


def _kink_or_face_rows(name, rays, tau=2e-3):
    """Coarse samples whose density (+ noise) lies within tau max|sigma| of the relu kink, or whose grid coordinate lies
    within 1e-5 cells of a cell face: the rows of d points (and d z) the fp16 streams may put on the other side."""
    case, _ = rg.CASES[name]
    gen = _cases.build_mirror(rg.base_case(case), "cpu")
    run = rg.oracle_run(case, {k: v.contiguous() for k, v in rays.items()})
    b, n, s = rays["points"].shape[:3]
    raw = run["out"]["stages"]["raw_coarse"]
    sig = raw[..., -1]
    if case.cfg["nerf_noise"] and case.cfg["clamp_mode"] == "relu" and not case.hierarchical:
        sig = sig + run["draws"][-1][1][..., 0] * case.cfg["nerf_noise"]
    kink = (sig.abs() <= tau * sig.abs().max()) if case.cfg["clamp_mode"] == "relu" else torch.zeros_like(sig, dtype=torch.bool)
    spec = gen.siren.field_spec()
    face = torch.zeros_like(kink)
    if spec.grid_channels:
        i = (rays["points"].double() * spec.input_scale + 1) / 2 * (spec.grid_res - 1)
        face = ((i - i.round()).abs() < 1e-5).any(-1)
    return kink | face


#: the precisions each field's rays-in backward serves (bridges: no split forward; P: exact and split only)
def _precisions(model):
    modes = [("exact", {}), ("guard", {}), ("split", {}), ("split", {"grad_precision": "split"})]
    if model in "MN":
        return modes[:2]
    if model == "P":
        return [modes[0], modes[2], modes[3]]
    return modes


GOLDEN_RUNS = [(n, p, e) for n, (c, _) in sorted(rg.CASES.items()) for p, e in _precisions(c.model)]
#: max |gpu - reference| / max |reference| per ray tensor, measured on an H100 80GB HBM3 (700 W): exact / split at most
#: 6.4e-5 (D's points); guard, with the kink and cell-face rows excluded (at most KINK_SHARE of them), at most 1.3e-2
#: except pf_b_vardirs' points, 3.9e-2 at one sample that is neither (the fp16 gradient streams)
BOUNDS = {"exact": 1e-4, "split": 1e-4, "guard": 5e-2}
BOUNDS_P = {"exact": 4e-3, "split": 4e-3}
KINK_SHARE = 0.05


@gpu
@pytest.mark.parametrize("name,precision,extra", GOLDEN_RUNS, ids=["%s-%s%s" % (n, p, "-gs" if e else "") for n, p, e in GOLDEN_RUNS])
def test_goldens(name, precision, extra):
    rays, gold, _ = rg.load_golden(name)
    got = _gpu_grads(name, rays, precision, **extra)
    bound = (BOUNDS_P if rg.CASES[name][0].model == "P" else BOUNDS)[precision]
    skip = _kink_or_face_rows(name, rays) if precision == "guard" else None
    if skip is not None:
        assert skip.float().mean().item() <= KINK_SHARE
    for k in rg.RAY_KEYS:
        assert (got[k] is None) == (gold[k] is None), (k, got[k] is None)
        if gold[k] is None:
            continue
        g, w = got[k].cpu().double(), gold[k].double()
        if skip is not None and k in ("points", "z_vals"):
            keep = ~skip.reshape(g.shape[:3])
            g, w = g[keep], w[keep]
        err = rg.rel(g, w)
        worst = (g - w).abs().reshape(-1, g.shape[-1]).amax(-1).argmax().item()
        print("%s %s%s %s: rel err %.2e%s, worst row %d" % (name, precision, "+gs" if extra else "", k, err,
              "" if skip is None else " (%d kink / face rows excluded)" % skip.sum().item(), worst))
        assert err <= bound, (k, err)


@gpu
@pytest.mark.parametrize("name", sorted(rg.EXTRA_CASES))
@pytest.mark.parametrize("precision", ["exact", "guard"])
def test_single_latent_fields_match_the_restatement(name, precision):
    """The grid in the trunk (L: layer 0's feature columns) and a 129-channel field without hierarchical sampling (K:
    the wide compositing body's depth gradient), through render_rays_with_grad."""
    rays = rg.make_rays(name)
    got = _gpu_grads(name, rays, precision)
    want = rg.chain_grads(name, DEV, rays=rays)
    for k in rg.RAY_KEYS:
        assert (got[k] is None) == (want[k] is None), k
        if want[k] is not None:
            err = rg.rel(got[k], want[k])
            print("%s %s %s: rel err %.2e" % (name, precision, k, err))
            assert err <= (5e-2 if precision == "guard" else 1e-4), (k, err)


@gpu
def test_the_gpu_comparison_catches_depth_ordered_fine_directions():
    rays, gold, _ = rg.load_golden("pf_b_vardirs")
    got = _gpu_grads("pf_b_vardirs", rays, "exact")
    want = rg.chain_grads("pf_b_vardirs", DEV, rays=rays, fault="sorted_dirs")
    assert rg.rel(got["dirs"], want["dirs"]) > 5 * BOUNDS["exact"]


@gpu
@pytest.mark.parametrize("name", ["pf_b_vardirs", "pf_b_nohier_lastback"])
def test_ray_grad_only_adds_outputs(name):
    """Under torch.use_deterministic_algorithms the film / parameter gradients and the pixels with ray_grad=True are
    bit for bit those of the same call without it; without the keyword none of the new kernels runs."""
    case = pf.CASE_BY_NAME[name]
    run = pf.oracle_run(case)
    out = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for with_rg in (False, True):
            gen = _cases.build_mirror(pf.base_case(case), DEV)
            r = {k: v.to(DEV).clone().requires_grad_(with_rg) for k, v in run["rays"].items()}
            latents = [z.to(DEV).requires_grad_(True) for z in run["latents"]]
            l0 = _lib.launch_count()
            px = gen.point_forward(r["points"], r["dirs"], r["origins"], r["ray_dirs"], r["z_vals"], *latents,
                                   **dict(pf.call_kwargs(case), precision="guard", _rng=vr.ReplayRng(run["draws"], DEV),
                                          **({"ray_grad": True} if with_rg else {})))
            (px * _cases.loss_weights(px.shape).to(DEV)).sum().backward()
            torch.cuda.synchronize()
            launches = _lib.launch_count() - l0
            grads = [z.grad for z in latents] + [p.grad for p in gen.parameters() if p.grad is not None]
            out.append((px.detach(), grads, launches))
    finally:
        torch.use_deterministic_algorithms(prev)
    (px0, g0, n0), (px1, g1, n1) = out
    assert torch.equal(px0, px1)
    assert len(g0) == len(g1) and all(torch.equal(a, b) for a, b in zip(g0, g1))
    assert n1 > n0


@gpu
def test_expanded_directions_get_the_per_ray_sum():
    """Per-ray directions given as an expand() and the same values given per sample: the expand's gradient is the
    per-sample gradient summed over S."""
    rays, _, _ = rg.load_golden("rg_b_expand")
    got_expand = _gpu_grads("rg_b_expand", rays, "exact")
    got_sample = _gpu_grads("rg_b_expand", dict(rays, dirs=rays["dirs"].contiguous()), "exact")
    want = got_sample["dirs"].sum(2)
    assert (got_expand["dirs"] - want).abs().max().item() <= 1e-5 * want.abs().max().item()
    assert rg.rel(got_expand["points"], got_sample["points"]) <= 1e-5


@gpu
def test_ray_grads_are_reproducible_across_processes(tmp_path):
    """Two fresh processes under torch.use_deterministic_algorithms(True) give bitwise-equal ray gradients."""
    child = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ray_grad_det_child.py")
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    outs = []
    for i in range(2):
        path = str(tmp_path / ("run%d.pt" % i))
        subprocess.run([sys.executable, child, path], check=True, env=env, timeout=900)
        outs.append(torch.load(path))
    assert outs[0].keys() == outs[1].keys() and len(outs[0]) > 0
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


def _yaw_rays(rays, yaw):
    c, s = torch.cos(yaw), torch.sin(yaw)
    zero, one = torch.zeros_like(yaw), torch.ones_like(yaw)
    rot = torch.stack([torch.stack([c, zero, s]), torch.stack([zero, one, zero]), torch.stack([-s, zero, c])])
    return {k: (v if k == "z_vals" else v.to(yaw.dtype) @ rot.t()) for k, v in rays.items()}


@gpu
def test_a_learnable_yaw():
    """A camera yaw builds the rays with torch ops; its gradient through point_forward (exact) against the float64 chain."""
    name = "pf_b_vardirs"
    case, _ = rg.CASES[name]
    rays, _, _ = rg.load_golden(name)
    with torch.no_grad():
        rot = _yaw_rays(rays, torch.tensor(0.2))
    run = rg.oracle_run(case, {k: v.contiguous() for k, v in rot.items()})
    yaw = torch.tensor(0.2, device=DEV, requires_grad=True)
    call = _yaw_rays({k: v.to(DEV) for k, v in rays.items()}, yaw)
    px = _gpu_call(name, call, [z.to(DEV) for z in run["latents"]], run, "exact")
    (px * _cases.loss_weights(px.shape).to(DEV)).sum().backward()
    yaw64 = torch.tensor(0.2, device=DEV, dtype=torch.float64, requires_grad=True)
    px64 = rg.chain(case, run, _yaw_rays({k: v.to(DEV).double() for k, v in rays.items()}, yaw64), DEV)
    (px64 * _cases.loss_weights(px64.shape).to(DEV).double()).sum().backward()
    err = abs(yaw.grad.item() - yaw64.grad.item()) / abs(yaw64.grad.item())
    print("yaw grad %.6e vs float64 %.6e: rel err %.2e" % (yaw.grad.item(), yaw64.grad.item(), err))
    assert err <= 1e-4, err


class _ReplayDraws:
    """oracle-style draws replayed from given tensors, in order."""

    def __init__(self, tensors):
        self.t, self.log = list(tensors), []

    def _next(self, kind, shape):
        t = self.t.pop(0)
        assert tuple(t.shape) == tuple(shape), (kind, t.shape, shape)
        self.log.append((kind, t))
        return t

    def rand(self, *shape):
        return self._next("rand", shape)

    def randn(self, *shape):
        return self._next("randn", shape)


#: B = 4, 128^2 rays per image, 24 + 24 steps, directions varying along each ray, per-ray origins; the float64 chain on
#: the first and last 48 rays of every image (the last rays of the buffer included)
PROD = pf.PointCase("rg_prod", "B", 4, 421, img_size=128, num_steps=24, vary_dirs=0.3, origin_jitter=0.01, cfg=dict(rg._KW))


@gpu
@pytest.mark.parametrize("hier", [True, False])
def test_production_shape_on_a_ray_subset(hier):
    case = dataclasses.replace(PROD, hierarchical=hier)
    rays = pf.make_rays(case)
    b, n, s = rays["points"].shape[:3]
    g = torch.Generator().manual_seed(7)
    draws = [("randn", torch.randn((b, n, s, 1), generator=g)), ("rand", torch.rand((b * n, s), generator=g))] if hier else []
    draws.append(("randn", torch.randn((b, n, 2 * s if hier else s, 1), generator=g)))
    idx = torch.cat([torch.arange(48), torch.arange(n - 48, n)])
    gen = _cases.build_mirror(pf.base_case(case), "cpu")
    latents = _cases.make_latents(pf.base_case(case))
    film = oracle.film_from_latents(gen.siren, latents)
    sub = {k: v[:, idx].contiguous() for k, v in rays.items()}
    sub_draws = [(k, t[:, idx] if t.shape[0] == b else t.reshape(b, n, s)[:, idx].reshape(-1, s)) for k, t in draws]
    out = pf.restate_point_forward(gen.siren, film, sub["points"], sub["dirs"], sub["origins"], sub["ray_dirs"],
                                   sub["z_vals"], pf.oracle_cfg(case), draws=_ReplayDraws([t for _, t in sub_draws]))
    run = dict(film=film, draws=sub_draws, out=out, latents=latents)
    w_full = torch.zeros((b, n, 21))
    w_full[:, idx] = _cases.loss_weights((b, len(idx), 21))
    leaves, call = rg.leaf_rays(rays, device=DEV)
    gpu_gen = _cases.build_mirror(pf.base_case(case), DEV)
    px = gpu_gen.point_forward(call["points"], call["dirs"], call["origins"], call["ray_dirs"], call["z_vals"],
                               *[z.to(DEV) for z in latents], **dict(pf.call_kwargs(case), precision="exact",
                                                                    _rng=vr.ReplayRng(draws, DEV), ray_grad=True))
    (px * w_full.to(DEV)).sum().backward()
    leaves64, call64 = rg.leaf_rays(sub, torch.float64, DEV)
    px64 = rg.chain(case, run, call64, DEV)
    (px64 * w_full[:, idx].to(DEV).double()).sum().backward()
    rest = torch.ones(n, dtype=torch.bool)
    rest[idx] = False
    for k in rg.RAY_KEYS:
        want = leaves64[k].grad
        assert (leaves[k].grad is None) == (want is None), k
        if want is None:
            continue
        got = leaves[k].grad
        assert torch.count_nonzero(got[:, rest.to(DEV)]).item() == 0, k      # rays outside the subset carry no gradient
        err = rg.rel(got[:, idx.to(DEV)], want)
        print("production %s %s: rel err %.2e" % ("hier" if hier else "nohier", k, err))
        # hierarchical: the fine depths are the CPU oracle's fp32 sample_pdf on its own coarse outputs, the kernel's on its
        # own; their last-bit differences move the fine samples, which shade the coarse ones behind them
        assert err <= (1e-3 if hier else 1e-4), (k, err)
