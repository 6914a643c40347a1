"""Parity of the CUDA path with the CPU oracle (and, through it, with the reference).  -m gpu.

Every comparison replays the oracle's recorded RNG draws into the CUDA path and goes through the
C-ABI (ctypes, fenerf_b200/ops.py) -- stage by stage first, then end to end through the generator
class API, then against the reference's committed golden outputs.

Tolerances (fp32; BASELINE.json north_star: 1e-3 max-abs on pixels, indices exact):
  ray set-up 2e-6 | field EXACT 5e-5 | resample depths 2e-5 / inds >= 99.9 % identical on the
  well-conditioned (opaque) fixture, 5e-4 / 99 % on the near-empty one (see the test) | compositing 2e-5 | end-to-end pixels 1e-3 (EXACT mode: 2e-4).
The reference's last compositing interval is 1e10 wide, so a pixel is a step function of
sign(sigma_far): rays whose oracle |sigma_far| is below ILL_TAU are ill-conditioned for ANY fp32
implementation (an ulp of summation order flips them) and are excluded, with their count bounded.
"""
import copy
import functools
import gc
import os
import weakref

import numpy as np
import pytest
import torch

import _cases
import _harness
from _fp64 import _film, _rel, _siren
from _harness import DEV, runs  # noqa: F401  (runs: the module's oracle-run fixture)
from _harness import cuda as _cuda
from fenerf_b200 import _lib, ops
from fenerf_b200.generators.volumetric_rendering import ReplayRng
from fenerf_b200.siren import siren as siren_mod

pytestmark = pytest.mark.gpu


def _desc(case, precision="exact", staged=False):
    c = case.cfg
    return ops.make_render_desc(
        batch=case.batch, img_size=c["img_size"], num_steps=c["num_steps"], hierarchical=c["hierarchical_sample"],
        clamp_mode=c["clamp_mode"], nerf_noise=c["nerf_noise"], fov=c["fov"], last_back=c.get("last_back", False),
        white_back=c.get("white_back", False), black_back=c.get("black_back", False),
        fill_mode=c.get("fill_mode") if staged else None, fill_color=c.get("fill_color", "black"),
        lock_view_dependence=c.get("lock_view_dependence", False), precision=precision)


def test_library_loads_and_counts_launches():
    lib = _lib.lib()
    assert lib.fenerf_abi_version() == _lib.ABI_VERSION
    assert _lib.launch_count() >= 0


@pytest.mark.parametrize("name", ["a_small", "a_lockview_uniform", "b_small"])
def test_ray_setup_stage(runs, name):
    case, run = runs(name)
    st = run["out"]["stages"]
    from fenerf_b200.generators import volumetric_rendering as vr
    c = case.cfg
    x_lin, y_lin, z_lin = vr.ray_tables(c["img_size"], c["num_steps"], c["ray_start"], c["ray_end"], DEV)
    rd = _desc(case)
    pts, z, dirs, org = ops.ray_setup(rd, x_lin, y_lin, z_lin, _cuda(st["cam2world"]), _cuda(run["draws"][0][1]))
    assert (pts.cpu() - st["points_coarse"]).abs().max() <= 2e-6
    assert (z.cpu() - st["z_coarse"]).abs().max() <= 2e-6
    assert (dirs.cpu() - st["dirs"]).abs().max() <= 2e-6
    assert (org.cpu() - st["origins"]).abs().max() <= 2e-6


@pytest.mark.parametrize("name", ["a_small", "b_small", "b_small_opaque", "c_small", "d_small"])
def test_field_exact_stage(runs, name):
    case, run = runs(name)
    st = run["out"]["stages"]
    gen = _cases.build_mirror(case, DEV)
    b, n, s = case.batch, case.cfg["img_size"] ** 2, case.cfg["num_steps"]
    with torch.no_grad():
        raw = ops.siren_points(gen.siren, _cuda(st["points_coarse"].reshape(b, n * s, 3)), _cuda(run["film"]),
                               _cuda(st["dirs"]), precision="exact")
    err = (raw.cpu().reshape(b, n, s, -1) - st["raw_coarse"]).abs()
    assert err.max() <= 5e-5, "max|field - oracle| = %g (per channel %s)" % (err.max(), err.amax((0, 1, 2)))


@pytest.mark.parametrize("name", ["a_small", "b_small", "b_small_opaque", "c_small", "d_small"])
def test_field_fast_stage(runs, name):
    """wgmma path vs oracle on the raw field outputs: fp16 operand rounding through 9-11 FiLM
    layers (gain ~1 per layer) stays at the few-1e-4 level (SURVEY.md section 7, hard part 1)."""
    case, run = runs(name)
    st = run["out"]["stages"]
    gen = _cases.build_mirror(case, DEV)
    b, n, s = case.batch, case.cfg["img_size"] ** 2, case.cfg["num_steps"]
    with torch.no_grad():
        raw = ops.siren_points(gen.siren, _cuda(st["points_coarse"].reshape(b, n * s, 3)), _cuda(run["film"]),
                               _cuda(st["dirs"]), precision="fast")
    err = (raw.cpu().reshape(b, n, s, -1) - st["raw_coarse"]).abs()
    assert err.max() <= 3e-3, "max|fast field - oracle| = %g (per channel %s)" % (err.max(), err.amax((0, 1, 2)))


#: one parity case per field class A-H (E: e_staged_debug's 23-channel D)
FIELD_CASES = ["a_small", "b_small", "c_small", "d_small", "e_staged_debug", "f_small", "g_small", "h_small"]


def _tile_test_inputs(n_points, seed):
    """(batch, points per image, how directions are passed) of a point count or of a named _cases.TILE_LAYOUTS schedule.
    The named schedules pass one direction per 24-sample ray, or one locked (0, 0, -1) per image, in turn."""
    if isinstance(n_points, int):
        return 2, n_points, "per_point"
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    mode = ("per_point", "dir_group24", "lock_dirs")[seed % 3]
    batch, ppb = _cases.tile_layout(n_points, sms, 24 if mode == "dir_group24" else 1)
    return batch, ppb, mode


def _tile_test_dirs(batch, ppb, mode, g):
    n = {"per_point": ppb, "dir_group24": ppb // 24, "lock_dirs": 1}[mode]
    dirs = torch.nn.functional.normalize(torch.randn(batch, n, 3, device=DEV, generator=g), dim=-1)
    if mode == "lock_dirs":
        dirs = torch.zeros_like(dirs)
        dirs[..., 2] = -1
    return dirs


@pytest.mark.parametrize("model", FIELD_CASES)
@pytest.mark.parametrize("n_points", [1, 127, 128, 129, 256, 389] + list(_cases.TILE_LAYOUTS))
def test_field_fast_tile_counts_against_the_fp32_path(model, n_points):
    """One tile, a lone odd tile, a ragged last tile, and the persistent schedules of the device's own SM count (one pair
    per CTA, a lone tile in a second pair, two pairs per CTA, pairs across image borders): the wgmma kernel against the
    fp32 path of the same library on the same points, and the density-only entry against the full evaluation.  (Round 2
    found that results depended on how the issuer warps' lanes left their barrier waits once the issue instructions
    became warp-level: a single tile was enough to show it.)"""
    case = _cases.CASE_BY_NAME[model]
    gen = _cases.build_mirror(case, DEV)
    seed = n_points if isinstance(n_points, int) else _cases.TILE_LAYOUTS.index(n_points) + FIELD_CASES.index(model)
    batch, ppb, mode = _tile_test_inputs(n_points, seed)
    g = torch.Generator(device=DEV).manual_seed(seed)
    pts = (torch.rand(batch, ppb, 3, device=DEV, generator=g) - 0.5) * 0.3
    dirs = _tile_test_dirs(batch, ppb, mode, g)
    zs = [torch.randn(batch, 256, device=DEV, generator=g) for _ in range(_cases.n_latents(case.model))]
    with torch.no_grad():
        film = gen.siren.film_from_latents(*zs)
        fast = ops.siren_points(gen.siren, pts, film, dirs, precision="fast")
        again = ops.siren_points(gen.siren, pts, film, dirs, precision="fast")
        exact = ops.siren_points(gen.siren, pts, film, dirs, precision="exact")
        sigma = ops.siren_sigma(gen.siren, pts, film, precision="fast")
    assert torch.equal(fast, again), "two launches on the same inputs differ"
    assert torch.equal(sigma, fast[..., -1:]), "the density-only entry differs from the full evaluation"
    err = (fast - exact).abs().amax((0, 1))
    assert torch.isfinite(fast).all() and err.max() <= 5e-3, "max|fast - exact| per channel %s (%s)" % (err, mode)


def _oracle_cdf(st, s):
    """The CDF sample_pdf searches (volumetric_rendering.py:273-277), from the oracle's coarse weights with the
    same torch ops on the same host, i.e. bit-identical to what the oracle's searchsorted saw."""
    w = st["coarse_weights"][:, 1:-1] + 1e-5
    pdf = w / torch.sum(w, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    return torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)


@pytest.mark.parametrize("name,z_tol,inds_frac,tie_tol", [
    ("a_small_opaque", 2e-5, 0.999, 2e-6), ("b_small_opaque", 2e-5, 0.999, 2e-6), ("a_small", 5e-4, 0.99, 2e-4),
    ("a_small_noise", 5e-4, 0.99, 2e-4), ("b_small", 5e-4, 0.99, 2e-4), ("a_hier_softplus", 5e-4, 0.99, 2e-4),
    ("a_cfg2", 5e-4, 0.99, 2e-4)])
def test_resample_stage(runs, name, z_tol, inds_frac, tie_tol):
    """`inds` = searchsorted(cdf, u) is an integer function of floating-point inputs: it can only differ from
    the oracle's where u sits within the CDF's own rounding error of a CDF entry.  The test records the
    exact-match rate and PROVES every mismatch is such a near-tie: the two indices are adjacent and
    |u - cdf_oracle[edge between them]| <= tie_tol.  tie_tol is the conditioning of the reference's own fp32
    formula, not slack for the kernel: alpha = 1 - exp(-delta * sigma) cancels catastrophically for the
    sigma ~ 0.03 of a random-init field (alpha ~ 4e-4: one ulp of exp() is 1.4e-4 relative -- torch's
    vectorised CPU exp and CUDA's expf both stay within their 1-2 ulp but are not the same function), the
    opaque fixtures (alpha ~ 1e-2) pin it 100x tighter.  z_fine is continuous across such a flip."""
    case, run = runs(name)
    st = run["out"]["stages"]
    rd = _desc(case)
    s = case.cfg["num_steps"]
    noise = _cuda(run["draws"][3][1]) if case.cfg["nerf_noise"] else None
    u = run["draws"][4][1]
    z_f, pts_f, inds = ops.resample(rd, _cuda(st["raw_coarse"]), _cuda(st["z_coarse"]), _cuda(st["dirs"]),
                                    _cuda(st["origins"]), noise, _cuda(u), want_inds=True)
    got, want = inds.cpu(), st["inds"]
    same = (got == want)
    zerr = (z_f.cpu() - st["z_fine"]).abs().max().item()
    perr = (pts_f.cpu() - st["points_fine"]).abs().max().item()
    mism = ~same
    n_mis = int(mism.sum())
    worst_tie, adjacent = 0.0, True
    if n_mis:
        cdf = _oracle_cdf(st, s)
        edge = torch.minimum(got, want)[mism]                # the CDF entry the two answers disagree about
        rows = mism.nonzero()[:, 0]
        adjacent = bool(((got - want).abs()[mism] == 1).all())
        worst_tie = float((u[mism] - cdf[rows, edge]).abs().max())
    rate = float(same.float().mean())
    msg = "inds identical %.4f %% (%d of %d differ), worst |u - cdf_edge| %.3g, max|dz| %.3g, max|dp| %.3g" % (
        100 * rate, n_mis, got.numel(), worst_tie, zerr, perr)
    assert adjacent, msg
    assert worst_tie <= tie_tol, msg
    assert rate >= inds_frac, msg
    assert zerr <= z_tol, msg
    assert perr <= z_tol, msg


@pytest.mark.parametrize("name", ["a_lockview_uniform", "a_small", "a_cam_hybrid", "a_cam_hybrid2", "a_cam_truncgauss",
                                  "a_cam_spherical", "a_nohier_softplus"])
def test_camera_modes(runs, name):
    """camera_kernel (every sample_dist mode of volumetric_rendering.py:179-228) against the oracle's poses."""
    case, run = runs(name)
    c = case.cfg
    rng = ReplayRng(run["draws"][1:], DEV)            # the camera draws follow draw #1
    c2w, pitch, yaw = ops.camera_poses(case.batch, c.get("sample_dist"), c["h_stddev"], c["v_stddev"], c["h_mean"],
                                       c["v_mean"], rng, torch.device(DEV))
    st = run["out"]["stages"]
    assert (c2w.cpu() - st["cam2world"]).abs().max() <= 2e-6
    assert (torch.cat([pitch, yaw], -1).cpu() - run["out"]["poses"]).abs().max() <= 2e-6


@pytest.mark.parametrize("name", ["a_small", "a_small_noise", "a_small_opaque", "a_nohier_softplus",
                                  "a_lockview_uniform", "b_small"])
def test_composite_stage(runs, name):
    case, run = runs(name)
    st = run["out"]["stages"]
    rd = _desc(case)
    hier = case.cfg["hierarchical_sample"]
    noise = _cuda(run["draws"][-1][1]) if case.cfg["nerf_noise"] else None
    px, depth, wsum, weights, sidx = ops.composite(
        rd, _cuda(st["raw_coarse"]), _cuda(st["z_coarse"]), _cuda(st["raw_fine"]) if hier else None,
        _cuda(st["z_fine"]) if hier else None, noise, want_weights=True, want_sort_idx=True)
    if hier:
        assert torch.equal(sidx.cpu().long(), st["sort_order"].squeeze(-1)), "merge order differs"
    assert (weights.cpu() - st["weights"]).abs().max() <= 2e-6
    assert (wsum.cpu() - run["out"]["weights_sum"]).abs().max() <= 2e-5
    assert (depth.cpu() - run["out"]["depth"]).abs().max() <= 2e-5
    assert (px.cpu() - run["out"]["pixels"]).abs().max() <= 2e-5


def _serves(model, precision):
    return precision in _cases.model_data(model, "precisions")


@pytest.mark.parametrize("case", _cases.CASES, ids=lambda c: c.name)
def test_end_to_end_exact(runs, case):
    case, run = runs(case.name)
    gen, pixels, poses, depth_map = _harness.end_to_end(case, run, "exact")
    tol = _cases.bound(case.model, "render_exact")
    _harness.check_pixels(case, run, pixels, tol)
    if poses is not None:
        assert (poses - run["out"]["poses"]).abs().max() <= 1e-5
    if depth_map is not None:
        r = case.cfg["img_size"]
        assert (depth_map - run["out"]["depth"].reshape(case.batch, r, r)).abs().max() <= tol


@pytest.mark.parametrize("case", [c for c in _cases.CASES if _serves(c.model, "guard")], ids=lambda c: c.name)
def test_end_to_end_default_precision(runs, case):
    """The default (wgmma + guard refinement) mode against the north-star bound."""
    case, run = runs(case.name)
    gen, pixels, poses, depth_map = _harness.end_to_end(case, run, "guard")
    tol = _cases.bound(case.model, "render_guard")
    if case.probed:
        tol = max(tol, _cases.bound(case.model, "render_guard_cfg2_labels"))
    _harness.check_pixels(case, run, pixels, tol)


_GOLDEN_RUNS = [(c, p) for c in _cases.CASES for p in ("exact", "guard") if _serves(c.model, p)]


@pytest.mark.parametrize("case,precision", _GOLDEN_RUNS, ids=["%s-%s" % (c.name, p) for c, p in _GOLDEN_RUNS])
def test_against_reference_golden(runs, case, precision):
    """CUDA output vs the reference's own committed output (no oracle in between): every well-conditioned pixel, or the
    probe of a probed golden; the label channels of a probed case in the default mode within their own bound."""
    gold = np.load(_cases.golden_path(case))
    case, run = runs(case.name)       # only for the RNG draws, latents and the ill-conditioned mask
    l0 = _lib.launch_count()
    gen, pixels, poses, depth_map = _harness.end_to_end(case, run, precision)
    assert _lib.launch_count() > l0
    got, want, idx = _harness.golden_pixels(pixels, gold)
    err = (got - want).abs()
    ill_rays = _harness.ill_conditioned_pixels(case, run)
    assert int(ill_rays.sum()) <= max(2, 0.002 * ill_rays.numel())
    ill = ill_rays.unsqueeze(1).expand_as(pixels).reshape(-1)
    chan = torch.arange(pixels.numel()) // (pixels.shape[2] * pixels.shape[3]) % pixels.shape[1]
    if idx is not None:
        ill, chan = ill[idx], chan[idx]
    labels = chan < pixels.shape[1] - 3
    tol = _cases.bound(case.model, "render_" + precision)
    label_tol = _cases.bound(case.model, "render_guard_cfg2_labels") if (case.probed and precision == "guard") else tol
    print("%s %s: max err %.3g" % (case.name, precision, err[~ill].max()))
    assert err[~ill & ~labels].max() <= tol
    if labels.any():
        assert err[~ill & labels].max() <= label_tol
    if poses is not None:
        assert (poses - torch.from_numpy(gold["poses"])).abs().max() <= 1e-5
    if depth_map is not None:
        # depth = sum w_i z_i is not bounded by the north star; with fp16 densities it holds to ~1e-3 of the ray span
        assert (depth_map - torch.from_numpy(gold["depth_map"])).abs()[~ill_rays].max() <= 3e-3


def test_missing_clamp_mode_is_a_keyerror_and_bad_one_a_typeerror():
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(1, 256, device=DEV)
    kw = dict(case.cfg)
    kw.pop("clamp_mode")
    with torch.no_grad():
        with pytest.raises(KeyError):
            gen(z, **kw)
        with pytest.raises(TypeError):
            gen(z, **dict(case.cfg, clamp_mode="nope"))


def test_extra_curriculum_kwargs_are_swallowed_and_max_batch_size_ignored():
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(1, 256, device=DEV)
    with torch.no_grad():
        px, poses = gen(z, **case.cfg, batch_size=24, gen_lr=6e-5, dataset='CelebA', topk_v=0.6)
        px2, depth, third = gen.staged_forward(z, **case.cfg, max_batch_size=7)
    assert px.shape == (1, 3, 16, 16) and poses.shape == (1, 2)
    assert px2.shape == (1, 3, 16, 16) and depth.shape == (1, 16, 16) and not depth.is_cuda


_GRAD_RUNS = [(n, p) for n in _cases.GRAD_PARAMS for p in ("exact", "guard") if _serves(_cases.CASE_BY_NAME[n].model, p)]


@pytest.mark.parametrize("name,precision", _GRAD_RUNS, ids=["%s-%s" % r for r in _GRAD_RUNS])
def test_backward_matches_reference_gradients(runs, name, precision):
    """The differentiable call (train_double_latent_semantic.py:411-446) against the reference's own autograd:
    d sum(pixels * W) / d (latents, field weights, mapping networks, feature grid), stored by
    tests/golden/make_goldens.py --grads.  Backward = fenerf_b200/backward.py over the CUDA library."""
    import dataclasses
    case = _cases.CASE_BY_NAME[name]
    if case.method != "forward":
        # the gradient goldens come from forward() under manual_seed(case.seed): no avg-frequency draws first
        case = dataclasses.replace(case, method="forward", cfg={k: v for k, v in case.cfg.items() if k != "fill_mode"})
        run = _harness.oracle_run(case)
    else:
        case, run = runs(name)
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "grad_%s.npz" % name))
    gen = _cases.build_mirror(case, DEV)
    latents = [_cuda(z).requires_grad_(True) for z in run["latents"]]
    kw = {k: v for k, v in case.cfg.items() if k != "fill_mode"}
    l0 = _lib.launch_count()
    pixels, _ = gen(*latents, **dict(kw, _rng=ReplayRng(run["draws"], DEV), precision=precision))
    assert pixels.requires_grad
    if case.method == "forward":
        assert (pixels.detach().cpu() - run["out"]["pixels"]).abs().max() <= 1e-3
    loss = (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum()
    assert abs(loss.item() - float(gold["loss"])) <= 2e-3 * max(1.0, abs(float(gold["loss"])))
    loss.backward()
    assert _lib.launch_count() - l0 > 20, "the backward did not go through the CUDA library"
    got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({k: p.grad for k, p in gen.named_parameters()})
    # exact mode (fp32 streams, fp32 GEMMs) pins the algorithm; the default runs its activation / gradient
    # streams in fp16 between the tensor-core GEMMs (what the reference's own AMP training does,
    # train_double_latent_semantic.py:408): u = f z + p with f ~ 30-50 amplifies the 3e-4 of a
    # recomputed z into ~1e-2 of phase, so individual entries sit within 1e-2 of the tensor's largest entry
    relu = case.cfg["clamp_mode"] == "relu"
    b = _cases.model_data(case.model, "bounds")
    worst = _harness.compare_grads(gold, got, rel=b["grad_" + precision], kink_rel=b["kink_" + precision] if relu else None)
    if "grid_probe" in gold.files:
        g = gen.siren.spatial_embeddings.grad.reshape(-1).cpu()
        want = torch.from_numpy(gold["grid_probe"])
        if "grid_probe_idx" in gold.files:          # the reference's largest entries
            gscale = want.abs().max().item()
            idx = torch.from_numpy(gold["grid_probe_idx"])
        else:
            gscale = max(want.abs().max().item(), float(gold["grid_abs_sum"]) / g.numel() * 50)
            idx = _cases.grid_probe_index(g.numel(), len(gold["grid_probe"]))
        # (the reference's own gradient is an fp32 sum of trilinear scatter contributions in another order)
        worst["grid_probe"] = (g[idx] - want).abs().max().item() / gscale
        assert worst["grid_probe"] <= 1e-2, "grid gradient at the probe: %.2e" % worst["grid_probe"]
        worst["grid_abs_sum"] = abs(g.abs().sum().item() - float(gold["grid_abs_sum"])) / float(gold["grid_abs_sum"])
        assert worst["grid_abs_sum"] <= b["grid_abs_sum_" + precision]
    print("gradients %s %s: %s" % (name, precision, {k: "%.1e" % v for k, v in worst.items()}))


@pytest.mark.parametrize("name", list(_cases.GRADFREQ))
def test_inversion_gradients_through_forward_with_frequencies(runs, name):
    """inverse_render_double_semantic.py:385-407: gradients w.r.t. the FiLM frequencies / phase shifts, in exact mode;
    _cases.GRADFREQ's rows (the label FiLM row, the feature heads' rows) also within the bound on their own."""
    case, run = runs(name)
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "gradfreq_%s.npz" % name))
    gen = _cases.build_mirror(case, DEV)
    with torch.no_grad():
        leaves, order = _cases.frequency_leaves(gen.siren, [_cuda(z) for z in run["latents"]], case.model)
    fp = [t.clone().requires_grad_(True) for t in leaves]
    for p in gen.parameters():
        p.requires_grad_(False)                       # the inversion optimises the offsets only
    pixels, _ = gen.forward_with_frequencies(*[fp[i] for i in order],
                                             **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    loss = (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum()
    loss.backward()
    rel = _cases.bound(case.model, "grad_exact")
    worst = _harness.compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=rel)
    assert all(p.grad is None for p in gen.parameters())
    rows = _cases.GRADFREQ[name]
    if rows:
        cols = slice(256 * rows[0], 256 * rows[1])
        worst["rows"] = max(_rel(t.grad[:, cols].cpu(), torch.from_numpy(gold["arg%d" % i])[:, cols])
                            for i, t in enumerate(fp))
        assert worst["rows"] <= rel
    print("inversion %s: %s" % (name, worst))


@pytest.mark.parametrize("precision,rel", [("exact", 5e-4), ("guard", 2e-2)])
def test_inversion_gradients_at_zero_frequencies(runs, precision, rel):
    """As above for a_small, with raw frequencies of exactly -2.0 (table frequency 15 x + 30 = 0) and -2.0 +- a few ulps
    (table frequencies of a few 2^-19) in four FiLM layers, in both images and in image 0 only
    (tests/golden/make_goldens.py --zero-freq): finite gradients, equal to the reference's within `rel` of each tensor's
    largest entry."""
    case, run = runs("a_small")
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "gradfreq_a_small_zero_f.npz"))
    gen = _cases.build_mirror(case, DEV)
    fp = [torch.from_numpy(gold[k]).to(DEV).requires_grad_(True) for k in ("freq_in", "phase_in")]
    assert int(((fp[0] * 15 + 30) == 0).sum()) == 12
    for p in gen.parameters():
        p.requires_grad_(False)
    pixels, _ = gen.forward_with_frequencies(*fp, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision=precision))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    errs = {}
    for i, t in enumerate(fp):
        assert torch.isfinite(t.grad).all(), "arg%d" % i
        want = torch.from_numpy(gold["arg%d" % i])
        errs["arg%d" % i] = (t.grad.cpu() - want).abs().max().item() / want.abs().max().item()
    print("inversion at f = 0 (%s): %s" % (precision, errs))
    assert max(errs.values()) <= rel, errs


def test_part_forward_ray_subset_training(monkeypatch):
    """generators.py:858-910 (`grad_points`): every ray rendered, a random 3/8 of them carry the gradient.  Frames,
    poses and gradients against the reference's own part_forward, its draws (per ray subset) replayed."""
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "part_d_small.npz"))
    case = _cases.CASE_BY_NAME["d_small"]
    draws = []
    for i in range(int(gold["n_draws"])):
        key = next(k for k in gold.files if k.startswith("draw%d_" % i))
        draws.append((key.split("_", 1)[1], torch.from_numpy(gold[key])))
    gen = _cases.build_mirror(case, DEV)
    latents = [_cuda(z).requires_grad_(True) for z in _cases.make_latents(case)]
    pixels, poses = gen(*latents, **dict(case.cfg, grad_points=int(gold["grad_points"]), _rng=ReplayRng(draws, DEV)))
    err = (pixels.detach().cpu() - torch.from_numpy(gold["pixels"])).abs().amax(1)
    assert int((err > 1e-3).sum()) <= 2, "pixels beyond 1e-3: %d (max %g)" % (int((err > 1e-3).sum()), float(err.max()))
    assert (poses.detach().cpu() - torch.from_numpy(gold["poses"])).abs().max() <= 1e-5
    loss = (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum()
    loss.backward()
    got = {"g_latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({"g_" + k: p.grad for k, p in gen.named_parameters()})
    worst = {}
    for key in (k for k in gold.files if k.startswith("g_")):
        want = torch.from_numpy(gold[key])
        worst[key] = ((got[key].detach().cpu() - want).abs().max() / want.abs().max()).item()
    bad = {k: "%.2e" % v for k, v in worst.items() if v > (0.3 if k[2:] in _harness.KINK_KEYS else 2e-2)}
    assert not bad, "part_forward gradients: %s (all %s)" % (bad, {k: "%.1e" % v for k, v in worst.items()})
    # and the no_grad flavour of the same call renders the same frames.  Both flavours run the same fenerf_render_forward
    # on the same draws; only the FiLM table differs: under no_grad it comes from the fused mapping kernels, with
    # autograd from the torch modules.  From the modules' table the no_grad render is bit-identical to the grad one ...
    from fenerf_b200.siren import siren as siren_mod
    zs = [z.detach() for z in latents]
    kw = dict(case.cfg, grad_points=int(gold["grad_points"]))
    with torch.no_grad():
        px2, _ = gen(*zs, **kw, _rng=ReplayRng(draws, DEV))
        film_fused = gen.siren.film_from_latents(*zs)
        with monkeypatch.context() as m:
            m.setattr(siren_mod, "_fused_mapping_ok", lambda *a: False)
            film_mod = gen.siren.film_from_latents(*zs)
            px3, _ = gen(*zs, **kw, _rng=ReplayRng(draws, DEV))
    assert torch.equal(px3, pixels.detach()), float((px3 - pixels.detach()).abs().max())
    # ... and the two tables agree to fp32 rounding (different summation orders of the same fp32 products) ...
    ferr = float(((film_fused - film_mod).abs() / film_mod.abs().clamp_min(1.0)).max())
    assert ferr <= 1e-5, "fused vs module FiLM table: %g" % ferr
    # ... which the fp16 operands of the default point network turn into one-ulp flips of a few fp16 activations.  Those
    # move a handful of pixels by ~1e-4 (on H100: 3 pixels beyond 1e-4, the largest 2.1e-4); none may reach the parity bound.
    d = (px2 - pixels.detach()).abs().amax(1)
    msg = "no_grad vs grad frames differ: %d pixels beyond 1e-4 (max %g; FiLM tables %g apart)" % (
        int((d > 1e-4).sum()), float(d.max()), ferr)
    assert int((d > 1e-4).sum()) <= 4, msg
    assert float(d.max()) <= 1e-3, msg


def test_backward_under_autocast_and_gradscaler():
    """The G step runs under torch.cuda.amp.autocast with a GradScaler (train_double_latent_semantic.py:405-446):
    the render node casts its inputs to fp32, returns fp32 pixels and survives a 2^16-scaled upstream gradient."""
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(2, 256, device=DEV)
    w = _cases.loss_weights((2, 3, 16, 16)).to(DEV)
    torch.manual_seed(3)
    px, _ = gen(z, **case.cfg)
    (px * w).sum().backward()
    ref = {k: p.grad.clone() for k, p in gen.named_parameters()}
    gen.zero_grad()
    scaler = torch.amp.GradScaler("cuda", init_scale=65536.0)
    torch.manual_seed(3)
    with torch.autocast("cuda", dtype=torch.float16):
        px2, _ = gen(z, **case.cfg)
        assert px2.dtype == torch.float32
        loss = (px2 * w).sum()
    scaler.scale(loss).backward()
    for k, p in gen.named_parameters():
        if "mapping_network" in k:
            continue                                   # the mapping network itself runs in fp16 under autocast
        got = p.grad / 65536.0
        scale = ref[k].abs().max().item()
        # loose on purpose: under autocast the mapping network's Linears run in fp16, so the two renders do not even
        # share their FiLM table to better than 1e-3; what is checked is dtype handling and the unscaling
        assert (got - ref[k]).abs().max().item() <= 0.2 * scale + 1e-12, k


def test_point_network_entry_is_forward_only():
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    pts = torch.randn(1, 64, 3, device=DEV) * 0.1
    with pytest.raises(NotImplementedError):
        gen.siren(pts, torch.randn(1, 256, device=DEV), ray_directions=torch.randn(1, 64, 3, device=DEV))
    with torch.no_grad():
        out = gen.siren(pts, torch.randn(1, 256, device=DEV), ray_directions=torch.randn(1, 64, 3, device=DEV))
    assert out.shape == (1, 64, 4)


def test_ema_style_data_copy_is_seen_by_staged_forward():
    """torch_ema's copy_to / restore write with `param.data.copy_` (no version bump, same storage): the
    staged methods fingerprint the raw parameters on the device and repack (ADVICE r1, medium)."""
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(1, 256, device=DEV)
    kw = dict(case.cfg)
    with torch.no_grad():
        torch.manual_seed(5); a = gen.staged_forward(z, **kw)[0].cpu()
        versions = [p._version for p in gen.parameters()]
        saved = [p.detach().clone() for p in gen.parameters()]
        for p in gen.parameters():                      # ema.copy_to
            p.data.copy_(p.data * 1.25 + 0.01)
        assert versions == [p._version for p in gen.parameters()], "the write was meant to be invisible to torch"
        torch.manual_seed(5); b = gen.staged_forward(z, **kw)[0].cpu()
        for p, s_ in zip(gen.parameters(), saved):       # ema.restore
            p.data.copy_(s_)
        torch.manual_seed(5); c = gen.staged_forward(z, **kw)[0].cpu()
        gen.siren.final_layer.bias.data.add_(0.5)        # plain forward: needs the explicit invalidation
        gen.siren.invalidate_packed()
        torch.manual_seed(5); d, _ = gen(z, **kw)
    assert (a - b).abs().max() > 1e-3, "EMA-style write was not picked up"
    assert torch.equal(a, c), "restore was not picked up"
    assert (d.cpu() - a).abs().max() > 1e-3


def test_render_script_call_sequence(runs, tmp_path):
    """render_multiview_images_double_semantic.py:43-65 replayed on the mirror: whole-module checkpoint ->
    torch.load -> attribute pokes -> ema.copy_to -> set_device -> eval -> staged_forward(**curriculum),
    against the reference's own golden for that render (b_staged_segpad).  The checkpoint holds perturbed
    weights and the EMA shadow the golden's, so a stale weight pack fails the comparison."""
    import fenerf_b200
    fenerf_b200.install()
    case, run = runs("b_staged_segpad")
    gold = np.load(_cases.golden_path(case))
    src = _cases.build_mirror(case, "cpu")
    shadow = [p.detach().clone() for p in src.parameters()]              # ExponentialMovingAverage.shadow_params
    with torch.no_grad():
        for p in src.parameters():
            p.mul_(0.9)
    path = str(tmp_path / "generator.pth")
    torch.save(src, path)                                                 # train_double_latent_semantic.py:523
    generator = torch.load(path, map_location=torch.device(DEV), weights_only=False)   # :58
    assert type(generator).__module__ == "generators.generators"
    generator.softmax_label = False
    generator.neural_renderer_img = None
    generator.neural_renderer_seg = None
    with torch.no_grad():
        torch.manual_seed(0)
        generator.set_device(DEV)
        pre, _ = generator.staged_forward(*[_cuda(z) for z in run["latents"]], **dict(case.cfg, psi=case.psi, max_batch_size=2400000))
        for s_param, param in zip(shadow, generator.parameters()):        # ema.copy_to(generator.parameters())
            param.data.copy_(s_param.data)
    generator.set_device(DEV)
    generator.eval()
    curriculum = dict(case.cfg, psi=case.psi, max_batch_size=2400000, lock_view_dependence=False,
                      batch_size=24, dataset_path="unused", topk_v=0.6)   # the whole curriculum dict goes in (:79-81)
    avg = ReplayRng([("randn", t) for t in run["avg_draws"]], DEV)
    with torch.no_grad():
        img, depth_map = generator.staged_forward(*[_cuda(z) for z in run["latents"]], _rng=ReplayRng(run["draws"], DEV),
                                                  _avg_rng=avg, **curriculum)
    assert not img.is_cuda and not depth_map.is_cuda                      # the reference returns CPU tensors (:644)
    err = (img - torch.from_numpy(gold["pixels"])).abs()
    ill = _harness.ill_conditioned_pixels(case, run).unsqueeze(1).expand_as(err)
    assert err[~ill].max() <= 1e-3, float(err[~ill].max())
    assert (pre - torch.from_numpy(gold["pixels"])).abs().max() > 1e-2, "the perturbed checkpoint should not match"
    rgb, segmap = img[:, -3:], img[:, :-3]                                # generate_img, :26-27
    assert rgb.shape[1] == 3 and segmap.shape[1] == img.shape[1] - 3


#: model A built with another latent width (ImplicitGenerator3d(TALLSIREN, z_dim, 4)): 512 is the `CelebA` curriculum's
#: latent_dim (the first layer's K = 512 loads fill the kernel's 512-float rows), 4 the narrowest accepted, 36 and 508
#: not multiples of the 128 floats one pass of a warp's loads covers
_Z_DIMS = {"a_z512": 512, "a_z4": 4, "a_z36": 36, "a_z508": 508}


@functools.lru_cache(maxsize=None)
def _generator_with_z_dim(z_dim):
    from fenerf_b200.generators import generators as g
    from fenerf_b200.siren import siren as s
    with torch.random.fork_rng(devices=[]):          # seeded initialisation; the session's RNG stream is left alone
        torch.manual_seed(0)
        gen = g.ImplicitGenerator3d(s.TALLSIREN, z_dim, 4)
    gen.eval()
    return gen


def _mapping_case_generator(name):
    if name in _Z_DIMS:
        gen = copy.deepcopy(_generator_with_z_dim(_Z_DIMS[name])).to(DEV)
        gen.device = gen.siren.device = DEV
        return gen, "A", _Z_DIMS[name]
    case = _cases.CASE_BY_NAME[name]
    return _cases.build_mirror(case, DEV), case.model, 256


def _film64(sir, zs, psi=1.0, avg=None):
    """The FiLM table of the mapping network(s) in float64, with the psi truncation towards `avg` (film_from_latents'
    order of the averages)."""
    ref = copy.deepcopy(sir).double()
    if len(zs) == 1:
        f, p = ref.mapping_network(zs[0].double())
        if avg is not None:
            f, p = avg[0].double() + psi * (f - avg[0].double()), avg[1].double() + psi * (p - avg[1].double())
        return torch.stack([(f * 15 + 30).reshape(f.shape[0], -1, 256), p.reshape(f.shape[0], -1, 256)], 2)
    fg, pg = ref.geo_mapping_network(zs[0].double())
    fa, pa = ref.app_mapping_network(zs[1].double())
    if avg is not None:
        a = [t.double() for t in avg]
        fg, pg, fa, pa = a[0] + psi * (fg - a[0]), a[1] + psi * (pg - a[1]), a[2] + psi * (fa - a[2]), a[3] + psi * (pa - a[3])
    b = fg.shape[0]
    f = torch.cat([(fg * 15 + 30).reshape(b, -1, 256), (fa * 15 + 30).reshape(b, -1, 256)], 1)
    return torch.stack([f, torch.cat([pg.reshape(b, -1, 256), pa.reshape(b, -1, 256)], 1)], 2)


@pytest.mark.parametrize("name,batch", [("a_small", 3), ("b_small", 2), ("h_small", 5), ("a_small", 37), ("a_z512", 1),
                                        ("a_z512", 32), ("a_z512", 37), ("a_z4", 3), ("a_z36", 5), ("a_z508", 33)])
def test_fused_mapping_network_matches_the_modules(name, batch):
    """fenerf_mapping_film (cluster kernel + wide last layer) against CustomMappingNetwork + film_table in PyTorch, and
    against the mapping network in float64, with and without the psi truncation of staged_forward: within 2e-5 of the
    table's largest entry.  Measured against float64 on an H100 80GB HBM3 (700 W power limit): at most 1.3e-7 of it,
    z_dim 512 included.  The a_z* rows are model A with another latent width (_Z_DIMS); at z_dim 512 one no_grad
    forward of the generator must equal render_forward on the same draws with the table the fused kernel wrote, bit
    for bit (test_fused_mapping_at_z_dim_512_feeds_the_render)."""
    gen, model, z_dim = _mapping_case_generator(name)
    sir = gen.siren
    g = torch.Generator(device=DEV).manual_seed(1)
    zs = [torch.randn(batch, z_dim, device=DEV, generator=g) for _ in range(_cases.n_latents(model))]
    nets = [sir.mapping_network] if len(zs) == 1 else [sir.geo_mapping_network, sir.app_mapping_network]
    with torch.no_grad():
        assert all(siren_mod._fused_mapping_ok(n, z) for n, z in zip(nets, zs)), "the fused mapping path is not taken"
        print("%s: z_dim %d on the fused mapping path (fenerf_mapping_film)" % (name, z_dim))
        got = sir.film_from_latents(*zs)
        if len(zs) == 1:
            f, p = sir.mapping_network(zs[0])
            want = sir.film_table(f, p)
            avg = (f.mean(0, keepdim=True) * 0.9, p.mean(0, keepdim=True) * 1.1)
            want_t = sir.film_table(avg[0] + 0.7 * (f - avg[0]), avg[1] + 0.7 * (p - avg[1]))
        else:
            fg, pg = sir.geo_mapping_network(zs[0]); fa, pa = sir.app_mapping_network(zs[1])
            want = sir.film_table(fg, fa, pg, pa)
            avg = (fg.mean(0, keepdim=True), pg.mean(0, keepdim=True) * 1.1, fa.mean(0, keepdim=True) * 0.9, pa.mean(0, keepdim=True))
            want_t = sir.film_table(avg[0] + 0.7 * (fg - avg[0]), avg[2] + 0.7 * (fa - avg[2]), avg[1] + 0.7 * (pg - avg[1]),
                                    avg[3] + 0.7 * (pa - avg[3]))
        got_t = sir.film_from_latents(*zs, psi=0.7, avg=avg)
    assert got.shape == want.shape
    assert (got - want).abs().max() <= 2e-5 * want.abs().max(), float((got - want).abs().max())
    assert (got_t - want_t).abs().max() <= 2e-5 * want_t.abs().max(), float((got_t - want_t).abs().max())
    w64, w64_t = _film64(sir, zs), _film64(sir, zs, 0.7, avg)
    e64, e64_t = _rel(got, w64), _rel(got_t, w64_t)
    print("%s B=%d z_dim %d: fused mapping vs float64 %.3g, with psi %.3g (of the table's maximum)" % (name, batch, z_dim,
                                                                                                       e64, e64_t))
    assert max(e64, e64_t) <= 2e-5, (e64, e64_t)
    # with autograd on, the PyTorch modules run (the latent / mapping network must stay differentiable)
    z = zs[0].clone().requires_grad_(True)
    film = sir.film_from_latents(z, *zs[1:])
    assert film.requires_grad


@pytest.mark.parametrize("m", [1, 24, 63, 128, 128 + 24, 1000, 128 * 149 + 17])
def test_wgmma_gemm_nt_cos_gate_against_fp32_matmul(m):
    """fenerf_gemm_nt_f16 (fp32 / fp16 output, the optional output * gate epilogue, and row ranges of one output written by
    separate launches, as the backward's per-image chain products do) and fenerf_gemm_nt_film, whose gate is cos(u) --
    no factor f, so that no FiLM gradient has to divide by it.  M = 1, 24 and 63 fill less than one 64-row half of a
    128-row tile (24: the one-ray trailing chunk of a flat 24-step 256² backward, backward.CHUNK_POINTS), 128 + 24 a
    second tile with that ragged tail.  The FiLM epilogue runs on two images of (M + 1) / 2 rows and on one image of M
    rows: at M = 24 that is the trailing chunk's own shape."""
    g = torch.Generator(device=DEV).manual_seed(m)
    a = (torch.randn(m, 256, device=DEV, generator=g) * 0.5).half()
    w = (torch.randn(256, 256, device=DEV, generator=g) * 0.1).half()
    want = a.float() @ w.float().t()
    got32 = ops.gemm_nt(a, w, torch.float32)
    got16 = ops.gemm_nt(a, w, torch.float16)
    scale = want.abs().max()
    assert (got32 - want).abs().max() <= 2e-5 * scale, float((got32 - want).abs().max() / scale)
    assert (got16.float() - want).abs().max() <= 1e-3 * scale
    split = torch.empty_like(got16)                                       # rows [0, r) and [r, m) by two launches
    r = m // 2 // 8 * 8
    for rows in (slice(0, r), slice(r, m)):
        if rows.stop > rows.start:
            ops.gemm_nt(a[rows], w, torch.float16, out=split[rows])
    assert torch.equal(split, got16)
    gate = (torch.randn(m, 256, device=DEV, generator=g) * 5).half()      # optional epilogue: output * gate
    gated = ops.gemm_nt(a, w, torch.float16, gate=gate)
    assert (gated.float() - want * gate.float()).abs().max() <= 2e-3 * (want * gate.float()).abs().max()
    # the fused FiLM epilogue, on two images and on one image of m rows (m = 24: the trailing chunk's one ray)
    for B, ppb in ((2, (m + 1) // 2), (1, m)):
        mm = B * ppb
        a2 = (torch.randn(mm, 256, device=DEV, generator=g) * 0.5).half()
        film = torch.stack([torch.rand(B, 3, 256, device=DEV, generator=g) * 40 + 10, torch.randn(B, 3, 256, device=DEV, generator=g)], 2).contiguous()
        bias = torch.randn(256, device=DEV, generator=g) * 0.1
        act, gate = ops.gemm_nt_film(a2, w, bias, film, 0, 1, ppb)
        z = (a2.float() @ w.float().t() + bias).reshape(B, ppb, 256)
        u = film[:, 1, 0].unsqueeze(1) * z + film[:, 1, 1].unsqueeze(1)
        assert (act.float().reshape(B, ppb, 256) - torch.sin(u)).abs().max() <= 2e-3
        assert (gate.float().reshape(B, ppb, 256) - torch.cos(u)).abs().max() <= 2e-3              # the gate is cos(u), without f
        # ... with a narrow fifth k-chunk (35 of 64 columns used)
        xn = torch.zeros(mm, 64, device=DEV).half(); xn[:, :35] = (torch.randn(mm, 35, device=DEV, generator=g) * 0.3).half()
        wn = torch.zeros(256, 64, device=DEV).half(); wn[:, :35] = (torch.randn(256, 35, device=DEV, generator=g) * 0.1).half()
        act2, gate2 = ops.gemm_nt_film(a2, w, bias, film, 0, 1, ppb, narrow_in=xn, narrow_w=wn)
        u2 = film[:, 1, 0].unsqueeze(1) * (z + (xn.float() @ wn.float().t()).reshape(B, ppb, 256)) + film[:, 1, 1].unsqueeze(1)
        assert (act2.float().reshape(B, ppb, 256) - torch.sin(u2)).abs().max() <= 2e-3
        assert (gate2.float().reshape(B, ppb, 256) - torch.cos(u2)).abs().max() <= 2e-3


@pytest.mark.parametrize("batch,ppb,slices", [(1, 1, None), (1, 24, None), (2, 24, 3), (3, 63, None), (1, 64, 1), (2, 200, 3),
                                              (3, 4096 * 3 + 5, None)])
def test_tcgen05_gemm_tn_against_fp32_bmm(batch, ppb, slices):
    """Per-image X_b^T Y_b and the column sums of X.  ppb = 1, 24 and 63 fill less than one 64-point stage (24: the
    one-ray trailing chunk of a flat 24-step 256² backward); (2, 24, 3) leaves two slices of each image without a stage,
    so their partials must be zero."""
    g = torch.Generator(device=DEV).manual_seed(ppb)
    x = (torch.randn(batch * ppb, 256, device=DEV, generator=g) * 0.5).half()
    y = (torch.randn(batch * ppb, 256, device=DEV, generator=g) * 0.5).half()
    want = torch.bmm(x.float().reshape(batch, ppb, 256).transpose(1, 2), y.float().reshape(batch, ppb, 256))
    got = ops.gemm_tn(x, y, batch, ppb, slices)
    scale = want.abs().max()
    assert (got - want).abs().max() <= 5e-5 * scale, float((got - want).abs().max() / scale)
    got2, cs = ops.gemm_tn(x, y, batch, ppb, slices, colsum=True)         # optional: column sums of X ride along
    assert torch.equal(got2, got)
    want_cs = x.float().reshape(batch, ppb, 256).sum(1)
    assert (cs - want_cs).abs().max() <= 1e-4 * max(1.0, float(want_cs.abs().max()))


def test_fused_mapping_at_z_dim_512_feeds_the_render():
    """Model A built with z_dim 512 (the `CelebA` curriculum's latent_dim): one no_grad forward of the generator equals,
    bit for bit, render_forward on the same draws with the FiLM table the fused mapping kernel wrote -- the render takes
    the fused table, not the PyTorch modules' (which differ from it in the last bits)."""
    gen, _, z_dim = _mapping_case_generator("a_z512")
    sir = gen.siren
    cfg = dict(_cases.BASE, img_size=32, num_steps=12, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.5)
    b, n, s = 2, 32 * 32, 12
    g = torch.Generator(device=DEV).manual_seed(512)
    z = torch.randn(b, z_dim, device=DEV, generator=g)
    draws = [("rand", torch.rand(b, n, s, 1, device=DEV, generator=g)), ("randn", torch.randn(b, 1, device=DEV, generator=g)),
             ("randn", torch.randn(b, 1, device=DEV, generator=g)), ("randn", torch.randn(b, n, s, 1, device=DEV, generator=g)),
             ("rand", torch.rand(b * n, s, device=DEV, generator=g)), ("randn", torch.randn(b, n, 2 * s, 1, device=DEV, generator=g))]
    with torch.no_grad():
        assert siren_mod._fused_mapping_ok(sir.mapping_network, z)
        px, _ = gen(z, _rng=ReplayRng(draws, DEV), **cfg)
        film = sir.film_from_latents(z)
        f, p = sir.mapping_network(z)
        assert not torch.equal(film, sir.film_table(f, p)), "the fused and the PyTorch tables agree bit for bit: no witness"
        rd = ops.make_render_desc(batch=b, img_size=32, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.5, fov=12)
        c2w = ops.camera_poses(b, "gaussian", 0.3, 0.155, cfg["h_mean"], cfg["v_mean"], ReplayRng(draws[1:3], DEV),
                               torch.device(DEV))[0]
        x_lin, y_lin, z_lin = ops.ray_tables(32, s, 0.88, 1.12, DEV)
        want = ops.render_forward(sir, rd, film, x_lin, y_lin, z_lin, c2w, draws[0][1].contiguous(), draws[3][1], draws[4][1],
                                  draws[5][1])[0]
    print("z_dim 512: generator forward on the fused mapping path, frame bit-identical to render_forward on its table")
    assert torch.equal(px, want), float((px - want).abs().max())


def test_frame_consumers_match_the_reference_loops():
    """mask2color (train_double_latent_semantic.py:66-72) and save_image's quantisation (fid_evaluation.py:149)."""
    from fenerf_b200 import frames
    from oracle import render_oracle as oracle
    g = torch.Generator().manual_seed(5)
    masks = torch.randn(3, 19, 37, 29, generator=g)
    want = oracle.mask2color(masks)
    got_gpu = frames.mask2color(masks.to(DEV))
    assert got_gpu.is_cuda and torch.equal(got_gpu.cpu(), want)
    got_cpu = frames.mask2color(masks)                       # CPU in -> CPU out, as the reference's callers expect
    assert not got_cpu.is_cuda and torch.equal(got_cpu, want)
    wide = torch.randn(2, 22, 8, 8, generator=g)
    sliced = wide.to(DEV)[:, :18]                            # a channel slice: not contiguous
    assert not sliced.is_contiguous()
    assert torch.equal(frames.mask2color(sliced).cpu(), oracle.mask2color(wide[:, :18]))
    img = torch.rand(2, 21, 33, 31, generator=g) * 2.4 - 1.2   # a little outside [-1, 1]: clamped
    u8 = frames.frames_to_uint8(img.to(DEV)).cpu()
    for b in range(2):
        assert torch.equal(u8[b], oracle.save_image_bytes(img[b, -3:]))


def test_guard_self_check_widens_the_threshold_on_large_weights():
    """The GUARD threshold was calibrated on the reference's initialisation (VERDICT r1, weak #4).  The refinement
    reports max |sigma_fp32 - sigma_wgmma| over the samples it re-evaluates; staged_* widens tau when that error
    comes within 3x of it.  Scaling the density head by 30 scales the fp16 error with it."""
    import warnings
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(2, 256, device=DEV)
    with torch.no_grad():
        torch.manual_seed(1)
        gen.staged_forward(z, **case.cfg)
        rep = ops.guard_stats(DEV)
        assert rep["refined"] > 0 and 0 < rep["max_abs_delta"] < rep["tau"] / 3 and abs(rep["tau"] - 1.5e-3) < 1e-9
        assert not hasattr(gen.siren, "_guard_tau")
        gen.siren.final_layer.weight.mul_(30.0)
        gen.siren.final_layer.bias.mul_(30.0)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.manual_seed(1)
            a = gen.staged_forward(z, **case.cfg)[0].cpu()
        assert any("guard_tau" in str(x.message) for x in w), "no widening on 30x weights"
        assert gen.siren._guard_tau > 1.5e-3
        torch.manual_seed(1)
        b = gen.staged_forward(z, **dict(case.cfg, precision="exact"))[0].cpu()
    assert ((a - b).abs() > 1e-3).float().mean() < 0.02     # the widened guard keeps the step function right


def test_repack_after_inplace_weight_update():
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(1, 256, device=DEV)
    with torch.no_grad():
        torch.manual_seed(5); a, _ = gen(z, **case.cfg)
        gen.siren.final_layer.bias += 0.5      # what an optimizer step / EMA copy_to does
        torch.manual_seed(5); b, _ = gen(z, **case.cfg)
    assert (a - b).abs().max() > 1e-3, "packed weights were not refreshed after an in-place update"


_REPACK = [m for m in _cases.MODELS if _cases.model_data(m, "repack")]


@pytest.mark.parametrize("model", _REPACK)
def test_staged_forward_sees_parameter_writes(model):
    """torch_ema's copy_to writes through param.data without a version bump: a write to each of the model's repack
    parameters alone (or to some of its columns, _cases.MODEL_DATA) must reach staged_forward -- the fingerprint covers
    it -- and after invalidate_packed() the render is the same."""
    case = _cases.CASE_BY_NAME["%s_small_opaque" % model.lower()]     # (white-filled at the plain init: nothing would move)
    gen = _cases.build_mirror(case, DEV)
    params = dict(gen.named_parameters())
    g = torch.Generator().manual_seed(8)
    z = [torch.randn(1, 256, generator=g).to(DEV) for _ in range(_cases.n_latents(model))]
    kw = dict(case.cfg, psi=0.7, max_batch_size=2400000, precision="exact")

    def render():
        torch.manual_seed(1)
        return torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(*z, **kw)[:2]])
    with torch.no_grad():
        for name, cols, factor in _cases.model_data(model, "repack"):
            w = params[name]
            cols = cols or slice(None)
            a = render()
            w.data[:, cols].copy_(w.detach()[:, cols] * factor)
            b = render()
            gen.siren.invalidate_packed()
            assert not torch.equal(a, b), name
            assert torch.equal(b, render()), name


_GUARD = [m for m in _cases.MODELS if _cases.model_data(m, "guard")]


@pytest.mark.parametrize("model", _GUARD)
def test_guard_refinement(model):
    """GUARD with every ray's far sample refined (tau huge): those densities equal the exact kernel's bit for bit, every
    other value of the row (labels and features included) is the fast pass's, and the self-check's max |delta| stays
    within the model's bound (_cases.MODEL_DATA)."""
    img, delta_bound = _cases.model_data(model, "guard")
    siren = _siren(model, DEV)
    film = _film(siren, 2, 77)
    c = siren.field_spec().out_dim
    rd = ops.make_render_desc(batch=2, img_size=img, num_steps=12, hierarchical=False, clamp_mode="relu", nerf_noise=0.0,
                              fov=12, precision="guard", guard_tau=1e9)
    x_lin, y_lin, z_lin = ops.ray_tables(img, 12, 0.88, 1.12, DEV)
    c2w = torch.eye(4, device=DEV).repeat(2, 1, 1)
    c2w[:, 2, 3] = 1.0
    rng = torch.rand(2, img * img, 12, 1, generator=torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        st = ops.render_forward_stages(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
        pts, dirs = st["points_c"].reshape(2, -1, 3), st["dirs"]
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast").reshape(2, img * img, 12, c)
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact").reshape(2, img * img, 12, c)
        pixels = ops.render_forward(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)[0]
    rep = ops.guard_stats(DEV)
    print("guard %s: %s" % (model, rep))
    if delta_bound is not None:
        assert rep["refined"] >= 2 * img * img and rep["max_abs_delta"] < delta_bound
    raw = st["raw_c"]
    assert torch.equal(raw[:, :, :-1], fast[:, :, :-1])
    assert torch.equal(raw[:, :, -1, -1], exact[:, :, -1, -1])
    assert torch.equal(raw[:, :, -1, :-1], fast[:, :, -1, :-1])
    assert torch.isfinite(pixels).all()


def test_neural_renderer_modules_run_on_the_unit_frame(runs):
    """generators.py:102-118, 231-248: with `neural_renderer_img` attached the caller's module runs on the [0, 1]
    frame and `* 2 - 1` follows; checked against the same module applied to the reference's golden frame, for
    `forward`, `staged_forward`, and with autograd through the module into the field's weights."""
    torch.manual_seed(9)
    up = torch.nn.Sequential(torch.nn.Upsample(scale_factor=2.), torch.nn.Conv2d(3, 3, 3, 1, 1), torch.nn.Sigmoid()).to(DEV)
    for name in ("a_small", "a_staged_white"):
        case, run = runs(name)
        gold = torch.from_numpy(np.load(_cases.golden_path(case))["pixels"])
        with torch.no_grad():
            want = (up(((gold + 1) * 0.5).to(DEV)) * 2 - 1).cpu()
        gen = _cases.build_mirror(case, DEV)
        gen.neural_renderer_img = up
        kw = dict(case.cfg, precision="guard", _rng=ReplayRng(run["draws"], DEV))
        with torch.no_grad():
            if case.method == "staged_forward":
                avg = ReplayRng([("randn", t) for t in run["avg_draws"]], DEV)
                got = gen.staged_forward(*[_cuda(z) for z in run["latents"]], psi=case.psi, _avg_rng=avg, **kw)[0].cpu()
            else:
                got = gen(*[_cuda(z) for z in run["latents"]], **kw)[0].cpu()
        r = case.cfg["img_size"]
        assert got.shape == (case.batch, 3, 2 * r, 2 * r)
        # a 3x3 convolution spreads an ill-conditioned ray over its neighbours: bound the bulk, not every pixel
        err = (got - want).abs()
        assert err.median() <= 1e-4 and (err > 1e-3).float().mean() <= 0.02
    case, run = runs("a_small")
    gen = _cases.build_mirror(case, DEV)
    gen.neural_renderer_img = up
    kw = dict(case.cfg, _rng=ReplayRng(run["draws"], DEV))
    frames, _ = gen(*[_cuda(z) for z in run["latents"]], **kw)
    assert frames.requires_grad
    frames.square().mean().backward()
    g = gen.siren.final_layer.weight.grad
    assert g is not None and torch.isfinite(g).all() and g.abs().sum() > 0
    assert up[1].weight.grad is not None and up[1].weight.grad.abs().sum() > 0


@pytest.mark.parametrize("name,kw", [("a_small", {}), ("b_small", dict(precision="exact")),
                                     ("b_small", dict(precision="split", grad_precision="split"))])
def test_backward_state_is_freed_without_the_cycle_collector(name, kw, monkeypatch):
    """The render backward's per-call state (_FieldBackward: the per-image accumulators, the stream's weight forms, the
    grid accumulator) is in no reference cycle: reference counting frees it, and its device memory, as soon as
    loss.backward() returns, so a training loop does not wait for Python's cycle collector to get that memory back."""
    from fenerf_b200 import backward
    case = _cases.CASE_BY_NAME[name]
    gen = _cases.build_mirror(case, DEV)
    zs = [torch.randn(case.batch, 256, device=DEV) for _ in range(_cases.n_latents(case.model))]
    made = []
    init = backward._FieldBackward.__init__

    def spy(self, *args, **kwargs):
        init(self, *args, **kwargs)
        made.append(weakref.ref(self))

    monkeypatch.setattr(backward._FieldBackward, "__init__", spy)
    gc.collect()
    gc.disable()
    try:
        px, _ = gen(*zs, **dict(case.cfg, **kw))
        px.sum().backward()
        assert len(made) == 1 and made[0]() is None
    finally:
        gc.enable()
