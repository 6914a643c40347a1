"""The reference scripts' own workloads against float64: the render scripts' 256² and 512² faces (buffers past 2^31
bytes), the shape extraction's 256³ grid, the inversion's flat 256² backward and model A's 512-wide latent (the
last in test_gpu_parity.py::test_fused_mapping_network_matches_the_modules).

Render scripts (render_multiview_images_double_semantic.py, render_video_interpolation_semantic.py): one face at
256² or 512², 48 steps times --ray_step_multiplier.  Model B at 512² x 96 + 96 holds raw_c and raw_f of 2.21 GB each
(262,144 x 96 x 22 floats), so every 32-bit byte or float offset in ray set-up, the point network's stores, the
resampler, GUARD and the compositor would land elsewhere for the buffer's tail.  A whole-image float64 reference of
such a render would not fit a shared card, so the float64 side runs on a fixed ray subset (ray_subset: the first and
last 4,096 rays of the buffer, the image's border rows and columns, a seeded random sample); the bit-for-bit checks
(stand-alone resampler = render, stand-alone compositor = render, points_f = o + d z_f) stay on the whole buffers.
At 512² x 96 x 22, float 2^29 lies 97 % into raw_c: the last 4,096 rays all sit past it.  The CPU tests show that
each subset reference equals the full-image reference on the subset, and that the tail rays' rows read from offsets
wrapped at the same fraction of the buffer move every stage past ten times its bound.

Shape extraction (extract_double_semantic_shapes.py): 256³ points of a cube of 0.3, evaluated in 24,000-point slices
(the last one 1,216 points) through forward_with_frequencies_phase_shifts, keeping sigma.  The script passes
directions (0, 0, -1); zero directions are what siren.density uses.  Sigma must be bit-identical across the slices,
one density call over all 16,777,216 points, and either direction, and within FWD_BOUND of float64 on a subset that
holds the last 65,536 voxels.

Inversion (inverse_render_double_semantic.py): forward_with_frequencies under autograd with the script's options
(flat 24 steps, 256², tensor h_mean / v_mean, fill_mode and fade_steps present), differentiated w.r.t. FiLM offsets.
One image is 1,572,864 points, above backward.CHUNK_POINTS: chunks of 524,280 points and a trailing chunk of 24
points (one ray), whose products run the wgmma GEMMs at M = 24 and ppb = 24.  The gradients are checked against the
float64 chain, the trailing ray on its own too, and against a two-halves chunk layout within LAYOUT_BOUND.

Every GPU test prints torch.cuda.max_memory_allocated() and keeps it under MEM_CAP.  The large ones (the 512² rows
and the inversion) print the free memory they find and skip when a shared card lacks what they need; with
FENERF_REQUIRE_SCRIPT_SHAPES=1 they fail instead, so that a run meant to cover them cannot pass without them.

Measured on an H100 80GB HBM3 (700 W power limit), all within the existing constants: ray set-up <= 2.7e-7
(RAY_BOUND 1e-6); the point network in guard <= 4.8e-4 (FWD_BOUND['fast'] 5e-3), in split 2.9e-6 (script512-B-split;
FWD_BOUND['exact'] 1e-5); CDF ratio <= 0.145 (1); refined far densities <= 7.4e-7 (1e-5); compositor <= 3.6e-6
(script512-B; COMPOSITE_FWD_BOUND 1e-5).  The grid's sigma 4.1e-4 in guard, 1.1e-6 in exact.  The inversion's
gradients 1.04e-2 in guard (FIELD_BOUND 2e-2; the trailing ray alone 1.44e-2), 1.5e-5 in exact (1e-4; the trailing ray
1.6e-5); two halves against the library's chunks 2.5e-5 in guard, 2.8e-6 in exact (LAYOUT_BOUND 5e-5).  Peak
allocation 10.4 GB for the 512² rows, 21.8 GB for the exact inversion.  The GPU tests of this file ran in 27 s.
"""
import copy
import gc
import math
import os

import pytest
import torch

from _fp64 import _film, _generator_cpu, _opt, field_ref, pass_dirs
import test_gpu_fp64_forward_stages as fs
from fenerf_b200 import backward, ops
from fenerf_b200.generators.volumetric_rendering import ReplayRng
from test_gpu_fp64_forward_stages import (COMPOSITE_FWD_BOUND, RAY_BOUND, _cpu_render, _cpu_ray_inputs, cdf_errors,
                                          check_composite, check_guard, check_points, check_ray_setup, check_resample,
                                          composite_subset_ref, guard_refined, ray_setup_ref, resample_ref)
from test_gpu_fp64_reference import FIELD_BOUND, FWD_BOUND, LAYOUT_BOUND, _grad_errors
from test_gpu_fp64_train_grads import camera_chain_vjp

DEV = "cuda:0"
gpu = pytest.mark.gpu
GIB = 1 << 30

#: peak torch.cuda.max_memory_allocated() of any test here
MEM_CAP = 24 * GIB
#: float 2^29 as a fraction of the 512² x 96 x 22 raw buffer: where a 32-bit byte offset of raw_c wraps
WRAP_FRACTION = 2 ** 29 / (512 * 512 * 96 * 22)


@pytest.fixture(autouse=True)
def _memory(request):
    """GPU tests: the peak allocation, printed and kept under MEM_CAP."""
    if request.node.get_closest_marker("gpu") is None:
        yield
        return
    torch.empty(1, device=DEV)                      # the caching allocator exists before its statistics are reset
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    peak = torch.cuda.max_memory_allocated(DEV)
    print("%s: max_memory_allocated %.2f GB" % (request.node.name, peak / 1e9))
    torch.cuda.empty_cache()
    assert peak <= MEM_CAP, "peak allocation %.2f GB above MEM_CAP" % (peak / 1e9)


def need_free(gib, what):
    """Skip when the card has less than `gib` GiB free -- a fail instead with FENERF_REQUIRE_SCRIPT_SHAPES=1, so that a
    run which must cover the large rows cannot pass without them.  Prints what it saw either way: the card's free and
    total memory, and what this process's allocator holds (live tensors of earlier tests included)."""
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(DEV)
    held = torch.cuda.memory_allocated(DEV)
    seen = "%s: %.1f GiB free of %.1f, this process holds %.1f GiB in live tensors, %.1f GiB needed" % (
        what, free / GIB, total / GIB, held / GIB, gib)
    print(seen)
    if free < gib * GIB:
        if os.environ.get("FENERF_REQUIRE_SCRIPT_SHAPES") == "1":
            pytest.fail("FENERF_REQUIRE_SCRIPT_SHAPES=1 and " + seen)
        pytest.skip(seen)


def ray_subset(r, edge=4096, n_random=1 << 14, seed=0, device=DEV):
    """Sorted ray indices (p = row * R + col) of one R² image: the first and last `edge` rays, the border rows and
    columns, and `n_random` seeded random rays."""
    n = r * r
    idx = torch.arange(r)
    parts = [torch.arange(min(edge, n)), torch.arange(max(0, n - edge), n), idx, (r - 1) * r + idx, idx * r,
             idx * r + r - 1, torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:n_random]]
    return torch.unique(torch.cat(parts)).to(device)


def wrap_rows(t, wrap_fraction=WRAP_FRACTION):
    """t (B, N, ...) as a kernel would see it whose flat offsets wrap at `wrap_fraction` of the buffer: the rays
    starting past the wrap point read the row of the ray their wrapped offset falls in.  -> (wrapped t, tail rays)."""
    b, n = t.shape[:2]
    per_ray = t[0, 0].numel()
    wrap = int(wrap_fraction * t.numel())
    g = torch.arange(b * n)
    tail = g * per_ray >= wrap
    src = torch.where(tail, (g * per_ray % wrap) // per_ray, g)
    return t.reshape(b * n, -1)[src.to(t.device)].reshape(t.shape), g[tail]


# --------------------------------------------------------------------------------------------
# the render scripts' faces
# --------------------------------------------------------------------------------------------
#: name -> a row of test_gpu_fp64_forward_stages._RENDERS: (model, batch, R, steps, hierarchical, options, precision,
#: lock_view_dependence)
_SCRIPT_RENDERS = {
    "script256-B": ("B", 1, 256, 48, True, _opt("relu"), "guard", False),
    "script256-B-lock": ("B", 1, 256, 48, True, _opt("relu"), "guard", True),
    "script512-B": ("B", 1, 512, 96, True, _opt("relu"), "guard", False),
    "script512-B-split": ("B", 1, 512, 96, True, _opt("relu"), "split", False),
    # 4 channels: the one-thread-per-ray compositor
    "script512-A": ("A", 1, 512, 72, True, _opt("relu", noise=0.5), "guard", False),
}


def check_stages(x, rays):
    """Every stage of render x against float64 on rays `rays`, the bit-for-bit checks on the whole buffers."""
    res = dict(rays=check_ray_setup(x, rays), points=check_points(x, rays))
    res.update(check_resample(x, rays))
    if x["precision"] == "guard":
        res["guard"] = check_guard(x, ops.DEFAULT_GUARD_TAU, refined_only=True)
    res.update(check_composite(x, rays))
    return res


@gpu
@pytest.mark.parametrize("name", list(_SCRIPT_RENDERS))
def test_script_render_stages_vs_fp64(name):
    """One face of a render script, every stage against float64 on ray_subset, the last 4,096 rays of the buffer
    included; the 512² rows hold raw_c and raw_f past 2^31 bytes."""
    spec = _SCRIPT_RENDERS[name]
    r = spec[2]
    if r == 512:
        need_free(12, name)          # peak measured 10.4 GB
    x = fs.render(name, spec=spec)
    raw_bytes = x["raw_c"].numel() * 4
    print("%s: %d rays, raw_c %d bytes (2^31 = %d), raw_f %d bytes" % (name, x["n"], raw_bytes, 2 ** 31,
                                                                       x["raw_f"].numel() * 4))
    if r == 512 and spec[0] == "B":
        assert raw_bytes > 2 ** 31 and x["raw_f"].numel() * 4 > 2 ** 31, raw_bytes
    elif r == 512:           # model A: 262,144 rays in one image on the one-thread-per-ray compositor (C <= 8)
        assert x["n"] == 1 << 18 and x["raw_c"].shape[-1] <= 8
    rays = ray_subset(r)
    assert rays[-1].item() == x["b"] * x["n"] - 1 and len(rays) < x["n"]
    res = check_stages(x, rays)
    print("script stages %s (%d rays of %d compared in float64): %s" % (name, len(rays), x["n"], res))


def _generator(model):
    """A device copy of the suite's generator of `model` (the field test_gpu_fp64_forward_stages renders)."""
    gen = copy.deepcopy(_generator_cpu(model)).to(DEV)
    gen.device = gen.siren.device = DEV
    return gen


def _truncated(siren, g, psi):
    """The script's truncated mapping outputs of model B: avg + psi (raw - avg), avg over 1,000 latents."""
    out = []
    with torch.no_grad():
        for net in (siren.geo_mapping_network, siren.app_mapping_network):
            f, p = net(torch.randn(1, 256, generator=g, device=DEV))
            fa, pa = (t.mean(0, keepdim=True) for t in net(torch.randn(1000, 256, generator=g, device=DEV)))
            out.append((fa + psi * (f - fa), pa + psi * (p - pa)))
    (fg, pg), (fa, pa) = out
    return fg, fa, pg, pa


@gpu
def test_staged_forward_with_frequencies_is_the_checked_render():
    """DoubleImplicitGenerator3d.staged_forward_with_frequencies of model B at 256², 48 + 48, psi 0.5, depth_map=True,
    on replayed draws: its frame and depth map equal, bit for bit, the stage-checked render on the same FiLM table and
    draws, whose stages are then checked against float64 on ray_subset."""
    gen = _generator("B")
    r, s, n = 256, 48, 256 * 256
    g = torch.Generator(device=DEV).manual_seed(256)
    freqs = _truncated(gen.siren, g, 0.5)
    draws = [("rand", torch.rand(1, n, s, 1, generator=g, device=DEV)), ("randn", torch.randn(1, n, s, 1, generator=g, device=DEV)),
             ("rand", torch.rand(n, s, generator=g, device=DEV)), ("randn", torch.randn(1, n, 2 * s, 1, generator=g, device=DEV))]
    h_mean = math.pi / 2 + 0.3
    frame, depth_map, _ = gen.staged_forward_with_frequencies(
        *freqs, img_size=r, fov=12, ray_start=0.88, ray_end=1.12, num_steps=s, h_stddev=0, v_stddev=0, h_mean=h_mean,
        v_mean=math.pi / 2, psi=0.5, depth_map=True, hierarchical_sample=True, sample_dist=None, clamp_mode="relu",
        nerf_noise=0, lock_view_dependence=False, _rng=ReplayRng(draws, DEV))
    with torch.no_grad():
        film = gen.siren.film_table(*freqs)
        c2w = ops.camera_poses(1, None, 0, 0, h_mean, math.pi / 2, None, torch.device(DEV))[0]
    inputs = dict(film=film, c2w=c2w, perturb=draws[0][1].reshape(1, n, s), noise_c=draws[1][1].reshape(1, n, s),
                  u=draws[2][1], noise_f=draws[3][1].reshape(1, n, 2 * s))
    x = fs.render("staged256-B", spec=("B", 1, r, s, True, _opt("relu"), "guard", False), inputs=inputs)
    assert torch.equal(frame, x["pixels"].cpu()), "staged_forward_with_frequencies' frame differs from the checked render"
    assert torch.equal(depth_map, x["depth"].reshape(1, r, r).cpu()), "its depth map differs"
    print("staged_forward_with_frequencies 256² x 48 + 48: frame and depth map bit-identical to the checked render")
    res = check_stages(x, ray_subset(r))
    print("staged256-B stages: %s" % res)


# --------------------------------------------------------------------------------------------
# the shape extraction's grid
# --------------------------------------------------------------------------------------------
def script_grid(n=256, cube=0.3):
    """The samples of extract_double_semantic_shapes.py's create_samples(N, voxel_origin=[0, 0, 0], cube_length),
    restated: index i -> (((i / N) / N) % N, (i / N) % N, i % N) in fp32 float division (the first two are not
    integers), times the voxel size, plus the corner at -cube / 2.  -> (1, N³, 3) fp32 on the CPU."""
    origin = -cube / 2
    size = cube / (n - 1)
    i = torch.arange(n ** 3)
    s = torch.zeros(n ** 3, 3)
    s[:, 2] = i % n
    s[:, 1] = (i.float() / n) % n
    s[:, 0] = ((i.float() / n) / n) % n
    return (s * size + origin).unsqueeze(0)


#: the script's slice of points per forward_with_frequencies_phase_shifts call
SLICE = 24000


@gpu
@pytest.mark.parametrize("precision", ["guard", "exact"])
@pytest.mark.parametrize("model", ["B", "A"])
def test_shape_grid_density_vs_fp64(model, precision):
    """256³ points of the shape extraction's grid: sigma of the script's 24,000-point slices with zero directions =
    one density call over all 16,777,216 points = the same points under the script's (0, 0, -1), bit for bit; within
    FWD_BOUND of float64 on the first and last 65,536 voxels (the whole last slice inside) and 65,536 random ones."""
    need_free(8, "the 256³ grid")
    siren = fs._field(model)
    g = torch.Generator(device=DEV).manual_seed(3)
    if model == "B":
        freqs = _truncated(siren, g, 0.5)
    else:
        with torch.no_grad():
            f, p = siren.mapping_network(torch.randn(1, 256, generator=g, device=DEV))
        freqs = (f, p)
    film = siren.film_table(*freqs)
    pts = script_grid().to(DEV)
    n_pts = pts.shape[1]
    assert n_pts == 1 << 24 and n_pts % SLICE == 1216
    old = ops.default_precision()
    ops.set_default_precision(precision)
    try:
        with torch.no_grad():
            sliced = torch.empty((1, n_pts, 1), device=DEV)
            zero_dirs = torch.zeros((1, SLICE, 3), device=DEV)
            for head in range(0, n_pts, SLICE):
                k = min(SLICE, n_pts - head)
                out = siren.forward_with_frequencies_phase_shifts(pts[:, head:head + k], *freqs, ray_directions=zero_dirs[:, :k])
                sliced[:, head:head + k] = out[..., -1:]
            full = siren.density(pts, film)
            locked = torch.tensor([[[0.0, 0.0, -1.0]]], device=DEV)
            sig_locked = ops.siren_points(siren, pts, film, locked, dir_group=n_pts)[..., -1:]
    finally:
        ops.set_default_precision(old)
    print("shape grid %s %s: %d points in one density call" % (model, precision, full.shape[1]))
    assert full.shape == (1, n_pts, 1)
    assert torch.equal(sliced, full), "24,000-point slices != one density call"
    assert torch.equal(sig_locked, full), "sigma under (0, 0, -1) != sigma under zero directions"
    edge = 1 << 16
    idx = torch.unique(torch.cat([torch.arange(edge), torch.arange(n_pts - edge, n_pts),
                                  torch.randperm(n_pts, generator=torch.Generator().manual_seed(4))[:edge]])).to(DEV)
    want = field_ref(siren, pts[:, idx], torch.zeros((1, len(idx), 3), device=DEV), film)[0][0, :, -1]
    err = (full[0, idx, 0].double() - want).abs().max().item()
    last = (full[0, n_pts - 1216:, 0].double() - want[-1216:]).abs().max().item()
    bound = FWD_BOUND["exact" if precision == "exact" else "fast"]
    print("shape grid %s %s: sigma vs fp64 on %d voxels %.3g, last slice %.3g (bound %g)" % (model, precision, len(idx),
                                                                                            err, last, bound))
    assert err <= bound, err


# --------------------------------------------------------------------------------------------
# the inversion's backward
# --------------------------------------------------------------------------------------------
def _inversion_options(draws, precision):
    """inverse_render_double_semantic.py's options dict, with the test's draws and precision."""
    return {'img_size': 256, 'fov': 12, 'ray_start': 0.88, 'ray_end': 1.12, 'num_steps': 24, 'h_stddev': 0, 'v_stddev': 0,
            'h_mean': torch.tensor(math.pi / 2).to(DEV), 'v_mean': torch.tensor(math.pi / 2).to(DEV),
            'hierarchical_sample': False, 'sample_dist': None, 'clamp_mode': 'relu', 'nerf_noise': 0, 'fade_steps': 10000,
            'z_app_lambda': 0, 'z_geo_lambda': 0, 'pos_lambda': 0, 'tok_interval': 2000, 'tok_v': 0.6, 'betas': (0, 0.9),
            'fill_mode': 'eval_seg_padding_background', '_rng': ReplayRng(draws, DEV), 'precision': precision}


def _inversion_grads(gen, ws, draws, precision, d_pixels, chunk_points, monkeypatch):
    """forward_with_frequencies(w + offsets) and the gradients of sum(frame * d_pixels) w.r.t. the four FiLM offsets and
    the field parameters, with backward.CHUNK_POINTS = chunk_points.  -> (frame, d film in the table's layout with the
    frequency rows times 15, {parameter name: gradient}, the chunk sizes the backward ran)."""
    siren = gen.siren
    monkeypatch.setattr(backward, "CHUNK_POINTS", chunk_points)
    chunks = []
    run_chunk = backward._FieldBackward._chunk

    def spy(self, points, *args):
        chunks.append(points.shape[1])
        return run_chunk(self, points, *args)

    monkeypatch.setattr(backward._FieldBackward, "_chunk", spy)
    offsets = [torch.zeros_like(w).requires_grad_(True) for w in ws]
    params = backward.FieldWeights(siren).parameters()
    names = {id(p): k for k, p in siren.named_parameters()}
    frame, _ = gen.forward_with_frequencies(*[w + o for w, o in zip(ws, offsets)], **_inversion_options(draws, precision))
    gr = torch.autograd.grad((frame * d_pixels).sum(), offsets + params)
    d_fg, d_fa, d_pg, d_pa = gr[:4]
    d_film = torch.stack([torch.cat([d_fg.reshape(1, -1, 256), d_fa.reshape(1, -1, 256)], 1),
                          torch.cat([d_pg.reshape(1, -1, 256), d_pa.reshape(1, -1, 256)], 1)], 2)
    return frame.detach(), d_film, {names[id(p)]: t for p, t in zip(params, gr[4:])}, chunks


def _check(tag, d_film, grads, want_film, want, bound):
    errs = _grad_errors(d_film, grads, want_film, want)         # (which also asserts one gradient set)
    worst = max(errs, key=errs.get)
    print("inversion %s: worst %s %.3g (bound %g)" % (tag, worst, errs[worst], bound))
    assert errs[worst] <= bound, {k: "%.2e" % v for k, v in errs.items() if v > bound}
    return errs[worst]


@gpu
@pytest.mark.parametrize("precision", ["guard", "exact"])
def test_inversion_backward_vs_fp64(monkeypatch, precision):
    """The inversion's differentiable render (model B, 1 x 256², flat 24 steps, the script's options) w.r.t. FiLM offsets
    and every field parameter, with the library's CHUNK_POINTS (three chunks of 524,280 points and a trailing chunk of
    24, one ray): against the float64 chain on a seeded upstream gradient, and on an upstream gradient on the trailing
    ray alone (a dropped last chunk leaves those gradients zero); then with the image split into two equal chunks,
    within LAYOUT_BOUND of the first run."""
    need_free(23 if precision == "exact" else 15, "the %s inversion backward" % precision)    # peaks 21.8 / 13.3 GB
    if precision == "exact":
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # exact mode's torch.mm stays fp32
    gen = _generator("B")
    siren = gen.siren
    r, s = 256, 24
    n = r * r
    ppb = n * s
    step = backward.CHUNK_POINTS // s * s
    assert ppb > backward.CHUNK_POINTS and ppb % step == 24, (ppb, backward.CHUNK_POINTS)
    g = torch.Generator(device=DEV).manual_seed(24)
    with torch.no_grad():
        fg, pg = siren.geo_mapping_network(torch.randn(1, 256, generator=g, device=DEV))
        fa, pa = siren.app_mapping_network(torch.randn(1, 256, generator=g, device=DEV))
    ws = [fg, fa, pg, pa]
    draws = [("rand", torch.rand(1, n, s, 1, generator=g, device=DEV)), ("randn", torch.randn(1, n, s, 1, generator=g, device=DEV))]
    c = siren.field_spec().out_dim
    d_pixels = torch.randn((1, c - 1, r, r), generator=g, device=DEV) / n
    frame, d_film, grads, chunks = _inversion_grads(gen, ws, draws, precision, d_pixels, backward.CHUNK_POINTS, monkeypatch)
    print("inversion %s: backward chunks %s (points per chunk; the last is one ray)" % (precision, chunks))
    assert chunks == [step] * (ppb // step) + [24], chunks
    # the render's own intermediates, on the same FiLM table and draws
    with torch.no_grad():
        film = siren.film_table(*ws)
        rd = ops.make_render_desc(batch=1, img_size=r, num_steps=s, hierarchical=False, clamp_mode="relu", nerf_noise=0,
                                  fov=12, precision=precision)
        x_lin, y_lin, z_lin = ops.ray_tables(r, s, 0.88, 1.12, DEV)
        c2w = ops.camera_poses(1, None, 0, 0, math.pi / 2, math.pi / 2, None, torch.device(DEV))[0]
        st = ops.render_forward_stages(siren, rd, film, x_lin, y_lin, z_lin, c2w, draws[0][1].contiguous(), None, None,
                                       draws[1][1])
    assert torch.equal(st["pixels"], frame), "render_forward_stages differs from the inversion's render"
    assert st["points_f"] is None
    bound = FIELD_BOUND["exact" if precision == "exact" else "default"]

    def chain(d):
        want_film, want = camera_chain_vjp(siren, film, st, False, _opt("relu"), None, d)
        want_film = want_film.clone()
        want_film[:, :, 0] *= 15                     # d offset = 15 d film of the frequency rows
        return want_film, want

    worst = _check("%s, seeded upstream gradient" % precision, d_film, grads, *chain(d_pixels), bound)
    d_last = torch.zeros_like(d_pixels)
    d_last[0, :, -1, -1] = torch.randn(c - 1, generator=g, device=DEV)
    _, d_film_l, grads_l, _ = _inversion_grads(gen, ws, draws, precision, d_last, backward.CHUNK_POINTS, monkeypatch)
    worst_l = _check("%s, the trailing ray alone" % precision, d_film_l, grads_l, *chain(d_last), bound)
    del st
    _, d_film2, grads2, chunks2 = _inversion_grads(gen, ws, draws, precision, d_pixels, ppb // 2, monkeypatch)
    assert chunks2 == [ppb // 2] * 2, chunks2
    inv = _grad_errors(d_film, grads, d_film2, grads2)
    w = max(inv, key=inv.get)
    print("inversion %s: two halves against the library's chunks: worst %s %.3g (LAYOUT_BOUND %g)" % (precision, w, inv[w],
                                                                                                      LAYOUT_BOUND))
    assert inv[w] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}
    print("inversion %s: fp64 %.3g, trailing ray %.3g, layout %.3g" % (precision, worst, worst_l, inv[w]))


# --------------------------------------------------------------------------------------------
# CPU: the subset references are the full ones restricted, and the subset sees a wrapped tail
# --------------------------------------------------------------------------------------------
def _cpu_x():
    """The stage dict of the oracle's render (model D, 2 x 8² rays, 12 + 12 samples, noise 0.5), as check_composite
    reads it."""
    st, draws, out = _cpu_render()
    o = _opt("relu", noise=0.5)
    return dict(opt=o, hier=True, raw_c=st["raw_coarse"], z_c=st["z_coarse"][..., 0], raw_f=st["raw_fine"],
                z_f=st["z_fine"][..., 0], noise_f=draws[5][..., 0], b=2, n=64, s=12)


def _cpu_subset():
    return ray_subset(8, edge=4, n_random=8, device="cpu")


def _resample_rows(b, n, rays):
    return (torch.arange(b)[:, None] * n + rays).reshape(-1)


def test_subset_references_equal_the_full_ones():
    """On the oracle's small render, every float64 reference on a ray subset equals the full-image reference restricted
    to that subset (to 1e-12: only the batching of the float64 sums differs)."""
    rays = _cpu_subset()
    assert rays[-1].item() == 63 and 4 < len(rays) < 64
    errs = {}
    args = _cpu_ray_inputs()
    full, sub = ray_setup_ref(*args), ray_setup_ref(*args, rays=rays)
    errs["ray set-up"] = max((f[:, rays] - s_).abs().max().item() for f, s_ in zip(full[:3], sub[:3]))
    errs["origins"] = (full[3] - sub[3]).abs().max().item()
    sig, z, u = fs._cpu_resample_inputs()
    rows = _resample_rows(2, 64, rays)
    rf, rs = resample_ref(sig, z, "relu", u), resample_ref(sig[rows], z[rows], "relu", u[rows])
    errs["resample"] = max((rf[k][rows] - rs[k]).abs().max().item() for k in ("cdf", "bins", "total", "z"))
    assert torch.equal(rf["inds"][rows], rs["inds"])
    x = _cpu_x()
    siren = fs._siren("D", "cpu")
    film = _film(siren, 2, 21)
    st, _, _ = _cpu_render()
    dirs = st["dirs"]
    f_full = field_ref(siren, st["points_coarse"].reshape(2, -1, 3), pass_dirs(dirs, 12, False), film)[0]
    f_full = f_full.reshape(st["raw_coarse"].shape)
    f_sub = field_ref(siren, st["points_coarse"][:, rays].reshape(2, -1, 3), pass_dirs(dirs[:, rays], 12, False), film)[0]
    errs["points"] = (f_full[:, rays].reshape(f_sub.shape) - f_sub).abs().max().item()
    for i in range(2):
        a, b_ = composite_subset_ref(x, i, None), composite_subset_ref(x, i, rays)
        errs["composite%d" % i] = max((a[0][:, :, rays] - b_[0]).abs().max().item(),
                                      *((p[:, rays] - q).abs().max().item() for p, q in zip(a[1:], b_[1:])))
    print("subset vs full references: %s" % errs)
    assert max(errs.values()) <= 1e-12, errs


def test_wrapped_tail_rays_exceed_every_bound():
    """A kernel whose offsets wrap at float 2^29 of a 512² x 96 x 22 buffer reads the rows of other rays for the
    buffer's last rays.  On the oracle's small render, the same wrap (WRAP_FRACTION of the buffer) applied to the
    float64 side moves ray set-up, the point network, resampling, the GUARD far densities and the compositor, measured
    on what each check compares (the ray subset; for GUARD its refined set), past ten times their bounds."""
    rays = _cpu_subset()
    st, draws, _ = _cpu_render()
    moved = {}
    pts, z, dirs, org = ray_setup_ref(*_cpu_ray_inputs())
    for tag, t in (("ray set-up points", pts), ("ray set-up depths", z)):
        bad, tail = wrap_rows(t)
        assert len(tail) and all(int(g) % 64 in rays.tolist() for g in tail), tail
        moved[tag] = (bad[:, rays] - t[:, rays]).abs().max().item() / RAY_BOUND
    siren = fs._siren("D", "cpu")
    film = _film(siren, 2, 21)
    raw = field_ref(siren, st["points_coarse"].reshape(2, -1, 3), pass_dirs(st["dirs"], 12, False), film)[0]
    raw = raw.reshape(st["raw_coarse"].shape)
    moved["points"] = (wrap_rows(raw)[0][:, rays] - raw[:, rays]).abs().max().item() / FWD_BOUND["fast"]
    # check_guard compares the refined far samples with float64 (the rest bit for bit with a fast pass), so the wrap is
    # measured on its refined set; at 512² its probe rays 256000, 258048 and 260096 lie past the wrap point
    far, noise_far = raw[:, :, -1, -1], draws[5][:, :, -1, 0].double() * 0.5
    sel = guard_refined(far, far + noise_far, ops.DEFAULT_GUARD_TAU)
    moved["guard far densities"] = (wrap_rows(raw)[0][:, :, -1, -1] - far)[sel].abs().max().item() / FWD_BOUND["exact"]
    n_rays = 512 * 512
    probes = guard_refined(torch.ones(1, n_rays), torch.ones(1, n_rays), 0.0).nonzero()[:, 1]
    past = probes[probes * 96 * 22 >= int(WRAP_FRACTION * n_rays * 96 * 22)]
    assert past.tolist() == [256000, 258048, 260096], past
    sig, zc, u = fs._cpu_resample_inputs()
    rows = _resample_rows(2, 64, rays)
    good = resample_ref(sig, zc, "relu", u)
    bad_z = wrap_rows(good["z"].reshape(2, 64, 12))[0].reshape(128, 12)
    moved["resample"] = cdf_errors({k: v[rows] for k, v in good.items()}, bad_z[rows], u[rows])[0].max().item()
    x = _cpu_x()
    bad_x = dict(x, raw_c=wrap_rows(x["raw_c"])[0], raw_f=wrap_rows(x["raw_f"])[0])
    comp = 0.0
    for i in range(2):
        a, b_ = composite_subset_ref(x, i, rays), composite_subset_ref(bad_x, i, rays)
        comp = max(comp, *((p - q).abs().max().item() for p, q in zip(a, b_)))
    moved["composite"] = comp / COMPOSITE_FWD_BOUND
    print("wrapped tail rays, x the bound: %s" % {k: "%.3g" % v for k, v in moved.items()})
    assert min(moved.values()) > 10, moved
