"""Renders with more than 64 samples per pass, up to the library's bound of 256 (512 merged): the reference's
``--ray_step_multiplier`` 3 and 4 on the production curriculum's 24 steps, and beyond.

CPU: the oracle against the reference's goldens (tests/golden/make_many_samples_goldens.py, cases in
tests/_many_samples.py); the descriptor check's bound.  GPU: the goldens end to end in exact and default precision,
the rays-in render, and gradients; every per-ray stage against float64 at S = 65 to 256, straddling the resampler's
switch from 128-ray to 64-ray blocks (S > 128) and the compositing backward's switch to rows read from global memory
(n C too large to stage); a CUDA-graph replay at S = 128.  The float64 checks are those of
test_gpu_fp64_forward_stages.py, test_gpu_fp64_rays.py and test_gpu_fp64_reference.py, with their bounds.
"""
import contextlib
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import _cases
import _many_samples as ms
import _point_forward as pf
import test_gpu_fp64_forward_stages as fs
import test_gpu_fp64_rays as fr
import test_gpu_fp64_reference as fref
import test_gpu_fp64_train_grads as tg
from _fp64 import _film, _opt, _siren, composite_ref
from fenerf_b200 import _lib, ops
from fenerf_b200.generators import volumetric_rendering as vr

gpu = pytest.mark.gpu
DEV = "cuda:0"
#: the oracle against the reference's goldens (tests/test_oracle.py's cross-host tolerance)
TOL = 2e-5


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ms.CASES, ids=lambda c: c.name)
def test_oracle_matches_the_reference_golden(case):
    import _harness
    gold = np.load(_cases.golden_path(case))
    run = _harness.oracle_run(case, keep_stages=False)
    got = run["out"]["pixels"].numpy()
    assert got.shape == gold["pixels"].shape
    err = np.abs(got - gold["pixels"]).max()
    assert err <= TOL, "max|oracle - reference| = %g" % err
    if "poses" in gold.files:
        assert np.abs(run["out"]["poses"].numpy() - gold["poses"]).max() <= 1e-6
    if "depth_map" in gold.files:
        r = case.cfg["img_size"]
        assert np.abs(run["out"]["depth"].reshape(case.batch, r, r).numpy() - gold["depth_map"]).max() <= TOL


@pytest.mark.parametrize("name", [c.name for c in ms.POINT_CASES])
def test_point_forward_oracle_matches_the_reference_golden(name):
    case = next(c for c in ms.POINT_CASES if c.name == name)
    gold = np.load(pf.golden_path(case))
    run = pf.oracle_run(case)
    assert run["out"]["pixels"].shape == gold["pixels"].shape
    err = (run["out"]["pixels"] - torch.from_numpy(gold["pixels"])).abs().max().item()
    assert err <= 1e-6, err


def _rays_call(num_steps, workspace_bytes=256):
    """fenerf_render_rays with non-NULL pointers that are never dereferenced: every check returns before the device."""
    lib = _lib.lib()
    rd = ops.make_rays_desc(batch=1, n_rays=16, num_steps=8, hierarchical=True, clamp_mode="relu", nerf_noise=0.0)
    rd.num_steps = num_steps
    fd = _lib.FieldDesc(trunk_layers=8, color_layers=1, label_dim=0, grid_channels=0, grid_res=0, out_dim=4,
                        input_scale=1.0, reserved=0)
    f = 1 << 20
    rc = lib.fenerf_render_rays(C.byref(rd), C.byref(fd), f, f, f, f, 1, f, f, f, f, f, f, f, 0, 0, f, workspace_bytes, None)
    return rc, lib.fenerf_last_error().decode(), lib.fenerf_rays_workspace_bytes(C.byref(rd), C.byref(fd), 1)


@pytest.mark.parametrize("num_steps,message", [(1, "num_steps 1 outside [2, 256]"), (257, "num_steps 257 outside [2, 256]")])
def test_descriptor_check_refuses_num_steps_outside_the_bound(num_steps, message):
    rc, err, _ = _rays_call(num_steps)
    assert rc == -1 and message in err, (rc, err)


@pytest.mark.parametrize("num_steps", [65, 128, 129, 256])
def test_descriptor_check_accepts_num_steps_up_to_256(num_steps):
    """Past the descriptor check, the call stops at the (too small) workspace; the planner's size grows with S."""
    rc, err, need = _rays_call(num_steps)
    assert rc == -4 and "workspace too small" in err, (rc, err)
    assert need > _rays_call(num_steps - 1)[2]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the goldens
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision,bound", [("exact", 2e-4), ("guard", 1e-3)])
@pytest.mark.parametrize("case", ms.CASES, ids=lambda c: c.name)
def test_goldens(case, precision, bound):
    """The generator API against the reference's output; rays whose far sample sits on the relu step (|sigma| below
    _harness.ILL_TAU, ill-conditioned for any fp32 render) are excluded, as the stock cases' tests do."""
    import _harness
    run = _harness.oracle_run(case)
    gold = np.load(_cases.golden_path(case))
    l0 = _lib.launch_count()
    _, pixels, poses, depth_map = _harness.end_to_end(case, run, precision)
    assert _lib.launch_count() > l0
    err = (pixels - torch.from_numpy(gold["pixels"])).abs()
    ill = _harness.ill_conditioned_pixels(case, run).unsqueeze(1).expand_as(err)
    assert int(ill[:, 0].sum()) <= max(2, 0.002 * ill[:, 0].numel())
    print("%s %s: max|gpu - reference| = %.2e (%d rays excluded)" % (case.name, precision, err[~ill].max(),
                                                                     int(ill[:, 0].sum())))
    assert err[~ill].max() <= bound
    if poses is not None:
        assert (poses - torch.from_numpy(gold["poses"])).abs().max() <= 1e-5


@gpu
@pytest.mark.parametrize("precision,bound", [("exact", 2e-4), ("guard", 1e-3), ("split", 2e-4)])
@pytest.mark.parametrize("name", [c.name for c in ms.POINT_CASES])
def test_point_forward_goldens(name, precision, bound):
    case = next(c for c in ms.POINT_CASES if c.name == name)
    run = pf.oracle_run(case)
    gold = torch.from_numpy(np.load(pf.golden_path(case))["pixels"])
    gen = _cases.build_mirror(pf.base_case(case), DEV)
    rays = {k: v.to(DEV) for k, v in run["rays"].items()}
    with torch.no_grad():
        px = gen.point_forward(rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"], rays["z_vals"],
                               *[z.to(DEV) for z in run["latents"]],
                               **dict(pf.call_kwargs(case), precision=precision, _rng=vr.ReplayRng(run["draws"], DEV)))
    err = (px.cpu() - gold).abs().max().item()
    print("%s %s: max|gpu - reference| = %.2e" % (name, precision, err))
    assert px.shape == gold.shape and err <= bound


@gpu
@pytest.mark.parametrize("precision,rel,kink", [("exact", 5e-4, 1e-2), ("guard", 2e-2, 0.3)])
def test_gradients_against_the_reference(precision, rel, kink):
    """forward() at 96 + 96 with autograd: the bounds of the stock gradient goldens (test_gpu_parity.py) and, in the
    default precision, the density bias measured against the density head's weight gradient (test_point_forward.py)."""
    import _harness
    case = ms.CASE_BY_NAME[ms.GRAD_CASE]
    run = _harness.oracle_run(case, keep_stages=False)
    gold = np.load(ms.grad_golden_path())
    gen = _cases.build_mirror(case, DEV)
    latents = [z.to(DEV).requires_grad_(True) for z in run["latents"]]
    pixels, _ = gen(*latents, **dict(case.cfg, _rng=vr.ReplayRng(run["draws"], DEV), precision=precision))
    loss = (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum()
    assert abs(loss.item() - float(gold["loss"])) <= 2e-3 * max(1.0, abs(float(gold["loss"])))
    loss.backward()
    got = pf.grad_record(latents, dict(gen.named_parameters()))
    keys = list(gold.files)
    if precision != "exact":
        bias = "siren.final_layer.bias"
        scale = np.abs(gold["siren.final_layer.weight"]).max()
        berr = (got[bias].detach().cpu() - torch.from_numpy(gold[bias])).abs().max().item() / scale
        print("final_layer.bias: %.2e of the weight gradient's largest entry" % berr)
        assert berr <= kink
        keys.remove(bias)
    kept = {k: gold[k] for k in keys}
    gold = type("Gold", (), {"files": keys, "__getitem__": lambda self, k: kept[k]})()
    worst = _harness.compare_grads(gold, got, rel=rel, kink_rel=kink)
    print("forward %s, 96 + 96: %s" % (precision, {k: "%.1e" % v for k, v in worst.items()}))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every per-ray stage against float64
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _registered(module, name, spec):
    """`name` in `module`'s render matrix while the block runs (its render() and checks are reused as they are)."""
    module._RENDERS[name] = spec
    try:
        yield
    finally:
        del module._RENDERS[name]


def _resample_pass(sms, s):
    """Rays one pass of the resampler's grid-stride loop covers at S: blocks <= num_sms * 8 of resample_block(S) rays."""
    return sms * 8 * (128 if s <= 128 else 64)


#: camera renders (fenerf_render_forward), as test_gpu_fp64_forward_stages._RENDERS: (model, batch (None: enough rays
#: for two passes of every grid-stride loop), R, S, hierarchical, options, precision, lock_view_dependence)
_RENDERS = {
    "s65-B": ("B", 2, 64, 65, True, _opt("relu", noise=0.5), "guard", False),
    "s96-D": ("D", 2, 64, 96, True, _opt("softplus", noise=0.3, softmax=True), "fast", False),
    "s128-B": ("B", 2, 64, 128, True, _opt("relu"), "guard", False),
    "s129-A": ("A", 2, 64, 129, True, _opt("relu", noise=0.5, black_back=True), "exact", False),
    "s200-D32": ("D32", 1, 64, 200, True, _opt("relu", softmax=True, last_back=True), "guard", False),
    "s256-B": ("B", 1, 64, 256, True, _opt("relu"), "guard", False),
    "s96-J": ("J", 1, 48, 96, True, _opt("relu", noise=0.5), "guard", False),
    "s256-K": ("K", 1, 32, 256, True, _opt("relu", softmax=True), "guard", False),
    "flat256-A": ("A", 2, 40, 256, False, _opt("softplus", white_back=True), "guard", True),
    "fill96-B-seg_padding-grey": ("B", 1, 64, 96, True, _opt(fill_mode="seg_padding_background", fill_color="grey"),
                                  "guard", False),
    "fill256-D-weight-softmax": ("D", 1, 48, 256, True, _opt(fill_mode="weight", softmax=True), "guard", False),
    "loop128-A": ("A", None, 256, 128, True, _opt("relu"), "guard", False),
    "loop256-A": ("A", None, 256, 256, True, _opt("relu", noise=0.5), "guard", False),
}


@gpu
@pytest.mark.parametrize("name", list(_RENDERS))
def test_forward_stages_vs_fp64(name):
    """Ray set-up, the resampler (bit for bit against the stand-alone entry, and in CDF space), the GUARD refinement and
    the compositor (against float64, and the stand-alone fenerf_composite bit for bit on the render's inputs).  The loop
    renders hold more rays than one pass of the resampler, the compositor and the guard scan covers on this device, at
    both resampler block sizes."""
    with _registered(fs, name, _RENDERS[name]):
        x = fs.render(name)
        if name.startswith("loop"):
            caps = dict(fs.one_pass_rays(fs._sms(), x["raw_c"].shape[-1]), resample=_resample_pass(fs._sms(), x["s"]))
            assert all(x["b"] * x["n"] > v for v in caps.values()), (x["b"], x["n"], caps)
        res = dict(rays=fs.check_ray_setup(x))
        if x["hier"]:
            res.update(fs.check_resample(x))
        if x["rd"].precision == _lib.PRECISION["guard"]:
            res["guard"] = fs.check_guard(x, ops.DEFAULT_GUARD_TAU)
        res.update(fs.check_composite(x))
        fs._far_fp64.cache_clear()
    print("forward stages %s (B=%d, S=%d): %s" % (name, x["b"], x["s"], res))


#: rays-in renders (fenerf_render_rays), as test_gpu_fp64_rays._RENDERS (+ directions 'sample' / 'ray')
_RAYS_RENDERS = {
    "s65-B": ("B", 2, 64, 65, True, _opt("relu"), "guard", "sample", False),
    "s128-D32": ("D32", 2, 48, 128, True, _opt("relu", noise=0.5, softmax=True, last_back=True), "exact", "sample", False),
    "s129-B": ("B", 2, 48, 129, True, _opt("relu"), "fast", "ray", False),
    "s200-K": ("K", 1, 32, 200, True, _opt("relu", softmax=True), "guard", "sample", False),
    "s256-B": ("B", 1, 48, 256, True, _opt("softplus", noise=0.5), "guard", "sample", False),
    "loop256-A": ("A", None, 256, 256, True, _opt("relu"), "guard", "sample", False),
}


@gpu
@pytest.mark.parametrize("name", list(_RAYS_RENDERS))
def test_rays_stages_vs_fp64(name):
    """The rays-in render's coarse pass, resampler (depths, fine points and the fine-direction slots, which at S > 255
    would no longer fit a byte), GUARD refinement, fine pass and ray-major compositor."""
    with _registered(fr, name, _RAYS_RENDERS[name]):
        x = fr.render(name)
        if name.startswith("loop"):
            caps = dict(fs.one_pass_rays(fr._sms(), x["c"]), resample=_resample_pass(fr._sms(), x["s"]))
            assert all(x["b"] * x["n"] > v for v in caps.values()), (x["b"], x["n"], caps)
        res = fr.check_coarse(x)
        res.update(fr.check_resample(x))
        fr.check_fine(x)
        res.update(fr.check_composite(x))
    print("rays stages %s (B=%d, N=%d, S=%d): %s" % (name, x["b"], x["n"], x["s"], res))


_COMPOSITE_MODEL = {4: "A", 22: "D", 32: "D32", 65: "J", 129: "K"}


@functools.lru_cache(maxsize=None)
def _composite_inputs(c, steps, hier, b=3, r=37):
    """test_gpu_fp64_reference._composite_inputs for every width: a field's exact outputs on render points, fine depths
    drawn inside the ray, some exactly equal to coarse ones."""
    siren = _siren(_COMPOSITE_MODEL[c], DEV)
    seed = 100 * c + steps
    film = _film(siren, b, seed)
    pts_c, z_c, dirs, org = fref._render_points(b, r, steps, seed)
    n = r * r
    with torch.no_grad():
        raw_c = ops.siren_points(siren, pts_c.reshape(b, n * steps, 3).to(DEV), film, dirs.to(DEV), precision="exact")
        out = dict(raw_c=raw_c.reshape(b, n, steps, c).contiguous(), z_c=z_c.to(DEV).contiguous(), raw_f=None, z_f=None)
        if hier:
            g = torch.Generator().manual_seed(seed)
            z_f = 0.88 + 0.24 * torch.sort(torch.rand(b, n, steps, generator=g), -1)[0]
            z_f[:, ::5, 0] = z_c[:, ::5, steps // 2]
            z_f[:, 1::7, -1] = z_c[:, 1::7, -1]
            pts_f = org.unsqueeze(2) + dirs.unsqueeze(2) * z_f.unsqueeze(-1)
            raw_f = ops.siren_points(siren, pts_f.reshape(b, n * steps, 3).to(DEV), film, dirs.to(DEV), precision="exact")
            out.update(raw_f=raw_f.reshape(b, n, steps, c).contiguous(), z_f=z_f.to(DEV).contiguous())
    return out


_STANDALONE_OPTS = {"relu": _opt("relu"), "softplus_noise": _opt("softplus", noise=0.5),
                    "softplus_last_back": _opt("softplus", last_back=True), "white_back": _opt("relu", white_back=True),
                    "black_back": _opt("relu", black_back=True), "softmax": _opt("relu", softmax=True),
                    "seg_padding_grey_softmax": _opt(fill_mode="seg_padding_background", fill_color="grey", softmax=True),
                    "eval_seg_padding_white": _opt(fill_mode="eval_seg_padding_background", fill_color="white"),
                    "debug": _opt(fill_mode="debug"), "weight_debug": _opt(fill_mode="weight_debug"),
                    "eval_white_back": _opt(fill_mode="eval_white_back"), "weight": _opt(fill_mode="weight")}
#: merged samples: 65 + 65, a flat 200, 128 + 128 and 129 + 129 (the resampler's switch), 256 + 256
_STANDALONE_N = [(130, True), (200, False), (256, True), (258, True), (512, True)]


def composite_bound(n):
    """COMPOSITE_FWD_BOUND, set on n <= 128 merged samples, grown with n: the fp32 rounding of the compositor's sums over
    the samples (transmittance product, weight and channel sums) accumulates linearly in n.  Measured on an H100 80GB
    HBM3: 1.5e-5 at n = 512 (C = 4, black_back), 1.05e-5 at n = 200."""
    return fs.COMPOSITE_FWD_BOUND * max(1.0, n / 128)


@gpu
@pytest.mark.parametrize("opt", list(_STANDALONE_OPTS))
@pytest.mark.parametrize("c", [4, 22, 32, 65, 129])
@pytest.mark.parametrize("n,hier", _STANDALONE_N, ids=["n%d" % n for n, _ in _STANDALONE_N])
def test_standalone_composite_vs_fp64(n, hier, c, opt):
    """fenerf_composite (samples in any order: above 384 merged samples its sort positions need the shared-memory opt-in)
    against float64 under every compositing and fill option, with the stable fine-first merge order."""
    steps = n // 2 if hier else n
    xi = _composite_inputs(c, steps, hier, b=2, r=24)
    o = _STANDALONE_OPTS[opt]
    g = torch.Generator().manual_seed(n + c)
    noise = torch.randn(2, 24 * 24, n, generator=g).to(DEV) if o["noise"] else None
    rd = ops.make_render_desc(batch=2, img_size=24, num_steps=steps, hierarchical=hier, clamp_mode=o["clamp"],
                              nerf_noise=o["noise"], fov=12, last_back=o["last_back"], white_back=o["white_back"],
                              black_back=o["black_back"], fill_mode=o["fill_mode"], fill_color=o["fill_color"],
                              softmax_label=o["softmax"])
    px, depth, wsum, weights, sidx = ops.composite(rd, xi["raw_c"], xi["z_c"], xi["raw_f"], xi["z_f"], noise,
                                                   want_weights=True, want_sort_idx=True)
    if hier:
        order = torch.sort(torch.cat([xi["z_f"], xi["z_c"]], 2), dim=2, stable=True)[1]
        assert torch.equal(sidx.long(), order), "merge order is not the stable fine-first one"
    px64, depth64, wsum64, w64 = composite_ref(xi["raw_c"].double(), xi["z_c"], xi["raw_f"].double() if hier else None,
                                               xi["z_f"], noise, o, full=True)
    keep = torch.ones_like(wsum64, dtype=torch.bool).reshape(-1)
    if o["fill_mode"] is not None:
        keep = ((wsum64 - 0.9).abs() >= fs.FILL_TIE).reshape(-1)
        assert int((~keep).sum()) <= max(1, fs.FILL_TIE_FRACTION * keep.numel())
    errs = dict(pixels=(px.double() - px64).abs().amax(1).reshape(-1)[keep].max().item(),
                depth=(depth[..., 0].double() - depth64).abs().max().item(),
                weights_sum=(wsum[..., 0].double() - wsum64).abs().max().item(),
                weights=(weights[..., 0].double() - w64).abs().max().item())
    print("stand-alone composite n=%d C=%d %s: %s" % (n, c, opt, errs))
    assert max(errs.values()) <= composite_bound(n), errs


#: (n merged, hierarchical, C, option), both entries.  The narrow kernel stages eight warps' raw blocks up to 227 KB
#: (C = 4 up to n = 512); beyond (n = 256 from C = 22, n = 512 from C = 8) the narrow fields take the wide kernel
_BACKWARD = [(n, hier, c, o) for n, hier in [(130, True), (256, False), (256, True), (400, True), (512, True)]
             for c, o in [(4, "relu"), (22, "softplus_noise"), (32, "softmax"), (65, "relu"), (129, "softmax")]]
_BACKWARD += [(512, True, 4, "softplus_last_back"), (512, True, 22, "white_back"), (258, True, 4, "black_back")]


@gpu
@pytest.mark.parametrize("n,hier,c,opt,entry", [pytest.param(n, h, c, o, e, id="n%d-%s-C%d-%s-%s" % (
    n, "hier" if h else "flat", c, o, e)) for n, h, c, o in _BACKWARD for e in fref.entries(h)])
def test_composite_backward_vs_fp64(n, hier, c, opt, entry):
    """fenerf_composite_backward and fenerf_composite_backward_rays against the float64 VJP (COMPOSITE_BOUND); the
    ray-major entry bit for bit equal to the NCHW one on the same upstream values.  Narrow fields whose raw block does
    not fit eight warps' shared memory (n = 256 from C = 22, n = 512 from C = 8) go through the wide kernel."""
    steps = n // 2 if hier else n
    x = _composite_inputs(c, steps, hier)
    o = _STANDALONE_OPTS[opt]
    g = torch.Generator().manual_seed(n * 64 + c)
    noise = torch.randn(3, 37 * 37, n, generator=g).to(DEV) if o["noise"] else None
    errs = fref.composite_backward_errors(o, steps, hier, x, noise, g, entry)[1]
    print("composite backward %s n=%d C=%d %s: %s" % (entry, n, c, opt, errs))
    assert not fref.over_bounds(errs), errs


# ---------------------------------------------------------------------------------------------------------------------
# GPU: gradients of the rays-in render at the bound, and a captured graph
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("model,s", [("B", 256), ("K", 160)])
def test_rays_gradients_vs_fp64(monkeypatch, model, s):
    """render_rays_with_grad at S = 256 (B: the narrow compositing backward's rows from global memory) and S = 160 (K):
    d film and every parameter gradient against the float64 VJP of the chain (test_gpu_fp64_rays.py's bound)."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    siren = fr._field(model)
    b, r = 1, 24
    n = r * r
    g = torch.Generator(device=DEV).manual_seed(4000 + s)
    rays = fr.edit_rays(*fr.camera_rays(b, r, s, g), g, True)
    o = _opt("relu", noise=0.5)
    draws = (torch.randn(b, n, s, generator=g, device=DEV), torch.rand(b * n, s, generator=g, device=DEV),
             torch.randn(b, n, 2 * s, generator=g, device=DEV))
    rd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=s, hierarchical=True, clamp_mode=o["clamp"], nerf_noise=o["noise"],
                            precision="exact")
    film = _film(siren, b, 4000 + s)
    c = siren.field_spec().out_dim
    weights = torch.randn(b, n, c - 1, generator=g, device=DEV)
    px, d_film, grads = fr.rays_grads(siren, rd, film, rays, draws, weights)
    with torch.no_grad():
        st = ops.render_rays_stages(siren, rd, film, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                                    rays["z_vals"], *draws)
    assert torch.equal(st["pixels"], px)
    want_film, want = fr.chain_vjp(siren, film, st, rays["dirs"].reshape(b, n * s, 3), st["dirs_f"], rays["z_vals"],
                                   draws[2], o, weights)
    errs = fref._grad_errors(d_film, {k: grads[k] for k in want}, want_film, want)
    worst = max(errs, key=errs.get)
    print("rays gradients %s S=%d: worst %s %.3g" % (model, s, worst, errs[worst]))
    assert errs[worst] <= fref.FIELD_BOUND["exact"], {k: "%.2e" % v for k, v in errs.items() if v > fref.FIELD_BOUND["exact"]}


@gpu
def test_camera_render_with_grad_at_256_steps(monkeypatch):
    """backward.render_with_grad at S = 256 (512 merged: the compositing backward reads the raw rows from global
    memory), model B, one image of 32², in exact and default precision: the differentiable render's pixels are the
    no_grad render's, and d film and every parameter gradient are within FIELD_BOUND of the float64 VJP of the camera
    render's chain on its own intermediates (test_gpu_fp64_train_grads.py)."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    for precision in ("exact", "guard"):
        x = tg.make_render("B", 1, 32, 256, _opt("relu"), precision, False, False, 256)
        px, d_film, grads = tg.camera_grads(x, x["d_pixels"])
        st = tg.stages(x)
        assert torch.equal(st["pixels"], px), "render_forward_stages differs from the differentiable render"
        want_film, want = tg.chain(x, st, x["d_pixels"])
        tg.check_against_chain(x, "S=256 %s" % precision, d_film, grads, want_film, want)


@gpu
def test_graphed_render_at_128_steps():
    """GraphedRender captures a render at S = 128 (the resampler's and compositor's shared-memory opt-ins happen at the
    first, eager launch) and its replay equals the eager render on the same draws."""
    from fenerf_b200.graphs import GraphedRender
    case = _cases.Case("graph128", "B", 2, 0, _cases._cfg(img_size=32, num_steps=128, h_stddev=0.3, v_stddev=0.155,
                                                           nerf_noise=0.0))
    gen = _cases.build_mirror(case, DEV)
    torch.manual_seed(5)
    z = [torch.randn(2, 256, device=DEV) for _ in range(2)]
    md = dict(case.cfg)
    graphed = GraphedRender(gen, z, md)
    state = torch.cuda.get_rng_state(DEV)
    out = graphed(*z)[0].clone()
    torch.cuda.set_rng_state(state, DEV)
    with torch.no_grad():
        eager = gen(*z, **md)[0]
    assert torch.equal(out, eager)
