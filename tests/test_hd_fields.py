"""The feature-head fields of the reference's neural-renderer path: SPATIALSIRENBASELINEHD (model "J", 65 channels) and
SPATIALSIRENSEMANTICHD (model "K", 129 channels), forward and backward (FENERF_FIELD_FEATURE_HEAD).

CPU: the mirror classes against the reference (init, state-dict keys, parameter order, pickles), the FiLM table, the
oracle (oracle.render_oracle.label_film_field_eval) against the reference's goldens, the flags word and packed sizes on
the host, and float64 restatements of the wide heads and the wide compositor that pass gradcheck.
GPU: end to end against the reference's goldens (exact <= 2e-4, default <= 1e-3), both point-network kernels against
float64 over the tile schedules, the GUARD refinement on a 64-label field, the wide compositor forward and backward
against float64 up to 64 + 64 samples and 129 channels, the stand-alone compositor bit-identical to the render's, the
gradients and the inversion gradients against the reference's autograd, and an ImplicitGenerator3d with caller-supplied
neural-renderer modules.
"""
import ctypes
import gzip
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
import _harness
import _hd_fields as HD
from _fp64 import _film, _opt, _rel, _siren, composite_ref, field_ref
from fenerf_b200 import _lib, ops, packing
from oracle import render_oracle as oracle
from test_dropin import _LOAD_WITH_MIRROR, _reference_checkpoint, _run
from test_gpu_fp64_reference import (COMPOSITE_BOUND, FIELD_BOUND, FWD_BOUND, LAYOUT_BOUND, _LAYOUTS, _field_backward,
                                     _field_points, _forward_inputs, _grad_errors, _per_point, _render_points,
                                     composite_backward_errors, over_bounds, with_entries)

DEV = "cuda:0"
gpu = pytest.mark.gpu
CASES = HD.CASES
GOLDEN = _cases.GOLDEN_DIR
TOL = 2e-5          # the oracle against the reference's goldens across hosts (test_oracle.py)
CHILDREN = {"J": ["network", "final_layer", "color_layer_sine", "color_layer_linear", "mapping_network", "gridwarper"],
            "K": ["network", "final_layer", "label_layer_sine", "label_layer_linear", "color_layer_sine", "color_layer_linear",
                  "mapping_network", "activation", "gridwarper"]}
SMALL = {"J": "j_small", "K": "k_small"}


def _gpu_parity():
    import test_gpu_parity
    return test_gpu_parity


# --------------------------------------------------------------------------------------------
# CPU: the mirror classes
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["J", "K"])
def test_mirror_init_and_state_dict_are_the_references(model):
    case = _cases.CASE_BY_NAME[SMALL[model]]
    gold = np.load(_cases.golden_path(case))
    gen = _cases.build_mirror(case, "cpu")
    assert _harness.state_digest(gen) == str(gold["state_digest"])
    with gzip.open(os.path.join(GOLDEN, "dropin_ref_%s.pth.meta.gz" % model), "rb") as f:
        meta = torch.load(io.BytesIO(f.read()), map_location="cpu", weights_only=False)
    assert list(gen.state_dict().keys()) == list(meta["state"].keys())
    assert [n for n, _ in gen.named_parameters()] == meta["names"]
    assert [n for n, _ in gen.siren.named_children()] == CHILDREN[model]
    spec = gen.siren.field_spec()
    assert spec.feature_head and spec.out_dim == (65 if model == "J" else 129) and spec.rgb_dim == 64
    if model == "K":
        assert gen.siren.max_batch_size == 2500 and isinstance(gen.siren.activation, torch.nn.Softmax)


@pytest.mark.parametrize("model", ["J", "K"])
def test_reference_pickle_loads_under_the_mirror(tmp_path, model):
    out = _run(_LOAD_WITH_MIRROR, _reference_checkpoint(tmp_path, model), ref="")
    assert "ok" in out


@pytest.mark.parametrize("model,rows", [("J", 9), ("K", 10)])
def test_film_table_rows(model, rows):
    siren = _cases.build_mirror(_cases.CASE_BY_NAME[SMALL[model]], "cpu").siren
    z = torch.randn(3, 256, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        film = siren.film_from_latents(z)
        f, p = siren.mapping_network(z)
    assert film.shape == (3, rows, 2, 256) and siren.film_rows() == rows
    for r in range(rows):
        assert torch.equal(film[:, r, 0], (f * 15 + 30)[:, 256 * r:256 * (r + 1)])
        assert torch.equal(film[:, r, 1], p[:, 256 * r:256 * (r + 1)])


# --------------------------------------------------------------------------------------------
# CPU: the C-ABI on the host (flags word, layout)
# --------------------------------------------------------------------------------------------
def _desc(flags, label_dim, grid=0, out_dim=None):
    return _lib.FieldDesc(trunk_layers=8, color_layers=1, label_dim=label_dim, grid_channels=grid, grid_res=16 if grid else 0,
                          out_dim=label_dim + 65 if out_dim is None else out_dim, input_scale=2 / 0.24, reserved=flags)


def test_feature_head_bit_only_in_the_reference_shapes():
    lib = _lib.lib()
    FH, LF = _lib.FIELD_FEATURE_HEAD, _lib.FIELD_LABEL_FILM
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(FH, 0))) > 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(FH | LF, 64))) > 0
    params = _lib.FieldParams()
    # a pre-multiplied label chain, other label widths, a grid field: no reference class, FENERF_E_UNSUPPORTED
    for d in (_desc(FH, 19), _desc(FH, 64), _desc(FH | LF, 19), _desc(FH | LF, 32), _desc(FH, 0, grid=32)):
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"FEATURE_HEAD" in lib.fenerf_last_error()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2
    # the channel count must be label_dim + 65; a plain field still stops at 32 labels
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(FH, 0, out_dim=4))) == 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(0, 64, out_dim=68))) == 0


def test_packed_sizes():
    """The feature-head sections are appended (fp32 copy + 32 KB image per 64-wide head); the label FiLM field's 32-row
    label image is not allocated; the mirror's descriptors give these sizes."""
    lib = _lib.lib()
    FH, LF = _lib.FIELD_FEATURE_HEAD, _lib.FIELD_LABEL_FILM
    head = ((64 * 256 + 64) * 4 + 1023) // 1024 * 1024 + 32768
    plain = lib.fenerf_packed_bytes(ctypes.byref(_desc(0, 0, out_dim=4)))
    label = lib.fenerf_packed_bytes(ctypes.byref(_desc(LF, 19, out_dim=23)))
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(FH, 0))) == plain + head
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(FH | LF, 64))) == label - 4 * 32 * 64 * 2 + 2 * head
    for model in ("J", "K"):
        spec = _cases.build_mirror(_cases.CASE_BY_NAME[SMALL[model]], "cpu").siren.field_spec()
        d = packing.field_desc(spec)
        assert d.reserved & FH and lib.fenerf_packed_bytes(ctypes.byref(d)) > 0


# --------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's goldens
# --------------------------------------------------------------------------------------------
def _golden_pixels(pixels, gold):
    pixels = pixels.cpu()
    if "pixel_probe" in gold.files:
        assert tuple(pixels.shape) == tuple(gold["pixels_shape"])
        idx = _cases.pixel_probe_index(pixels.numel())
        return pixels.reshape(-1)[idx], torch.from_numpy(gold["pixel_probe"]), idx
    assert tuple(pixels.shape) == gold["pixels"].shape
    return pixels.reshape(-1), torch.from_numpy(gold["pixels"]).reshape(-1), None


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_oracle_matches_reference_golden(case):
    gold = np.load(_cases.golden_path(case))
    run = _harness.oracle_run(case, keep_stages=False)
    got, want, _ = _golden_pixels(run["out"]["pixels"], gold)
    diff = (got - want).abs()
    assert diff.max() <= TOL, "max|oracle - reference| = %g" % diff.max()
    if "pixels_abs_sum" in gold.files:
        assert abs(run["out"]["pixels"].abs().sum().item() - float(gold["pixels_abs_sum"])) <= 1e-5 * float(gold["pixels_abs_sum"])
    if "depth_map" in gold.files:
        r = case.cfg["img_size"]
        assert np.abs(run["out"]["depth"].reshape(case.batch, r, r).numpy() - gold["depth_map"]).max() <= TOL


def test_gradient_goldens_cover_the_wide_heads():
    for model in ("J", "K"):
        gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % SMALL[model]))
        for k in HD.GRAD_PARAMS[model] + ["latent0"]:
            assert np.abs(gold[k]).max() > 0, k
    freq = np.load(os.path.join(GOLDEN, "gradfreq_k_small.npz"))
    for i in (0, 1):
        for row in (8, 9):
            assert np.abs(freq["arg%d" % i][:, 256 * row:256 * (row + 1)]).max() > 0


# --------------------------------------------------------------------------------------------
# CPU: float64 restatements that pass gradcheck
# --------------------------------------------------------------------------------------------
def _restated(siren, pts, film, dirs, fault=None):
    """The feature-head fields in float64, written out independently of the oracle: x, [labels,] features, sigma.
    `fault` applies one mistake: the old sigmoid on the features, the label and colour FiLM rows swapped, or the label
    head on the trunk output instead of the label FiLM layer's."""
    x = pts * siren.gridwarper.scale_factor
    for i, layer in enumerate(siren.network):
        x = torch.sin(film[:, i, 0].unsqueeze(1) * layer.layer(x) + film[:, i, 1].unsqueeze(1))
    semantic = hasattr(siren, "label_layer_sine")
    row_l, row_c = ((9, 8) if fault == "rows_swapped" else (8, 9)) if semantic else (None, 8)
    c = torch.sin(film[:, row_c, 0].unsqueeze(1) * siren.color_layer_sine.layer(torch.cat([dirs, x], -1))
                  + film[:, row_c, 1].unsqueeze(1))
    feat = siren.color_layer_linear[0](c)
    parts = [torch.sigmoid(feat) if fault == "sigmoid" else feat, siren.final_layer(x)]
    if semantic:
        lab = x if fault == "label_on_trunk" else torch.sin(film[:, row_l, 0].unsqueeze(1) * siren.label_layer_sine.layer(x)
                                                            + film[:, row_l, 1].unsqueeze(1))
        parts.insert(0, siren.label_layer_linear[0](lab))
    return torch.cat(parts, -1)


def _cpu_inputs(model, seed, n=200):
    siren = _cases.build_mirror(_cases.CASE_BY_NAME[SMALL[model]], "cpu").siren
    film = _film(siren, 2, seed).double()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).double()
    return siren.double(), film, pts, dirs


@pytest.mark.parametrize("model", ["J", "K"])
def test_restatement_is_the_oracle_and_passes_gradcheck(model):
    """The oracle's feature-head field evaluation (what the GPU tests compare the kernels and the backward with) equals
    the written-out restatement, and differentiates correctly through the FiLM table and every field parameter."""
    siren, film, pts, dirs = _cpu_inputs(model, 11)
    with torch.no_grad():
        assert torch.equal(_restated(siren, pts, film, dirs), oracle.field_eval(siren, pts, film, dirs))
    pts, dirs = pts[:, :2].contiguous(), dirs[:, :2].contiguous()
    names = [n for n, _ in siren.named_parameters() if "mapping_network" not in n]
    params = dict(siren.named_parameters())

    def fn(film_, *ps):
        saved = [params[n].data for n in names]
        mods = dict(siren.named_modules())
        for n, p in zip(names, ps):
            m, a = n.rsplit(".", 1)
            mods[m]._parameters[a] = p
        try:
            return oracle.field_eval(siren, pts, film_, dirs)
        finally:
            for n, d in zip(names, saved):
                m, a = n.rsplit(".", 1)
                mods[m]._parameters[a] = torch.nn.Parameter(d)
    inputs = (film.clone().requires_grad_(True),) + tuple(params[n].detach().clone().requires_grad_(True) for n in names)
    assert torch.autograd.gradcheck(fn, inputs, fast_mode=True, eps=1e-7, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("model,fault", [("J", "sigmoid"), ("K", "sigmoid"), ("K", "rows_swapped"), ("K", "label_on_trunk")])
def test_faults_exceed_the_bounds(model, fault):
    """Each fault moves the float64 forward past 10x the fast kernel's bound and the float64 gradients of the FiLM
    table past 10x the default backward bound."""
    siren, film, pts, dirs = _cpu_inputs(model, 12)
    film = film.requires_grad_(True)
    c = siren.field_spec().out_dim
    d_out = torch.randn(2, pts.shape[1], c, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    res = {}
    for k in (None, fault):
        film.grad = None
        out = _restated(siren, pts, film, dirs, fault=k)
        (out * d_out).sum().backward()
        res[k] = (out.detach(), film.grad.clone())
    fwd = (res[None][0] - res[fault][0]).abs().amax((0, 1)).max().item()
    grad = _rel(res[fault][1][:, 8:], res[None][1][:, 8:])
    print("fault %s %s: forward %.3g, gradient %.3g" % (model, fault, fwd, grad))
    assert fwd >= 10 * FWD_BOUND["fast"]
    assert grad >= 10 * FIELD_BOUND["default"]


@pytest.mark.parametrize("opt", [_opt("relu"), _opt("softplus", last_back=True), _opt("relu", softmax=True)],
                         ids=["relu", "last_back", "softmax_label"])
def test_wide_composite_reference_gradcheck(opt):
    """The float64 compositing VJP at 129 channels (softmax over the first 125) is the derivative of its own function."""
    g = torch.Generator().manual_seed(3)
    b, s, c = 1, 4, 129
    z_c = (0.88 + 0.24 * torch.sort(torch.rand(b, 1, s, generator=g), -1)[0]).float()
    z_f = (0.88 + 0.24 * torch.sort(torch.rand(b, 1, s, generator=g), -1)[0]).float()
    raw_c = torch.randn(b, 1, s, c, generator=g, dtype=torch.float64)
    raw_f = torch.randn(b, 1, s, c, generator=g, dtype=torch.float64)
    for r in (raw_c, raw_f):
        r[..., -1] = torch.where(r[..., -1] >= 0, r[..., -1] + 0.05, r[..., -1] - 0.05) * 20
    leaves = (raw_c.requires_grad_(True), raw_f.requires_grad_(True))
    assert torch.autograd.gradcheck(lambda rc, rf: composite_ref(rc, z_c, rf, z_f, None, opt), leaves, eps=1e-7, atol=1e-7,
                                    rtol=1e-5)


# --------------------------------------------------------------------------------------------
# GPU: end to end against the reference's goldens
# --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def runs():
    cache = {}

    def get(name):
        if name not in cache:
            case = _cases.CASE_BY_NAME[name]
            cache[name] = (case, _harness.oracle_run(case))
        return cache[name]
    return get


@gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("precision,tol", [("exact", 2e-4), ("guard", 1e-3)])
def test_end_to_end_against_reference_golden(runs, case, precision, tol):
    """forward / staged_forward with the far-sigma exclusion rule of test_gpu_parity.py, every channel (labels, features)."""
    p = _gpu_parity()
    gold = np.load(_cases.golden_path(case))
    case, run = runs(case.name)
    l0 = _lib.launch_count()
    gen, pixels, poses, depth_map = p._end_to_end(case, run, precision)
    assert _lib.launch_count() > l0
    got, want, idx = _golden_pixels(pixels, gold)
    err = (got - want).abs()
    ill_rays = p._ill_conditioned_pixels(case, run)
    assert int(ill_rays.sum()) <= max(2, 0.002 * ill_rays.numel())
    ill = ill_rays.unsqueeze(1).expand_as(pixels).reshape(-1)
    if idx is not None:
        ill = ill[idx]
    print("%s %s: max err %.3g" % (case.name, precision, err[~ill].max()))
    assert err[~ill].max() <= tol
    if poses is not None:
        assert (poses - torch.from_numpy(gold["poses"])).abs().max() <= 1e-5
    if depth_map is not None:
        assert (depth_map - torch.from_numpy(gold["depth_map"])).abs()[~ill_rays].max() <= 3e-3


# --------------------------------------------------------------------------------------------
# GPU: the point-network kernels
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("model", ["J", "K"])
@pytest.mark.parametrize("layout", _cases.TILE_LAYOUTS)
def test_point_network_vs_fp64(model, layout):
    """Both kernels against the oracle's field evaluation in float64 per channel (exact 1e-5, fast 5e-3); the fast kernel
    is bit-identical between launches and its density-only entry (the plain instantiation on the trunk view) equals its
    sigma channel."""
    siren = _siren(model, DEV)
    pts, dirs, film = _forward_inputs(siren, layout, 2200)
    with torch.no_grad():
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact")
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
        fast2 = ops.siren_points(siren, pts, film, dirs, precision="fast")
        sigma = ops.siren_sigma(siren, pts, film, precision="fast")
        sigma_x = ops.siren_sigma(siren, pts, film, precision="exact")
    want = field_ref(siren, pts, _per_point(dirs, pts.shape[1], False), film)[0]
    err = {k: (v.double() - want).abs().amax((0, 1)) for k, v in (("exact", exact), ("fast", fast))}
    print("forward %s %s: exact %.3g fast %.3g" % (model, layout, err["exact"].max(), err["fast"].max()))
    assert torch.isfinite(fast).all()
    for k in err:
        assert err[k].max() <= FWD_BOUND[k], "%s: max |out - fp64| per channel %s" % (k, err[k].tolist())
    assert torch.equal(fast, fast2)
    assert torch.equal(sigma, fast[..., -1:])
    assert torch.equal(sigma_x, exact[..., -1:])


_FIELD = [(lay, m, p) for lay in ("L1", "L2", "L3") for m in ("J", "K") for p in ("exact", "default")] + \
    [("L4", "K", p) for p in ("exact", "default")]


@gpu
@pytest.mark.parametrize("layout,model,precision", _FIELD, ids=["%s-%s-%s" % c for c in _FIELD])
def test_field_backward_vs_fp64(monkeypatch, layout, model, precision):
    """_FieldBackward against the float64 VJP under the chunk layouts of test_gpu_fp64_reference.py: the 64-wide colour
    head, K's (64 + 8)-row head block, head_grads_feature_kernel, and FiLM rows 8 / 9 from image b0 > 0 of a chunk (L2)
    and from images split into point chunks (L3, L4 = cfg2's pass); L2 / L3 also within LAYOUT_BOUND of a one-chunk run."""
    from fenerf_b200 import backward
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    exact = precision == "exact"
    if exact:
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    siren = _siren(model, DEV)
    seed = 3200 + 10 * (model == "K") + int(layout[1])
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film = _film(siren, batch, seed, edges=True)
    out_dim = siren.field_spec().out_dim
    d_raw = torch.randn(batch, ppb, out_dim, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    out64, want_film, want = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw)
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, False, raw, d_raw, exact)
    errs = _grad_errors(d_film, grads, want_film, want)
    worst = max(errs, key=errs.get)
    print("field %s %s %s: worst %s %.3g (colour head %.3g)" % (layout, model, precision, worst, errs[worst],
                                                              errs["color_layer_linear.0.weight"]))
    assert errs[worst] <= FIELD_BOUND[precision], {k: "%.2e" % v for k, v in errs.items() if v > FIELD_BOUND[precision]}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, False, raw, d_raw, exact)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        print("layout %s %s %s: worst %s %.3g" % (layout, model, precision, worst, inv[worst]))
        assert inv[worst] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


@gpu
def test_guard_refinement_on_a_64_label_field():
    """SEMANTICHD in guard precision: the refinement runs (non-zero count) through the plain exact kernel on the trunk
    view, its densities equal the exact kernel's, and the 128 other channels of the row stay the fast pass's."""
    siren = _siren("K", DEV)
    film = _film(siren, 2, 77)
    rd = ops.make_render_desc(batch=2, img_size=16, num_steps=12, hierarchical=False, clamp_mode="relu", nerf_noise=0.0,
                              fov=12, precision="guard", guard_tau=1e9)                      # every ray refined
    x_lin, y_lin, z_lin = ops.ray_tables(16, 12, 0.88, 1.12, DEV)
    c2w = torch.eye(4, device=DEV).repeat(2, 1, 1)
    c2w[:, 2, 3] = 1.0
    rng = torch.rand(2, 16 * 16, 12, 1, generator=torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        st = ops.render_forward_stages(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
        pts, dirs = st["points_c"].reshape(2, -1, 3), st["dirs"]
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast").reshape(2, 256, 12, 129)
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact").reshape(2, 256, 12, 129)
        pixels = ops.render_forward(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)[0]
    rep = ops.guard_stats(DEV)
    assert rep["refined"] >= 2 * 256 and rep["max_abs_delta"] < 1e-2
    raw = st["raw_c"]
    assert torch.equal(raw[:, :, :-1], fast[:, :, :-1])
    assert torch.equal(raw[:, :, -1, -1], exact[:, :, -1, -1])
    assert torch.equal(raw[:, :, -1, :-1], fast[:, :, -1, :-1])
    assert torch.isfinite(pixels).all()


# --------------------------------------------------------------------------------------------
# GPU: the wide compositor
# --------------------------------------------------------------------------------------------
_WB, _WR = 2, 23
_WIDE = [(n, hier, c, o) for n, hier in [(9, False), (33, False), (64, False), (48, True), (128, True)] for c in (65, 129)
         for o in ("relu", "softplus_noise")]
_WIDE += [(n, True, 129, o) for n in (48, 128) for o in ("relu_softmax", "softplus_last_back", "relu_white_back",
                                                          "relu_black_back")]
# just past the narrow kernels (C <= 32): the first widths on the wide ones
_WIDE += [(n, hier, c, o) for n, hier in [(33, False), (128, True)] for c in (33, 34, 36)
          for o in ("relu", "softplus_noise", "relu_softmax", "softplus_last_back")]
_WOPTS = {"relu": _opt("relu"), "softplus_noise": _opt("softplus", noise=0.5), "relu_softmax": _opt("relu", softmax=True),
          "softplus_last_back": _opt("softplus", last_back=True), "relu_white_back": _opt("relu", white_back=True),
          "relu_black_back": _opt("relu", black_back=True)}


def _wide_inputs(c, steps, hier, seed):
    g = torch.Generator().manual_seed(seed)
    _, z_c, _, _ = _render_points(_WB, _WR, steps, seed)
    n = _WR * _WR
    raw_c = torch.randn(_WB, n, steps, c, generator=g)
    raw_c[..., -1] *= 3
    x = dict(raw_c=raw_c.to(DEV).contiguous(), z_c=z_c.to(DEV).contiguous(), raw_f=None, z_f=None)
    if hier:
        z_f = 0.88 + 0.24 * torch.sort(torch.rand(_WB, n, steps, generator=g), -1)[0]
        z_f[:, ::5, 0] = z_c[:, ::5, steps // 2]
        raw_f = torch.randn(_WB, n, steps, c, generator=g)
        raw_f[..., -1] *= 3
        x.update(raw_f=raw_f.to(DEV).contiguous(), z_f=z_f.to(DEV).contiguous())
    return x


@gpu
@pytest.mark.parametrize("n,hier,c,opt,entry", with_entries(_WIDE, ["n%d-%s-C%d-%s" % (n, "hier" if h else "flat", c, o)
                                                                    for n, h, c, o in _WIDE]))
def test_wide_composite_vs_fp64(n, hier, c, opt, entry):
    """fenerf_composite (unsorted: the render's samples shuffled) and fenerf_composite_backward at 33 .. 129 channels
    against the float64 compositing and its VJP.  The gradient buffers start as NaN, and the density column is compared
    on its own as well: every entry must be written.  '-rays': fenerf_composite_backward_rays (ray-major d_pixels) in
    place of fenerf_composite_backward, bit for bit the NCHW entry's result on the same upstream value."""
    steps = n // 2 if hier else n
    o = _WOPTS[opt]
    x = _wide_inputs(c, steps, hier, 7 * n + c)
    g = torch.Generator().manual_seed(n * 64 + c)
    noise = torch.randn(_WB, _WR * _WR, n, generator=g).to(DEV) if o["noise"] else None
    rd = ops.make_render_desc(batch=_WB, img_size=_WR, num_steps=steps, hierarchical=hier, clamp_mode=o["clamp"],
                              nerf_noise=o["noise"], fov=12, last_back=o["last_back"], white_back=o["white_back"],
                              black_back=o["black_back"], softmax_label=o["softmax"])
    perm = torch.randperm(steps, generator=g).to(DEV)
    shuf = {k: (v.index_select(2, perm).contiguous() if v is not None else None) for k, v in x.items()}
    px = ops.composite(rd, shuf["raw_c"], shuf["z_c"], shuf["raw_f"], shuf["z_f"], noise)[0]
    # (hierarchical: the reference's stable sort of the shuffled lists -- a list may hold two equal fp32 depths, whose order
    # of appearance the shuffle decides; flat: the reference composites in the given order, the depth-sorted one)
    src = shuf if hier else x
    want = composite_ref(src["raw_c"].double(), src["z_c"], src["raw_f"].double() if hier else None, src["z_f"], noise, o)
    fwd = _rel(px, want)
    t, errs = composite_backward_errors(o, steps, hier, x, noise, g, entry, batch=_WB, img=_WR)
    errs.update(forward=fwd, d_sigma_c=_rel(t["d_c"][..., -1], t["w_c"][..., -1]))
    if hier:
        errs["d_sigma_f"] = _rel(t["d_f"][..., -1], t["w_f"][..., -1])
    assert all(v == v for v in errs.values()), errs          # (NaN: an entry was not written)
    print("wide composite %s n=%d C=%d %s: %s" % (entry, n, c, opt, errs))
    assert not over_bounds(errs), errs


@gpu
@pytest.mark.parametrize("case_name", ["k_small", "k_staged_softmax", "j_small"])
def test_standalone_composite_is_the_renders(runs, case_name):
    """fenerf_composite on the render's own intermediates (samples in any order) reproduces the render's pixels bit for
    bit, fill modes and softmax included."""
    case, run = runs(case_name)
    siren = _siren(case.model, DEV)
    film = _film(siren, 1, 5)
    cfg = case.cfg
    r, s = 16, 10
    fill = cfg.get("fill_mode") if case.method == "staged_forward" else None
    rd = ops.make_render_desc(batch=1, img_size=r, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.0, fov=12,
                              fill_mode=fill, softmax_label=cfg.get("softmax_label", False), precision="exact")
    x_lin, y_lin, z_lin = ops.ray_tables(r, s, 0.88, 1.12, DEV)
    c2w = torch.eye(4, device=DEV).unsqueeze(0).contiguous()
    c2w[:, 2, 3] = 1.0
    g = torch.Generator().manual_seed(9)
    rng = torch.rand(1, r * r, s, 1, generator=g).to(DEV)
    u = torch.rand(r * r, s, generator=g).to(DEV)
    with torch.no_grad():
        st = ops.render_forward_stages(siren, rd, film, x_lin, y_lin, z_lin, c2w, rng, None, u, None)
        pix = ops.render_forward(siren, rd, film, x_lin, y_lin, z_lin, c2w, rng, None, u, None)[0]
        alone = ops.composite(rd, st["raw_c"].contiguous(), st["z_c"].contiguous(), st["raw_f"].contiguous(),
                              st["z_f"].contiguous())[0]
    assert torch.equal(pix, alone)


# --------------------------------------------------------------------------------------------
# GPU: the backward
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("model", ["J", "K"])
@pytest.mark.parametrize("precision", ["exact", "guard"])
def test_backward_matches_reference_gradients(runs, model, precision):
    """Against the reference's autograd: <= 5e-4 of each tensor's max in exact mode, <= 2e-2 in the default mode."""
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    p = _gpu_parity()
    case, run = runs(SMALL[model])
    gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % SMALL[model]))
    gen = _cases.build_mirror(case, DEV)
    latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
    pixels, _ = gen(*latents, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision=precision))
    loss = (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum()
    loss.backward()
    got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({k: q.grad for k, q in gen.named_parameters()})
    worst = p._compare_grads(gold, got, rel=5e-4 if precision == "exact" else 2e-2,
                             kink_rel=1e-2 if precision == "exact" else 0.3)
    print("gradients %s %s: %s" % (model, precision, {k: "%.1e" % v for k, v in worst.items()}))


@gpu
def test_inversion_gradients_reach_rows_8_and_9(runs):
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    p = _gpu_parity()
    case, run = runs("k_small")
    gold = np.load(os.path.join(GOLDEN, "gradfreq_k_small.npz"))
    gen = _cases.build_mirror(case, DEV)
    with torch.no_grad():
        fp = [t.clone().requires_grad_(True) for t in gen.siren.mapping_network(p._cuda(run["latents"][0]))]
    for q in gen.parameters():
        q.requires_grad_(False)
    pixels, _ = gen.forward_with_frequencies(*fp, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=5e-4)
    rows = max(_rel(t.grad[:, 8 * 256:10 * 256].cpu(), torch.from_numpy(gold["arg%d" % i])[:, 8 * 256:10 * 256])
               for i, t in enumerate(fp))
    print("inversion: %s, rows 8-9 %.2e" % (worst, rows))
    assert rows <= 5e-4


# --------------------------------------------------------------------------------------------
# GPU: a neural-renderer generator with caller-supplied modules
# --------------------------------------------------------------------------------------------
class _Upsampler(torch.nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = torch.nn.Conv2d(cin, cout, 3, padding=1)
        self.up = torch.nn.Upsample(scale_factor=2, mode="bilinear", align_corners=False)

    def forward(self, x):
        return self.up(self.conv(x))


@gpu
def test_neural_renderer_generator():
    """ImplicitGenerator3d(SPATIALSIRENSEMANTICHD, 256, 129, neural_renderer_img=..., neural_renderer_seg=...): the output
    is the caller's modules applied to the [0, 1] frame split at channel 64 (generators.py:102-118), within the parity
    bound of the exact mode, and gradients reach the field through them."""
    from fenerf_b200.generators import generators as G
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    from fenerf_b200.siren import siren as S
    p = _gpu_parity()
    case = _cases.CASE_BY_NAME["k_small"]
    run = _harness.oracle_run(case)
    gold = torch.from_numpy(np.load(_cases.golden_path(case))["pixels"])
    torch.manual_seed(0)
    img_nr, seg_nr = _Upsampler(64, 3), _Upsampler(64, 19)
    torch.manual_seed(0)
    gen = G.ImplicitGenerator3d(S.SPATIALSIRENSEMANTICHD, 256, 129, neural_renderer_img=img_nr, neural_renderer_seg=seg_nr)
    ref = _cases.build_mirror(case, "cpu")
    gen.load_state_dict(ref.state_dict(), strict=False)
    gen.to(DEV)
    gen.set_device(DEV)
    latents = [p._cuda(z) for z in run["latents"]]
    out, _ = gen(*latents, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    unit = (gold.to(DEV) + 1) * 0.5                    # the golden frame before the reference's * 2 - 1
    with torch.no_grad():
        want = torch.cat([seg_nr(unit[:, :64]), img_nr(unit[:, 64:])], 1) * 2 - 1
    assert out.shape == want.shape == (2, 22, 24, 24)
    err = (out - want).abs().max().item()
    # the frame is within the exact mode's 2e-4 of the golden; (frame + 1) / 2 halves that, a convolution output moves by at
    # most its weights' absolute sum times it, the bilinear upsampling (a convex combination) not at all, * 2 doubles it
    gain = max(m.conv.weight.detach().abs().sum((1, 2, 3)).max().item() for m in (img_nr, seg_nr))
    print("neural renderer: max err %.3g, bound %.3g (largest absolute weight sum %.3g)" % (err, 2e-4 * gain, gain))
    assert err <= 2e-4 * gain
    gen.zero_grad()
    out.sum().backward()
    assert gen.siren.color_layer_linear[0].weight.grad.abs().max() > 0
    assert gen.siren.label_layer_linear[0].weight.grad.abs().max() > 0
