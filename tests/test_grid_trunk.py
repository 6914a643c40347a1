"""The grid-trunk field: pi-GAN's EmbeddingPiGAN256 (model "L"), whose 32 x 64^3 feature grid feeds the first trunk layer,
cat[feat, pos] -> 256, and not the colour branch (FENERF_FIELD_GRID_TRUNK), forward and backward.

CPU: the mirror class against the reference (init draws, state-dict keys, parameter names, pickling), the oracle
(tests/_grid_trunk.py) against the reference's goldens, the flag rules and the packed layout on the host, a float64
restatement that passes gradcheck, and three faults the bounds must catch.
GPU: end to end against the reference's goldens (exact <= 2e-4, default <= 1e-3), both point-network kernels against float64
over the tile schedules with the density-only entry bit-identical to the sigma channel, the GUARD refinement, the backward
against float64 and against the reference's autograd (grid probe, the first layer's feature columns), inversion through
forward_with_frequencies, and a staged_forward that sees an in-place write to the feature columns.

Measured maxima on an NVIDIA H100 80GB HBM3 (400 W power limit, SM clock up to 1980 MHz):
  end to end vs the reference    exact 2.4e-5 (l_small_opaque), guard 1.6e-4 (l_staged_white); l_cfg2 3.6e-6 / 7.8e-5
  point network vs float64       exact 1.34e-5 (sigma; rgb <= 6e-6), fast 4.1e-4 (sigma), over the four tile layouts
  GUARD self-check               max |delta| 2.7e-4 on the reference init (< tau / 3 = 5e-4), 0 sign flips
  _FieldBackward vs float64      exact: grid 1.17e-4, layer 0 6.1e-5, the rest <= 1e-4; default 4.1e-3
  gradients vs the reference     exact <= 4.8e-4 (final_layer.weight), grid's largest entries 8.0e-4, abs-sum 1.8e-5;
  (l_small_opaque)               default <= 7.7e-3, grid's largest entries 4.0e-3, abs-sum 5.3e-5
  inversion                      3.3e-4 (phases), 2.5e-4 (frequencies)
"""
import copy
import ctypes
import gzip
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
import _grid_trunk as GT
import _harness
from _fp64 import _film, _rel, _siren, field_ref
from fenerf_b200 import _lib, ops, packing
from oracle import render_oracle as oracle
from test_gpu_fp64_reference import (FIELD_BOUND, FWD_BOUND, LAYOUT_BOUND, _LAYOUTS, _field_backward, _field_points,
                                     _forward_inputs, _grad_errors, _per_point)
from test_hd_fields import _golden_pixels

DEV = "cuda:0"
gpu = pytest.mark.gpu
CASES = GT.CASES
GOLDEN = _cases.GOLDEN_DIR
TOL = 2e-5          # the oracle against the reference's goldens across hosts (test_oracle.py)
CHILDREN = ["network", "final_layer", "color_layer_sine", "color_layer_linear", "mapping_network", "gridwarper"]
SMALL = GT.CASE_BY_NAME["l_small"]
#: the exact kernel's density carries the fp32 trilinear features through a 35-term first layer at f ~ 30 and then every
#: trunk layer: measured 1.1e-5 .. 1.3e-5 on sigma (rgb 3e-6 .. 6e-6), against 1e-5 for fields whose trunk sees only the
#: position; the fast bound is the shared one
FWD_BOUND_L = {"exact": 3e-5, "fast": FWD_BOUND["fast"]}
#: the grid's gradient in exact mode reaches the grid through layer 0's fp32 chain and the fp32 scatter-add: measured
#: 1.1e-4 .. 1.2e-4 of its largest entry (every other tensor within the shared 1e-4)
GRID_BOUND_EXACT = 3e-4
GRAD_CASE = GT.CASE_BY_NAME[GT.GRAD_CASE]


def _gpu_parity():
    import test_gpu_parity
    return test_gpu_parity


# --------------------------------------------------------------------------------------------
# CPU: the mirror class
# --------------------------------------------------------------------------------------------
def test_mirror_init_and_state_dict_are_the_references():
    gold = np.load(_cases.golden_path(SMALL))
    gen = _cases.build_mirror(SMALL, "cpu")
    assert _harness.state_digest(gen) == str(gold["state_digest"])
    with gzip.open(os.path.join(GOLDEN, "dropin_ref_L.pth.meta.gz"), "rb") as f:
        meta = torch.load(io.BytesIO(f.read()), map_location="cpu", weights_only=False)
    assert {k: tuple(v.shape) for k, v in gen.state_dict().items()} == meta["state"]
    assert list(gen.state_dict().keys()) == list(meta["state"].keys())
    assert [n for n, _ in gen.named_parameters()] == meta["names"]
    assert [n for n, _ in gen.siren.named_children()] == CHILDREN
    siren = gen.siren
    spec = siren.field_spec()
    assert spec.grid_trunk and spec.grid_channels == 32 and spec.grid_res == 64 and spec.out_dim == 4
    assert siren.network[0].layer.weight.shape == (256, 35) and siren.network[0].layer.weight.abs().max() <= 1 / 3
    assert siren.color_layer_sine.layer.weight.shape == (256, 259) and siren.film_rows() == 9


def test_mirror_pickles_and_resolves_by_name():
    from fenerf_b200.siren import siren as S
    assert getattr(S, "EmbeddingPiGAN256") is S.EmbeddingPiGAN256
    gen = _cases.build_mirror(SMALL, "cpu")
    buf = io.BytesIO()
    torch.save(gen, buf)
    back = torch.load(io.BytesIO(buf.getvalue()), map_location="cpu", weights_only=False)
    assert type(back.siren) is S.EmbeddingPiGAN256
    assert all(torch.equal(a, b) for a, b in zip(gen.state_dict().values(), back.state_dict().values()))


# --------------------------------------------------------------------------------------------
# CPU: the C-ABI on the host (flag rules, layout)
# --------------------------------------------------------------------------------------------
def _desc(flags, label_dim=0, grid=32, out_dim=None, res=64):
    return _lib.FieldDesc(trunk_layers=8, color_layers=1, label_dim=label_dim, grid_channels=grid, grid_res=res if grid else 0,
                          out_dim=label_dim + 4 if out_dim is None else out_dim, input_scale=2 / 0.24, reserved=flags)


def test_grid_trunk_bit_only_in_the_reference_shape():
    lib = _lib.lib()
    GTF, LF, FH = _lib.FIELD_GRID_TRUNK, _lib.FIELD_LABEL_FILM, _lib.FIELD_FEATURE_HEAD
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(GTF))) > 0
    params = _lib.FieldParams()
    for d in (_desc(GTF | LF, 19), _desc(GTF | FH, out_dim=65), _desc(GTF, grid=0), _desc(GTF, 19), _desc(GTF | LF | FH, 64, out_dim=129)):
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"GRID_TRUNK" in lib.fenerf_last_error()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2


def test_packed_layout():
    """The first layer's fp32 copy grows by 32 rows (32 KB), the first colour layer's shrinks by as much (extra inputs 48
    -> 16 padded rows); the low parts of the feature weights add one 32 KB image.  The mirror's descriptor sets the flag."""
    lib = _lib.lib()
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(_lib.FIELD_GRID_TRUNK))) == \
        lib.fenerf_packed_bytes(ctypes.byref(_desc(0))) + 32768         # + the feature weights' low-part image
    d = packing.field_desc(_cases.build_mirror(SMALL, "cpu").siren.field_spec())
    assert d.reserved == _lib.FIELD_GRID_TRUNK and d.grid_channels == 32 and d.grid_res == 64
    assert lib.fenerf_packed_bytes(ctypes.byref(d)) > 0


# --------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's goldens
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_oracle_matches_reference_golden(case):
    if case.name in GT.BIG and not os.environ.get("FENERF_SLOW_TESTS") and not torch.cuda.is_available():
        pytest.skip("minutes of CPU oracle (FENERF_SLOW_TESTS=1 runs it)")
    gold = np.load(_cases.golden_path(case))
    run = GT.oracle_run(case, keep_stages=False)
    got, want, _ = _golden_pixels(run["out"]["pixels"], gold)
    diff = (got - want).abs()
    assert diff.max() <= TOL, "max|oracle - reference| = %g" % diff.max()
    if "pixels_abs_sum" in gold.files:
        assert abs(run["out"]["pixels"].abs().sum().item() - float(gold["pixels_abs_sum"])) <= 1e-5 * float(gold["pixels_abs_sum"])
    if "depth_map" in gold.files:
        r = case.cfg["img_size"]
        assert np.abs(run["out"]["depth"].reshape(case.batch, r, r).numpy() - gold["depth_map"]).max() <= TOL


def test_gradient_goldens_cover_the_feature_columns():
    gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % GT.GRAD_CASE))
    for k in GT.GRAD_PARAMS + ["latent0"]:
        assert np.abs(gold[k]).max() > 0, k
    assert np.abs(gold["siren.network.0.layer.weight"][:, :32]).max() > 0 and float(gold["grid_abs_sum"]) > 0
    # the grid probe holds the reference's largest entries, none of them zero
    assert np.abs(gold["grid_probe"]).min() > 0 and len(np.unique(gold["grid_probe_idx"])) == len(gold["grid_probe"])
    freq = np.load(os.path.join(GOLDEN, "gradfreq_%s.npz" % GT.GRAD_CASE))
    assert all(np.abs(freq["arg%d" % i][:, :256]).max() > 0 for i in (0, 1))
    # the render the gradients come from is not the empty background: the opaque field's colours vary over the image
    px = np.load(_cases.golden_path(GRAD_CASE))["pixels"]
    assert px.std() > 1e-2 and px.max() > -0.99


# --------------------------------------------------------------------------------------------
# CPU: a float64 restatement that passes gradcheck, and the faults the bounds catch
# --------------------------------------------------------------------------------------------
def _restated(siren, pts, film, dirs):
    """EmbeddingPiGAN256 in float64, written out independently of the oracle."""
    x = pts * siren.gridwarper.scale_factor
    g = siren.spatial_embeddings
    s = F.grid_sample(g.expand(x.shape[0], -1, -1, -1, -1), x.reshape(x.shape[0], 1, 1, -1, 3), mode="bilinear",
                      padding_mode="zeros", align_corners=True)
    feat = s.reshape(x.shape[0], g.shape[1], -1).transpose(1, 2)
    h = torch.cat([feat, x], -1)
    for i, layer in enumerate(siren.network):
        h = torch.sin(film[:, i, 0].unsqueeze(1) * layer.layer(h) + film[:, i, 1].unsqueeze(1))
    c = torch.sin(film[:, 8, 0].unsqueeze(1) * siren.color_layer_sine.layer(torch.cat([dirs, h], -1)) + film[:, 8, 1].unsqueeze(1))
    return torch.cat([torch.sigmoid(siren.color_layer_linear[0](c)), siren.final_layer(h)], -1)


def _cpu_inputs(seed, n=200, res=None):
    siren = copy.deepcopy(_cases.build_mirror(SMALL, "cpu").siren)
    if res:     # a coarse grid of the same statistics: gradcheck perturbs every entry
        g = torch.Generator().manual_seed(seed)
        siren.spatial_embeddings = torch.nn.Parameter(torch.randn(1, 32, res, res, res, generator=g) * 0.1)
    film = _film(siren, 2, seed).double()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).double()
    return siren.double(), film, pts, dirs


def test_restatement_is_the_oracle_and_passes_gradcheck():
    """The restatement equals the oracle's float64 evaluation (tests/_grid_trunk.py) and differentiates
    correctly through the FiLM table, every field parameter and the grid."""
    siren, film, pts, dirs = _cpu_inputs(11)
    with torch.no_grad():
        assert torch.allclose(_restated(siren, pts, film, dirs), GT.field_eval(siren, pts, film, dirs), rtol=0, atol=1e-12)
    siren, film, pts, dirs = _cpu_inputs(11, n=3, res=5)
    names = [n for n, _ in siren.named_parameters() if "mapping_network" not in n]
    params = dict(siren.named_parameters())

    def fn(film_, *ps):
        saved = [params[n].data for n in names]
        mods = dict(siren.named_modules())
        for n, p in zip(names, ps):
            m, a = n.rsplit(".", 1) if "." in n else ("", n)
            mods[m]._parameters[a] = p
        try:
            return GT.field_eval(siren, pts, film_, dirs)
        finally:
            for n, d in zip(names, saved):
                m, a = n.rsplit(".", 1) if "." in n else ("", n)
                mods[m]._parameters[a] = torch.nn.Parameter(d)
    inputs = (film.clone().requires_grad_(True),) + tuple(params[n].detach().clone().requires_grad_(True) for n in names)
    assert torch.autograd.gradcheck(fn, inputs, fast_mode=True, eps=1e-7, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("fault", ["no_feat", "feat_in_colour", "no_warp"])
def test_faults_exceed_the_bounds(fault):
    """Each fault moves the float64 forward past 10x the fast kernel's bound and the float64 FiLM-table gradients past 10x
    the default backward bound."""
    siren, film, pts, dirs = _cpu_inputs(12)
    film = film.requires_grad_(True)
    d_out = torch.randn(2, pts.shape[1], 4, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    res = {}
    for k in (None, fault):
        film.grad = None
        out = GT.field_eval(siren, pts, film, dirs, fault=k)
        (out * d_out).sum().backward()
        res[k] = (out.detach(), film.grad.clone())
    fwd = (res[None][0] - res[fault][0]).abs().amax((0, 1)).max().item()
    grad = _rel(res[fault][1], res[None][1])
    print("fault %s: forward %.3g, gradient %.3g" % (fault, fwd, grad))
    assert fwd >= 10 * FWD_BOUND["fast"]
    assert grad >= 10 * FIELD_BOUND["default"]


# --------------------------------------------------------------------------------------------
# GPU: end to end against the reference's goldens
# --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def runs():
    cache = {}

    def get(name):
        if name not in cache:
            case = GT.CASE_BY_NAME[name]
            cache[name] = (case, GT.oracle_run(case))
        return cache[name]
    return get


@gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("precision,tol", [("exact", 2e-4), ("guard", 1e-3)])
def test_end_to_end_against_reference_golden(runs, case, precision, tol):
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
@pytest.mark.parametrize("layout", _cases.TILE_LAYOUTS)
def test_point_network_vs_fp64(monkeypatch, layout):
    """Both kernels against the oracle's field evaluation in float64 per channel (exact 1e-5, fast 5e-3); back-to-back
    launches are bit-identical, and the density-only entry equals the sigma channel bit for bit in both modes -- the check
    that catches a density path without the grid gather."""
    siren = _siren("L", DEV)
    pts, dirs, film = _forward_inputs(siren, layout, 2300)
    with torch.no_grad():
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact")
        exact2 = ops.siren_points(siren, pts, film, dirs, precision="exact")
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
        fast2 = ops.siren_points(siren, pts, film, dirs, precision="fast")
        sigma = ops.siren_sigma(siren, pts, film, precision="fast")
        sigma_x = ops.siren_sigma(siren, pts, film, precision="exact")
    monkeypatch.setattr(oracle, "field_eval", GT.field_eval)
    want = field_ref(siren, monkeypatch, pts, _per_point(dirs, pts.shape[1], False), film)[0]
    err = {k: (v.double() - want).abs().amax((0, 1)) for k, v in (("exact", exact), ("fast", fast))}
    print("forward L %s: exact %.3g fast %.3g (sigma %.3g)" % (layout, err["exact"].max(), err["fast"].max(),
                                                              err["fast"][-1]))
    assert torch.isfinite(fast).all()
    for k in err:
        assert err[k].max() <= FWD_BOUND_L[k], "%s: max |out - fp64| per channel %s" % (k, err[k].tolist())
    assert torch.equal(fast, fast2) and torch.equal(exact, exact2)
    assert torch.equal(sigma, fast[..., -1:])
    assert torch.equal(sigma_x, exact[..., -1:])


@gpu
def test_guard_refinement():
    """GUARD on the reference init: every ray's far sample refined (tau huge) equals the stand-alone exact entry bit for
    bit, the other channels stay the fast pass's, and the self-check's max |delta| stays under tau / 3 of the default tau
    (1.5e-3), so that the generators' self-check never widens tau for this field."""
    siren = _siren("L", DEV)
    film = _film(siren, 2, 77)
    x_lin, y_lin, z_lin = ops.ray_tables(16, 12, 0.88, 1.12, DEV)
    c2w = torch.eye(4, device=DEV).repeat(2, 1, 1)
    c2w[:, 2, 3] = 1.0
    rng = torch.rand(2, 16 * 16, 12, 1, generator=torch.Generator().manual_seed(4)).to(DEV)
    rd = ops.make_render_desc(batch=2, img_size=16, num_steps=12, hierarchical=False, clamp_mode="relu", nerf_noise=0.0,
                              fov=12, precision="guard", guard_tau=1e9)
    with torch.no_grad():
        st = ops.render_forward_stages(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
        pts, dirs = st["points_c"].reshape(2, -1, 3), st["dirs"]
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast").reshape(2, 256, 12, 4)
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact").reshape(2, 256, 12, 4)
        ops.render_forward(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
    rep = ops.guard_stats(DEV)
    print("guard: %s" % rep)
    assert rep["refined"] >= 2 * 256 and rep["max_abs_delta"] < 1.5e-3 / 3
    raw = st["raw_c"]
    assert torch.equal(raw[:, :, :-1], fast[:, :, :-1])
    assert torch.equal(raw[:, :, -1, -1], exact[:, :, -1, -1])
    assert torch.equal(raw[:, :, -1, :-1], fast[:, :, -1, :-1])


# --------------------------------------------------------------------------------------------
# GPU: the backward
# --------------------------------------------------------------------------------------------
_FIELD = [(lay, p) for lay in ("L1", "L2", "L3") for p in ("exact", "default")]


@gpu
@pytest.mark.parametrize("layout,precision", _FIELD, ids=["%s-%s" % c for c in _FIELD])
def test_field_backward_vs_fp64(monkeypatch, layout, precision):
    """_FieldBackward against the float64 VJP under the chunk layouts of test_gpu_fp64_reference.py: the first layer's 35
    columns, the grid gradient through it, FiLM row 0 from image b0 > 0 of a chunk (L2) and from point chunks (L3)."""
    from fenerf_b200 import backward
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    exact = precision == "exact"
    if exact:
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    siren = _siren("L", DEV)
    seed = 3300 + int(layout[1])
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film = _film(siren, batch, seed, edges=True)
    d_raw = torch.randn(batch, ppb, 4, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    monkeypatch.setattr(oracle, "field_eval", GT.field_eval)
    out64, want_film, want = field_ref(siren, monkeypatch, pts, _per_point(dirs, ppb, False), film, d_raw)
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, False, raw, d_raw, exact)
    errs = _grad_errors(d_film, grads, want_film, want)
    worst = max(errs, key=errs.get)
    print("field %s %s: worst %s %.3g (layer 0 %.3g, grid %.3g)" % (layout, precision, worst, errs[worst],
                                                                   errs["network.0.layer.weight"], errs["spatial_embeddings"]))
    bound = {k: GRID_BOUND_EXACT if (exact and k == "spatial_embeddings") else FIELD_BOUND[precision] for k in errs}
    assert all(errs[k] <= bound[k] for k in errs), {k: "%.2e" % v for k, v in errs.items() if v > bound[k]}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, False, raw, d_raw, exact)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        assert inv[worst] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


@gpu
@pytest.mark.parametrize("precision", ["exact", "guard"])
def test_backward_matches_reference_gradients(runs, precision):
    """Against the reference's autograd on the opaque case: <= 5e-4 of each tensor's max in exact mode, <= 2e-2 in the
    default mode, the first layer's feature columns included; the grid's gradient at the reference's largest entries and
    in its absolute sum."""
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    p = _gpu_parity()
    case, run = runs(GT.GRAD_CASE)
    gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % GT.GRAD_CASE))
    gen = _cases.build_mirror(case, DEV)
    latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
    pixels, _ = gen(*latents, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision=precision))
    loss = (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum()
    loss.backward()
    got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({k: q.grad for k, q in gen.named_parameters()})
    rel = 5e-4 if precision == "exact" else 2e-2
    weights = {k: gold[k] for k in gold.files if k != "grid_probe_idx"}

    class _Gold(dict):
        files = list(weights)
    worst = p._compare_grads(_Gold(weights), got, rel=rel, kink_rel=1e-2 if precision == "exact" else 0.3)
    g = gen.siren.spatial_embeddings.grad.reshape(-1).cpu()
    want = torch.from_numpy(gold["grid_probe"])
    probe = (g[torch.from_numpy(gold["grid_probe_idx"])] - want).abs().max().item() / want.abs().max().item()
    worst["grid_probe"] = probe
    # (the bound test_gpu_parity.py gives model B's grid probe: the reference's own gradient is an fp32 sum of trilinear
    # scatter contributions in another order)
    assert probe <= 1e-2, "grid gradient at the reference's largest entries: %.2e of the largest" % probe
    grid_sum = abs(g.abs().sum().item() - float(gold["grid_abs_sum"])) / float(gold["grid_abs_sum"])
    print("gradients %s: %s, grid abs-sum %.1e" % (precision, {k: "%.1e" % v for k, v in worst.items()}, grid_sum))
    assert grid_sum <= (5e-3 if precision == "exact" else 2e-2)


@gpu
def test_inversion_gradients_through_forward_with_frequencies(runs):
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    p = _gpu_parity()
    case, run = runs(GT.GRAD_CASE)
    gold = np.load(os.path.join(GOLDEN, "gradfreq_%s.npz" % GT.GRAD_CASE))
    gen = _cases.build_mirror(case, DEV)
    with torch.no_grad():
        fp = [t.clone().requires_grad_(True) for t in gen.siren.mapping_network(p._cuda(run["latents"][0]))]
    for q in gen.parameters():
        q.requires_grad_(False)
    pixels, _ = gen.forward_with_frequencies(*fp, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=5e-4)
    print("inversion: %s" % worst)


@gpu
def test_staged_forward_sees_feature_column_writes():
    """torch_ema's copy_to writes through param.data without a version bump: a write to the first layer's feature columns
    alone must reach staged_forward (the fingerprint counts all 35 columns)."""
    case = GT.CASE_BY_NAME["l_small_opaque"]          # (white-filled at the plain init: nothing would move)
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(1, 256, generator=torch.Generator().manual_seed(8)).to(DEV)
    kw = dict(case.cfg, psi=0.7, max_batch_size=2400000, precision="exact")
    with torch.no_grad():
        torch.manual_seed(1)
        a = torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(z, **kw)[:2]])
        w = gen.siren.network[0].layer.weight
        new = w.detach().clone()
        new[:, :32] *= -1.0
        w.data.copy_(new)
        torch.manual_seed(1)
        b = torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(z, **kw)[:2]])
        gen.siren.invalidate_packed()
        torch.manual_seed(1)
        c = torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(z, **kw)[:2]])
    assert not torch.equal(a, b)
    assert torch.equal(b, c)
