"""The direction-free texture-grid field (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96, model P): the first
colour layer reads cat[feat, x] with U(+-1/3) weights and no ray direction.  CPU: the mirror against the reference's init,
the flag rules and the layout of the C-ABI, the oracle against the reference's goldens, the restatement's gradients and
the faults the bounds catch.  GPU: the exact point network against a float64 restatement, the refusal of the fp16 colour
path (and the density-only entry it leaves), the renders and gradients against the reference's goldens, the backward
against float64 under production chunk layouts, and repacking."""
import copy
import ctypes
import io
import json
import os

import numpy as np

import pytest
import torch
import torch.nn.functional as F

import _cases
import _harness
import _wo_dir_fields as WF
from _fp64 import _film, _siren, field_ref
from fenerf_b200 import _lib, backward, ops, packing
from fenerf_b200.siren import siren as S
from oracle import render_oracle as oracle
from test_gpu_fp64_reference import (_LAYOUTS, _field_backward, _field_points, _forward_inputs,
                                     _grad_errors, _per_point)

DEV = "cuda:0"
GOLDEN = _cases.GOLDEN_DIR
#: exact point network, max |out - fp64| over the (labels, rgb, sigma) channels.  Measured on an H100 80GB HBM3 (700 W
#: power limit): labels 8.1e-8, rgb 8.4e-5, sigma 7.6e-7.  The wgmma colour path is refused for this field: its rgb error
#: was 2.1e-2 at 2 x 2048 points, the fp16 trunk's own error amplified by the first colour layer's U(+-1/3) weights at
#: f ~ 30 (with those weights zeroed on the trunk columns it was 7.7e-5; DESIGN section 5).  The density alone stays on
#: the wgmma kernel: 2.9e-4 there.
EXACT_BOUND = (1e-5, 2e-4, 1e-5)
SIGMA_FAST_BOUND = 1e-3
#: the backward in the exact mode against float64, relative to each tensor's max (measured <= 1.7e-3: fp32 rounding through
#: the same amplification; FIELD_BOUND['exact'] = 1e-4 holds for the other fields).  It also bounds a chunked run against a
#: one-chunk run (measured 1.2e-3: the fp32 library GEMMs round differently for other row counts, and the first colour
#: layer amplifies that too; LAYOUT_BOUND = 5e-5 holds for the other fields)
BWD_BOUND = 3e-3


def _mirror(name, seed=0):
    torch.manual_seed(seed)
    return getattr(S, name)(**WF.KWARGS)


# --------------------------------------------------------------------------------------------
# CPU: the mirror classes, the flag, the layout
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", WF.CLASSES)
def test_mirror_init_and_state_dict_are_the_references(name):
    with open(os.path.join(GOLDEN, "wo_dir_init.json")) as f:
        gold = json.load(f)[name]
    siren = _mirror(name)
    assert torch.rand(1).item() == gold["next_draw"]          # the init drew exactly the reference's draws
    assert _harness.state_digest(siren) == gold["digest"]
    assert [n for n, _ in siren.named_parameters()] == gold["names"]
    assert {k: list(v.shape) for k, v in siren.state_dict().items()} == gold["state"]
    assert [n for n, _ in siren.named_children()] == gold["children"]
    spec = siren.field_spec()
    assert spec.wo_dir and spec.color_layers == 8 and spec.label_dim == 18 and spec.grid_channels == 32


@pytest.mark.parametrize("name", WF.CLASSES)
def test_mirror_pickles_and_resolves_by_name(name):
    import fenerf_b200
    fenerf_b200.install()
    import siren.siren as installed
    assert getattr(installed, name) is getattr(S, name)
    siren = _mirror(name)
    buf = io.BytesIO()
    torch.save(siren, buf)
    back = torch.load(io.BytesIO(buf.getvalue()), map_location="cpu", weights_only=False)
    assert type(back) is getattr(S, name)
    assert all(torch.equal(a, b) for a, b in zip(siren.state_dict().values(), back.state_dict().values()))


def _desc(flags, label_dim=18, grid=32, trunk=8, color=8):
    return _lib.FieldDesc(trunk_layers=trunk, color_layers=color, label_dim=label_dim, grid_channels=grid,
                          grid_res=96 if grid else 0, out_dim=label_dim + 4, input_scale=2 / 0.24, reserved=flags)


def test_wo_dir_flag_only_in_the_reference_shape():
    lib = _lib.lib()
    WD = _lib.FIELD_WO_DIR
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(WD))) > 0
    params = _lib.FieldParams()
    for d in (_desc(WD | _lib.FIELD_GRID_TRUNK), _desc(WD | _lib.FIELD_LABEL_FILM), _desc(WD | _lib.FIELD_BRIDGE),
              _desc(WD, grid=0), _desc(WD, label_dim=0), _desc(WD, color=3), _desc(WD, trunk=7)):
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"unknown field flag combination" in lib.fenerf_last_error()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2
    d = packing.field_desc(_mirror(WF.CLASSES[1]).field_spec())
    assert d.reserved == WD and d.grid_channels == 32 and d.color_layers == 8 and d.label_dim == 18


def test_hidden_width_128_is_refused():
    with pytest.raises(ValueError, match="hidden_dim=256"):
        packing.collect_params(_mirror(WF.CLASSES[0]), torch.device("cpu"))


def test_packed_layout_is_the_plain_grid_layout():
    """The direction-free field packs into the plain 8 + 8 grid layout (kx = 3 + G, zero direction rows): same sections,
    same sizes."""
    lib = _lib.lib()
    plain = lib.fenerf_packed_bytes(ctypes.byref(_desc(0)))
    mine = lib.fenerf_packed_bytes(ctypes.byref(_desc(_lib.FIELD_WO_DIR)))
    assert plain > 0 and mine == plain


# --------------------------------------------------------------------------------------------
# CPU: the restatement, its gradients and its faults
# --------------------------------------------------------------------------------------------
def _cpu_inputs(seed, n=1024):
    siren = _siren("P", "cpu")
    film = _film(siren, 2, seed)
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).double()
    return copy.deepcopy(siren).double(), film.double(), pts, dirs


def test_restatement_is_the_oracle_and_passes_gradcheck():
    siren, film, pts, dirs = _cpu_inputs(3, n=6)
    with torch.no_grad():
        assert torch.equal(oracle.field_eval(siren, pts, film, dirs), oracle.wo_dir_field_eval(siren, pts, film, dirs))
    c0 = len(siren.network)

    def f(sub):
        fl = film.clone()
        fl[:, c0, :, :3] = sub
        return oracle.wo_dir_field_eval(siren, pts, fl, dirs)[..., 18:21]
    sub = film[:, c0, :, :3].clone().requires_grad_(True)
    assert torch.autograd.gradcheck(f, (sub,), eps=1e-6, atol=1e-7)


@pytest.mark.parametrize("fault", ["fp16_first_colour", "with_dir", "feat_after_x"])
def test_faults_move_the_colours_past_the_exact_bound(fault):
    """At the reference init, fp16 operands in the first colour layer alone (emulated), the direction in the colour input
    and the features after x each move the colours past the exact kernel's rgb bound."""
    siren, film, pts, dirs = _cpu_inputs(5)
    with torch.no_grad():
        good = oracle.wo_dir_field_eval(siren, pts, film, dirs)
        bad = oracle.wo_dir_field_eval(siren, pts, film, dirs, fault=fault)
    err = (good - bad)[..., 18:21].abs().max().item()
    print("fault %s: max |rgb| move %.3g" % (fault, err))
    assert err > EXACT_BOUND[1]


@pytest.mark.parametrize("case", WF.CASES, ids=lambda c: c.name)
def test_oracle_matches_reference_golden(case):
    from test_hd_fields import _golden_pixels
    if case.name in WF.BIG and not os.environ.get("FENERF_SLOW_TESTS") and not torch.cuda.is_available():
        pytest.skip("minutes of CPU oracle (FENERF_SLOW_TESTS=1 runs it)")
    gold = np.load(_cases.golden_path(case))
    run = _harness.oracle_run(case, keep_stages=False)
    got, want, _ = _golden_pixels(run["out"]["pixels"], gold)
    assert (got - want).abs().max() <= 2e-5


# --------------------------------------------------------------------------------------------
# GPU: the point network against float64, the refused fp16 colour path
# --------------------------------------------------------------------------------------------
def _gpu_inputs(batch, ppb, seed=7):
    siren = _siren("P", DEV)
    film = _film(siren, batch, seed).contiguous()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(batch, ppb, 3, generator=g) - 0.5) * 0.3).to(DEV)
    dirs = F.normalize(torch.randn(batch, ppb, 3, generator=g), dim=-1).to(DEV)
    return siren, film, pts, dirs


def _want(siren, film, pts, dirs):
    s64 = copy.deepcopy(siren).double()
    with torch.no_grad():
        return oracle.wo_dir_field_eval(s64, pts.double(), film.double(), dirs.double())


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("shape", [64, 64 * 37 + 5, 20000] + list(_cases.TILE_LAYOUTS))
def test_points_match_float64(shape):
    """The exact point network against the float64 restatement per channel group (labels, rgb, sigma).  A second launch is
    bit-identical, other directions -- and the locked direction (0, 0, -1) -- give the same bits, and the density-only
    entries (exact, and fast on the wgmma kernel) match the sigma channel."""
    if isinstance(shape, int):
        siren, film, pts, dirs = _gpu_inputs(batch=2, ppb=shape)
        dir_group = 1
    else:
        siren = _gpu_inputs(batch=1, ppb=64)[0]
        pts, dirs, film = _forward_inputs(siren, shape, 2600)
        dir_group = None
    want = _want(siren, film, pts, _per_point(dirs, pts.shape[1], False))
    out = ops.siren_points(siren, pts, film, dirs, precision="exact", dir_group=dir_group)
    again = ops.siren_points(siren, pts, film, dirs, precision="exact", dir_group=dir_group)
    other = ops.siren_points(siren, pts, film, F.normalize(torch.randn_like(dirs), dim=-1), precision="exact",
                             dir_group=dir_group)
    locked = torch.zeros_like(dirs)
    locked[..., 2] = -1
    lock = ops.siren_points(siren, pts, film, locked, precision="exact", dir_group=dir_group)
    sigma = ops.siren_sigma(siren, pts, film, precision="exact")
    sigma_fast = siren.density(pts, film, precision="fast")
    torch.cuda.synchronize()
    err = (out.double() - want).abs().amax(dim=(0, 1))
    groups = (err[:18].max().item(), err[18:21].max().item(), err[21].item())
    fast_err = (sigma_fast.double() - want[..., -1:]).abs().max().item()
    print("forward P exact %s (B=%d, ppb %d): max|out - fp64| labels / rgb / sigma %s; fast density %.3g" % (
        shape, pts.shape[0], pts.shape[1], ["%.3g" % e for e in groups], fast_err))
    assert torch.isfinite(out).all()
    assert all(e <= b for e, b in zip(groups, EXACT_BOUND)), groups
    assert torch.equal(out, again) and torch.equal(out, other) and torch.equal(out, lock)
    assert torch.equal(sigma, out[..., -1:])
    assert fast_err <= SIGMA_FAST_BOUND


@pytest.mark.gpu
def test_fp16_colour_path_is_refused():
    """fast and guard renders and the default-mode backward raise with the reason, instead of returning colours ~2e-2 off."""
    siren, film, pts, dirs = _gpu_inputs(batch=1, ppb=64)
    with torch.no_grad(), pytest.raises(RuntimeError, match="FENERF_FIELD_WO_DIR"):
        ops.siren_points(siren, pts, film, dirs, precision="fast")
    x_lin, y_lin, z_lin = ops.ray_tables(16, 12, 0.88, 1.12, DEV)
    c2w = torch.eye(4, device=DEV).repeat(1, 1, 1)
    c2w[:, 2, 3] = 1.0
    rng = torch.rand(1, 16 * 16, 12, 1, generator=torch.Generator().manual_seed(4)).to(DEV)
    rd = ops.make_render_desc(batch=1, img_size=16, num_steps=12, hierarchical=False, clamp_mode="relu", nerf_noise=0.0,
                              fov=12, precision="guard")
    with torch.no_grad(), pytest.raises(RuntimeError, match="FENERF_FIELD_WO_DIR"):
        ops.render_forward(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
    one = torch.ones(1, device=DEV)
    with pytest.raises(RuntimeError, match="precision='exact' only"):
        backward._FieldBackward(siren, film, one, one, exact=False)


# --------------------------------------------------------------------------------------------
# GPU: the backward against float64 under the production chunk layouts
# --------------------------------------------------------------------------------------------
#: (layout, lock_dirs, planted): with `planted`, f = 0, +-2^-19 ... +-50 (test_gpu_fp64_film_edges.BACKWARD_FREQS: +-50 is
#: the top of what the mapping network gives these fields) are planted in every FiLM role, the first colour layer's row
#: included, within BWD_BOUND; then the full EDGE_FREQS with |f| = 150, where the first colour layer's U(+-1/3) weights
#: scale fp32 rounding five times further than at f ~ 30: finite, within EDGE_BOUND (measured 8.3e-3, the grid's
#: gradient; the library's default-mode bound for the other fields)
EDGE_BOUND = 2e-2
_BWD = [("L1", False, False), ("L2", False, False), ("L3", False, False), ("L1", True, False), ("L2", False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("layout,lock,edges", _BWD,
                         ids=["%s%s%s" % (lay, "-lock_dirs" if k else "", "-edges" if e else "") for lay, k, e in _BWD])
def test_backward_matches_float64_autograd(monkeypatch, layout, lock, edges):
    """``_FieldBackward`` (exact mode) against the float64 VJP of the restatement: every parameter gradient (the grid's
    included) and d film, per tensor and per FiLM layer, within BWD_BOUND; L2 / L3 also run as one chunk, within the same
    bound.  With planted edge frequencies every gradient is finite and each planted column is checked on its own."""
    import test_gpu_fp64_film_edges as FE
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    # TF32 on, a common training setting: the backward keeps this field's products fp32 itself
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", True)
    siren = _siren("P", DEV)
    seed = 6000 + int(layout[1])
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film, planted = (FE._edge_film(siren, batch, seed, FE.BACKWARD_FREQS) if edges
                     else (_film(siren, batch, seed, edges=True), []))
    d_raw = torch.randn(batch, ppb, 22, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    out64, want_film, want = field_ref(siren, pts, _per_point(dirs, ppb, lock), film, d_raw)
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, True)
    assert torch.isfinite(d_film).all() and all(torch.isfinite(g).all() for g in grads.values())
    errs = _grad_errors(d_film, grads, want_film, want)
    worst = max(errs, key=errs.get)
    c0 = {k: "%.2e" % v for k, v in errs.items() if k.startswith("color_layer_sine.0") or k == "spatial_embeddings"}
    print("wo_dir backward %s: worst %s %.3g; first colour layer / grid %s" % (layout, worst, errs[worst], c0))
    assert errs[worst] <= BWD_BOUND, {k: "%.2e" % v for k, v in errs.items() if v > BWD_BOUND}
    if edges:
        cols = FE._planted_errors(d_film, grads, want_film, want, planted, FE._layer_weights(siren))
        worst_col = max(cols, key=cols.get)
        print("wo_dir edge columns %s: worst %s %.3g" % (layout, worst_col, cols[worst_col]))
        assert cols[worst_col] <= BWD_BOUND, {k: "%.2e" % v for k, v in cols.items() if v > BWD_BOUND}
        film150, _ = FE._edge_film(siren, batch, seed)
        out150, want_film150, want150 = field_ref(siren, pts, _per_point(dirs, ppb, lock), film150, d_raw)
        d_film150, grads150 = _field_backward(siren, film150, pts, dirs, dir_group, lock, out150.float().contiguous(), d_raw,
                                              True)
        assert torch.isfinite(d_film150).all() and all(torch.isfinite(g).all() for g in grads150.values())
        e150 = _grad_errors(d_film150, grads150, want_film150, want150)
        worst150 = max(e150, key=e150.get)
        print("wo_dir edges up to |f| = 150 %s: worst %s %.3g" % (layout, worst150, e150[worst150]))
        assert e150[worst150] <= EDGE_BOUND, {k: "%.2e" % v for k, v in e150.items() if v > EDGE_BOUND}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, True)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        print("wo_dir layout %s: worst %s %.3g" % (layout, worst, inv[worst]))
        assert inv[worst] <= BWD_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > BWD_BOUND}


# --------------------------------------------------------------------------------------------
# GPU: renders and gradients against the reference's goldens
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


@pytest.mark.gpu
@pytest.mark.parametrize("case", WF.CASES, ids=lambda c: c.name)
def test_end_to_end_against_reference_golden(runs, case):
    """Exact renders against the reference's: measured on an H100 80GB HBM3 (700 W) <= 5.6e-4 (p_cfg2; 2.5e-4 .. 3.4e-4 on
    the small cases) -- the reference's own fp32 forward differs from float64 by the same amplification of its rounding."""
    import test_gpu_parity as p
    from test_hd_fields import _golden_pixels
    gold = np.load(_cases.golden_path(case))
    case, run = runs(case.name)
    gen, pixels, poses, depth_map = p._end_to_end(case, run, "exact")
    ill_rays = p._ill_conditioned_pixels(case, run)
    got, want, idx = _golden_pixels(pixels, gold)
    err = (got - want).abs()
    assert int(ill_rays.sum()) <= max(2, 0.002 * ill_rays.numel())
    ill = ill_rays.unsqueeze(1).expand_as(pixels).reshape(-1)
    if idx is not None:
        ill = ill[idx]
    print("%s exact: max err %.3g" % (case.name, err[~ill].max()))
    assert err[~ill].max() <= 1e-3
    if poses is not None:
        assert (poses - torch.from_numpy(gold["poses"])).abs().max() <= 1e-5


@pytest.mark.gpu
def test_generator_gradients_match_reference(runs):
    """forward() with autograd (exact mode) against the reference's autograd on the opaque case: <= 1e-2 of each tensor's
    max (measured <= 6.6e-3)."""
    import test_gpu_parity as p
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    case, run = runs(WF.GRAD_CASE)
    gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % WF.GRAD_CASE))
    gen = _cases.build_mirror(case, DEV)
    latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
    pixels, _ = gen(*latents, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({k: q.grad for k, q in gen.named_parameters()})
    worst = p._compare_grads(gold, got, rel=1e-2, kink_rel=1e-2)
    print("gradients P exact: %s" % ({k: "%.1e" % v for k, v in worst.items()},))


@pytest.mark.gpu
def test_inversion_gradients_through_forward_with_frequencies(runs):
    """d pixels / d (frequencies, phase shifts) through forward_with_frequencies, exact mode: <= 1e-2 (measured 5.9e-3)."""
    import test_gpu_parity as p
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    case, run = runs(WF.GRAD_CASE)
    gold = np.load(os.path.join(GOLDEN, "gradfreq_%s.npz" % WF.GRAD_CASE))
    gen = _cases.build_mirror(case, DEV)
    with torch.no_grad():
        lat = [p._cuda(z) for z in run["latents"]]
        fp = [t.clone().requires_grad_(True) for t in gen.siren.geo_mapping_network(lat[0]) + gen.siren.app_mapping_network(lat[1])]
    for q in gen.parameters():
        q.requires_grad_(False)
    pixels, _ = gen.forward_with_frequencies(fp[0], fp[2], fp[1], fp[3],
                                             **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=1e-2)
    print("inversion P: %s" % (worst,))


@pytest.mark.gpu
def test_staged_forward_sees_first_colour_layer_writes():
    """torch_ema's copy_to writes through param.data without a version bump: a write to color_layer_sine[0] alone -- its
    feature columns alone, too -- must reach staged_forward (the fingerprint covers all 288 columns)."""
    case = _cases.CASE_BY_NAME["p_small_opaque"]
    gen = _cases.build_mirror(case, DEV)
    s = gen.siren
    g = torch.Generator().manual_seed(8)
    z = [torch.randn(1, 256, generator=g).to(DEV) for _ in range(2)]
    kw = dict(case.cfg, psi=0.7, max_batch_size=2400000, precision="exact")
    w = s.color_layer_sine[0].layer.weight

    def render():
        torch.manual_seed(1)
        return torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(*z, **kw)[:2]])
    with torch.no_grad():
        for cols in (slice(None), slice(0, 32)):
            a = render()
            w.data[:, cols].copy_(w.detach()[:, cols] * -3.0)
            b = render()
            s.invalidate_packed()
            assert not torch.equal(a, b) and torch.equal(b, render())
