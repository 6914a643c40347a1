"""Bridge fields (SPATIALSIRENAUGDISENTANGLE, RESSIRENDISENTANGLE): the colour branch starts from a 3-wide v taken off the
trunk output.  CPU: the field spec, the flag rules of the C-ABI, the restatement's faults and the faults the backward's
bounds catch.  GPU: both point-network kernels under the tile schedules of a real SM count, the density-only entries, the
GUARD refinement, and the backward under the chunk layouts of production, against a float64 restatement.  The init,
oracle, drop-in, end-to-end, gradient, inversion and repack checks of these fields run with every other field's, in
test_oracle.py, test_dropin.py and test_gpu_parity.py."""
import copy
import ctypes

import pytest
import torch
import torch.nn.functional as F

import _cases
import test_gpu_fp64_film_edges as FE
from _fp64 import _film, _siren, field_ref
from fenerf_b200 import _lib, backward, ops, packing
from fenerf_b200.siren import siren as S
from oracle import render_oracle as oracle
from test_gpu_fp64_reference import (FIELD_BOUND, LAYOUT_BOUND, _LAYOUTS, _field_backward, _field_points, _forward_inputs,
                                     _grad_errors, _per_point)

DEV = "cuda:0"
CLASSES = _cases.INIT_GOLDENS["bridge_init.json"][1]
#: point network forward, max |out - fp64| over the rgb / the sigma channels, per model.  Measured on an H100 80GB HBM3
#: (132 SMs, 400 W power limit) at up to 20,000 points per image and under the four tile schedules (up to 33,691 points
#: per image): exact <= 1.1e-6 (rgb, AUG at 4sms_minus_1), 8.4e-7 (AUG sigma), 9.7e-6 (RES sigma, scaled chain); fast
#: <= 3.6e-4 (AUG), 2.0e-4 (RES rgb), 1.6e-8 (RES sigma at the reference init, where |a| ~ 1e-6) and 3.6e-3 (RES sigma
#: with the chain scaled so that a . v is O(1): v's error from the fp16 trunk, times |a| = 1)
FWD_BOUND = {"exact": 1e-5, "fast": 5e-3}
FAST_BOUND = {"aug": (6e-4, 6e-4), "res": (3e-4, 1e-6), "res_scaled": (3e-4, 5e-3)}
EXACT_BOUND = {"aug": (2e-6, 2e-6), "res": (2e-6, 1e-7), "res_scaled": (2e-6, 2e-5)}


def _mirror(name, seed=0):
    torch.manual_seed(seed)
    return _cases.construct_field(S, name)


@pytest.mark.parametrize("name", CLASSES)
def test_field_spec(name):
    spec = _mirror(name).field_spec()
    assert spec.bridge and spec.bridge_res == (name == "RESSIRENDISENTANGLE") and spec.out_dim == 4


# --------------------------------------------------------------------------------------------
# CPU: the mirror classes
# --------------------------------------------------------------------------------------------
def _desc(flags, label_dim=0, grid=0, color=8):
    return _lib.FieldDesc(trunk_layers=8, color_layers=color, label_dim=label_dim, grid_channels=grid,
                          grid_res=64 if grid else 0, out_dim=label_dim + 4, input_scale=2 / 0.24, reserved=flags)


def test_bridge_bits_only_in_the_reference_shapes():
    lib = _lib.lib()
    BR, RES = _lib.FIELD_BRIDGE, _lib.FIELD_BRIDGE_RES
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(BR))) > 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(BR | RES, color=6))) > 0
    params = _lib.FieldParams()
    for d in (_desc(RES), _desc(BR | _lib.FIELD_LABEL_FILM, 19), _desc(BR, 19), _desc(BR, grid=32),
              _desc(BR | _lib.FIELD_GRID_TRUNK, grid=32), _desc(BR | _lib.FIELD_FEATURE_HEAD)):
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"unknown field flag combination" in lib.fenerf_last_error()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2
    # a RES field's density chain and color_layer_pre come in fenerf_bridge_params only
    buf = (ctypes.c_uint8 * 2048)()
    aligned = (ctypes.addressof(buf) + 1023) // 1024 * 1024
    assert lib.fenerf_pack_field(ctypes.byref(_desc(BR | RES, color=6)), ctypes.byref(params), aligned, 1, None) == -1
    assert b"fenerf_bridge_params" in lib.fenerf_last_error()
    for name in CLASSES:
        d = packing.field_desc(_mirror(name).field_spec())
        assert d.reserved == (BR | RES if name == "RESSIRENDISENTANGLE" else BR)
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) > 0


def _cpu_inputs(name, seed, n=64, scaled=False):
    siren = _mirror(name, seed).double()
    if scaled:
        _cases.scale_density(siren)
    film = _film(siren.float(), 2, seed).double()
    siren.double()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).double()
    return siren, film, pts, dirs


@pytest.mark.parametrize("name,fault", [("SPATIALSIRENAUGDISENTANGLE", "no_bridge_bias"), ("SPATIALSIRENAUGDISENTANGLE", "swap"),
                                        ("RESSIRENDISENTANGLE", "no_bridge_bias"), ("RESSIRENDISENTANGLE", "no_pos"),
                                        ("RESSIRENDISENTANGLE", "swap")])
def test_faults_move_the_restatement_past_the_bounds(name, fault):
    """A dropped bias of v, RES's v without the position and swapped dir / v columns each move an output channel by more
    than the fast kernel's bound (RES with the scaled density chain, so that sigma depends on v)."""
    siren, film, pts, dirs = _cpu_inputs(name, 5, scaled=name == "RESSIRENDISENTANGLE")
    with torch.no_grad():     # a bias of v a dropped one visibly moves (the default init's is U(+-1/16))
        lin = siren.res_coord_layer if name == "RESSIRENDISENTANGLE" else siren.color_layer_pre[0]
        lin.bias.copy_(torch.tensor([0.1, -0.1, 0.1], dtype=lin.bias.dtype))
        good = oracle.bridge_field_eval(siren, pts, film, dirs)
        bad = oracle.bridge_field_eval(siren, pts, film, dirs, fault=fault)
    assert (good - bad).abs().max() > FWD_BOUND["fast"]


def test_restatement_runs_the_mirror_forward():
    """The mirror's module structure is what the restatement reads: every parameter meets the output."""
    for name in CLASSES:
        siren, film, pts, dirs = _cpu_inputs(name, 3, n=8, scaled=name == "RESSIRENDISENTANGLE")
        out = oracle.bridge_field_eval(siren, pts, film, dirs)
        out.sum().backward()
        missing = [n for n, p in siren.named_parameters() if "mapping" not in n and (p.grad is None or p.grad.abs().max() == 0)]
        assert missing == [], missing


def _c0_freqs_of_image0(field, points, film, dirs):
    """The restatement with image 0's frequencies of the first colour row used for every image (a wrong b0 in dv)."""
    c0 = len(field.network)
    f = film.clone()
    f[1:, c0, 0] = film[0, c0, 0]
    return oracle.bridge_field_eval(field, points, f, dirs)


def _sigma_from_detached_v(field, points, film, dirs):
    return oracle.bridge_field_eval(field, points, film, dirs, fault="sigma_from_detached_v")


_BWD_FAULTS = [("aug", "c0_freqs_of_image0"), ("res_scaled", "c0_freqs_of_image0"), ("res_scaled", "sigma_from_detached_v"),
               ("aug", "dirs_one_ray_off"), ("res_scaled", "dirs_one_ray_off")]


@pytest.mark.parametrize("model,fault", _BWD_FAULTS, ids=["%s-%s" % f for f in _BWD_FAULTS])
def test_backward_faults_exceed_the_bounds(monkeypatch, model, fault):
    """Faults of the bridge's backward, each applied to the float64 restatement: image 0's colour-row-c0 frequencies
    used in every image's dv, RES's density from v.detach() (dv without d sigma . a, on the scaled chain where sigma
    depends on v), and directions sliced one ray off in image 1's second point chunk.  The first two must move some
    gradient past 10x the default-mode bound; the direction fault past 10x the layout-invariance bound, the check that
    sees it in default mode, and past the exact-mode bound."""
    siren = _bridge_siren(model, "cpu")
    batch, ppb, dir_group = 2, 480, 24
    pts, dirs = _field_points(batch, ppb, dir_group, 13)
    film = _film(siren, batch, 13, edges=True)
    d_raw = torch.randn(batch, ppb, 4, generator=torch.Generator().manual_seed(13)) * 1e-3
    _, film_g, good = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw)
    if fault == "dirs_one_ray_off":
        shifted = dirs.clone()
        half = dirs.shape[1] // 2
        shifted[1, half:-1] = dirs[1, half + 1:]
        _, film_b, bad = field_ref(siren, pts, _per_point(shifted, ppb, False), film, d_raw)
    else:
        monkeypatch.setattr(oracle, "field_eval", _c0_freqs_of_image0 if fault == "c0_freqs_of_image0" else _sigma_from_detached_v)
        _, film_b, bad = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw)
    errs = _grad_errors(film_b, bad, film_g, good)
    worst = max(errs, key=errs.get)
    print("bridge backward fault %s %s: %s moves %.3g" % (model, fault, worst, errs[worst]))
    if fault == "dirs_one_ray_off":
        assert errs[worst] > 10 * LAYOUT_BOUND and errs[worst] > FIELD_BOUND["exact"], errs[worst]
    else:
        assert errs[worst] > 10 * FIELD_BOUND["default"], errs[worst]


# --------------------------------------------------------------------------------------------
# GPU: the kernels against the float64 restatement
# --------------------------------------------------------------------------------------------
MODELS = [("SPATIALSIRENAUGDISENTANGLE", False), ("RESSIRENDISENTANGLE", False), ("RESSIRENDISENTANGLE", True)]
_IDS = ["aug", "res", "res_scaled"]


def _gpu_inputs(name, scaled, batch, ppb, seed=7):
    siren = _mirror(name, seed)
    if scaled:
        _cases.scale_density(siren)
    siren = siren.to(DEV)
    film = _film(siren, batch, seed).contiguous()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(batch, ppb, 3, generator=g) - 0.5) * 0.3).to(DEV)
    dirs = F.normalize(torch.randn(batch, ppb, 3, generator=g), dim=-1).to(DEV)
    return siren, film, pts, dirs


def _want(siren, film, pts, dirs):
    s64 = copy.deepcopy(siren).double()
    with torch.no_grad():
        return oracle.bridge_field_eval(s64, pts.double(), film.double(), dirs.double())


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("shape", [64, 64 * 37 + 5, 20000] + list(_cases.TILE_LAYOUTS))
@pytest.mark.parametrize("model", MODELS, ids=_IDS)
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_points_match_float64(model, precision, shape):
    """The point network against the float64 restatement per channel, within the model's own bound.  An int shape is
    points per image with one direction per point (one tile, an odd count, a ragged last tile); a tile layout is one
    of the schedules derived from the device's SM count, with its direction mode (test_gpu_fp64_reference._FWD_DIRS:
    per point, one per 24-sample ray, one per image).  A second launch is bit-identical, and the density-only entries
    (ops.siren_sigma, siren.density) equal the sigma channel bit for bit -- for RES, the density rebuilt from v."""
    if isinstance(shape, int):
        siren, film, pts, dirs = _gpu_inputs(*model, batch=2, ppb=shape)
        dir_group = 1
    else:
        siren = _gpu_inputs(*model, batch=1, ppb=64)[0]
        pts, dirs, film = _forward_inputs(siren, shape, 2400 + MODELS.index(model))
        dir_group = None
    want = _want(siren, film, pts, _per_point(dirs, pts.shape[1], False))
    out = ops.siren_points(siren, pts, film, dirs, precision=precision, dir_group=dir_group)
    again = ops.siren_points(siren, pts, film, dirs, precision=precision, dir_group=dir_group)
    sigma = ops.siren_sigma(siren, pts, film, precision=precision)
    density = siren.density(pts, film, precision=precision)
    torch.cuda.synchronize()
    err = (out.double() - want).abs().amax(dim=(0, 1))
    print("forward %s %s %s (B=%d, ppb %d): max|out - fp64| per channel %s" % (
        _IDS[MODELS.index(model)], precision, shape, pts.shape[0], pts.shape[1], err.tolist()))
    rgb_bound, sigma_bound = (EXACT_BOUND if precision == "exact" else FAST_BOUND)[_IDS[MODELS.index(model)]]
    assert torch.isfinite(out).all()
    assert err[:3].max() <= rgb_bound and err[3] <= sigma_bound, err.tolist()
    assert torch.equal(out, again)
    assert torch.equal(sigma, out[..., -1:]) and torch.equal(density, out[..., -1:])


#: backward cases: (layout of test_gpu_fp64_reference._LAYOUTS, model, lock_dirs, planted edge frequencies).  L2 with
#: planted frequencies on res_scaled: the reference init leaves RES's |a| ~ 1e-6, so only the scaled chain puts the
#: planted colour-row-c0 columns' dv next to a dsigma a of the same size.  The shared bounds hold for every tensor,
#: color_layer_pre and the density chain included.  Measured on an H100 80GB HBM3 (400 W power limit): exact <= 1.8e-5
#: (L4 aug, a FiLM frequency gradient; color_layer_pre <= 1.0e-5, the density chain <= 4.5e-6), default <= 1.24e-2
#: (L1 aug; color_layer_pre <= 9.4e-3); planted columns 5.0e-6 / 4.4e-3; chunked against one chunk 1.3e-5 (exact) and
#: 7.8e-6 (default; 2.8e-4 while dv W_v reached the trunk from a skinny library product, see fenerf_b200/backward.py).
_BWD = ([(lay, m, False, False) for lay in ("L1", "L2", "L3") for m in _IDS]
        + [("L1", m, True, False) for m in _IDS]
        + [("L4", m, False, False) for m in ("aug", "res_scaled")]
        + [("L2", "res_scaled", False, True)])


def _bridge_siren(model_id, device):
    """The generator's field (the seed protocol of _fp64._siren); res_scaled with the density chain scaled."""
    name, scaled = MODELS[_IDS.index(model_id)]
    siren = _siren("M" if name == CLASSES[0] else "N", device)
    return _cases.scale_density(siren) if scaled else siren


@pytest.mark.gpu
@pytest.mark.parametrize("layout,model,lock,edges", _BWD,
                         ids=["%s-%s%s%s" % (lay, m, "-lock_dirs" if k else "", "-edges" if e else "") for lay, m, k, e in _BWD])
@pytest.mark.parametrize("precision", ["exact", "default"])
def test_backward_matches_float64_autograd(monkeypatch, layout, model, lock, edges, precision):
    """``_FieldBackward`` against the float64 VJP of the restatement under the production chunk layouts: every parameter
    gradient (RES's color_layer_pre and density chain unfolded in finish()) and d film, per tensor and per FiLM layer.
    L2 has chunks whose image b0 > 0 reads its own colour-row-c0 frequencies in dv; L3 splits each image into point
    chunks (directions sliced at p0 // dir_group, d a / d c summed over every chunk); L4 is cfg2's pass.  L2 / L3 also
    run as one chunk, within LAYOUT_BOUND.  With `edges`, f = 0, tiny and large |f| are planted in every FiLM role, and
    each planted column is checked on its own."""
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    exact = precision == "exact"
    if exact:
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # exact mode's torch.mm stays fp32
    siren = _bridge_siren(model, DEV)
    seed = 5000 + 10 * _IDS.index(model) + int(layout[1])
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film, planted = FE._edge_film(siren, batch, seed, FE.BACKWARD_FREQS) if edges else (_film(siren, batch, seed, edges=True), [])
    d_raw = torch.randn(batch, ppb, 4, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    out64, want_film, want = field_ref(siren, pts, _per_point(dirs, ppb, lock), film, d_raw)
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, exact)
    assert torch.isfinite(d_film).all() and all(torch.isfinite(g).all() for g in grads.values())
    errs = _grad_errors(d_film, grads, want_film, want)
    bound = FIELD_BOUND[precision]
    worst = max(errs, key=errs.get)
    bridge = {k: "%.2e" % v for k, v in errs.items() if k.split(".")[0] in ("color_layer_pre", "density_layer_linear",
                                                                           "res_coord_layer", "final_layer")}
    print("bridge field %s %s %s: worst %s %.3g; bridge tensors %s" % (layout, model, precision, worst, errs[worst], bridge))
    assert errs[worst] <= bound, {k: "%.2e" % v for k, v in errs.items() if v > bound}
    if edges:
        cols = FE._planted_errors(d_film, grads, want_film, want, planted, FE._layer_weights(siren))
        worst_col = max(cols, key=cols.get)
        print("bridge edge columns %s %s %s: worst %s %.3g" % (layout, model, precision, worst_col, cols[worst_col]))
        assert cols[worst_col] <= FIELD_BOUND[precision], {k: "%.2e" % v for k, v in cols.items() if v > FIELD_BOUND[precision]}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, exact)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        print("bridge layout %s %s %s: worst %s %.3g" % (layout, model, precision, worst, inv[worst]))
        assert inv[worst] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS, ids=_IDS)
def test_guard_refinement(model):
    """GUARD: every ray's far sample refined (tau huge) equals the stand-alone exact entry bit for bit -- RES's density
    rebuilt from v in the GUARD kernel -- and the other channels stay the fast pass's.  The self-check's max |delta|
    stays under tau / 3 of the default tau (1.5e-3) for AUG and for RES at the reference init; with RES's density chain
    scaled so that a . v is O(1) it is v's fp16 error times |a| (measured 3.0e-3 on an H100, no sign flips), above tau / 3: the
    generators' self-check then widens tau for such weights (README, DESIGN section 5), and the bound here is the fast
    kernel's sigma bound."""
    siren, _, _, _ = _gpu_inputs(*model, batch=2, ppb=64)
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
    print("guard %s: %s" % (model, rep))
    assert rep["refined"] >= 2 * 256
    bound = 1.5e-3 / 3 if _IDS[MODELS.index(model)] != "res_scaled" else FAST_BOUND["res_scaled"][1]
    assert rep["max_abs_delta"] < bound
    raw = st["raw_c"]
    assert torch.equal(raw[:, :, :-1], fast[:, :, :-1])
    assert torch.equal(raw[:, :, -1, -1], exact[:, :, -1, -1])
    assert torch.equal(raw[:, :, -1, :-1], fast[:, :, -1, :-1])


# --------------------------------------------------------------------------------------------
# render level: the oracle and the library against the reference's goldens
# --------------------------------------------------------------------------------------------