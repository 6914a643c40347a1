"""``_FieldBackward`` and the point network at the edges of the FiLM frequency range, against float64.

The FiLM tables of test_gpu_fp64_reference.py keep |f| >= 0.25.  Here plant_frequencies() writes f = 0, -0, ±2^-19 (one
ulp of the table's 15 x + 30 near 0), ±1e-5, ±1e-3, ±0.05 and ±150 (±50 for the backward, see BACKWARD_FREQS) into
the first, a middle and the last trunk layer, the label FiLM layer (models I, K), and the first colour layer (its narrow
[dir, grid] inputs; the grid gradient of model H; the [dir, v] inputs of the bridge fields M, N, whose dv takes this
row's frequencies; [dir] alone for model L, whose grid feeds layer 0) and the last one: each value in one column of
every image and in another column of the last image only, so that image b0 > 0 of a multi-image chunk sees it.  The
committed bounds of test_gpu_fp64_reference.py apply unchanged, to every tensor and to each planted column on its own
(relative to its layer's maximum, so that a wrong column cannot hide behind a right maximum); model L keeps its own
exact-mode bounds for the grid gradient and the forward (tests/_cases.py, MODEL_DATA).

Measured on an H100 80GB HBM3 (400 W): backward exact 1.7e-5, default 1.07e-2 (model H, L2; planted columns 8.0e-3),
layout invariance within LAYOUT_BOUND; forward exact 2.2e-6, fast 7.9e-4 (model K).  Models J, L, M, N on the same
card and power limit: backward exact 1.3e-5 (N, L3; L's grid gradient 1.1e-4), default 1.05e-2 (N, L3), layout
invariance 1.3e-5; forward exact 1.4e-5 (L), fast 8.5e-4 (J).  Before the backward stopped dividing by f, every L1
case gave NaN FiLM gradients at f = 0 in both precisions.
"""
import pytest
import torch

import _cases
from _fp64 import EDGE_FREQS, _film, _siren, field_ref, film_rows, plant_frequencies
from fenerf_b200 import backward, ops
from test_gpu_fp64_reference import (FIELD_BOUND, LAYOUT_BOUND, _LAYOUTS, _field_backward, _field_points,
                                     _grad_errors, _per_point)

DEV = "cuda:0"
gpu = pytest.mark.gpu

#: I: label FiLM; J, K: feature heads; L: the grid in the trunk; M, N: the bridge fields ([dir, v] as the first colour
#: layer's only inputs, FiLM role color_first)
MODELS = ("A", "D", "H", "I", "K", "J", "L", "M", "N")
#: the backward's planted values: EDGE_FREQS with |f| = 150 replaced by 50, the top of what the mapping network gives
#: these fields (|f| <= 54 over their tables).  At |f| = 150 the default mode measured 4.6e-2 (model H, L2: a bias
#: gradient, whose largest entry is then f dp at that column, with dp carrying the fp16 recompute's error of u = f z + p
#: scaled by f) and the exact mode's layout invariance 1.1e-4 (model A, L3: the fp32 library GEMMs' other summation
#: orders, scaled the same way); nothing overflows.  The forward test below keeps +-150.
BACKWARD_FREQS = EDGE_FREQS[:-2] + (50.0, -50.0)
_CASES = ([(lay, m, p) for lay in ("L1", "L2", "L3") for m in MODELS for p in ("exact", "default")]
          + [("L4", "A", p) for p in ("exact", "default")])


def _edge_film(siren, batch, seed, freqs=EDGE_FREQS):
    film = _film(siren, batch, seed, edges=True)
    rows = [r for r in film_rows(siren).values() if r is not None]
    return plant_frequencies(film, rows, freqs)


def _layer_weights(siren):
    """(weight name, bias name) of each FiLM row, in FiLM-row order."""
    names = ["network.%d.layer" % i for i in range(len(siren.network))]
    if hasattr(siren, "label_layer_sine"):
        names.append("label_layer_sine.layer")
    color = siren.color_layer_sine
    if isinstance(color, torch.nn.ModuleList):
        names += ["color_layer_sine.%d.layer" % j for j in range(len(color))]
    else:
        names.append("color_layer_sine.layer")
    return [(n + ".weight", n + ".bias") for n in names]


def _planted_errors(d_film, grads, want_film, want, planted, layers):
    """max error of each planted column (its FiLM freq / phase gradient, its weight row and bias entry) relative to the
    maximum of its layer's whole tensor."""
    errs = {}

    def rel(got, ref, scale):
        s = scale.abs().max().item()
        return (got.double() - ref.double()).abs().max().item() / (s if s > 0 else 1.0)

    for row, col, img in planted:
        imgs = slice(None) if img is None else slice(img, img + 1)
        tag = "row%d.col%d%s" % (row, col, "" if img is None else ".img%d" % img)
        for k, name in ((0, "freq"), (1, "phase")):
            errs["%s.%s" % (tag, name)] = rel(d_film[imgs, row, k, col], want_film[imgs, row, k, col], want_film[:, row, k])
        wn, bn = layers[row]
        errs[tag + ".weight"] = rel(grads[wn][col], want[wn][col], want[wn])
        errs[tag + ".bias"] = rel(grads[bn][col], want[bn][col], want[bn])
    return errs


def _grad_bounds(names, precision):
    """FIELD_BOUND, except the exact mode's grid gradient: model L's bound (_cases.MODEL_DATA)."""
    return {n: _cases.bound("L", "grid_exact") if (precision == "exact" and n == "spatial_embeddings") else FIELD_BOUND[precision]
            for n in names}


def _fwd_bound(model, precision):
    return _cases.bound(model, "fwd_" + precision)


@gpu
@pytest.mark.parametrize("layout,model,precision", _CASES, ids=["%s-%s-%s" % c for c in _CASES])
def test_field_backward_at_edge_frequencies(monkeypatch, layout, model, precision):
    """``_FieldBackward`` with f = 0, tiny and large |f| planted: finite everywhere, every tensor and every planted
    column within FIELD_BOUND, and the L2 / L3 chunked run within LAYOUT_BOUND of a one-chunk run."""
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    exact = precision == "exact"
    if exact:
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    siren = _siren(model, DEV)
    seed = 3000 + 10 * MODELS.index(model) + int(layout[1])
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film, planted = _edge_film(siren, batch, seed, BACKWARD_FREQS)
    out_dim = siren.field_spec().out_dim
    d_raw = torch.randn(batch, ppb, out_dim, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    out64, want_film, want = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw)
    assert torch.isfinite(want_film).all() and all(torch.isfinite(g).all() for g in want.values())
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, False, raw, d_raw, exact)
    bad = [n for n, g in grads.items() if not torch.isfinite(g).all()]
    assert torch.isfinite(d_film).all() and not bad, ("non-finite gradients", bad, (~torch.isfinite(d_film)).nonzero()[:8].tolist())
    bound = FIELD_BOUND[precision]
    errs = _grad_errors(d_film, grads, want_film, want)
    bounds = _grad_bounds(errs, precision)
    cols = _planted_errors(d_film, grads, want_film, want, planted, _layer_weights(siren))
    worst, worst_col = max(errs, key=errs.get), max(cols, key=cols.get)
    print("edge field %s %s %s: worst %s %.3g, planted %s %.3g" % (layout, model, precision, worst, errs[worst], worst_col,
                                                                 cols[worst_col]))
    assert all(errs[k] <= bounds[k] for k in errs), {k: "%.2e" % v for k, v in errs.items() if v > bounds[k]}
    assert cols[worst_col] <= bound, {k: "%.2e" % v for k, v in cols.items() if v > bound}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, False, raw, d_raw, exact)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        print("edge layout %s %s %s: worst %s %.3g" % (layout, model, precision, worst, inv[worst]))
        assert inv[worst] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


@gpu
@pytest.mark.parametrize("model", MODELS)
def test_point_network_at_edge_frequencies(model):
    """Both point-network kernels on the planted tables against float64 within FWD_BOUND, per output channel; at |f| =
    150 the pre-activations reach the hundreds (the fast kernel's sin.approx and its fp16 operands)."""
    siren = _siren(model, DEV)
    seed = 4000 + MODELS.index(model)
    batch, ppb = 2, 6000
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, 24, seed))
    film, _ = _edge_film(siren, batch, seed)
    with torch.no_grad():
        got = {p: ops.siren_points(siren, pts, film, dirs, precision=p) for p in ("exact", "fast")}
    want = field_ref(siren, pts, _per_point(dirs, ppb, False), film)[0]
    err = {k: (v.double() - want).abs().amax((0, 1)) for k, v in got.items()}
    print("edge forward %s: exact %.3g fast %.3g" % (model, err["exact"].max(), err["fast"].max()))
    for k in err:
        assert torch.isfinite(got[k]).all(), k
        assert err[k].max() <= _fwd_bound(model, k), "%s: max |out - fp64| per channel %s" % (k, err[k].tolist())
