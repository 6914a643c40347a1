"""grad_precision='split': the backward of precision='split' / 'exact' renders with its 256-wide products on the split
kernels of csrc/gemm_split.cu (fp16 hi / lo operands scaled by powers of two, fp32 accumulation).

CPU: the restatement of tools/split_backward_precision.py against float64 within its bounds and the faults they catch,
the keyword's validation and refusals, the new C-ABI symbols.  GPU: each kernel against float64 products (odd, ragged and
single-tile row counts, multi-image chunks, cfg2's 393216-row pass, dU rows spanning 1e-8 .. 1e2), ``_FieldBackward`` in
split mode against the float64 VJP under the chunk layouts, gradients through renders against the reference's goldens,
the default backward untouched without the keyword, and the refusals through the generators."""
import math
import os

import numpy as np
import pytest
import torch

import _cases
import _harness
import _wo_dir_fields as WF
from _fp64 import _film, _siren, field_ref
from fenerf_b200 import _lib, backward, ops
from fenerf_b200.generators.volumetric_rendering import ReplayRng
from test_gpu_fp64_reference import (FIELD_BOUND, FIELD_MODELS, LAYOUT_BOUND, _LAYOUTS, _field_points, _grad_errors,
                                     _per_point)
from tools import split_backward_precision as SB

DEV = "cuda:0"
gpu = pytest.mark.gpu
SPLIT_SYMBOLS = ("fenerf_gemm_nt_split", "fenerf_gemm_nt_film_split", "fenerf_gemm_tn_split", "fenerf_absmax_f32")
#: variants the split kernels do not serve: label FiLM (I, K), feature head (J, K), grid trunk (L), bridge (M, N)
REFUSED = ("I", "J", "K", "L", "M", "N")


# --------------------------------------------------------------------------------------------
# CPU: the restatement against float64 and its faults (tools/split_backward_precision.py)
# --------------------------------------------------------------------------------------------
#: largest error over the trunk's layers (activations absolute; M_b, dA' relative to each layer's max), 2 latents x 512
#: points at the reference's init.  The tool's rows at this size: A (3.1e-6, 1.0e-6, 1.2e-6), B (3.6e-6, 1.1e-6,
#: 1.3e-6); the bounds are about 1.4x those.  The faults move B past them by >= 3x (sinf, unscaled) and >= 1000x (dropped
#: terms).
CPU_BOUND = {"A": (4.4e-6, 1.5e-6, 1.7e-6), "B": (5.1e-6, 1.6e-6, 1.9e-6)}


@pytest.fixture(scope="module")
def cpu_fields():
    out = {}
    for m in CPU_BOUND:
        siren, film, pts, _ = SB.inputs(m, latents=2, points=512)
        out[m] = (siren, film, pts)
    return out


def _groups(e):
    return e["act"], e["m_b"], e["d_a"]


@pytest.mark.parametrize("model", sorted(CPU_BOUND))
def test_restatement_within_bound(cpu_fields, model):
    e = SB.errors(*cpu_fields[model])
    print("%s split backward: %s" % (model, {k: "%.3g" % v for k, v in e.items()}))
    assert all(g <= b for g, b in zip(_groups(e), CPU_BOUND[model])), e


@pytest.mark.parametrize("fault", SB.FAULTS)
def test_faults_move_the_restatement_past_the_bound(cpu_fields, fault):
    """A dropped lo.hi or hi.lo term, dU split without its power-of-two scale, or __sinf in the recompute each move the
    restatement past its bound."""
    e = SB.errors(*cpu_fields["B"], fault=fault)
    print("B %s: %s" % (fault, {k: "%.3g" % v for k, v in e.items()}))
    assert any(g > b for g, b in zip(_groups(e), CPU_BOUND["B"])), e


# --------------------------------------------------------------------------------------------
# CPU: the keyword, the refusals, the C-ABI
# --------------------------------------------------------------------------------------------
def _rd(precision):
    return ops.make_render_desc(batch=1, img_size=4, num_steps=4, hierarchical=False, clamp_mode="relu", nerf_noise=0.0,
                                fov=12, precision=precision)


@pytest.mark.parametrize("precision", ["exact", "split"])
@pytest.mark.parametrize("model", ["A", "B", "P"])
def test_grad_precision_accepted(model, precision):
    siren = _siren(model, "cpu")
    backward.check_grad_precision(siren, "split", precision)
    backward.check_grad_precision(siren, "split", _lib.PRECISION[precision])
    for p in ("exact", "split", "fast", "guard"):
        backward.check_grad_precision(siren, None, p)        # no keyword: every precision, as before


@pytest.mark.parametrize("precision", ["fast", "guard"])
def test_grad_precision_refused_with_the_fp16_backward(precision):
    siren = _siren("A", "cpu")
    with pytest.raises(RuntimeError, match="grad_precision='split' differentiates precision='split' or 'exact'"):
        backward.check_grad_precision(siren, "split", precision)
    with pytest.raises(RuntimeError, match="precision='split' or 'exact'"):     # before anything reaches the device
        backward.render_with_grad(siren, _rd(precision), None, None, None, None, None, None, None, None, None,
                                  grad_precision="split")


@pytest.mark.parametrize("model", REFUSED)
def test_grad_precision_refused_for_fields_the_split_kernels_do_not_serve(model):
    siren = _siren(model, "cpu")
    with pytest.raises(RuntimeError, match="grad_precision='split' is not built for fields with"):
        backward.check_grad_precision(siren, "split", "exact")
    with pytest.raises(RuntimeError, match="is not built for fields with"):
        backward.render_with_grad(siren, _rd("split"), None, None, None, None, None, None, None, None, None,
                                  grad_precision="split")


def test_unknown_grad_precision_is_a_value_error():
    with pytest.raises(ValueError, match="grad_precision must be one of"):
        backward.check_grad_precision(_siren("A", "cpu"), "fp16", "exact")


def test_split_abi_symbols_resolve():
    lib = _lib.lib()
    header = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "fenerf_b200.h")).read()
    for name in SPLIT_SYMBOLS:
        assert name in _lib.EXPORTS and hasattr(lib, name), name
        assert "int %s(" % name in header, name
    assert lib.fenerf_abi_version() == _lib.ABI_VERSION


def test_split_weights_scale_and_parts():
    """ops.split_weights: max |s W| in [2^14, 2^15), s a power of two, hi + lo = s W to fp32 rounding of the lo part."""
    g = torch.Generator().manual_seed(3)
    w = torch.randn(3, 256, 256, generator=g) * torch.tensor([6e-3, 1e-8, 30.0]).reshape(3, 1, 1)
    hi, lo, amax = ops.split_weights(w)
    s = torch.ldexp(torch.ones(3), ops.split_scale_exp(amax))
    top = (w.abs().amax(dim=(1, 2)) * s)
    assert torch.all((top >= 2 ** 14) & (top < 2 ** 15)), top
    resid = (hi.double() + lo.double() - w.double() * s.double().reshape(3, 1, 1)).abs().amax(dim=(1, 2))
    assert torch.all(resid <= top.double() * 2.0 ** -22), resid


# --------------------------------------------------------------------------------------------
# GPU: the kernels against float64 products
# --------------------------------------------------------------------------------------------
#: max |out - fp64| / max |fp64| of one product, measured on an H100 80GB HBM3.  dA' (K = 256): the fp16 pairs carry 22
#: bits and the lo.lo term (2^-22) is dropped; measured <= 1.6e-6.  M_b: the same per product, then fp32 accumulation over
#: the ~6000 points a CTA sums at cfg2 (the fp32 library product has the same kind of error); measured 2.2e-5.  A dropped
#: lo term is ~2e-3 (tools/split_backward_precision.py).
GEMM_BOUND = 4e-6
TN_BOUND = 5e-5
#: recompute: max |a - fp64|, |gate - fp64| with u = f (z + b) + p, |f| up to ~100: f times the 2^-22 of z, and the fp32
#: rounding of u; measured 2.6e-5
FILM_BOUND = 5e-5
_ROWS = [1, 64, 127, 128, 64 * 37 + 5, 393216]


def _wide_rows(m, seed, lo=-8.0, hi=2.0):
    """(m, 256) fp32 whose row magnitudes are spread log-uniformly over 10^lo .. 10^hi."""
    g = torch.Generator().manual_seed(seed)
    mag = torch.pow(10.0, lo + (hi - lo) * torch.rand(m, 1, generator=g))
    return (torch.randn(m, 256, generator=g) * mag).float()


def _weights(seed, n=1):
    g = torch.Generator().manual_seed(seed)
    f = 30.0 + 15.0 * torch.randn(n, 256, 1, generator=g)
    w = (torch.rand(n, 256, 256, generator=g) * 2 - 1) * math.sqrt(6 / 256) / 25
    return (f * w).float()


def _sines(m, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.sin(torch.randn(m, 256, generator=g) * 3).float()


@gpu
@pytest.mark.parametrize("rows", _ROWS)
@pytest.mark.parametrize("spread", [False, True], ids=["sines", "dU_1e-8_1e2"])
def test_nt_split_vs_fp64(rows, spread):
    """dA' = dU diag(f) W (and z = a W^T): rows of A either sines or spanning 1e-8 .. 1e2."""
    a = (_wide_rows(rows, rows) if spread else _sines(rows, rows)).to(DEV)
    bmat = _weights(rows + 1)[0].to(DEV)
    hi, lo, bmax = ops.split_weights(bmat)
    amax = ops.absmax(a) if spread else None
    if spread:
        assert amax.item() == a.abs().max().item()
    out = ops.gemm_nt_split(a, hi, lo, bmax, a_amax=amax)
    want = a.double() @ bmat.double().t()
    err = (out.double() - want).abs().max().item() / want.abs().max().item()
    print("nt split M=%d %s: %.3g" % (rows, "spread" if spread else "sines", err))
    assert torch.isfinite(out).all() and err <= GEMM_BOUND
    assert torch.equal(out, ops.gemm_nt_split(a, hi, lo, bmax, a_amax=amax))
    if spread and rows >= 128:      # rows far below the maximum: within the fp32 sums' share of the largest rows
        small = (a.abs().amax(1) < 1e-6 * a.abs().max())
        if small.any():
            assert (out.double() - want)[small].abs().max().item() <= GEMM_BOUND * want.abs().max().item()


@gpu
@pytest.mark.parametrize("rows,ppb", [(1, 1), (127, 127), (3 * 1000, 1000), (2 * 64 * 37 + 10, 64 * 37 + 5),
                                      (2 * 393216, 393216)])
def test_nt_film_split_vs_fp64(rows, ppb):
    """The recompute with its FiLM epilogue: each image of a multi-image chunk takes its own FiLM rows (from b0 = 1)."""
    n_img = rows // ppb
    a = _sines(rows, rows).to(DEV)
    w = (_weights(rows + 2)[0] / 30).to(DEV)
    hi, lo, wmax = ops.split_weights(w)
    g = torch.Generator().manual_seed(rows)
    film = torch.randn(n_img + 1, 3, 2, 256, generator=g)
    film[:, :, 0] = 30 + 15 * film[:, :, 0]
    film = film.to(DEV)
    bias = (torch.rand(256, generator=g) * 0.1).to(DEV)
    act, gate = ops.gemm_nt_film_split(a, hi, lo, wmax, bias, film, 1, 2, ppb)
    z = a.double() @ w.double().t()
    img = torch.arange(rows, device=DEV) // ppb + 1
    u = film[img, 2, 0].double() * (z + bias.double()) + film[img, 2, 1].double()
    ea, eg = (act.double() - torch.sin(u)).abs().max().item(), (gate.double() - torch.cos(u)).abs().max().item()
    print("nt film split M=%d ppb=%d: sin %.3g cos %.3g" % (rows, ppb, ea, eg))
    assert ea <= FILM_BOUND and eg <= FILM_BOUND


@gpu
@pytest.mark.parametrize("batch,ppb", [(1, 1), (1, 63), (2, 64), (3, 64 * 37 + 5), (2, 393216)])
def test_tn_split_vs_fp64(batch, ppb):
    """M_b = dU_b^T a per image, split-K: dU rows spanning 1e-8 .. 1e2, a sines."""
    x = _wide_rows(batch * ppb, ppb + batch).to(DEV)
    y = _sines(batch * ppb, ppb).to(DEV)
    amax = ops.absmax(x)
    out = ops.gemm_tn_split(x, y, batch, ppb, x_amax=amax)
    want = torch.bmm(x.double().view(batch, ppb, 256).transpose(1, 2), y.double().view(batch, ppb, 256))
    err = max((out[b].double() - want[b]).abs().max().item() / want[b].abs().max().item() for b in range(batch))
    with backward._NoTF32():
        f32 = torch.bmm(x.view(batch, ppb, 256).transpose(1, 2), y.view(batch, ppb, 256))
    err32 = max((f32[b].double() - want[b]).abs().max().item() / want[b].abs().max().item() for b in range(batch))
    print("tn split B=%d ppb=%d: %.3g (fp32 library %.3g)" % (batch, ppb, err, err32))
    assert torch.isfinite(out).all() and err <= TN_BOUND
    if ppb <= 4096:     # one CTA per image and row half (a longer fp32 sum in one accumulator loses more bits)
        one = ops.gemm_tn_split(x, y, batch, ppb, x_amax=amax, slices=1)
        err1 = max((one[b].double() - want[b]).abs().max().item() / want[b].abs().max().item() for b in range(batch))
        print("tn split B=%d ppb=%d, one slice: %.3g" % (batch, ppb, err1))
        assert err1 <= TN_BOUND


# --------------------------------------------------------------------------------------------
# GPU: _FieldBackward in split mode against the float64 VJP
# --------------------------------------------------------------------------------------------
#: P, the direction-free field: its first colour layer amplifies rounding (test_wo_dir_fields.BWD_BOUND = 3e-3 for the
#: exact mode).  Measured on an H100 80GB HBM3: split <= 4.1e-3, the exact mode 1.5e-3 on the same inputs -- the split
#: operands' 22 bits against fp32's 24, as in the forward (tests/test_split_precision.py).
P_BOUND = 6e-3
_FIELD = ([(lay, m) for lay in ("L1", "L2", "L3") for m in FIELD_MODELS + ("P",)] + [("L4", "A"), ("L4", "B")])


def _field_backward(siren, film, pts, dirs, dir_group, raw, d_raw, grad_split=True):
    with torch.no_grad(), backward._NoTF32():
        m = d_raw.abs().max()
        scale = torch.exp2(4.0 - torch.ceil(torch.log2(m.clamp_min(1e-30)))).float().reshape(1)   # as backward._field_backward
        fb = backward._FieldBackward(siren, film, scale, (1.0 / scale).float().reshape(1), exact=True, grad_split=grad_split)
        fb.add_points(pts, dirs, dir_group, False, raw, d_raw)
        d_film, grads = fb.finish()
    return d_film, {n: grads[id(p)].reshape(p.shape) for n, p in siren.named_parameters() if id(p) in grads}


@gpu
@pytest.mark.parametrize("layout,model", _FIELD, ids=["%s-%s" % f for f in _FIELD])
def test_field_backward_split_vs_fp64(monkeypatch, layout, model):
    """Every parameter gradient, the whole grid gradient and d film within the exact mode's bound of the float64 VJP, at
    FiLM tables with edge frequencies; the chunked layouts (L2, L3) agree with one chunk within LAYOUT_BOUND."""
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    siren = _siren(model, DEV)
    seed = 3000 + 10 * (FIELD_MODELS + ("P",)).index(model) + int(layout[1])
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film = _film(siren, batch, seed, edges=True)
    out_dim = siren.field_spec().out_dim
    d_raw = torch.randn(batch, ppb, out_dim, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    out64, want_film, want = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw)
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    l0 = _lib.launch_count()
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, raw, d_raw)
    assert _lib.launch_count() > l0
    errs = _grad_errors(d_film, grads, want_film, want)
    worst = max(errs, key=errs.get)
    print("field split %s %s: worst %s %.3g" % (layout, model, worst, errs[worst]))
    if model == "P":
        ex = _grad_errors(*_field_backward(siren, film, pts, dirs, dir_group, raw, d_raw, grad_split=False), want_film, want)
        wex = max(ex, key=ex.get)
        print("field exact %s %s: worst %s %.3g" % (layout, model, wex, ex[wex]))
    bound = P_BOUND if model == "P" else FIELD_BOUND["exact"]
    assert errs[worst] <= bound, {k: "%.2e" % v for k, v in errs.items() if v > bound}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, raw, d_raw)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        print("layout split %s %s: worst %s %.3g" % (layout, model, worst, inv[worst]))
        bound = P_BOUND if model == "P" else LAYOUT_BOUND
        assert inv[worst] <= bound, {k: "%.2e" % v for k, v in inv.items() if v > bound}


# --------------------------------------------------------------------------------------------
# GPU: gradients through renders against the reference's goldens
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


def _latent_grads(runs, name, precision, **extra):
    import test_gpu_parity as p
    case, run = runs(name)
    gen = _cases.build_mirror(case, DEV)
    latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
    kw = {k: v for k, v in case.cfg.items() if k != "fill_mode"}
    pixels, _ = gen(*latents, **dict(kw, _rng=ReplayRng(run["draws"], DEV), precision=precision, **extra))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({k: q.grad for k, q in gen.named_parameters()})
    return got


@gpu
@pytest.mark.parametrize("name", ["a_small", "b_small"])
@pytest.mark.parametrize("precision", ["exact", "split"])
def test_render_gradients_against_reference(runs, name, precision):
    """forward() with grad_precision='split' after an exact or split forward: within the exact mode's 5e-4 (the density
    head's relu kink: 1e-2, as the exact test) of the reference's gradients."""
    import test_gpu_parity as p
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "grad_%s.npz" % name))
    l0 = _lib.launch_count()
    got = _latent_grads(runs, name, precision, grad_precision="split")
    assert _lib.launch_count() - l0 > 20
    worst = p._compare_grads(gold, got, rel=5e-4, kink_rel=1e-2)
    print("%s %s + grad split: %s" % (name, precision, {k: "%.2e" % v for k, v in worst.items()}))


@gpu
@pytest.mark.parametrize("name", ["a_small", "d_small"])
def test_inversion_gradients_against_reference(runs, name):
    """forward_with_frequencies with grad_precision='split': the FiLM-offset gradients within 5e-4."""
    import test_gpu_parity as p
    case, run = runs(name)
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "gradfreq_%s.npz" % name))
    gen = _cases.build_mirror(case, DEV)
    with torch.no_grad():
        if case.model == "A":
            fp = list(gen.siren.mapping_network(p._cuda(run["latents"][0])))
        else:
            fg, pg = gen.siren.geo_mapping_network(p._cuda(run["latents"][0]))
            fa, pa = gen.siren.app_mapping_network(p._cuda(run["latents"][1]))
            fp = [fg, fa, pg, pa]
    fp = [t.clone().requires_grad_(True) for t in fp]
    for q in gen.parameters():
        q.requires_grad_(False)
    pixels, _ = gen.forward_with_frequencies(*fp, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="split",
                                                         grad_precision="split"))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=5e-4)
    print("%s inversion grad split: %s" % (name, {k: "%.2e" % v for k, v in worst.items()}))


@gpu
@pytest.mark.parametrize("golden", ["grad", "gradfreq"])
def test_direction_free_gradients_against_reference(runs, golden):
    """The direction-free field (P) through forward() and forward_with_frequencies with grad_precision='split': within the
    1e-2 of each tensor's largest entry that its split-render gradient test uses."""
    import test_gpu_parity as p
    case, run = runs(WF.GRAD_CASE)
    gold = np.load(os.path.join(_cases.GOLDEN_DIR, "%s_%s.npz" % (golden, WF.GRAD_CASE)))
    gen = _cases.build_mirror(case, DEV)
    kw = dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="split", grad_precision="split")
    if golden == "grad":
        latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
        pixels, _ = gen(*latents, **kw)
        (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
        got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
        got.update({k: q.grad for k, q in gen.named_parameters()})
        worst = p._compare_grads(gold, got, rel=1e-2, kink_rel=1e-2)
    else:
        with torch.no_grad():
            lat = [p._cuda(z) for z in run["latents"]]
            fp = [t.clone().requires_grad_(True)
                  for t in gen.siren.geo_mapping_network(lat[0]) + gen.siren.app_mapping_network(lat[1])]
        for q in gen.parameters():
            q.requires_grad_(False)
        pixels, _ = gen.forward_with_frequencies(fp[0], fp[2], fp[1], fp[3], **kw)
        (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
        worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=1e-2)
    print("%s P grad split: %s" % (golden, {k: "%.2e" % v for k, v in worst.items()}))


# --------------------------------------------------------------------------------------------
# GPU: no keyword, no change; refusals through the generators
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", ["exact", "split"])
def test_without_the_keyword_the_backward_is_unchanged(monkeypatch, runs, precision):
    """Without grad_precision (or with None) the backward never reaches the split kernels and launches as many kernels as
    before; two runs agree to the last bits that the column-sum and grid atomics leave to the order of arrival."""
    l0 = _lib.launch_count()
    first = _latent_grads(runs, "b_small", precision)
    n_first = _lib.launch_count() - l0

    def refuse(*a, **k):
        raise AssertionError("the split kernels ran without grad_precision='split'")
    for name in ("gemm_nt_split", "gemm_nt_film_split", "gemm_tn_split", "absmax"):
        monkeypatch.setattr(ops, name, refuse)
    l0 = _lib.launch_count()
    again = _latent_grads(runs, "b_small", precision, grad_precision=None)
    assert _lib.launch_count() - l0 == n_first
    for k, v in first.items():
        assert (v is None) == (again[k] is None), k
        if v is not None:
            assert (v - again[k]).abs().max().item() <= 1e-5 * v.abs().max().item(), k


@gpu
@pytest.mark.parametrize("name,precision", [("a_small", "fast"), ("a_small", "guard"), ("b_small", "guard")])
def test_generators_refuse_grad_split_with_the_fp16_backward(runs, name, precision):
    case, run = runs(name)
    gen = _cases.build_mirror(case, DEV)
    latents = [t.to(DEV).requires_grad_(True) for t in run["latents"]]
    kw = {k: v for k, v in case.cfg.items() if k != "fill_mode"}
    with pytest.raises(RuntimeError, match="precision='split' or 'exact'"):
        gen(*latents, **dict(kw, _rng=ReplayRng(run["draws"], DEV), precision=precision, grad_precision="split"))
    with torch.no_grad():       # no autograd: the keyword is ignored
        gen(*[t.detach() for t in latents], **dict(kw, _rng=ReplayRng(run["draws"], DEV), precision="exact",
                                                   grad_precision="split"))


@gpu
@pytest.mark.parametrize("model", REFUSED)
def test_field_backward_refuses_unserved_fields(model):
    siren = _siren(model, DEV)
    film = _film(siren, 1, 3).contiguous()
    one = torch.ones(1, device=DEV)
    with pytest.raises(RuntimeError, match="is not built for fields with"):
        backward._FieldBackward(siren, film, one, one, exact=True, grad_split=True)
    with pytest.raises(RuntimeError, match="precision='split' or 'exact'"):
        backward._FieldBackward(_siren("A", DEV), _film(_siren("A", DEV), 1, 3), one, one, exact=False, grad_split=True)
