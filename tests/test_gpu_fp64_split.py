"""precision='split' and grad_precision='split' against float64 where their other tests do not reach.

The point network of every served plain field is in test_split_precision.py (GPU_BOUND: A-H, D32 and P under the tile
schedules), and every stage of split camera renders, the point-network outputs included, in
test_gpu_fp64_forward_stages.py (the '-split' rows of _RENDERS, check_points).  This file adds:

  * the split point network at the edge FiLM frequencies of test_gpu_fp64_film_edges.py (f = 0, -0, +-2^-19, +-1e-5,
    +-1e-3, +-0.05 and +-150 planted in the first, middle and last trunk layer and the first and last colour layer, in a
    column of every image and another of the last image only) for models A, B, D, H, D32 and P: all values at once,
    and each planted (row, value) on its own table, so that a planted column's error is measured apart from the
    others', beside the unplanted table and the exact kernel on every table.  Bound: the exact kernel's,
    FWD_BOUND['exact'], on every table; P 2e-4 (its exact bound) on each single-column table and 3e-4 with every value
    planted at once (EDGE_P_BOUND: the measured cause);
  * the training backward: backward.render_with_grad(..., grad_precision='split') after a split forward, against the
    float64 VJP of the camera render's chain on its own intermediates (test_gpu_fp64_train_grads.py), at the training
    step (8 x 64², 24 + 24 samples, chunks of 5 + 3 images, so FiLM rows come from b0 = 5), with softplus and noise,
    with an opaque field, at cfg2 (A, 4 x 128²), under lock_view_dependence, for D and H at 64² and P at 48².  Every
    tensor within FIELD_BOUND['exact'] (test_split_backward.P_BOUND for P), and so is each image's own d film under the
    GAN-shaped spread of upstream gradients (1e-3 ... 1 of the batch's largest): the split hi / lo operands are floating
    point and keep ~22 bits of each value until the fp16 low part goes subnormal, ~2^-18 of the layer's largest entry;
  * the backward's properties in split: d pixels x 2^k (k = -20, 16, 24) gives gradients x 2^k (the per-layer
    power-of-two scale of fenerf_absmax_f32 absorbs 2^k, so the hi / lo parts are bit-identical) up to twice the
    run-to-run spread; an inf or a nan in one image's d pixels makes every parameter gradient non-finite (the render's
    global scale, from max |d raw|, is already non-finite); under a finite global scale, a nan in a dU stream, which
    absmax_kernel's fmaxf skips, still reaches the split products through its own hi / lo parts, and leaves every
    other entry bit-identical; an image with zero upstream gradient gets a d film of exactly zero; grad_rays on a
    random 3/8 of the rays matches the chain on the masked d pixels.

CPU: check_points, applied to the float64 reference with a typical fault, moves past FWD_BOUND['exact'] at least
tenfold: the coarse pass left unlocked under lock_view_dependence, image b + 1's FiLM rows used for image b.

Measured on an H100 80GB HBM3 (700 W power limit), this file's GPU part in about 20 s:
  * edge frequencies: A, B, D, H and D32 <= 2.9e-6 (model H, every value planted; one planted row <= 2.1e-6; the
    exact kernel <= 1.3e-6), P 1.52e-4 for one planted row and 2.16e-4 for all (the exact kernel 8.5e-5: EDGE_P_BOUND);
  * training backward, max |grad - fp64| / max |grad fp64| over every tensor: <= 7.3e-5 (H-split: d film of FiLM row
    9's frequencies; train-B 3.3e-5, train-B-noise 3.7e-5, train-B-opaque 3.8e-5, cfg2-A 1.9e-5, lock-A 2.4e-5,
    D 4.0e-5), P 5.1e-3; each image's own d film <= 7.3e-5 (P 7.6e-3: P_IMAGE_BOUND), so a split render's FiLM
    gradients need no per-image care whatever the spread of the upstream gradients;
  * loss scales 2^-20, 2^16, 2^24: 21 of 34 tensors bit-identical, the rest (the biases, d film: the atomics) within
    5.6e-7 of their maximum against a run-to-run spread of 6.3e-7; an inf or a nan makes all 33 parameter gradients
    non-finite; in the split products a nan leaves the absmax scale at its other entries' 1e-3 and makes its dA row
    and its M row non-finite (256 of 256 each), an inf makes the scale inf; the zeroed image's d film is exactly zero
    (the others 4.9e-5); grad_rays 4.1e-5.
"""
import pytest
import torch

from _fp64 import EDGE_FREQS, _film, _opt, _siren, field_ref, film_rows, plant_frequencies
from fenerf_b200 import backward, ops
from test_gpu_fp64_film_edges import _edge_film
from test_gpu_fp64_forward_stages import point_errors, point_refs
from test_gpu_fp64_reference import FIELD_BOUND, FWD_BOUND, _field_points, _grad_errors, _per_point
from test_gpu_fp64_train_grads import (_all, _moved, _oracle_render, camera_grads, chain, check_against_chain,  # noqa: F401
                                       film_errors_per_image, fp32_products, make_render, ray_mask, stages)
from test_split_backward import P_BOUND, _sines, _weights

DEV = "cuda:0"
gpu = pytest.mark.gpu


# --------------------------------------------------------------------------------------------
# GPU: the split point network at edge FiLM frequencies
# --------------------------------------------------------------------------------------------
EDGE_MODELS = ("A", "B", "D", "H", "D32", "P")
#: P, max |out - fp64| (rgb): each planted (row, value) on its own within the exact kernel's bound for this field, 2e-4;
#: every value planted at once within 3e-4.  Measured: the unplanted table 8.8e-5 (the exact kernel 4.7e-5); |f| = 150
#: alone in one row 9.9e-5 ... 1.52e-4 (the middle trunk row; the exact kernel <= 5.9e-5 on every table); every value at
#: once 2.16e-4 (exact 8.5e-5).  At a planted column u = f (z + b) + p carries f times the error of z, which split's
#: products leave at ~2^-22 of the terms against fp32's 2^-24; the first colour layer's U(+-1/3) weights amplify it
#: into rgb (test_wo_dir_fields.py), and the rows' increments over the unplanted table add up when all are planted.
EDGE_P_BOUND = {"column": 2e-4, "all": 3e-4}


def _edge_errors(siren, pts, dirs, film):
    """(split, exact): max |out - fp64| over every point and channel of one FiLM table, and split's per image."""
    want = field_ref(siren, pts, _per_point(dirs, pts.shape[1], False), film)[0]
    split, exact = ((ops.siren_points(siren, pts, film, dirs, precision=p).double() - want).abs() for p in ("split", "exact"))
    assert torch.isfinite(split).all()
    return split.max().item(), exact.max().item(), split.amax((1, 2))


@gpu
@torch.no_grad()
@pytest.mark.parametrize("model", EDGE_MODELS)
def test_split_point_network_at_edge_frequencies(model):
    """At |f| = 150 the pre-activations reach the hundreds: soft_sinf's range reduction and the fp32 fold of f b + p.
    The tables: the unplanted one, every value planted at once (_edge_film), and each planted (row, value) on its own,
    in its column of every image and its column of the last image, so that each planted column's error is its own and
    not the field's.  The exact kernel runs on every table beside split."""
    siren = _siren(model, DEV)
    seed = 5000 + EDGE_MODELS.index(model)
    batch, ppb = 2, 6000
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, 24, seed))
    film0 = _film(siren, batch, seed, edges=True)           # the table _edge_film plants into
    rows = sorted({r for r in film_rows(siren).values() if r is not None})
    tables = {"none": film0, "all": _edge_film(siren, batch, seed)[0]}
    for r in rows:
        for v in EDGE_FREQS:
            tables[(r, v)] = plant_frequencies(film0, [r], (v,))[0]
    errs = {k: _edge_errors(siren, pts, dirs, t) for k, t in tables.items()}
    print("edge forward %s: split / exact kernel: unplanted %.3g / %.3g; all planted %.3g / %.3g (per image %s)" % (
        model, *errs["none"][:2], *errs["all"][:2], ["%.3g" % e for e in errs["all"][2].tolist()]))
    for r in rows:
        big = max(errs[(r, v)][0] for v in EDGE_FREQS[-2:])
        rest = max(errs[(r, v)][0] for v in EDGE_FREQS[:-2])
        print("  row %d alone: |f| = 150 %.3g / %.3g, the other values <= %.3g / %.3g" % (
            r, big, max(errs[(r, v)][1] for v in EDGE_FREQS[-2:]), rest, max(errs[(r, v)][1] for v in EDGE_FREQS[:-2])))
    bound = {k: (EDGE_P_BOUND["all" if k == "all" else "column"] if model == "P" else FWD_BOUND["exact"]) for k in errs}
    over = {str(k): "%.3g" % e[0] for k, e in errs.items() if e[0] > bound[k]}
    assert not over, over


# --------------------------------------------------------------------------------------------
# GPU: the training backward in split against the float64 chain
# --------------------------------------------------------------------------------------------
#: name -> (model, B, R, S, options, lock_view_dependence, opaque field); precision='split', grad_precision='split'
_CASES = {
    "train-B-split": ("B", 8, 64, 24, _opt("relu"), False, False),
    "train-B-noise-split": ("B", 8, 64, 24, _opt("softplus", noise=0.5), False, False),
    "train-B-opaque-split": ("B", 4, 64, 24, _opt("relu"), False, True),
    "cfg2-A-split": ("A", 4, 128, 24, _opt("relu"), False, False),
    "lock-A-split": ("A", 4, 64, 24, _opt("relu"), True, False),
    "D-split": ("D", 4, 64, 24, _opt("relu"), False, False),
    "H-split": ("H", 4, 64, 24, _opt("relu"), False, False),
    "P-split": ("P", 3, 48, 24, _opt("relu"), False, False),
}


def split_render(model, b, r, s, o, lock, opaque, seed):
    return dict(make_render(model, b, r, s, o, "split", lock, opaque, seed), model=model)


def split_case(name):
    model, b, r, s, o, lock, opaque = _CASES[name]
    return split_render(model, b, r, s, o, lock, opaque, sum(map(ord, name)))


#: P's own d film per image, relative to that image's largest entry.  Measured 7.6e-3 (the tensors 5.1e-3, P_BOUND
#: 6e-3), and 7.6e-3 again with the spread of upstream gradients taken out, so the shared scale costs nothing; the
#: exact backward gets 2.9e-3 per image (2.5e-3 over the tensors) on the same render.  The field's amplification of
#: rounding (P_BOUND), not the split streams' scaling, sets it.
P_IMAGE_BOUND = 1e-2


def check_split(x, tag, d_film, grads, want_film, want):
    """check_against_chain at the split bound (P_BOUND for P, FIELD_BOUND['exact'] otherwise), and each image's own
    d film, relative to its own largest entry, within FIELD_BOUND['exact'] (P_IMAGE_BOUND for P)."""
    p = x["model"] == "P"
    check_against_chain(x, tag, d_film, grads, want_film, want, bound=P_BOUND if p else FIELD_BOUND["exact"])
    per_image = film_errors_per_image(d_film, want_film)
    bound = P_IMAGE_BOUND if p else FIELD_BOUND["exact"]
    assert per_image.max().item() <= bound, ["%.2e" % v for v in per_image.tolist()]


@gpu
@pytest.mark.parametrize("name", list(_CASES))
def test_split_train_gradients_vs_fp64(fp32_products, name):
    """render_with_grad in split with grad_precision='split' on a GAN-shaped d pixels: d film and every parameter
    gradient against the float64 VJP of the chain on the render's own intermediates."""
    x = split_case(name)
    px, d_film, grads = camera_grads(x, x["d_pixels"], grad_precision="split")
    st = stages(x)
    assert torch.equal(st["pixels"], px), "render_forward_stages differs from the differentiable render"
    want_film, want = chain(x, st, x["d_pixels"])
    if x["model"] == "P":       # the exact backward on the same render, for comparison
        _, film_ex, grads_ex = camera_grads(x, x["d_pixels"])
        ex = _grad_errors(film_ex, {k: grads_ex[k] for k in want}, want_film, want)
        print("train grads %s, exact backward: worst %.3g; d film per image %s" % (
            name, max(ex.values()), ["%.2g" % v for v in film_errors_per_image(film_ex, want_film).tolist()]))
        d_flat = x["d_pixels"] / x["d_pixels"].abs().amax((1, 2, 3), keepdim=True)     # the spread taken out
        _, film_fl, _ = camera_grads(x, d_flat, grad_precision="split")
        print("train grads %s, no spread: d film per image %s" % (
            name, ["%.2g" % v for v in film_errors_per_image(film_fl, chain(x, st, d_flat)[0]).tolist()]))
    check_split(x, name, d_film, grads, want_film, want)


# --------------------------------------------------------------------------------------------
# GPU: properties of the split backward
# --------------------------------------------------------------------------------------------
def _grads(x, d, **kw):
    return _all(*camera_grads(x, d, grad_precision="split", **kw)[1:])


@gpu
def test_split_loss_scale_homogeneity(fp32_products):
    """d pixels x 2^k (k = -20, 16, 24) gives every gradient x 2^k, within twice the run-to-run spread of three runs of
    g(d) (test_gpu_fp64_train_grads.test_loss_scale_homogeneity): the absmax scales shift by k, so the hi / lo parts
    are bit-identical, and only the order of the backward's atomics can differ."""
    x = split_case("train-B-split")
    d = x["d_pixels"]
    g1 = _grads(x, d)
    runs = [_moved(_grads(x, d), g1) for _ in range(2)]
    spread = max(max(r.values()) for r in runs)
    print("split homogeneity: run-to-run spread %.3g; tensors that differ between runs: %s" % (
        spread, sorted({k for r in runs for k, v in r.items() if v > 0})))
    for k in (-20, 16, 24):
        moved = _moved({n: v * 2.0 ** -k for n, v in _grads(x, d * 2.0 ** k).items()}, g1)
        worst = max(moved, key=moved.get)
        print("split homogeneity 2^%d: worst %s %.3g (twice the spread %.3g); bit-identical %d of %d tensors" % (
            k, worst, moved[worst], 2 * spread, sum(v == 0 for v in moved.values()), len(moved)))
        assert moved[worst] <= 2 * spread, (k, {n: v for n, v in moved.items() if v > 2 * spread})


@gpu
@pytest.mark.parametrize("value", ["inf", "nan"])
def test_split_non_finite_upstream_reaches_the_parameters(value):
    """One inf (or nan) in d pixels of one image leaves every parameter gradient non-finite, so GradScaler skips the
    step.  In a render the backward's global scale, from max |d raw| (torch's max keeps a nan; an inf gives scale 0
    and inv_scale inf), is non-finite before any per-layer absmax runs; test_split_products_carry_a_non_finite_entry
    covers the split products under a finite global scale."""
    x = split_case("train-B-split")
    d = x["d_pixels"].clone()
    d[6, 3, 17, 41] = float(value)
    _, d_film, grads = camera_grads(x, d, grad_precision="split")
    bad = [k for k, v in grads.items() if not torch.isfinite(v).all()]
    print("split non-finite %s: %d of %d parameter gradients non-finite, d film finite: %s" % (
        value, len(bad), len(grads), bool(torch.isfinite(d_film).all())))
    assert len(bad) == len(grads), sorted(set(grads) - set(bad))


@gpu
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_split_products_carry_a_non_finite_entry(value):
    """The split products' own scales, fenerf_absmax_f32 per dU stream, with one non-finite entry in image 1's dU (2
    images of 300 points).  absmax_kernel's fmaxf skips a nan, so the stream keeps the scale of its other entries; the
    nan's own hi / lo parts (f16(nan) is nan) then carry it: its row of dU W^T and its column's row of image 1's
    dU^T a are nan, and every other entry is bit-identical to the products of the stream with a 0 in its place.  An
    inf makes the scale inf: its row and its column's row are non-finite."""
    batch, ppb, row, col = 2, 300, 317, 40
    du = (_sines(batch * ppb, 61) * 1e-3).to(DEV)
    du[row, col] = 0.0
    bad = du.clone()
    bad[row, col] = float(value)
    hi, lo, wmax = ops.split_weights(_weights(62)[0].to(DEV))
    a = _sines(batch * ppb, 63).to(DEV)
    amax, amax_bad = ops.absmax(du), ops.absmax(bad)
    nt, nt_bad = (ops.gemm_nt_split(t, hi, lo, wmax, a_amax=m) for t, m in ((du, amax), (bad, amax_bad)))
    tn, tn_bad = (ops.gemm_tn_split(t, a, batch, ppb, x_amax=m) for t, m in ((du, amax), (bad, amax_bad)))
    print("split products, a %s in dU: absmax %g (without it %g); its dA row finite %d of 256, its M row %d of 256" % (
        value, amax_bad.item(), amax.item(), int(torch.isfinite(nt_bad[row]).sum()), int(torch.isfinite(tn_bad[1, col]).sum())))
    assert not torch.isfinite(nt_bad[row]).any() and not torch.isfinite(tn_bad[1, col]).any()
    if value == "nan":
        assert torch.equal(amax_bad, amax)
        others = torch.arange(batch * ppb, device=DEV) != row
        assert torch.equal(nt_bad[others], nt[others])
        keep = torch.ones(batch, 256, dtype=torch.bool, device=DEV)
        keep[1, col] = False
        assert torch.equal(tn_bad[keep], tn[keep])
    else:
        assert torch.isinf(amax_bad).all()


@gpu
def test_split_image_isolation(fp32_products):
    """Image 6 (second chunk [5, 8)) with d pixels = 0 gets a d film of exactly zero; the others stay within the bound."""
    x = split_case("train-B-split")
    assert backward.CHUNK_POINTS // (x["r"] ** 2 * x["s"]) == 5
    d = x["d_pixels"].clone()
    d[6] = 0
    _, d_film, grads = camera_grads(x, d, grad_precision="split")
    assert torch.equal(d_film[6], torch.zeros_like(d_film[6])), "image 6's d film is not zero: max %g" % d_film[6].abs().max()
    want_film, want = chain(x, stages(x), d)
    check_split(x, "split isolation", d_film, grads, want_film, want)


@gpu
def test_split_grad_rays_vs_fp64(fp32_products):
    """grad_rays with a random 3/8 of the rays (not a symmetric set) against the chain on the masked d pixels."""
    x = split_render("B", 8, 64, 24, _opt("relu"), False, False, 5151)
    n = x["r"] ** 2
    rays = torch.randperm(n, generator=torch.Generator().manual_seed(52))[:3 * n // 8].to(DEV)
    mask = ray_mask(rays, x["r"])
    assert not torch.equal(mask, mask.t())
    _, d_film, grads = camera_grads(x, x["d_pixels"], grad_rays=rays, grad_precision="split")
    want_film, want = chain(x, stages(x), x["d_pixels"] * mask)
    check_split(x, "split grad_rays", d_film, grads, want_film, want)


# --------------------------------------------------------------------------------------------
# CPU: check_points catches faults
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fault", ["coarse_pass_unlocked", "film_rows_of_the_next_image"])
def test_point_check_faults_exceed_the_bound(fault):
    """point_refs (check_points' reference) on the oracle's render (model D, 2 x 8² rays, 12 + 12 samples) reproduces its
    raw outputs within FWD_BOUND['exact']; with the fault it moves them past 10 x that bound."""
    lock = fault == "coarse_pass_unlocked"
    siren, film, st, _, _ = _oracle_render(lock)
    b = film.shape[0]
    rays = torch.arange(st["dirs"].shape[1])
    good = point_refs(siren, film, st, lock, rays)
    assert point_errors([st["raw_c"], st["raw_f"]], good) <= FWD_BOUND["exact"]
    kw = dict(lock_coarse=False) if lock else dict(film_rows=[(i + 1) % b for i in range(b)])
    moved = point_errors(point_refs(siren, film, st, lock, rays, **kw), good)
    print("point check fault %s: moved %.3g (FWD_BOUND exact x %.0f)" % (fault, moved, moved / FWD_BOUND["exact"]))
    assert moved > 10 * FWD_BOUND["exact"], moved
