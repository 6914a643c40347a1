"""The training backward end to end against float64: differentiable camera renders (backward.render_with_grad, what
``generator(z, ...)`` runs under autograd) in the default precision, at the shapes training runs.

Every render here runs backward.render_with_grad with the library's own CHUNK_POINTS on an upstream gradient shaped like
a GAN's: randn / R² (bench.py's training step) times a per-image factor spread over 1e-3 ... 1, as the softplus
derivative of a discriminator's loss spreads over a batch.  d film and every parameter gradient (the whole feature grid
included) are checked against the float64 VJP of the whole chain, evaluated on the render's own intermediates
(ops.render_forward_stages: points, depths, raw_c, raw_f and the draws): composite_vjp of the NCHW pixels (the
``* 2 - 1`` included), then field_ref on both passes with the directions each pass used: each ray's direction repeated
over its samples, or (0, 0, -1) on both passes under lock_view_dependence, as the reference's camera render locks
them.  d raw comes from the kernel's own raw outputs, so the relu switch is the kernel's and no row needs a bound of its
own: FIELD_BOUND holds as it is, 2e-2 for the fp16 gradient streams, 1e-4 for exact.

The matrix: model B at bench.py's training step (8 images of 64², 24 + 24 samples: chunks of 5 + 3 images, so FiLM rows
come from b0 = 5), with softplus and nerf_noise, with an opaque field (weights concentrate at a surface, so d raw
spans more decades) and in exact; cfg2 (model A, 4 x 128²) and model B in fast precision; lock_view_dependence; the
label FiLM (I), 129-channel feature-head (K: the wide NCHW compositing backward), grid-trunk (L) and bridge (N) fields.
S = 256 is in test_many_samples.py::test_camera_render_with_grad_at_256_steps.  The per-image error of d film (each
image's FiLM gradients relative to that image's own largest entry) is printed beside the asserted figures.

Properties that need no reference: scaling d pixels by 2^k scales every gradient by 2^k exactly (the power-of-two
scale of the fp16 streams and fp32 rounding commute), up to the run-to-run spread of the backward's atomics, also
under torch.autocast with a GradScaler; an inf or a nan in one image's d pixels reaches the parameter gradients, so
GradScaler skips the step; an image whose d pixels are zero gets a d film of exactly zero; ``grad_rays`` (part_forward)
matches the chain on the masked d pixels, and, in exact, the full-ray backward on the same masked d pixels.

CPU tests show that the chain's forward reproduces the oracle's pixels (with and without lock_view_dependence), that
its VJP is the derivative of its forward (gradcheck), and that typical faults of the path, applied to the float64
chain, exceed FIELD_BOUND['default'] at least tenfold: the factor 2 of ``* 2 - 1`` dropped (25x), the coarse pass left
unlocked under lock_view_dependence (11x: the first colour layer's weight gradient), the grad_rays mask with x and y
swapped (82x), image b + 1's FiLM rows used for image b (112x).

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), max |grad - fp64| / max |grad fp64| over every tensor:
default precision 1.57e-2 (train-B: d film of layer 0's frequencies; train-B-noise 1.02e-2, train-B-opaque 1.18e-2,
cfg2-B-fast 1.14e-2, bridge-N 1.07e-2, the others <= 8.2e-3, S = 256 1.15e-2; FIELD_BOUND 2e-2); exact 1.43e-5
(train-B-exact; S = 256 1.86e-5; FIELD_BOUND 1e-4); grad_rays 9.1e-3 in guard, 1.64e-5 in exact, 8.7e-6 from the
full-ray backward (LAYOUT_BOUND 5e-5).  Loss scales 2^-20, 2^16, 2^24 and autocast + GradScaler: 26 of 34 tensors
bit-identical, the other eight (the biases of layers 0-5, d film and the grid, the ones the atomics reach) within
8.5e-7 of their maximum, against a run-to-run spread of 9.0e-7.  The GPU part of this file ran in 40 s there (the
homogeneity test 13 s of it).

Limitation, printed and not asserted: the fp16 streams share one power-of-two scale, taken from the largest |d raw| of
the whole batch, so an image whose upstream gradient is 1e-3 of the batch's largest keeps fewer significant bits.  Its
own d film, relative to its own largest entry, measured up to 6.3e-2 (train-B-noise; cfg2-A 6.2e-2, bridge-N 3.2e-2)
while the images at the top of the spread stay near 1e-2.  FIELD_BOUND, per tensor over the batch, holds; a caller who
needs each image's FiLM gradient to 2e-2 of itself (an inversion whose images' losses differ by decades) differentiates
in exact, or a precision='split' render with grad_precision='split' (each image's d film within 7.3e-5 of itself under
the same spread, test_gpu_fp64_split.py), or renders those images in separate calls.
"""
import copy
import functools
import math

import pytest
import torch

from _fp64 import _film, _opt, _rel, _siren, composite_ref, field_ref, noise_offset, pass_dirs
from fenerf_b200 import backward, ops
from fenerf_b200.generators import volumetric_rendering as vr
from oracle import render_oracle as oracle
from test_gpu_fp64_forward_stages import COMPOSITE_FWD_BOUND, _CPU_CFG, _DeviceDraws
from test_gpu_fp64_reference import FIELD_BOUND, FWD_BOUND, LAYOUT_BOUND, _grad_errors, composite_vjp

DEV = "cuda:0"
gpu = pytest.mark.gpu

#: float64 rows per field_ref chunk: the float64 autograd of one chunk stays a few GB at any batch
CHAIN_ROWS = 1 << 17


# --------------------------------------------------------------------------------------------
# the float64 chain of the camera render
# --------------------------------------------------------------------------------------------
def camera_chain(siren, film, st, lock, opt, noise, offset=None):
    """float64 pixels (B, C - 1, R, R) of the camera render from the FiLM table: field_ref on both passes (directions as
    pass_dirs), then composite_ref.  st: points_c, z_c, dirs, points_f, z_f (the render's own).  Differentiable in film
    where film requires grad; `offset` fixes the fp32 noise offset (noise_offset) for gradcheck.  A flat render has
    points_f None."""
    b, n, s = st["z_c"].shape
    outs = []
    for pts, locked in ((st["points_c"], lock), (st["points_f"], lock)):
        if pts is None:
            outs.append(None)
            continue
        d = pass_dirs(st["dirs"], s, locked).double()
        outs.append(oracle.field_eval(siren, pts.reshape(b, -1, 3).double(), film, d).reshape(b, n, s, -1))
    return composite_ref(outs[0], st["z_c"], outs[1], st["z_f"], noise, opt, offset)


def camera_chain_vjp(siren, film, st, lock, opt, noise, d_pixels, lock_coarse=None, film_rows=None):
    """The float64 VJP of the camera render on its own intermediates st (points_c, z_c, dirs, raw_c, points_f, z_f,
    raw_f): composite_vjp of the NCHW pixels, then field_ref on each pass with the directions it used.  lock_coarse and
    film_rows exist for the fault checks (a coarse pass locked otherwise than the fine one; image i reading the FiLM rows
    of image film_rows[i]).  A flat render has points_f, z_f and raw_f None.  -> (d film, {parameter name: gradient})."""
    b, n, s, c = st["raw_c"].shape
    d_c, d_f = composite_vjp(st["raw_c"], st["z_c"], st["raw_f"], st["z_f"], noise, opt, d_pixels)
    lock_c = lock if lock_coarse is None else lock_coarse
    chunk = max(1, CHAIN_ROWS // b)
    _, film_c, want = field_ref(siren, st["points_c"].reshape(b, -1, 3), pass_dirs(st["dirs"], s, lock_c), film,
                                d_c.reshape(b, -1, c), film_rows, chunk)
    if st["points_f"] is None:
        return film_c, want
    _, film_f, want_f = field_ref(siren, st["points_f"].reshape(b, -1, 3), pass_dirs(st["dirs"], s, lock), film,
                                  d_f.reshape(b, -1, c), film_rows, chunk)
    for k, v in want_f.items():
        want[k] = want[k] + v if k in want else v
    return film_c + film_f, want


def ray_mask(rays, r, transposed=False):
    """(R, R) mask of the rays `rays` (ray p = row * R + col, the layout of the NCHW pixels); transposed: x and y
    swapped (a fault)."""
    m = torch.zeros(r * r, dtype=torch.bool, device=rays.device)
    m[rays] = True
    m = m.reshape(r, r)
    return m.t() if transposed else m


def film_errors_per_image(d_film, want_film):
    """(B,) max over FiLM layers and frequency / phase of the error relative to that image's own largest entry."""
    err = (d_film.double() - want_film.double()).abs().amax(-1)
    scale = want_film.double().abs().amax(-1)
    return (err / torch.where(scale > 0, scale, torch.ones_like(scale))).flatten(1).amax(1)


# --------------------------------------------------------------------------------------------
# GPU: render_with_grad against the chain
# --------------------------------------------------------------------------------------------
#: name -> (model, B, R, S, options, precision, lock_view_dependence, opaque field)
_CASES = {
    "train-B": ("B", 8, 64, 24, _opt("relu"), "guard", False, False),
    "train-B-noise": ("B", 8, 64, 24, _opt("softplus", noise=0.5), "guard", False, False),
    "train-B-opaque": ("B", 4, 64, 24, _opt("relu"), "guard", False, True),
    "train-B-exact": ("B", 8, 64, 24, _opt("relu"), "exact", False, False),
    "cfg2-A": ("A", 4, 128, 24, _opt("relu"), "guard", False, False),
    "cfg2-B-fast": ("B", 4, 128, 24, _opt("relu"), "fast", False, False),
    "lock-A": ("A", 4, 64, 24, _opt("relu"), "guard", True, False),
    "label-I": ("I", 4, 64, 24, _opt("relu"), "guard", False, False),
    "wide-K": ("K", 2, 48, 24, _opt("relu"), "guard", False, False),
    "grid-L": ("L", 3, 64, 24, _opt("relu"), "guard", False, False),
    "bridge-N": ("N", 3, 64, 24, _opt("relu"), "guard", False, False),
}


@functools.lru_cache(maxsize=2)
def _field(model, opaque=False):
    """The field of `model` on the device; opaque: the suite's opaque field (density bias + 0.5) with the density
    head's weight x 8, so that the weights of most rays concentrate at a surface."""
    siren = _siren(model, DEV, sigma_bias_shift=0.5 if opaque else 0.0)
    if opaque:
        with torch.no_grad():
            siren.final_layer.weight *= 8
    return siren


def gan_d_pixels(b, c_img, r, g):
    """randn / R² (bench.py's training step) times a per-image factor spread over 1e-3 ... 1, in shuffled order."""
    spread = 10.0 ** (-3.0 * torch.arange(b, dtype=torch.float64) / max(1, b - 1))
    factor = spread[torch.randperm(b, generator=torch.Generator().manual_seed(b))].float().to(DEV)
    return torch.randn((b, c_img, r, r), generator=g, device=DEV) / (r * r) * factor.reshape(b, 1, 1, 1)


def make_render(model, b, r, s, o, precision, lock, opaque, seed):
    """A camera render's descriptor, field, FiLM table, draws (render_with_grad's arguments after the FiLM table) and a
    GAN-shaped upstream gradient."""
    siren = _field(model, opaque)
    g = torch.Generator(device=DEV).manual_seed(seed)
    n = r * r
    rd = ops.make_render_desc(batch=b, img_size=r, num_steps=s, hierarchical=True, clamp_mode=o["clamp"],
                              nerf_noise=o["noise"], fov=12, lock_view_dependence=lock, precision=precision)
    x_lin, y_lin, z_lin = vr.ray_tables(r, s, 0.88, 1.12, DEV)
    c2w = ops.camera_poses(b, "gaussian", 0.3, 0.155, math.pi / 2, math.pi / 2, _DeviceDraws(g), torch.device(DEV))[0]
    args = (x_lin, y_lin, z_lin, c2w, torch.rand(b, n, s, 1, generator=g, device=DEV),
            torch.randn(b, n, s, 1, generator=g, device=DEV), torch.rand(b * n, s, generator=g, device=DEV),
            torch.randn(b, n, 2 * s, 1, generator=g, device=DEV))
    c = siren.field_spec().out_dim
    return dict(siren=siren, rd=rd, film=_film(siren, b, seed), args=args, opt=o, lock=lock, b=b, r=r, s=s, c=c,
                precision=precision, d_pixels=gan_d_pixels(b, c - 1, r, g))


def render_case(name):
    model, b, r, s, o, precision, lock, opaque = _CASES[name]
    return make_render(model, b, r, s, o, precision, lock, opaque, sum(map(ord, name)))


def camera_grads(x, d_pixels, grad_rays=None, grad_precision=None):
    """render_with_grad and the gradients of sum(pixels * d_pixels): (pixels, d film, {parameter name: gradient})."""
    siren = x["siren"]
    params = backward.FieldWeights(siren).parameters()
    names = {id(p): k for k, p in siren.named_parameters()}
    f = x["film"].clone().requires_grad_(True)
    px = backward.render_with_grad(siren, x["rd"], f, *x["args"], grad_rays=grad_rays, grad_precision=grad_precision)
    gr = torch.autograd.grad((px * d_pixels).sum(), [f] + params)
    return px.detach(), gr[0], {names[id(p)]: t for p, t in zip(params, gr[1:])}


def stages(x):
    with torch.no_grad():
        return ops.render_forward_stages(x["siren"], x["rd"], x["film"], *x["args"])


def chain(x, st, d_pixels):
    noise = x["args"][-1][..., 0] if x["opt"]["noise"] else None
    return camera_chain_vjp(x["siren"], x["film"], st, x["lock"], x["opt"], noise, d_pixels)


def bound_of(precision):
    """A 'split' render's backward runs on fp32 streams, with or without grad_precision='split'."""
    return FIELD_BOUND["exact" if precision in ("exact", "split") else "default"]


def check_against_chain(x, tag, d_film, grads, want_film, want, bound=None):
    """Every parameter tensor and each FiLM layer's frequency and phase gradient within `bound` (None: the precision's
    bound)."""
    assert set(want) <= set(grads), sorted(set(want) - set(grads))
    errs = _grad_errors(d_film, {k: grads[k] for k in want}, want_film, want)
    worst = max(errs, key=errs.get)
    per_image = film_errors_per_image(d_film, want_film)
    bound = bound_of(x["precision"]) if bound is None else bound
    print("train grads %s: worst %s %.3g (bound %g); d film per image %.3g %s" % (
        tag, worst, errs[worst], bound, per_image.max().item(), ["%.2g" % v for v in per_image.tolist()]))
    assert errs[worst] <= bound, {k: "%.2e" % v for k, v in errs.items() if v > bound}
    return errs


@pytest.fixture
def fp32_products(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # exact mode's torch.mm stays fp32


@gpu
@pytest.mark.parametrize("name", list(_CASES))
def test_train_gradients_vs_fp64(fp32_products, name):
    """render_with_grad (the library's CHUNK_POINTS) on a GAN-shaped d pixels: d film and every parameter gradient
    against the float64 VJP of the camera render's chain on its own intermediates."""
    x = render_case(name)
    px, d_film, grads = camera_grads(x, x["d_pixels"])
    st = stages(x)
    assert torch.equal(st["pixels"], px), "render_forward_stages differs from the differentiable render"
    want_film, want = chain(x, st, x["d_pixels"])
    check_against_chain(x, name, d_film, grads, want_film, want)


# --------------------------------------------------------------------------------------------
# GPU: properties of the backward
# --------------------------------------------------------------------------------------------
def _all(d_film, grads):
    return dict(grads, film=d_film)


def _moved(got, ref):
    """{tensor: max |got - ref| / max |ref|}"""
    return {k: _rel(got[k], ref[k]) for k in ref}


@gpu
def test_loss_scale_homogeneity(fp32_products):
    """d pixels x 2^k (k = -20, 16, 24) gives every gradient x 2^k: the backward's own power-of-two scale absorbs 2^k, so
    its fp16 streams are bit-identical and only the run order of its atomics (the gate's column sums, the grid scatter)
    can differ.  The run-to-run spread is measured on three runs of g(d): the largest max |g_i - g_1| / max |g_1| over
    the tensors and the two pairs.  Every tensor's max |g(2^k d) / 2^k - g(d)| / max |g(d)| must stay within twice that
    spread (twice: the spread of a few runs is itself a draw; the atomics reach a few tensors only, and which of those
    happen to agree bit for bit between two runs is chance).  The training step's torch.autocast +
    GradScaler(init_scale=2^16), on a FiLM table made outside autocast, must give the plain call's gradients once
    unscaled, within the same bound."""
    x = render_case("train-B")
    d = x["d_pixels"]
    g1 = _all(*camera_grads(x, d)[1:])
    runs = [_moved(_all(*camera_grads(x, d)[1:]), g1) for _ in range(2)]
    spread = max(max(r.values()) for r in runs)
    print("homogeneity: run-to-run spread %.3g; tensors that differ between runs: %s" % (
        spread, sorted({k for r in runs for k, v in r.items() if v > 0})))

    def check(tag, got):
        moved = _moved(got, g1)
        worst = max(moved, key=moved.get)
        print("homogeneity %s: worst %s %.3g (twice the spread %.3g); bit-identical %d of %d tensors" % (
            tag, worst, moved[worst], 2 * spread, sum(v == 0 for v in moved.values()), len(moved)))
        assert moved[worst] <= 2 * spread, (tag, {k: v for k, v in moved.items() if v > 2 * spread})

    for k in (-20, 16, 24):
        got = _all(*camera_grads(x, d * 2.0 ** k)[1:])
        check("2^%d" % k, {n: v * 2.0 ** -k for n, v in got.items()})

    siren = x["siren"]
    params = backward.FieldWeights(siren).parameters()
    names = {id(p): k for k, p in siren.named_parameters()}
    f = x["film"].clone().requires_grad_(True)
    opt = torch.optim.SGD([f] + params, lr=0.0)
    opt.zero_grad(set_to_none=True)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    try:
        with torch.autocast("cuda", dtype=torch.float16):
            px = backward.render_with_grad(siren, x["rd"], f, *x["args"])
            loss = (px * d).sum()
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        assert all(torch.isfinite(p.grad).all() for p in [f] + params)
        check("autocast + GradScaler", dict({names[id(p)]: p.grad.clone() for p in params}, film=f.grad.clone()))
    finally:
        opt.zero_grad(set_to_none=True)


@gpu
@pytest.mark.parametrize("value", ["inf", "nan"])
def test_non_finite_upstream_reaches_the_parameters(value):
    """One inf (or nan) in d pixels of one image leaves non-finite parameter gradients, so GradScaler skips the step."""
    x = render_case("train-B")
    d = x["d_pixels"].clone()
    d[6, 3, 17, 41] = float(value)
    _, d_film, grads = camera_grads(x, d)
    bad = [k for k, v in grads.items() if not torch.isfinite(v).all()]
    print("non-finite %s: %d of %d parameter gradients non-finite, d film finite: %s" % (
        value, len(bad), len(grads), bool(torch.isfinite(d_film).all())))
    assert bad, "a %s in d pixels left every parameter gradient finite" % value


@gpu
def test_image_isolation(fp32_products):
    """Image 6 of the training step (second chunk [5, 8): its FiLM rows come from b0 = 5) with d pixels = 0 gets a d film
    of exactly zero; the other images stay within the bound of the float64 chain."""
    x = render_case("train-B")
    assert backward.CHUNK_POINTS // (x["r"] ** 2 * x["s"]) == 5
    d = x["d_pixels"].clone()
    d[6] = 0
    px, d_film, grads = camera_grads(x, d)
    assert torch.equal(d_film[6], torch.zeros_like(d_film[6])), "image 6's d film is not zero: max %g" % d_film[6].abs().max()
    want_film, want = chain(x, stages(x), d)
    check_against_chain(x, "isolation", d_film, grads, want_film, want)


@gpu
@pytest.mark.parametrize("precision", ["guard", "exact"])
def test_grad_rays_vs_fp64(fp32_products, precision):
    """render_with_grad(grad_rays=...) with a random 3/8 of the rays (not a symmetric set, so that a transposed mask
    would show), at the training step's shape: against the chain on d pixels masked to those rays, within the
    precision's bound; in exact also against the full-ray backward on the same masked d pixels (LAYOUT_BOUND: the fp32
    library products sum other row counts in other orders)."""
    x = make_render("B", 8, 64, 24, _opt("relu"), precision, False, False, 5150)
    n = x["r"] ** 2
    rays = torch.randperm(n, generator=torch.Generator().manual_seed(51))[:3 * n // 8].to(DEV)
    mask = ray_mask(rays, x["r"])
    assert not torch.equal(mask, mask.t())
    d = x["d_pixels"] * mask
    px, d_film, grads = camera_grads(x, x["d_pixels"], grad_rays=rays)
    want_film, want = chain(x, stages(x), d)
    check_against_chain(x, "grad_rays %s" % precision, d_film, grads, want_film, want)
    if precision == "exact":
        _, d_film1, grads1 = camera_grads(x, d)
        inv = _grad_errors(d_film, {k: grads[k] for k in want}, d_film1, {k: grads1[k] for k in want})
        worst = max(inv, key=inv.get)
        print("grad_rays exact against the full-ray backward: worst %s %.3g" % (worst, inv[worst]))
        assert inv[worst] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


# --------------------------------------------------------------------------------------------
# CPU: the chain reproduces the oracle, is the derivative of its forward, and its bound catches faults
# --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _oracle_render(lock, hier=True):
    """The fp32 oracle's render of model D (2 images, 8² rays, 12 + 12 samples, noise 0.5), as test_gpu_fp64_forward_
    stages._cpu_render, with or without lock_view_dependence, or flat (12 samples); its stages in the chain's names."""
    siren = _siren("D", "cpu")
    film = _film(siren, 2, 21)
    torch.manual_seed(21)
    out = oracle.render(siren, film, dict(_CPU_CFG, lock_view_dependence=lock, hierarchical_sample=hier), keep_stages=True)
    s = out["stages"]
    st = dict(points_c=s["points_coarse"], z_c=s["z_coarse"][..., 0], dirs=s["dirs"], raw_c=s["raw_coarse"],
              points_f=None, z_f=None, raw_f=None)
    if hier:
        st.update(points_f=s["points_fine"], z_f=s["z_fine"][..., 0], raw_f=s["raw_fine"])
    noise = out["draws"][-1][1][..., 0]            # the compositor's draw, the last one
    return siren, film, st, noise, out["pixels"]


_CPU_OPT = _opt("relu", noise=_CPU_CFG["nerf_noise"])


@pytest.mark.parametrize("lock", [False, True], ids=["free", "lock_view_dependence"])
def test_camera_chain_matches_the_oracle(lock):
    """field_ref on both passes with pass_dirs reproduces the oracle's raw outputs within FWD_BOUND['exact'] (under
    lock_view_dependence, both passes locked, as the oracle's and the reference's camera render lock them), and the
    chain's pixels reproduce the oracle's."""
    _check_chain_against_the_oracle(lock, True)


def test_flat_camera_chain_matches_the_oracle():
    """The same for a flat render (no fine pass: points_f None), the inversion's render."""
    _check_chain_against_the_oracle(False, False)


def _check_chain_against_the_oracle(lock, hier):
    siren, film, st, noise, pixels = _oracle_render(lock, hier)
    b, n, s, c = st["raw_c"].shape
    errs = {}
    for tag, pts, raw in (("coarse", st["points_c"], st["raw_c"]), ("fine", st["points_f"], st["raw_f"])):
        if pts is None:
            continue
        out = field_ref(siren, pts.reshape(b, -1, 3), pass_dirs(st["dirs"], s, lock), film)[0]
        errs[tag] = (out - raw.reshape(b, -1, c).double()).abs().max().item()
    with torch.no_grad():
        px = camera_chain(copy_double(siren), film.double(), st, lock, _CPU_OPT, noise)
    errs["pixels"] = (px - pixels.double()).abs().max().item()
    print("camera chain vs oracle (%s, %s): %s" % ("locked" if lock else "free", "hierarchical" if hier else "flat", errs))
    assert max(v for k, v in errs.items() if k != "pixels") <= FWD_BOUND["exact"], errs
    assert errs["pixels"] <= COMPOSITE_FWD_BOUND, errs


def copy_double(siren):
    return copy.deepcopy(siren).double()


def _tiny_chain_inputs(hier=True):
    """Model A on 1 image of 3² rays, 4 + 4 samples (or 4, flat) from the oracle's set-up, its float64 field outputs as
    raw."""
    siren = _siren("A", "cpu")
    film = _film(siren, 1, 31).double()
    cfg = dict(_CPU_CFG, img_size=3, num_steps=4, hierarchical_sample=hier)
    torch.manual_seed(31)
    out = oracle.render(siren, film.float(), cfg, keep_stages=True)
    s = out["stages"]
    st = dict(points_c=s["points_coarse"], z_c=s["z_coarse"][..., 0], dirs=s["dirs"], points_f=None, z_f=None, raw_f=None)
    if hier:
        st.update(points_f=s["points_fine"], z_f=s["z_fine"][..., 0])
    b, n, k = st["z_c"].shape
    ref = copy_double(siren)
    for tag, pts in (("c", st["points_c"]), ("f", st["points_f"])):
        if pts is None:
            continue
        with torch.no_grad():
            st["raw_" + tag] = oracle.field_eval(ref, pts.reshape(b, -1, 3).double(), film,
                                                 pass_dirs(st["dirs"], k, False).double()).reshape(b, n, k, -1)
    noise = out["draws"][-1][1][..., 0]            # the compositor's draw, the last one
    return siren, ref, film, st, noise


def test_camera_chain_gradcheck():
    """The chain's forward passes gradcheck in the FiLM table (fast mode), and camera_chain_vjp is its derivative: d film
    and every parameter gradient equal the float64 autograd of the whole chain to 1e-10."""
    _check_chain_gradcheck(True)


def test_flat_camera_chain_gradcheck():
    """The same for a flat render (points_f None), the inversion's render."""
    _check_chain_gradcheck(False)


def _check_chain_gradcheck(hier):
    siren, ref, film, st, noise = _tiny_chain_inputs(hier)
    off = noise_offset(st["raw_c"], st["z_c"], st["raw_f"], st["z_f"], noise, _CPU_OPT["noise"])
    fn = lambda f: camera_chain(ref, f, st, False, _CPU_OPT, noise, off)       # noqa: E731
    assert torch.autograd.gradcheck(fn, (film.clone().requires_grad_(True),), fast_mode=True, eps=1e-7, atol=1e-6,
                                    rtol=1e-4)
    d_pixels = torch.randn(fn(film).shape, generator=torch.Generator().manual_seed(32), dtype=torch.float64)
    f = film.clone().requires_grad_(True)
    params = {k: p for k, p in ref.named_parameters() if "mapping_network" not in k}
    for p in params.values():
        p.grad = None
    (fn(f) * d_pixels).sum().backward()
    got_film, got = camera_chain_vjp(siren, film, st, False, _CPU_OPT, noise, d_pixels)
    assert set(got) == {k for k, p in params.items() if p.grad is not None}
    errs = _grad_errors(got_film, got, f.grad, {k: params[k].grad for k in got})
    assert max(errs.values()) <= 1e-10, errs


_FAULTS = ["factor_two_dropped", "coarse_pass_unlocked", "grad_rays_mask_transposed", "film_rows_of_the_next_image"]


@pytest.mark.parametrize("fault", _FAULTS)
def test_train_faults_exceed_the_bound(fault):
    """Each fault, applied to the float64 chain on the oracle's render (model D, 2 x 8² rays, 12 + 12 samples), moves d
    film or a parameter gradient past 10 x FIELD_BOUND['default'].  The grad_rays faults use a random 3/8 of the rays."""
    lock = fault == "coarse_pass_unlocked"
    siren, film, st, noise, _ = _oracle_render(lock)
    b, r = film.shape[0], _CPU_CFG["img_size"]
    c = st["raw_c"].shape[-1]
    d_pixels = torch.randn(b, c - 1, r, r, generator=torch.Generator().manual_seed(33))
    kw = dict(lock_coarse=False) if fault == "coarse_pass_unlocked" else {}
    if fault == "grad_rays_mask_transposed":
        rays = torch.randperm(r * r, generator=torch.Generator().manual_seed(34))[:3 * r * r // 8]
        d_pixels, bad_d = d_pixels * ray_mask(rays, r), d_pixels * ray_mask(rays, r, transposed=True)
    else:
        bad_d = d_pixels / 2 if fault == "factor_two_dropped" else d_pixels
    if fault == "film_rows_of_the_next_image":
        kw = dict(film_rows=[(i + 1) % b for i in range(b)])
    good_film, good = camera_chain_vjp(siren, film, st, lock, _CPU_OPT, noise, d_pixels)
    bad_film, bad = camera_chain_vjp(siren, film, st, lock, _CPU_OPT, noise, bad_d, **kw)
    errs = _grad_errors(bad_film, bad, good_film, good)
    worst = max(errs, key=errs.get)
    print("train fault %s: %s moved %.3g (FIELD_BOUND default x %.1f)" % (fault, worst, errs[worst],
                                                                         errs[worst] / FIELD_BOUND["default"]))
    assert errs[worst] > 10 * FIELD_BOUND["default"], (worst, errs[worst])
