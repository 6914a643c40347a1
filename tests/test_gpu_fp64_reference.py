"""The backward and the point network against float64 references, at the shapes training runs.

The parity tests elsewhere compare whole renders at 12²-16² pixels with 9-12 samples per pass.  Here each kernel is
checked on its own against a float64 restatement of the same operation, at the shapes where it changes behaviour:

  A. ``fenerf_composite_backward`` with 8-128 merged samples (the 32-sample scan chunks and their carry, the dynamic
     shared-memory opt-in beyond 48 KB), 4-32 channels, every compositing option, exact depth ties; and, as a second
     entry ('-rays'), ``fenerf_composite_backward_rays`` (ray-major pixels in [0, 1]: its own kernel and opt-in), bit
     for bit the NCHW entry's result on the same upstream value (measured: 2.3e-6 at n = 128, C = 22, softplus + noise);
     and on flat renders a third ('-rays_dz'), ``fenerf_composite_backward_rays_dz``: the same d raw bit for bit, and the
     gradient w.r.t. the coarse depths against float64 autograd, from S = 2 up to the 256-step limit on both sides of
     the narrow body's shared-memory limit (248 / 249 samples at C = 22);
  B. ``_FieldBackward`` for every field class under the chunk layouts of production: several images per chunk
     (FiLM rows of image b0 > 0) and one image split into point chunks (directions sliced at p0 // dir_group);
  C. the point network forward (exact and fast kernels) under the tile schedules of a real SM count.

D. The bounds are shown to catch faults: each fault is applied to the float64 reference (not to a kernel) and must move
the result past the committed bound.  Those checks and the references' own gradchecks run on the CPU.

E. The FiLM-gradient algebra of finish() restated in float64 from autograd pieces, at f = 0, tiny and large |f| (CPU);
   the kernels at those frequencies are in test_gpu_fp64_film_edges.py.

Bounds: measured on an H100 80GB HBM3 (132 SMs); each constant below states the measured maximum.
"""
import copy
import ctypes
import functools
import math

import pytest
import torch
import torch.nn.functional as F

import _cases
from _fp64 import (EDGE_FREQS, _ZeroDraws, _film, _opt, _rel, _siren, composite_ref, field_ref,
                   noise_offset, plant_frequencies)
from fenerf_b200 import _lib, backward, ops
from oracle import render_oracle as oracle

DEV = "cuda:0"
gpu = pytest.mark.gpu

#: composite backward, max |d_raw - fp64| / max |d_raw fp64| per tensor (coarse and fine).  Measured: 2.5e-6 (n = 128,
#: C = 22, softplus + noise); 1.6e-6 at n = 96, 9.9e-7 at n = 48, <= 8.3e-7 up to 33.  The faults of D move it by >= 4.4e-3.
COMPOSITE_BOUND = 1e-5
#: the depth gradient of fenerf_composite_backward_rays_dz, max |d z - fp64| / max |d z fp64|.  Measured: 6.7e-5 (n = 256,
#: C = 4, opaque, black_back), 3.2e-5 at n = 248, <= 1.0e-5 up to n = 64: each sample's d z is the difference of its two
#: intervals' terms d alpha act exp(-delta act), which cancel where the density is high and the intervals short, so
#: d alpha's fp32 rounding (COMPOSITE_BOUND's) grows relative to d z with S.
DEPTH_BOUND = 2e-4
#: field backward, max |grad - fp64| / max |grad fp64| per parameter tensor, the whole grid and each FiLM layer's
#: frequency and phase gradients.  Measured: exact 3.1e-5 (model H, L1: d film of colour layer 5), 1.0e-5 at L4;
#: default 1.21e-2 (model H, L1), 5.5e-3 at L4 -- the fp16 streams (u = f z + p recomputed from them, f ~ 30) set it.
FIELD_BOUND = {"exact": 1e-4, "default": 2e-2}
#: the same gradients from a chunked run (L2 / L3) and a one-chunk run of the same kernels, relative to the tensor's
#: maximum.  Measured: exact 1.7e-5 (model H: the fp32 library GEMMs pick other algorithms for other row counts, and 16
#: FiLM layers carry that forward), default 8.4e-6 (layer 0's weight gradient, an fp32 sum of 7,200 cancelling terms).
#: A wrong FiLM image moves the float64 gradients by 1.3, directions one ray off by 3.2e-2 (test_field_backward_faults_*).
LAYOUT_BOUND = 5e-5
#: point network forward, max |out - fp64| per channel.  Measured: exact 9.5e-7, fast 4.2e-4 (model H); the fast bound is
#: the one its comparison with the fp32 path has always had.  The faults of D move an output channel by >= 0.13.
FWD_BOUND = {"exact": 1e-5, "fast": 5e-3}


# --------------------------------------------------------------------------------------------
# fields, FiLM tables, points
# --------------------------------------------------------------------------------------------
STOCK_FIELD_MODELS = ("A", "B", "C", "D", "E", "F", "G", "H", "D32")   # S shares A's field; D32: the widest renderable head
#: and the field families: label FiLM, feature heads, grid trunk
FIELD_MODELS = STOCK_FIELD_MODELS + ("I", "J", "K", "L")


def _fwd_seed(model):
    return _cases.model_data(model, "fwd_seed") or 2000 + FIELD_MODELS.index(model)


def _bwd_seed(model, layout):
    return (_cases.model_data(model, "bwd_seed") or 1000 + 10 * FIELD_MODELS.index(model)) + int(layout[1])


def _render_points(batch, img, steps, seed):
    """Jittered sample points of a render (the oracle's ray set-up, gaussian poses): points (B, R², S, 3),
    depths (B, R², S), directions (B, R², 3), origins (B, R², 3); CPU fp32."""
    torch.manual_seed(seed)
    d = oracle.Draws()
    pts, z, dirs = oracle.camera_rays(batch, img, steps, 12, 0.88, 1.12)
    pts, z = oracle.jitter(pts, z, dirs, d)
    origin, _, _ = oracle.camera_pose(batch, 0.3, 0.155, math.pi / 2, math.pi / 2, "gaussian", d)
    pts, dirs, org = oracle.to_world(pts, z, dirs, oracle.look_at(oracle.unit(-origin), origin))
    return pts, z[..., 0], dirs, org


def _field_points(batch, ppb, dir_group, seed):
    """ppb render points per image, dir_group consecutive samples per ray: (B, ppb, 3), (B, ppb / dir_group, 3)."""
    rays = ppb // dir_group
    pts, _, dirs, _ = _render_points(batch, math.isqrt(rays - 1) + 1, dir_group, seed)
    return pts[:, :rays].reshape(batch, ppb, 3).contiguous(), dirs[:, :rays].contiguous()


def _per_point(dirs, ppb, lock):
    if lock:
        d = torch.zeros((dirs.shape[0], ppb, 3), dtype=dirs.dtype, device=dirs.device)
        d[..., 2] = -1
        return d
    return dirs.repeat_interleave(ppb // dirs.shape[1], dim=1)


# --------------------------------------------------------------------------------------------
# 0. float64 references
# --------------------------------------------------------------------------------------------
def composite_vjp(raw_c, z_c, raw_f, z_f, noise, opt, d_pixels, ray_major=False, want_z=False):
    """(d raw_c, d raw_f) in float64 for the upstream gradient d_pixels (NCHW, or (B, N, C - 1) with ray_major);
    want_z (no fine samples): (d raw_c, d z_c), the coarse depths a float64 leaf as well."""
    assert not (want_z and raw_f is not None), "the depth gradient is that of a non-hierarchical render"
    leaves = [raw_c.double().requires_grad_(True)] + ([raw_f.double().requires_grad_(True)] if raw_f is not None else [])
    z_c = z_c.double().requires_grad_(True) if want_z else z_c
    px = composite_ref(leaves[0], z_c, leaves[1] if raw_f is not None else None, z_f, noise, opt, ray_major=ray_major)
    grads = torch.autograd.grad((px * d_pixels.double()).sum(), leaves + ([z_c] if want_z else []))
    return grads[0], grads[1] if (raw_f is not None or want_z) else None


# --------------------------------------------------------------------------------------------
# the references' own checks (CPU)
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", [
    _opt("relu"), _opt("softplus"), _opt("relu", noise=0.5), _opt("softplus", last_back=True), _opt("relu", white_back=True),
    _opt("softplus", black_back=True), _opt("relu", softmax=True), _opt("softplus", noise=0.3, softmax=True, last_back=True)],
    ids=["relu", "softplus", "noise", "last_back", "white_back", "black_back", "softmax_label", "softmax_noise_last_back"])
@pytest.mark.parametrize("hier", [False, True], ids=["flat", "hier"])
def test_composite_reference_gradcheck(opt, hier):
    """The float64 compositing VJP is the derivative of its own function: 2 rays (2 images of one ray), 5 samples per
    pass, 6 channels (2 labels), with an exact depth tie between a fine and a coarse sample."""
    g = torch.Generator().manual_seed(3)
    b, s, c = 2, 5, 6
    z_c = (0.88 + 0.24 * torch.sort(torch.rand(b, 1, s, generator=g), -1)[0]).float()
    z_f = (0.88 + 0.24 * torch.sort(torch.rand(b, 1, s, generator=g), -1)[0]).float() if hier else None
    if hier:
        z_f[0, 0, 2] = z_c[0, 0, 1]                                    # exact tie
    n = 2 * s if hier else s
    raw_c = torch.randn(b, 1, s, c, generator=g, dtype=torch.float64)
    raw_f = torch.randn(b, 1, s, c, generator=g, dtype=torch.float64) if hier else None
    for r in (raw_c, raw_f):                                           # densities away from the relu kink
        if r is not None:
            r[..., -1] = torch.where(r[..., -1] >= 0, r[..., -1] + 0.05, r[..., -1] - 0.05) * 20
    noise = torch.randn(b, 1, n, generator=g) if opt["noise"] else None
    off = noise_offset(raw_c, z_c, raw_f, z_f, noise, opt["noise"]) if opt["noise"] else None
    leaves = (raw_c.requires_grad_(True),) + ((raw_f.requires_grad_(True),) if hier else ())
    fn = (lambda rc, rf: composite_ref(rc, z_c, rf, z_f, noise, opt, off)) if hier else \
        (lambda rc: composite_ref(rc, z_c, None, None, noise, opt, off))
    assert torch.autograd.gradcheck(fn, leaves, eps=1e-7, atol=1e-7, rtol=1e-5)


def test_composite_reference_keeps_the_tie_rule_and_matches_the_oracle():
    """Equal depths merge fine-first, and in fp32 the reference is the oracle's own compositing."""
    g = torch.Generator().manual_seed(4)
    z_c = torch.sort(torch.rand(1, 1, 4, generator=g), -1)[0]
    z_f = z_c.clone()                                                  # every fine depth ties with a coarse one
    raw_c = torch.randn(1, 1, 4, 4, generator=g).double()
    raw_f = torch.randn(1, 1, 4, 4, generator=g).double()
    opt = _opt("softplus")
    px = composite_ref(raw_c, z_c, raw_f, z_f, None, opt)
    order = [0, 4, 1, 5, 2, 6, 3, 7]                                   # fine i (index i) before coarse i (4 + i)
    raw = torch.cat([raw_f, raw_c], 2)[:, :, order]
    z = torch.cat([z_f, z_c], 2)[:, :, order]
    want = oracle.alpha_composite(raw.float(), z.unsqueeze(-1), _ZeroDraws(z), 0.0, "softplus")[0]
    assert (px.reshape(-1) - (want.double() * 2 - 1).reshape(-1)).abs().max() <= 1e-6


def test_grid_lookup_is_the_references_in_fp32_and_passes_gradcheck_in_float64():
    """fp32 coordinates take the reference's sample_from_3dgrid (its .float() casts included) bit for bit; float64
    coordinates sample in float64, which the float64 references differentiate."""
    g = torch.Generator().manual_seed(5)
    grid = torch.randn(1, 3, 4, 4, 4, generator=g)
    coords = torch.rand(2, 7, 3, generator=g) * 2.4 - 1.2
    s = F.grid_sample(grid.float().expand(2, -1, -1, -1, -1), coords.float().reshape(2, 1, 1, -1, 3), mode='bilinear',
                      padding_mode='zeros', align_corners=True)
    assert torch.equal(s.permute(0, 4, 3, 2, 1).reshape(2, 7, 3), oracle.grid_lookup(coords, grid))
    assert torch.autograd.gradcheck(oracle.grid_lookup, (coords.double().requires_grad_(True),
                                                         grid.double().requires_grad_(True)))


@pytest.mark.parametrize("model,edges", [("A", False), ("D", False), ("A", True), ("D", True)],
                         ids=["A", "D", "A-zero_tiny_f", "D-zero_tiny_f"])
def test_field_reference_gradcheck(model, edges):
    """The float64 field VJP (every parameter and the FiLM table) on 2 points, checked in gradcheck's fast mode
    (random projections of the full Jacobian); with `edges`, every FiLM row also holds f = 0, -0, tiny and large |f|."""
    siren = _siren(model, "cpu")
    film = _film(siren, 1, 6).double()
    if edges:
        film = plant_frequencies(film, range(film.shape[1]))[0]
    pts, dirs = _field_points(1, 2, 2, 7)
    ref = copy.deepcopy(siren).double()
    names = [n for n, p in ref.named_parameters() if "mapping_network" not in n]
    params = dict(ref.named_parameters())

    pts64, dirs64 = pts.double(), _per_point(dirs, 2, False).double()

    def fn(film_, *ps):
        return _eval_with(ref, names, ps, pts64, film_, dirs64)

    inputs = (film.requires_grad_(True),) + tuple(params[n].detach().clone().requires_grad_(True) for n in names)
    assert torch.autograd.gradcheck(fn, inputs, fast_mode=True, eps=1e-7, atol=1e-6, rtol=1e-4)


def _eval_with(ref, names, ps, pts, film, dirs):
    saved = {}
    mods = dict(ref.named_modules())
    for n, p in zip(names, ps):
        mod_name, attr = n.rsplit(".", 1)
        mod = mods[mod_name]
        saved[n] = mod._parameters[attr]
        mod._parameters[attr] = p
    try:
        return oracle.field_eval(ref, pts, film, dirs)
    finally:
        for n in names:
            mod_name, attr = n.rsplit(".", 1)
            mods[mod_name]._parameters[attr] = saved[n]


# --------------------------------------------------------------------------------------------
# A. composite backward
# --------------------------------------------------------------------------------------------
_OPTS = {"relu": _opt("relu"), "softplus_noise": _opt("softplus", noise=0.5), "softplus_last_back": _opt("softplus", last_back=True),
         "relu_white_back": _opt("relu", white_back=True), "relu_black_back": _opt("relu", black_back=True),
         "relu_softmax": _opt("relu", softmax=True), "softplus_noise_softmax": _opt("softplus", noise=0.5, softmax=True)}
#: merged samples per ray: flat n = S from the descriptor's least 2 steps; hierarchical n = 2 S (12+12, cfg2's 24+24,
#: cfg5's 48+48, 64+64)
_SAMPLES = [(2, False), (3, False), (8, False), (31, False), (32, False), (33, False), (64, False), (24, True), (48, True),
            (96, True), (128, True)]
_COMPOSITE = [(n, hier, c, o, opaque) for n, hier in _SAMPLES
              for c, o, opaque in [(4, "relu", False), (22, "softplus_noise", False), (32, "relu", True)]]
_COMPOSITE += [(n, hier, c, o, opaque) for n, hier in [(33, False), (96, True), (128, True)]
               for c, o, opaque in [(23, "softplus_last_back", False), (4, "relu_white_back", True), (22, "relu_black_back", False),
                                    (22, "relu_softmax", False), (23, "softplus_noise_softmax", True)]]
#: the flat ends of the library's 256 steps: C = 22's narrow body at S = 248 and its spill to the wide one at 249
#: (narrow_pass_limit), S = 256 narrow at C = 4 and wide at C = 22
_COMPOSITE += [(248, False, 22, "softplus_noise", False), (249, False, 22, "relu_white_back", False),
               (256, False, 4, "relu_black_back", True), (256, False, 22, "relu_softmax", False)]
_COMPOSITE_MODEL = {4: "A", 22: "D", 23: "E", 32: "D32"}
_B, _R = 3, 37          # 37² rays per image: not a multiple of the 8 rays of a composite_backward block
#: the entries of the compositing backward: NCHW pixels * 2 - 1 (fenerf_composite_backward, the ids without a suffix),
#: ray-major pixels in [0, 1] (fenerf_composite_backward_rays, the rays-in render's; ids '-rays') and the same with the
#: depth gradient of a non-hierarchical render (fenerf_composite_backward_rays_dz, point_forward(..., ray_grad=True)'s;
#: ids '-rays_dz')
ENTRIES = ("nchw", "rays", "rays_dz")


def entries(hier):
    """The compositing-backward entries a case runs on: the depth gradient is built for flat renders only."""
    return ENTRIES if not hier else ENTRIES[:2]


def with_entries(cases, ids):
    """Every case (n, hier, ...) on each of its compositing-backward entries; the NCHW entry keeps the case's id."""
    return [pytest.param(*case, e, id=i + ("" if e == "nchw" else "-" + e)) for case, i in zip(cases, ids)
            for e in entries(case[1])]


def narrow_pass_limit(c):
    """The most merged samples whose raw blocks, eight warps' of them, composite_backward stages in the narrow body's
    227 KB of shared memory at C channels; beyond, the wide body reads rows from global memory.  A restatement of
    composite_backward's plan (csrc/composite.cu: narrow_floats and the `wide` test after it): keep the two in step."""
    fits = lambda n: 8 * ((7 * ((n + 3) & ~3) + 64 + n * c + 3) & ~3) * 4 <= 227 * 1024      # noqa: E731
    return max(n for n in range(1, 513) if fits(n))


@functools.lru_cache(maxsize=None)
def _composite_inputs(c, steps, hier, opaque):
    """The mirror field's (exact path) outputs on render points of 3 images; fine depths drawn inside the ray, some
    set exactly equal to coarse ones."""
    siren = _siren(_COMPOSITE_MODEL[c], DEV, sigma_bias_shift=0.5 if opaque else 0.0)
    seed = 100 * c + steps
    film = _film(siren, _B, seed)
    pts_c, z_c, dirs, org = _render_points(_B, _R, steps, seed)
    n = _R * _R
    with torch.no_grad():
        raw_c = ops.siren_points(siren, pts_c.reshape(_B, n * steps, 3).to(DEV), film, dirs.to(DEV), precision="exact")
        out = dict(raw_c=raw_c.reshape(_B, n, steps, c).contiguous(), z_c=z_c.to(DEV).contiguous(), raw_f=None, z_f=None)
        if hier:
            g = torch.Generator().manual_seed(seed)
            z_f = 0.88 + 0.24 * torch.sort(torch.rand(_B, n, steps, generator=g), -1)[0]
            z_f[:, ::5, 0] = z_c[:, ::5, steps // 2]                     # exact ties with coarse depths
            z_f[:, 1::7, -1] = z_c[:, 1::7, -1]
            pts_f = org.unsqueeze(2) + dirs.unsqueeze(2) * z_f.unsqueeze(-1)
            raw_f = ops.siren_points(siren, pts_f.reshape(_B, n * steps, 3).to(DEV), film, dirs.to(DEV), precision="exact")
            out.update(raw_f=raw_f.reshape(_B, n, steps, c).contiguous(), z_f=z_f.to(DEV).contiguous())
    return out


def _composite_backward(opt, steps, hier, x, noise, d_pixels, entry="nchw", batch=_B, img=_R):
    """One entry of the compositing backward; the gradient buffers start as NaN (an entry not written stays NaN).
    'rays' / 'rays_dz': the rays-in render's descriptor, img_h = 1 and img_w = the img² rays per image; 'rays_dz'
    returns (d raw_c, d z_c)."""
    c = x["raw_c"].shape[-1]
    rd = ops.make_render_desc(batch=batch, img_size=img, num_steps=steps, hierarchical=hier, clamp_mode=opt["clamp"],
                              nerf_noise=opt["noise"], fov=12, last_back=opt["last_back"], white_back=opt["white_back"],
                              black_back=opt["black_back"], softmax_label=opt["softmax"])
    lib = _lib.lib()
    d_c = torch.full_like(x["raw_c"], float("nan"))
    p = lambda t: t.data_ptr() if t is not None else 0                  # noqa: E731
    stream = torch.cuda.current_stream().cuda_stream
    if entry != "nchw":
        rd.img_h, rd.img_w = 1, img * img
    if entry == "rays_dz":
        d_z = torch.full_like(x["z_c"], float("nan"))
        _lib.check(lib.fenerf_composite_backward_rays_dz(ctypes.byref(rd), c, p(x["raw_c"]), p(x["z_c"]), p(noise),
                                                         p(d_pixels), p(d_c), p(d_z), stream))
        return d_c, d_z
    fn = lib.fenerf_composite_backward_rays if entry == "rays" else lib.fenerf_composite_backward
    d_f = torch.full_like(x["raw_f"], float("nan")) if hier else None
    _lib.check(fn(ctypes.byref(rd), c, p(x["raw_c"]), p(x["z_c"]), p(x["raw_f"]), p(x["z_f"]), p(noise), p(d_pixels), p(d_c),
                  p(d_f), stream))
    return d_c, d_f


def composite_backward_errors(o, steps, hier, x, noise, g, entry, batch=_B, img=_R):
    """The compositing backward of `entry` on a d_pixels drawn from `g`, against composite_vjp -> (dict of the kernel's
    d_c, d_f and the float64 w_c, w_f; relative errors).
    'rays' is also run on the NCHW entry with d_pixels permuted to NCHW and halved: that entry doubles what it reads, so
    both kernels see the same upstream value exactly, and their results must agree bit for bit.  'rays_dz' must give the
    'rays' entry's d raw bit for bit, and its depth gradient ('d_z', in place of d_f) is checked against float64 autograd
    w.r.t. the coarse depths."""
    c = x["raw_c"].shape[-1]
    if entry == "nchw":
        d_pixels = torch.randn(batch, c - 1, img, img, generator=g).to(DEV)
    else:
        d_pixels = torch.randn(batch, img * img, c - 1, generator=g).to(DEV)
    d_c, d_f = _composite_backward(o, steps, hier, x, noise, d_pixels, entry, batch, img)
    w_c, w_f = composite_vjp(x["raw_c"], x["z_c"], x["raw_f"], x["z_f"], noise, o, d_pixels, ray_major=entry != "nchw",
                             want_z=entry == "rays_dz")
    if entry == "rays":
        nchw = (0.5 * d_pixels).permute(0, 2, 1).reshape(batch, c - 1, img, img).contiguous()
        e_c, e_f = _composite_backward(o, steps, hier, x, noise, nchw, "nchw", batch, img)
        assert torch.equal(d_c, e_c), "ray-major d_raw_c differs from the NCHW entry's on the same upstream value"
        assert not hier or torch.equal(d_f, e_f), "ray-major d_raw_f differs from the NCHW entry's on the same upstream value"
    if entry == "rays_dz":
        e_c = _composite_backward(o, steps, hier, x, noise, d_pixels, "rays", batch, img)[0]
        assert torch.equal(d_c, e_c), "the depth-gradient entry's d_raw_c differs from the ray-major entry's"
    errs = {"d_raw_c": _rel(d_c, w_c)}
    if hier or entry == "rays_dz":
        errs["d_z" if entry == "rays_dz" else "d_raw_f"] = _rel(d_f, w_f)
    assert all(v == v for v in errs.values()), errs          # (NaN: an entry was not written)
    return dict(d_c=d_c, d_f=d_f, w_c=w_c, w_f=w_f), errs


def over_bounds(errs):
    """The entries of a composite_backward_errors() result past their bound: DEPTH_BOUND for d z, COMPOSITE_BOUND else."""
    return {k: v for k, v in errs.items() if v > (DEPTH_BOUND if k == "d_z" else COMPOSITE_BOUND)}


_COMPOSITE_IDS = ["n%d-%s-C%d-%s%s" % (n, "hier" if h else "flat", c, o, "-opaque" if q else "") for n, h, c, o, q in _COMPOSITE]


def test_flat_cases_straddle_the_narrow_body_limit():
    """The flat cases put C = 22 on both sides of the narrow body's limit and S = 256 in the narrow body at C = 4."""
    assert narrow_pass_limit(22) == 248 and narrow_pass_limit(4) >= 256
    flat22 = {n for n, hier, c, _, _ in _COMPOSITE if c == 22 and not hier}
    assert {248, 249, 256} <= flat22 and (256, False, 4) in {case[:3] for case in _COMPOSITE}


@gpu
@pytest.mark.parametrize("n,hier,c,opt,opaque,entry", with_entries(_COMPOSITE, _COMPOSITE_IDS))
def test_composite_backward_vs_fp64(n, hier, c, opt, opaque, entry):
    """``fenerf_composite_backward`` as RenderFunction.backward calls it for a camera render, and
    ``fenerf_composite_backward_rays`` as it does for a rays-in render, against the float64 VJP of the compositing:
    B = 3, 37² rays, n merged samples (more than 32 carry the transmittance scan from chunk to chunk; the shared memory
    of n = 48 with C = 32 and of n >= 96 with C >= 22 is beyond 48 KB and needs the opt-in, which each entry's kernel
    makes for itself)."""
    steps = n // 2 if hier else n
    x = _composite_inputs(c, steps, hier, opaque)
    o = _OPTS[opt]
    g = torch.Generator().manual_seed(n * 64 + c)
    noise = torch.randn(_B, _R * _R, n, generator=g).to(DEV) if o["noise"] else None
    errs = composite_backward_errors(o, steps, hier, x, noise, g, entry)[1]
    print("composite %s n=%d C=%d %s: %s" % (entry, n, c, opt, errs))
    assert not over_bounds(errs), errs


# --------------------------------------------------------------------------------------------
# B. field backward
# --------------------------------------------------------------------------------------------
#: layout -> (B, points per image, dir_group, CHUNK_POINTS or None for the library's own)
_LAYOUTS = {
    "L1": (2, 3000, 24, None),          # every image in one chunk, b0 = 0
    "L2": (5, 1000, 20, 3000),          # chunks of images [0, 3) and [3, 5): FiLM rows from b0 = 3, a ragged last chunk
    "L3": (2, 7200, 12, 2999),          # each image in point chunks of 2988, 2988, 1224; image 1's chunks have b0 = 1
    "L4": (2, 393216, 24, None),        # cfg2's pass (128² rays x 24): one image per chunk, so b0 = 1
}
_FIELD = ([(lay, m, p, False) for lay in ("L1", "L2", "L3") for m in FIELD_MODELS for p in ("exact", "default")]
          + [("L4", m, p, False) for m in ("A", "B", "K") for p in ("exact", "default")]
          + [("L1", "A", p, True) for p in ("exact", "default")])


def _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, exact):
    with torch.no_grad():
        m = d_raw.abs().max()
        scale = torch.exp2(4.0 - torch.ceil(torch.log2(m.clamp_min(1e-30)))).float().reshape(1)   # as backward._field_backward
        fb = backward._FieldBackward(siren, film, scale, (1.0 / scale).float().reshape(1), exact=exact)
        fb.add_points(pts, dirs, dir_group, lock, raw, d_raw)
        d_film, grads = fb.finish()
    return d_film, {n: grads[id(p)].reshape(p.shape) for n, p in siren.named_parameters() if id(p) in grads}


def _grad_errors(d_film, grads, want_film, want):
    """max relative error per parameter tensor and per FiLM layer's frequency / phase gradient."""
    assert set(grads) == set(want), sorted(set(grads) ^ set(want))
    errs = {n: _rel(grads[n], want[n]) for n in want}
    for layer in range(d_film.shape[1]):
        errs["film%d.freq" % layer] = _rel(d_film[:, layer, 0], want_film[:, layer, 0])
        errs["film%d.phase" % layer] = _rel(d_film[:, layer, 1], want_film[:, layer, 1])
    return errs


@gpu
@pytest.mark.parametrize("layout,model,precision,lock", _FIELD,
                         ids=["%s-%s-%s%s" % (lay, m, p, "-lock_dirs" if k else "") for lay, m, p, k in _FIELD])
def test_field_backward_vs_fp64(monkeypatch, layout, model, precision, lock):
    """``_FieldBackward`` (recompute, gate, the per-image dW and finish()) against the float64 VJP of the field: every
    parameter gradient, the whole feature-grid gradient and d film.  L2 / L3 also run as one chunk: each row's fp16
    values do not depend on the chunk, so the two runs differ only by fp32 summation order; a wrong FiLM offset or a
    mis-sliced direction would be O(1)."""
    batch, ppb, dir_group, chunk = _LAYOUTS[layout]
    exact = precision == "exact"
    if exact:
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # exact mode's torch.mm stays fp32
    siren = _siren(model, DEV)
    seed = _bwd_seed(model, layout)
    pts, dirs = (t.to(DEV) for t in _field_points(batch, ppb, dir_group, seed))
    film = _film(siren, batch, seed, edges=True)
    out_dim = siren.field_spec().out_dim
    d_raw = torch.randn(batch, ppb, out_dim, generator=torch.Generator().manual_seed(seed)).to(DEV) * 1e-3
    out64, want_film, want = field_ref(siren, pts, _per_point(dirs, ppb, lock), film, d_raw)
    raw = out64.float().contiguous()
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
    d_film, grads = _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, exact)
    errs = _grad_errors(d_film, grads, want_film, want)
    worst = max(errs, key=errs.get)
    print("field %s %s %s: worst %s %.3g" % (layout, model, precision, worst, errs[worst]))
    bound = {k: _cases.bound(model, "grid_exact") if (exact and k == "spatial_embeddings") else FIELD_BOUND[precision]
             for k in errs}
    assert all(errs[k] <= bound[k] for k in errs), {k: "%.2e" % v for k, v in errs.items() if v > bound[k]}
    if chunk:
        monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
        d_film1, grads1 = _field_backward(siren, film, pts, dirs, dir_group, lock, raw, d_raw, exact)
        inv = _grad_errors(d_film, grads, d_film1, grads1)
        worst = max(inv, key=inv.get)
        print("layout %s %s %s: worst %s %.3g" % (layout, model, precision, worst, inv[worst]))
        assert inv[worst] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


# --------------------------------------------------------------------------------------------
# C. point network forward
# --------------------------------------------------------------------------------------------
#: how each tile layout passes directions: one per point, one per 24-sample ray, or one locked (0, 0, -1) per image
_FWD_DIRS = {"one_pair_per_cta": "per_point", "lone_tile_in_second_pair": "dir_group24", "4sms_minus_1": "lock_dirs",
             "b3_pairs_straddle_images": "dir_group24"}


def _forward_inputs(siren, layout, seed):
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    mode = _FWD_DIRS[layout]
    batch, ppb = _cases.tile_layout(layout, sms, 24 if mode == "dir_group24" else 1)
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(batch, ppb, 3, generator=g) - 0.5) * 0.24).to(DEV)
    n_dirs = {"per_point": ppb, "dir_group24": ppb // 24, "lock_dirs": 1}[mode]
    dirs = F.normalize(torch.randn(batch, n_dirs, 3, generator=g), dim=-1).to(DEV)
    if mode == "lock_dirs":
        dirs = _per_point(dirs, 1, True)
    return pts, dirs, _film(siren, batch, seed)


@gpu
@pytest.mark.parametrize("layout", _cases.TILE_LAYOUTS)
@pytest.mark.parametrize("model", FIELD_MODELS)
def test_point_network_vs_fp64(model, layout):
    """Both point-network kernels against oracle.field_eval in float64, per output channel, under tile schedules derived
    from the device's SM count (one pair per CTA, a lone tile in a second pair, two pairs per CTA with the last half
    empty, pairs across image borders); both kernels are bit-identical between launches, and the density-only entries
    are bit-equal to the full evaluations' sigma channel (the check that catches a density path without a grid gather)."""
    siren = _siren(model, DEV)
    pts, dirs, film = _forward_inputs(siren, layout, _fwd_seed(model))
    with torch.no_grad():
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact")
        exact2 = ops.siren_points(siren, pts, film, dirs, precision="exact")
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
        fast2 = ops.siren_points(siren, pts, film, dirs, precision="fast")
        sigma = ops.siren_sigma(siren, pts, film, precision="fast")
        sigma_x = ops.siren_sigma(siren, pts, film, precision="exact")
    want = field_ref(siren, pts, _per_point(dirs, pts.shape[1], False), film)[0]
    err = {k: (v.double() - want).abs().amax((0, 1)) for k, v in (("exact", exact), ("fast", fast))}
    print("forward %s %s: exact %.3g fast %.3g (sigma %.3g / %.3g)" % (model, layout, err["exact"].max(), err["fast"].max(),
                                                                      err["exact"][-1], err["fast"][-1]))
    assert torch.isfinite(fast).all()
    for k in err:
        assert err[k].max() <= _cases.bound(model, "fwd_" + k), "%s: max |out - fp64| per channel %s" % (k, err[k].tolist())
    assert torch.equal(fast, fast2) and torch.equal(exact, exact2)
    assert torch.equal(sigma, fast[..., -1:])
    assert torch.equal(sigma_x, exact[..., -1:])


# --------------------------------------------------------------------------------------------
# D. the bounds catch faults (CPU: each fault is applied to the float64 reference)
# --------------------------------------------------------------------------------------------
def _chunked_cumprod(x, dim):
    """torch.cumprod with the running product restarted every 32 samples: a lost scan carry."""
    return torch.cat([_TRUE_CUMPROD(c, dim) for c in x.split(32, dim)], dim)


class _ShiftedScanCumprod(torch.autograd.Function):
    """Correct cumprod forward; its reverse scan (the backward) read one sample late."""

    @staticmethod
    def forward(ctx, x, dim):
        ctx.save_for_backward(x)
        ctx.dim = dim
        return _TRUE_CUMPROD(x, dim)

    @staticmethod
    def backward(ctx, grad):
        x, = ctx.saved_tensors
        with torch.enable_grad():
            xx = x.detach().requires_grad_(True)
            g, = torch.autograd.grad(_TRUE_CUMPROD(xx, ctx.dim), xx, grad)
        n = g.shape[ctx.dim]
        return torch.cat([g.narrow(ctx.dim, 1, n - 1), torch.zeros_like(g.narrow(ctx.dim, 0, 1))], ctx.dim), None


_TRUE_CUMPROD = torch.cumprod


def _cpu_composite_inputs(n, hier):
    """Model A's fp32 oracle outputs on 36 render rays of one image."""
    siren = _siren("A", "cpu")
    film = _film(siren, 1, 9)
    steps = n // 2 if hier else n
    pts_c, z_c, dirs, org = _render_points(1, 6, steps, 9)
    with torch.no_grad():
        raw_c = oracle.field_eval(siren, pts_c.reshape(1, -1, 3), film, _per_point(dirs, 36 * steps, False)).reshape(1, 36, steps, 4)
        raw_f = z_f = None
        if hier:
            z_f = 0.88 + 0.24 * torch.sort(torch.rand(1, 36, steps, generator=torch.Generator().manual_seed(9)), -1)[0]
            pts_f = org.unsqueeze(2) + dirs.unsqueeze(2) * z_f.unsqueeze(-1)
            raw_f = oracle.field_eval(siren, pts_f.reshape(1, -1, 3), film, _per_point(dirs, 36 * steps, False)).reshape(1, 36, steps, 4)
    return raw_c, z_c, raw_f, z_f


@pytest.mark.parametrize("fault", ["carry_reset_every_32", "reverse_scan_one_sample_late"])
@pytest.mark.parametrize("n,hier", [(64, False), (48, True), (96, True)], ids=["n64-flat", "n48-hier", "n96-hier"])
def test_composite_faults_exceed_the_bound(monkeypatch, fault, n, hier):
    raw_c, z_c, raw_f, z_f = _cpu_composite_inputs(n, hier)
    opt = _opt("relu")
    d_pixels = torch.randn(1, 3, 6, 6, generator=torch.Generator().manual_seed(n))
    good = composite_vjp(raw_c, z_c, raw_f, z_f, None, opt, d_pixels)
    monkeypatch.setattr(torch, "cumprod", _chunked_cumprod if fault == "carry_reset_every_32" else _ShiftedScanCumprod.apply)
    bad = composite_vjp(raw_c, z_c, raw_f, z_f, None, opt, d_pixels)
    moved = max(_rel(b, g) for b, g in zip(bad, good) if g is not None)
    print("composite fault %s n=%d: %.3g" % (fault, n, moved))
    assert moved > 10 * COMPOSITE_BOUND, moved


def _cpu_field_case(model):
    siren = _siren(model, "cpu")
    batch, ppb, dir_group = 2, 480, 24
    pts, dirs = _field_points(batch, ppb, dir_group, 11)
    film = _film(siren, batch, 11, edges=True)
    d_raw = torch.randn(batch, ppb, siren.field_spec().out_dim, generator=torch.Generator().manual_seed(11)) * 1e-3
    return siren, pts, dirs, film, d_raw


@pytest.mark.parametrize("model", ["A", "D"])
def test_field_backward_faults_exceed_the_bounds(model):
    """Image 0's FiLM rows used for every image (a wrong b0 in gemm_nt_film / _stash / _gate) and directions sliced one ray
    off in image 1's second point chunk (a wrong p0 // dir_group).  Both must exceed the default-mode bound; the
    direction fault must exceed the layout-invariance bound, which is the check that sees it in default mode."""
    siren, pts, dirs, film, d_raw = _cpu_field_case(model)
    batch, ppb = pts.shape[:2]
    _, film_g, good = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw)
    _, film_b, bad = field_ref(siren, pts, _per_point(dirs, ppb, False), film, d_raw, film_rows=[0] * batch)
    moved_film = max(_grad_errors(film_b, bad, film_g, good).values())
    shifted = dirs.clone()
    half = dirs.shape[1] // 2
    shifted[1, half:-1] = dirs[1, half + 1:]
    _, film_d, bad_d = field_ref(siren, pts, _per_point(shifted, ppb, False), film, d_raw)
    moved_dirs = max(_grad_errors(film_d, bad_d, film_g, good).values())
    print("field faults %s: film rows %.3g, directions %.3g" % (model, moved_film, moved_dirs))
    assert moved_film > 10 * FIELD_BOUND["default"], moved_film
    assert moved_dirs > 10 * LAYOUT_BOUND and moved_dirs > FIELD_BOUND["exact"], moved_dirs


@pytest.mark.parametrize("model", ["A", "D"])
def test_forward_faults_exceed_the_bounds(model):
    """The neighbouring image's FiLM rows, and the bias of feature half 1 (features 128-255) left out of every FiLM
    layer: both must move some output channel past the fast kernel's bound."""
    siren, pts, dirs, film, _ = _cpu_field_case(model)
    dirs_pp = _per_point(dirs, pts.shape[1], False)
    good = field_ref(siren, pts, dirs_pp, film)[0]
    swapped = field_ref(siren, pts, dirs_pp, film, film_rows=[1, 0])[0]
    no_bias = copy.deepcopy(siren)
    with torch.no_grad():
        layers = list(no_bias.network) + (list(no_bias.color_layer_sine) if isinstance(no_bias.color_layer_sine, torch.nn.ModuleList)
                                          else [no_bias.color_layer_sine])
        for layer in layers:
            layer.layer.bias[128:] = 0
    dropped = field_ref(no_bias, pts, dirs_pp, film)[0]
    moved = {k: float((v - good).abs().amax((0, 1)).max()) for k, v in (("film_rows", swapped), ("bias_half1", dropped))}
    print("forward faults %s: %s" % (model, moved))
    assert min(moved.values()) > 10 * FWD_BOUND["fast"], moved


# --------------------------------------------------------------------------------------------
# E. the FiLM-gradient algebra of finish() at the frequency edges (CPU, float64)
# --------------------------------------------------------------------------------------------
def _record_film_layers(monkeypatch):
    log = []

    def film_layer(linear, x, freq, phase):
        u = freq.unsqueeze(1) * linear(x) + phase.unsqueeze(1)
        u.retain_grad()
        log.append((linear, x.detach(), u))
        return torch.sin(u)
    monkeypatch.setattr(oracle, "_film", film_layer)
    return log


def _film_grads_new(f, w, b, a, du):
    """finish()'s algebra: M_b = dU_b^T a, dp_b = sum dU_b -> (d freq, d phase, dW, db), no division by f."""
    m = torch.einsum("bpf,bpk->bfk", du, a)
    dp = du.sum(1)
    return torch.einsum("fk,bfk->bf", w, m) + b * dp, dp, torch.einsum("bf,bfk->fk", f, m), (f * dp).sum(0)


def _film_grads_divided(f, w, b, a, du):
    """The earlier algebra: from dZ = dU f, dp = db_b / f and df = rowsum(W dW_b) / f + b dp."""
    dz = du * f.unsqueeze(1)
    dw_b = torch.einsum("bpf,bpk->bfk", dz, a)
    db_b = dz.sum(1)
    dp = db_b / f
    return torch.einsum("fk,bfk->bf", w, dw_b) / f + b * dp, dp, dw_b.sum(0), db_b.sum(0)


@pytest.mark.parametrize("model", ["A", "D", "I", "K"])
def test_film_gradient_algebra_at_edge_frequencies(monkeypatch, model):
    """finish()'s FiLM-gradient algebra, restated from float64 autograd pieces (each layer's input and dL/du), equals
    the autograd gradients of the FiLM table and of every FiLM layer's weight and bias, with f in EDGE_FREQS planted in
    every FiLM row (in all images and in image 1 only).  The algebra that divided by f gives NaN at f = 0 and -0."""
    siren = copy.deepcopy(_siren(model, "cpu")).double()
    n = 300
    pts, dirs = _field_points(2, n, 3, 21)
    pts, dirs = pts.double(), _per_point(dirs, n, False).double()
    film0 = _film(_siren(model, "cpu"), 2, 21, edges=True).double()
    film, planted = plant_frequencies(film0, range(film0.shape[1]))
    film.requires_grad_(True)
    log = _record_film_layers(monkeypatch)
    out = oracle.field_eval(siren, pts, film, dirs)
    d_out = torch.randn(out.shape, generator=torch.Generator().manual_seed(22), dtype=torch.float64)
    (out * d_out).sum().backward()
    assert len(log) == film.shape[1]
    zero_cols = [(r, c) for r, c, img in planted if img is None and EDGE_FREQS[(c - 5) // 17] == 0.0]
    for row, (linear, a, u) in enumerate(log):
        f = film.detach()[:, row, 0]
        w, b = linear.weight.detach(), linear.bias.detach()
        want = (film.grad[:, row, 0], film.grad[:, row, 1], linear.weight.grad, linear.bias.grad)
        got = _film_grads_new(f, w, b, a, u.grad)
        for name, g, wv in zip(("freq", "phase", "weight", "bias"), got, want):
            assert torch.isfinite(wv).all() and torch.isfinite(g).all(), (row, name)
            assert _rel(g, wv) <= 1e-12, (row, name, _rel(g, wv))
        old = _film_grads_divided(f, w, b, a, u.grad)
        cols = [c for r, c in zero_cols if r == row]
        assert torch.isnan(old[0][:, cols]).all() and torch.isnan(old[1][:, cols]).all(), row
        assert torch.isfinite(want[0][:, cols]).all() and torch.isfinite(want[1][:, cols]).all()
