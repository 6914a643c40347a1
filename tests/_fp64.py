"""float64 restatements shared by the float64 reference tests (test_gpu_fp64_reference.py, test_gpu_fp64_forward_stages.py):
fields and FiLM tables, the depth merge, the final compositing with every background / fill option, and the point network."""
import copy
import functools
import math

import torch
import torch.nn.functional as F

import _cases
from oracle import render_oracle as oracle


@functools.lru_cache(maxsize=None)
def _generator_cpu(model):
    if model != "D32":
        return _cases._mirror_generator_cached(model, False)
    from fenerf_b200.generators import generators as g
    from fenerf_b200.siren import siren as s
    torch.manual_seed(0)
    gen = g.DoubleImplicitGenerator3d(s.SIRENBASELINESEMANTICDISENTANGLE, 256, 256, 32)   # 28 labels
    gen.eval()
    return gen


def _siren(model, device, sigma_bias_shift=0.0):
    gen = copy.deepcopy(_generator_cpu(model))
    if sigma_bias_shift:
        with torch.no_grad():
            gen.siren.final_layer.bias += sigma_bias_shift
    gen.to(device)
    gen.device = device
    gen.siren.device = device
    return gen.siren


def _film(siren, batch, seed, edges=False):
    """FiLM table (B, L, 2, 256) from random latents.  edges: 10 % of the frequencies negated and 5 % set to
    0.25 <= |f| <= 1, so that the backward sees frequencies away from f ~ 30 (plant_frequencies() adds f = 0, tiny and
    large |f| in chosen columns)."""
    g = torch.Generator().manual_seed(seed)
    n_lat = 2 if hasattr(siren, "geo_mapping_network") else 1
    zs = [torch.randn(batch, 256, generator=g) for _ in range(n_lat)]
    dev = next(siren.parameters()).device
    with torch.no_grad():
        film = siren.film_from_latents(*[z.to(dev) for z in zs]).clone()
    if edges:
        f = film[:, :, 0]
        u = torch.rand(f.shape, generator=g).to(dev)
        mag = (0.25 + 0.75 * torch.rand(f.shape, generator=g)).to(dev) * torch.sign(f)
        f[u < 0.1] = -f[u < 0.1]
        small = (u >= 0.1) & (u < 0.15)
        f[small] = mag[small]
    return film.contiguous()


#: frequencies at the edges of the FiLM gradient algebra: zero of either sign (the table's 15 x + 30 is exactly 0 at
#: x = -2), one ulp of 30 (2^-19, the smallest non-zero |f| the table can hold near 0), values where the fp16 gate and
#: gradient streams would go subnormal if they carried f, and a large |f| where |u| reaches the hundreds
EDGE_FREQS = (0.0, -0.0, 2.0 ** -19, -2.0 ** -19, 1e-5, -1e-5, 1e-3, -1e-3, 0.05, -0.05, 150.0, -150.0)


def film_rows(siren):
    """FiLM rows by role: first / middle / last trunk layer, the label FiLM layer (or None), first / last colour layer."""
    t = len(siren.network)
    lf = int(hasattr(siren, "label_layer_sine"))
    color = siren.color_layer_sine
    n_color = len(color) if isinstance(color, torch.nn.ModuleList) else 1
    return dict(trunk_first=0, trunk_mid=t // 2, trunk_last=t - 1, label=t if lf else None, color_first=t + lf,
                color_last=t + lf + n_color - 1)


def plant_frequencies(film, rows, freqs=EDGE_FREQS):
    """Writes each frequency of `freqs` into every row of `rows` twice: in column 17 i + 5 of every image, and in
    column 17 i + 13 of the last image only (image b0 > 0 of a multi-image chunk).  -> (film, [(row, col, image or None)])"""
    film = film.clone()
    planted = []
    last = film.shape[0] - 1
    for row in sorted(set(rows)):
        for i, v in enumerate(freqs):
            film[:, row, 0, 17 * i + 5] = v
            film[last, row, 0, 17 * i + 13] = v
            planted += [(row, 17 * i + 5, None), (row, 17 * i + 13, last)]
    return film.contiguous(), planted


def pass_dirs(dirs, s, lock):
    """(B, N * S, 3) per-point directions of one pass of a camera render: each ray's direction (B, N, 3) repeated over
    its S samples, or (0, 0, -1) under lock_view_dependence."""
    if lock:
        d = torch.zeros((dirs.shape[0], dirs.shape[1] * s, 3), dtype=dirs.dtype, device=dirs.device)
        d[..., 2] = -1
        return d
    return dirs.repeat_interleave(s, dim=1)


def _rel(got, want):
    s = want.abs().max().item()
    return (got.double() - want.double()).abs().max().item() / (s if s > 0 else 1.0)


def _opt(clamp="relu", noise=0.0, last_back=False, white_back=False, black_back=False, softmax=False, fill_mode=None,
         fill_color="black"):
    return dict(clamp=clamp, noise=noise, last_back=last_back, white_back=white_back, black_back=black_back, softmax=softmax,
                fill_mode=fill_mode, fill_color=fill_color)


class _ZeroDraws:
    """alpha_composite's noise draw: zero (the noise is added to sigma beforehand, in fp32)."""

    def __init__(self, like):
        self.like = like

    def randn(self, *shape):
        return torch.zeros(shape, dtype=self.like.dtype, device=self.like.device)


def _merge(raw_c, z_c, raw_f, z_f):
    """Stable sort on depth, fine samples first (composite.cu's tie rule)."""
    if raw_f is None:
        return raw_c, z_c
    raw, z = torch.cat([raw_f, raw_c], 2), torch.cat([z_f, z_c], 2)
    z, order = torch.sort(z, dim=2, stable=True)
    return torch.gather(raw, 2, order.to(raw.device).unsqueeze(-1).expand(-1, -1, -1, raw.shape[-1])), z


def noise_offset(raw_c, z_c, raw_f, z_f, noise, std):
    """(sigma + noise * std) - sigma per merged sample, with the sum formed in fp32 as the reference and the kernel form it."""
    sig = _merge(raw_c, z_c, raw_f, z_f)[0][..., -1].detach().float()
    return (sig + noise.to(sig.device) * std).double() - sig.double()


PAD_FILL_MODES = ("seg_padding_background", "eval_seg_padding_background")


def _fill(out, wsum, fill_mode, fill_color):
    """The fill modes of oracle.alpha_composite (volumetric_rendering.py:53-102) on any device and dtype: rays with
    weights_sum < 0.9 are 'empty'; the seg-padding modes put a background channel in front of the colours / labels."""
    empty = (wsum < 0.9).unsqueeze(-1)
    n_ch = out.shape[-1]
    if fill_mode in ("debug", "weight_debug"):
        out = torch.where(empty, F.one_hot(torch.zeros((), dtype=torch.long), n_ch).to(out), out)
    elif fill_mode in PAD_FILL_MODES:
        out = torch.cat([torch.zeros_like(out[..., :1]), out], -1)
        if fill_color in oracle._FILL_VALUE:
            fill = torch.full((n_ch + 1,), oracle._FILL_VALUE[fill_color], dtype=out.dtype, device=out.device)
            fill[0] = 1
            out = torch.where(empty, fill, out)
    elif fill_mode == "eval_white_back":
        out = torch.where(empty, torch.ones_like(out), out)
    return out


def composite_ref(raw_c, z_c, raw_f, z_f, noise, opt, offset=None, full=False, ray_major=False):
    """float64 pixels (B, C_img, R, R) of the final compositing.  raw_* float64 (B, N, S, C), possibly requiring grad;
    z_* (B, N, S) and noise (B, N, n) are the kernel's own fp32 inputs (noise is in merged-sample order).

    Merge fine-first; sigma + noise * std formed in fp32 and then upcast (noise_offset; fixed by `offset` where the
    function must stay smooth under perturbation), so the relu sees the same sign as in the kernel.  Then
    oracle.alpha_composite in float64, the fill mode (C_img = C - 1, or C with the seg-padding background channel), the
    label softmax over the channels before the last three (so over [background, labels] with padding) and `* 2 - 1` to
    NCHW.  ray_major: the rays-in render's pixels instead, (B, N, C - 1) in [0, 1] for any N (no `* 2 - 1`, no
    reshape).  full: -> (pixels, depth (B, N), weights_sum (B, N), weights (B, N, n)) instead."""
    raw, z = _merge(raw_c, z_c, raw_f, z_f)
    sig = raw[..., -1]
    if noise is not None:
        sig = sig + (offset if offset is not None else noise_offset(raw_c, z_c, raw_f, z_f, noise, opt["noise"]))
    raw = torch.cat([raw[..., :-1], sig.unsqueeze(-1)], -1)
    z = z.to(raw.device).to(raw.dtype).unsqueeze(-1)
    px, depth, weights, wsum = oracle.alpha_composite(raw, z, _ZeroDraws(raw), 0.0, opt["clamp"], last_back=opt["last_back"],
                                                      white_back=opt["white_back"], black_back=opt["black_back"])
    px = _fill(px, wsum[..., 0], opt.get("fill_mode"), opt.get("fill_color", "black"))
    if opt["softmax"]:
        px = torch.cat([torch.softmax(px[..., :-3], -1), px[..., -3:]], -1)
    if not ray_major:
        b, n = px.shape[:2]
        r = math.isqrt(n)
        px = px.reshape(b, r, r, -1).permute(0, 3, 1, 2) * 2 - 1
    if not full:
        return px
    return px, depth[..., 0], wsum[..., 0], weights[..., 0]


def field_ref(siren, points, dirs_pp, film, d_raw=None, film_rows=None, chunk=1 << 15):
    """oracle.field_eval on a float64 copy of `siren`, on the tensors' device, in point chunks.
    -> (out (B, P, C) float64, d_film, {parameter name: float64 gradient}); the gradients (the VJP with d_raw, accumulated
    over the chunks) only when d_raw is given.  film_rows: image index whose FiLM rows each image uses (fault checks)."""
    ref = copy.deepcopy(siren).double()
    want_grad = d_raw is not None
    # a copy even of a float64 film: two calls must not accumulate into one .grad of the caller's tensor
    film64 = film.detach().to(torch.float64, copy=True).requires_grad_(want_grad)
    for p in ref.parameters():
        p.requires_grad_(want_grad)
    outs = []
    with torch.set_grad_enabled(want_grad):
        for p0 in range(0, points.shape[1], chunk):
            p1 = min(points.shape[1], p0 + chunk)
            fl = film64 if film_rows is None else film64[film_rows]
            out = oracle.field_eval(ref, points[:, p0:p1].double(), fl, dirs_pp[:, p0:p1].double())
            if want_grad:
                (out * d_raw[:, p0:p1].double()).sum().backward()
            outs.append(out.detach())
    out = torch.cat(outs, 1)
    if not want_grad:
        return out, None, None
    return out, film64.grad, {n: p.grad for n, p in ref.named_parameters() if p.grad is not None}
