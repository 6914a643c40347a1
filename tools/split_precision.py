"""The split-precision point network (precision='split') restated on the CPU against float64, at the reference's init and
random latents.  It computes what the split kernel computes:
  - every weight matrix (first layer, hidden layers, heads) scaled by a power of two s with max |s W| in [0.5, 1);
  - each 256-wide layer and head as hi * W_hi + lo * W_hi + hi * W_lo, with hi = f16(v), lo = f16(v - hi) in both
    operands, the sum divided by s again (the lo * lo term is dropped);
  - the grid features taken from the fp32 grid and split the same way;
  - every FiLM sine through the kernel's software sine (soft_sinf, restated in float32 arithmetic).
Products are summed in float64; the kernel sums them in fp32, which this restatement leaves out.

Why the scale: the hidden layers' frequency_init weights are |w| <= sqrt(6 / 256) / 25 = 6.1e-3.  Unscaled, w - f16(w)
falls below fp16's smallest normal (2^-14) and its low part keeps only a few bits; the 'unscaled' row shows what that
costs the direction-free field, whose first colour layer amplifies every error in its inputs.

For each field (A: TALLSIREN, B: TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96, P: its direction-free sibling) a
row gives the rms / max error of the FiLM sine arguments over all layers and the max error of the labels, rgb and sigma
against float64.  The fault rows are what the GPU tests' bounds must catch:
  - no_lo_w, no_w_lo: a dropped lo * W_hi or hi * W_lo term;
  - fp16_grid: the grid features from the fp16 copy (the fast path's);
  - sinf: __sinf in place of soft_sinf, modelled as sin.approx after a float32 a / 2 pi, plus an error of 2^-21 that
    varies with the argument (PTX documents sin.approx to 2^-20.9 on [-pi, pi]).
The diagnostic rows: lo_lo adds the dropped lo * W_lo term, f32_sine uses float64 sin rounded to float32.

    python tools/split_precision.py [--points N] [--latents B]
"""
import argparse
import copy
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
from _fp64 import _film, _siren  # noqa: E402
from oracle import render_oracle as oracle  # noqa: E402

FAULTS = ("no_lo_w", "no_w_lo", "fp16_grid", "sinf")
DIAGNOSTICS = ("unscaled", "lo_lo", "f32_sine")
_SIN64 = torch.sin


def f16(t):
    return t.half().to(t.dtype)


def f32(t):
    return t.float().to(t.dtype)


_SOFT = [-2.041572245e-08, 2.701100129e-06, -1.980991656e-04, 8.332454599e-03, -1.666656137e-01, 9.999996424e-01]


def _c(v):
    return float(torch.tensor(v, dtype=torch.float32))


def soft_sin(a):
    """soft_sinf (csrc/siren_fast.cuh) in float32 arithmetic: each fmaf is one float64 evaluation rounded to float32 (the
    product of two float32 values is exact in float64)."""
    a = f32(a)
    n = f32(a * _c(0.159154943) + 12582912.0) - 12582912.0
    r = f32(-n * _c(6.28318548) + a)
    r = f32(-n * _c(-1.74845553e-7) + r)
    r2 = f32(r * r)
    p = torch.full_like(r, _c(_SOFT[0]))
    for c in _SOFT[1:]:
        p = f32(p * r2 + _c(c))
    return f32(r * p)


def approx_sin(a):
    """__sinf: sin.approx of a float32 argument reduced by a float32 product a * (1 / 2 pi), plus an absolute error of
    2^-21 that varies with the argument (a model: PTX documents 2^-20.9 at most on [-pi, pi])."""
    t = f32(f32(a) * _c(0.5 / torch.pi))
    return _SIN64(2 * torch.pi * t) + 2.0 ** -21 * _SIN64(1000.0 * t)


def split_mm(a, w, fault=None):
    """a @ w.T from fp16 hi / lo parts of both operands, w scaled by a power of two first (unless fault='unscaled')."""
    scale = 1.0
    if fault != "unscaled":
        mx = w.abs().max().item()
        if mx > 0:
            scale = 2.0 ** -torch.frexp(torch.tensor(mx, dtype=torch.float64)).exponent.item()
    w = w * scale
    ah, wh = f16(a), f16(w)
    al, wl = f16(a - ah), f16(w - wh)
    z = ah @ wh.t()
    if fault != "no_lo_w":
        z = z + al @ wh.t()
    if fault != "no_w_lo":
        z = z + ah @ wl.t()
    if fault == "lo_lo":
        z = z + al @ wl.t()
    return z / scale


def patch_split(setattr_, fault=None, args=None):
    """Makes oracle.field_eval and the direction-free restatement compute as the split kernel does, through the setter
    `setattr_(obj, name, value)` -- pytest's monkeypatch.setattr, or a Patcher, which undoes its patches on exit.
    `args` collects every FiLM sine argument (float64) when given."""
    def linear(self, x):
        return split_mm(x, self.weight, fault) + self.bias

    def sine(a):
        if args is not None:
            args.append(a.detach().reshape(-1))
        if fault == "f32_sine":
            return f32(_SIN64(f32(a)))
        return approx_sin(a) if fault == "sinf" else soft_sin(a)

    setattr_(torch.nn.Linear, "forward", linear)
    setattr_(torch, "sin", sine)
    if fault == "fp16_grid":           # the fast path's copy: fp16 voxels, the interpolated feature rounded to fp16
        lookup = oracle.grid_lookup
        setattr_(oracle, "grid_lookup", lambda coords, g: f16(lookup(coords, f16(g))))


class Patcher:
    """setattr with undo, for use outside pytest: `with Patcher() as p: patch_split(p, ...)`."""

    def __init__(self):
        self.saved = []

    def __call__(self, obj, name, value):
        self.saved.append((obj, name, getattr(obj, name)))
        setattr(obj, name, value)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for obj, name, value in reversed(self.saved):
            setattr(obj, name, value)
        self.saved.clear()


def inputs(model, latents=2, points=4096, seed=3):
    siren = _siren(model, "cpu")
    film = _film(siren, latents, seed).double()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(latents, points, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(latents, points, 3, generator=g), dim=-1).double()
    return copy.deepcopy(siren).double(), film, pts, dirs


def evaluate(setattr_, siren, film, pts, dirs, mode=None, fault=None, args=None):
    """mode None: float64 (sine arguments into `args`); 'split': the split kernel's arithmetic (with `fault`)."""
    with torch.no_grad():
        if mode is None:
            if args is not None:
                setattr_(torch, "sin", lambda a: (args.append(a.detach().reshape(-1)), _SIN64(a))[1])
        else:
            patch_split(setattr_, fault, args)
        return oracle.field_eval(siren, pts, film, dirs)


def errors(siren, film, pts, dirs, fault=None, setattr_=None):
    """-> dict: sine-argument rms / max and the max error of labels, rgb, sigma against float64.  `setattr_`: the
    patching setter (pytest's monkeypatch.setattr); a Patcher per evaluation when None."""
    got_args, ref_args = [], []
    with Patcher() as p:
        want = evaluate(setattr_ or p, siren, film, pts, dirs, args=ref_args)
    with Patcher() as p:
        got = evaluate(setattr_ or p, siren, film, pts, dirs, "split", fault, got_args)
    d = torch.cat([g - w for g, w in zip(got_args, ref_args)]).abs()
    n_lab = got.shape[-1] - 4
    e = (got - want).abs()
    return dict(arg_rms=d.pow(2).mean().sqrt().item(), arg_max=d.max().item(),
                labels=e[..., :n_lab].max().item() if n_lab else 0.0, rgb=e[..., n_lab:n_lab + 3].max().item(),
                sigma=e[..., -1].max().item())


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--latents", type=int, default=2)
    a = ap.parse_args()
    print("%-6s %-10s %10s %10s %10s %10s %10s" % ("field", "variant", "arg rms", "arg max", "labels", "rgb", "sigma"))
    for model in ("A", "B", "P"):
        siren, film, pts, dirs = inputs(model, a.latents, a.points)
        for fault in (None,) + FAULTS + DIAGNOSTICS:
            if fault == "fp16_grid" and not hasattr(siren, "spatial_embeddings"):
                continue
            r = errors(siren, film, pts, dirs, fault)
            print("%-6s %-10s %10.3g %10.3g %10.3g %10.3g %10.3g" % (model, fault or "split", r["arg_rms"], r["arg_max"],
                                                                 r["labels"], r["rgb"], r["sigma"]))


if __name__ == "__main__":
    main()
