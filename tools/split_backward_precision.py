"""The split-precision backward (grad_precision='split') restated on the CPU against float64, at the reference's init and
random latents.  Through the trunk's 256-wide FiLM layers it computes what csrc/gemm_split.cu computes:
  - recompute    z = a W^T with a = the fp32 sine stream (scale 2^14: |a| <= 1) and W scaled by its power of two, then
                 u = fmaf(f, z + b, p) in float32 and a' = sin(u), gate = cos(u) through a precise float32 sine (float64
                 sine rounded to float32);
  - gate         dU = dA * gate in float32;
  - M_b          dU_b^T a_{l-1}, dU scaled by the power of two of its largest magnitude;
  - dA'          dU diag(f_b) W, the per-image (diag(f_b) W)^T scaled by its own power of two.
Every operand is scaled by s = 2^(15 - e) (largest magnitude m 2^e, m in [0.5, 1)) and split into hi = f16(s x),
lo = f16(s x - hi); each product is hi.hi + lo.hi + hi.lo (lo.lo dropped), summed in float64 (the kernels sum in fp32,
which this restatement leaves out).  The float64 reference runs the same chain with float64 operands and sines.

The top dU is 1e-3 randn, the size of an unscaled loss gradient: without the per-layer scale ('unscaled'), most of
s dU = dU lies below 0.125, where lo = dU - f16(dU) is an fp16 subnormal with few bits.

A row per field gives the largest error, over the trunk's layers, of the recomputed activations (absolute; |a| <= 1),
of M_b and of dA' (each relative to that layer's largest float64 entry).  The fault rows are what the bounds of
tests/test_split_backward.py must catch:
  - no_lo_w, no_w_lo: a dropped lo.hi or hi.lo term in all three products;
  - unscaled: dU split without its power-of-two scale;
  - sinf: __sinf in the recompute (tools/split_precision.approx_sin's model of sin.approx).

    python tools/split_backward_precision.py [--points N] [--latents B]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tools.split_precision import approx_sin, f16, f32, inputs  # noqa: E402

FAULTS = ("no_lo_w", "no_w_lo", "unscaled", "sinf")


def scale_exp(amax):
    """The kernels' scale exponent (fenerf_b200.ops.split_scale_exp) of an operand whose largest magnitude is amax."""
    e = torch.frexp(torch.as_tensor(amax, dtype=torch.float64)).exponent
    return int((15 - e).clamp(-126, 126))


def split(x, amax=None):
    """x (float64 holding float32 values) -> (hi, lo, s): s x split into fp16 parts; amax None: |x| <= 1."""
    s = 2.0 ** scale_exp(1.0 if amax is None else amax)
    xs = x * s
    hi = f16(xs)
    return hi, f16(xs - hi), s


def split_prod(xa, xb, fault):
    """sum of the three fp16 products of two split operands (hi, lo, s), unscaled: (hi.hi + lo.hi + hi.lo) / (s_a s_b);
    xa @ xb (batched when 3-D)."""
    (ah, al, sa), (bh, bl, sb) = xa, xb
    p = ah @ bh
    if fault != "no_lo_w":
        p = p + al @ bh
    if fault != "no_w_lo":
        p = p + ah @ bl
    return p / (sa * sb)


def _trunk(siren):
    return [(l.layer.weight.detach().double(), l.layer.bias.detach().double()) for l in siren.network]


def chain(siren, film, pts, mode=None, fault=None, seed=5):
    """The trunk's recompute and backward.  mode None: float64; 'split': the split kernels' arithmetic (with `fault`).
    -> list over layers l = 1 .. T-1 of (a_l, M_b, dA')."""
    layers = _trunk(siren)
    B, N, _ = pts.shape
    f = film[:, :, 0].unsqueeze(1)            # (B, 1, L, 256)
    p = film[:, :, 1].unsqueeze(1)
    split_mode = mode == "split"
    sin = (approx_sin if fault == "sinf" else lambda u: f32(torch.sin(u))) if split_mode else torch.sin
    cos = (lambda u: f32(torch.cos(u))) if split_mode else torch.cos
    w0, b0 = layers[0]
    a = torch.sin(f[:, :, 0] * (pts @ w0.t() + b0) + p[:, :, 0])        # layer 0: narrow inputs, fp32 in the kernels
    if split_mode:
        a = f32(a)
    acts, gates = [a], [None]
    for l in range(1, len(layers)):
        w, b = layers[l]
        if split_mode:
            z = f32(split_prod(split(acts[-1]), split(w.t(), w.abs().max()), fault))
            u = f32(f[:, :, l] * f32(z + b) + p[:, :, l])
        else:
            u = f[:, :, l] * (acts[-1] @ w.t() + b) + p[:, :, l]
        acts.append(sin(u))
        gates.append(cos(u))
    g = torch.Generator().manual_seed(seed)
    dA = (torch.randn(B, N, 256, generator=g) * 1e-3).double()
    if split_mode:
        dA = f32(dA)
    out = []
    for l in range(len(layers) - 1, 0, -1):
        w, _ = layers[l]
        dU = f32(dA * gates[l]) if split_mode else dA * gates[l]
        fw = f[:, 0, l].unsqueeze(2) * w                                  # (B, 256, 256): diag(f_b) W
        if split_mode:
            if fault == "unscaled":
                hi = f16(dU)
                lo, s = f16(dU - hi), 1.0
            else:
                hi, lo, s = split(dU, dU.abs().max().item())
            m_b = split_prod((hi.transpose(1, 2), lo.transpose(1, 2), s), split(acts[l - 1]), fault)
            dA = torch.stack([f32(split_prod((hi[i], lo[i], s), split(fw[i], fw[i].abs().max().item()), fault))
                              for i in range(B)])
        else:
            m_b = dU.transpose(1, 2) @ acts[l - 1]
            dA = dU @ fw
        out.append((acts[l], m_b, dA))
    return out[::-1]


def _rel(got, want):
    s = want.abs().max().item()
    return (got - want).abs().max().item() / (s if s > 0 else 1.0)


def errors(siren, film, pts, fault=None):
    """-> dict: the largest error over the trunk's layers of the activations (absolute), M_b and dA' (relative)."""
    with torch.no_grad():
        want = chain(siren, film, pts)
        got = chain(siren, film, pts, "split", fault)
    return dict(act=max((g[0] - w[0]).abs().max().item() for g, w in zip(got, want)),
                m_b=max(_rel(g[1], w[1]) for g, w in zip(got, want)),
                d_a=max(_rel(g[2], w[2]) for g, w in zip(got, want)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--latents", type=int, default=2)
    a = ap.parse_args()
    print("%-6s %-10s %10s %10s %10s" % ("field", "variant", "act", "M_b", "dA'"))
    for model in ("A", "B", "P"):
        siren, film, pts, _ = inputs(model, a.latents, a.points)
        for fault in (None,) + FAULTS:
            r = errors(siren, film, pts, fault)
            print("%-6s %-10s %10.3g %10.3g %10.3g" % (model, fault or "split", r["act"], r["m_b"], r["d_a"]))


if __name__ == "__main__":
    main()
