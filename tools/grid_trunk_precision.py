"""Error of the first layer of a grid-trunk field (EmbeddingPiGAN256) when its 32 grid features enter the wgmma kernel as
fp16 operands, on the CPU: the sine argument f (W [feat, x] + b) + p in float64 against

  fp16      what the kernel computes: the grid stored in fp16, the trilinear features rounded to fp16, the feature columns
            of W in fp16 (the position keeps its hi / lo split), exact products summed in float64
  split     features and feature weights both hi / lo split (hi*hi + lo*hi + hi*lo), the grid in fp32

and, for scale, the same error of hidden layer 1 (fp16 activations and weights), at the reference's init and random
latents, on points spread over the grid's box (a cfg2 render's samples lie inside it).

    python tools/grid_trunk_precision.py [--points N]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fenerf_b200.siren import siren as S  # noqa: E402


def f16(t):
    return t.half().double()


def split(t):
    hi = t.half().double()
    return hi, (t - hi).half().double()


def lookup(grid, x):
    """sample_from_3dgrid in float64: (1, P, 3) -> (1, P, C)."""
    s = torch.nn.functional.grid_sample(grid, x.reshape(1, 1, 1, -1, 3), mode='bilinear', padding_mode='zeros',
                                        align_corners=True)
    return s.reshape(grid.shape[1], -1).t().unsqueeze(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=200000)
    args = ap.parse_args()
    torch.manual_seed(0)
    field = S.EmbeddingPiGAN256(input_dim=3, z_dim=256, output_dim=4)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        film = field.film_from_latents(torch.randn(4, 256, generator=g)).double()
        pts = (torch.rand(1, args.points, 3, generator=g, dtype=torch.float64) - 0.5) * 0.24
        x = pts * (2 / 0.24)
        grid = field.spatial_embeddings.detach().double()
        feat = lookup(grid, x)[0]                                 # float64 lookup of the fp32 grid
        feat16 = f16(lookup(f16(grid), x)[0])                     # fp16 grid, fp16 operand
        W = field.network[0].layer.weight.detach().double()       # (256, 35): [feat, pos]
        b = field.network[0].layer.bias.detach().double()
        Wf, Wp = W[:, :32], W[:, 32:]
        pos_term = x[0] @ Wp.t()                                  # the position's split is fp32-accurate in every variant
        exact = feat @ Wf.t() + pos_term + b
        fast = feat16 @ f16(Wf).t() + pos_term + b
        fh, fl = split(feat)
        wh, wl = split(Wf)
        spl = fh @ wh.t() + fl @ wh.t() + fh @ wl.t() + pos_term + b
        W1 = field.network[1].layer.weight.detach().double()
        rows = {"fp16 features": [], "split features": [], "hidden layer 1 (fp16)": []}
        for i in range(film.shape[0]):
            f0, p0 = film[i, 0, 0], film[i, 0, 1]
            rows["fp16 features"].append(((fast - exact) * f0).abs())
            rows["split features"].append(((spl - exact) * f0).abs())
            a0 = torch.sin(f0 * exact + p0)
            z1 = a0 @ W1.t()
            z1h = f16(a0) @ f16(W1).t()
            rows["hidden layer 1 (fp16)"].append(((z1h - z1) * film[i, 1, 0]).abs())
    print("sine-argument error, %d points x %d latents (radians)" % (args.points, film.shape[0]))
    print("%-24s %10s %10s %10s" % ("", "rms", "p99.9", "max"))
    for k, v in rows.items():
        v = torch.cat([t.reshape(-1) for t in v])
        print("%-24s %10.3g %10.3g %10.3g" % (k, v.pow(2).mean().sqrt(), v.quantile(0.999) if v.numel() < 1 << 24 else
                                              v[torch.randperm(v.numel(), generator=g)[:1 << 23]].quantile(0.999), v.max()))


if __name__ == "__main__":
    main()
