"""Where the colour error of the direction-free texture-grid field (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96)
comes from, on the CPU, against float64: the first colour layer's sine argument f (W [feat, x] + b) + p and the rgb
output, at the reference's init and random latents, on points spread over the grid's box.

A layer "in fp16" rounds both of its operands (activations, weights) to fp16 and sums exact products in float64, as the
wgmma kernel does; "split" is hi*hi + lo*hi + hi*lo with hi = f16(v), lo = f16(v - hi) in both operands (features,
trunk output and weights).  The variants:

  fp16 trunk, fp16 c0      what the plain wgmma kernel computes: trunk layers 1..7, the first colour layer (features
                           from the fp16 grid) and colour layers 1..7 in fp16
  fp16 trunk, split c0     the same with the first colour layer split hi / lo in both operands
  exact trunk, fp16 c0     float64 everywhere but the first colour layer, in fp16
  exact trunk, split c0    float64 everywhere but the first colour layer, split
  fp32 throughout          the field evaluated in float32 (what the exact kernel and the reference's own fp32 forward do)

The first trunk layer keeps its fp32-accurate position split in every variant.  A second table gives the error of the
field's vector-Jacobian product (random output weights) evaluated in float32 -- the exact kernels' and the reference's
own precision -- against float64, per parameter tensor relative to its largest entry: the same amplification reaches the
gradients.

    python tools/wo_dir_precision.py [--points N] [--latents B]
"""
import argparse
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fenerf_b200.siren import siren as S  # noqa: E402


def f16(t):
    return t.half().to(t.dtype)


def split_mm(a, w):
    """a @ w.T from hi / lo fp16 parts of both operands (the lo * lo term dropped)."""
    ah, wh = f16(a), f16(w)
    al, wl = f16(a - ah), f16(w - wh)
    return ah @ wh.t() + al @ wh.t() + ah @ wl.t()


def lookup(grid, x):
    """sample_from_3dgrid: (B, P, 3) -> (B, P, C) in the grid's dtype."""
    b = x.shape[0]
    s = torch.nn.functional.grid_sample(grid.expand(b, -1, -1, -1, -1), x.reshape(b, 1, 1, -1, 3), mode='bilinear',
                                        padding_mode='zeros', align_corners=True)
    return s.reshape(b, grid.shape[1], -1).transpose(1, 2)


def evaluate(field, film, x, trunk16, c0):
    """-> (first colour layer's sine argument, rgb).  trunk16: trunk layers 1..7 and colour layers 1..7 in fp16; c0:
    'exact', 'fp16' or 'split' for the first colour layer."""
    dt = x.dtype

    def layer(i, h, fp16):
        lin = field.network[i].layer if i < 8 else field.color_layer_sine[i - 8].layer
        w, b = lin.weight.to(dt), lin.bias.to(dt)
        z = (f16(h) @ f16(w).t() if fp16 else h @ w.t()) + b
        return torch.sin(film[:, i, 0].unsqueeze(1) * z + film[:, i, 1].unsqueeze(1))

    grid = field.spatial_embeddings.detach().to(dt)
    h = layer(0, x, False)
    for i in range(1, 8):
        h = layer(i, h, trunk16)
    lin = field.color_layer_sine[0].layer
    w, b = lin.weight.to(dt), lin.bias.to(dt)
    if c0 == "fp16":
        c = torch.cat([lookup(f16(grid), x), h], dim=-1)        # the wgmma kernel reads the fp16 copy of the grid
        z = f16(c) @ f16(w).t() + b
    elif c0 == "split":
        z = split_mm(torch.cat([lookup(grid, x), h], dim=-1), w) + b
    else:
        z = torch.cat([lookup(grid, x), h], dim=-1) @ w.t() + b
    arg = film[:, 8, 0].unsqueeze(1) * z + film[:, 8, 1].unsqueeze(1)
    c = torch.sin(arg)
    for i in range(9, 16):
        c = layer(i, c, trunk16)
    head = field.color_layer_linear[0]
    return arg, torch.sigmoid(c @ head.weight.to(dt).t() + head.bias.to(dt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--latents", type=int, default=2)
    args = ap.parse_args()
    torch.manual_seed(0)
    field = S.TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96(input_dim=3, z_geo_dim=256, z_app_dim=256,
                                                                        output_dim=22)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        film = field.film_from_latents(torch.randn(args.latents, 256, generator=g),
                                       torch.randn(args.latents, 256, generator=g)).double()
        pts = (torch.rand(args.latents, args.points, 3, generator=g, dtype=torch.float64) - 0.5) * 0.24
        x = pts * (2 / 0.24)
        arg64, rgb64 = evaluate(field, film, x, False, "exact")
        rows = {}
        for name, trunk16, c0 in (("fp16 trunk, fp16 c0", True, "fp16"), ("fp16 trunk, split c0", True, "split"),
                                  ("exact trunk, fp16 c0", False, "fp16"), ("exact trunk, split c0", False, "split")):
            rows[name] = evaluate(field, film, x, trunk16, c0)
        arg32, rgb32 = evaluate(field, film.float(), x.float(), False, "exact")
        rows["fp32 throughout"] = (arg32.double(), rgb32.double())
    print("TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96, reference init, %d latents x %d points, against float64"
          % (args.latents, args.points))
    print("%-24s %12s %12s %12s %12s" % ("", "arg rms", "arg max", "rgb rms", "rgb max"))
    for name, (arg, rgb) in rows.items():
        da, dr = (arg - arg64).abs(), (rgb - rgb64).abs()
        print("%-24s %12.3g %12.3g %12.3g %12.3g" % (name, da.pow(2).mean().sqrt(), da.max(), dr.pow(2).mean().sqrt(),
                                                     dr.max()))
    grad_table(field, film, x, g)


def vjp(field, film, x, d_rgb):
    """Gradients of sum(rgb * d_rgb) with respect to the field's colour-branch and trunk parameters and the FiLM table."""
    film = film.clone().requires_grad_(True)
    params = dict((n, p) for n, p in field.named_parameters() if "mapping" not in n and p.requires_grad)
    _, rgb = evaluate(field, film, x, False, "exact")
    names = [n for n in params if not n.startswith(("final_layer", "label_layer"))]
    grads = torch.autograd.grad((rgb * d_rgb).sum(), [params[n] for n in names] + [film], allow_unused=True)
    return dict(zip(names + ["film"], grads))


def grad_table(field, film, x, g):
    d_rgb = torch.randn(x.shape[0], x.shape[1], 3, generator=g, dtype=torch.float64)
    f64 = copy.deepcopy(field).double()
    want = vjp(f64, film, x, d_rgb)
    got = vjp(copy.deepcopy(field).float(), film.float(), x.float(), d_rgb.float())
    rel = {k: ((got[k].double() - want[k]).abs().max() / want[k].abs().max()).item()
           for k in want if want[k] is not None and want[k].abs().max() > 0}
    worst = sorted(rel.items(), key=lambda kv: -kv[1])
    print("\nfloat32 VJP of the rgb against float64, max |error| / max |gradient| per tensor (worst five of %d)" % len(rel))
    for k, v in worst[:5]:
        print("  %-40s %10.3g" % (k, v))


if __name__ == "__main__":
    main()
