"""Ray-sharded renders (fenerf_b200.dist.render_sharded_rays), shared by tests/test_shard_rays.py and its child processes.

A virtual-rank run renders every rank's pixel rows in turn in one process (dist.RayShard with collective=False), each
from the same seeded generator state, and assembles the windows; its gradients are the sum of the windows' own.
"""
import random

import numpy as np
import torch

import _cases
from fenerf_b200 import dist as fdist

#: curriculum of the sharded renders: small enough to run many, with every per-ray option the render has
BASE = dict(fov=12, ray_start=0.88, ray_end=1.12, num_steps=12, h_stddev=0.3, v_stddev=0.155, h_mean=np.pi * 0.5,
            v_mean=np.pi * 0.5, hierarchical_sample=True, sample_dist='gaussian', clamp_mode='relu', nerf_noise=0.0)


def kwargs(img_size, **kw):
    d = dict(BASE, img_size=img_size)
    d.update(kw)
    return d


def seed(s):
    torch.manual_seed(s)
    random.seed(s)


def latents(model, batch, device, s=1000):
    g = torch.Generator().manual_seed(s)
    return [torch.randn(batch, 256, generator=g).to(device) for _ in range(_cases.n_latents(model))]


def film_inputs(gen, zs):
    """The FiLM tables of forward_with_frequencies / staged_forward_with_frequencies for latents zs (double-latent
    generators: frequencies geo, app, phase shifts geo, app)."""
    with torch.no_grad():
        fg, pg = gen.siren.geo_mapping_network(zs[0])
        fa, pa = gen.siren.app_mapping_network(zs[1])
    return [fg, fa, pg, pa]


def call(gen, method, inputs, kw, s, shard=None):
    seed(s)
    extra = dict(_ray_shard=shard) if shard is not None else {}
    return getattr(gen, method)(*inputs, **kw, **extra)


def rows_dim(t):
    """Pixel rows of a returned image-shaped tensor: (B, C, R, R) or (B, R, R) -> dim -2; poses (B, 2) have none."""
    return t.dim() - 2 if t.dim() >= 3 else None


def assemble(outs, img_size, world):
    """Per-rank returns of a virtual-rank run -> the whole: every image-shaped tensor takes each rank's rows from that
    rank; the rest (poses) must be the same on every rank."""
    whole = []
    for i, first in enumerate(outs[0]):
        d = rows_dim(first)
        if d is None:
            for o in outs[1:]:
                assert torch.equal(o[i], first), "output %d differs between ranks" % i
            whole.append(first)
            continue
        t = torch.empty_like(first)
        for r, o in enumerate(outs):
            lo, hi = fdist.row_bounds(img_size, r, world)
            t.narrow(d, lo, hi - lo).copy_(o[i].narrow(d, lo, hi - lo))
        whole.append(t)
    return whole


def virtual_forward(gen, method, inputs, kw, world, s, per_rank=None):
    """The returns of a virtual-rank run, assembled; per_rank(rank) runs after each rank's render."""
    outs = []
    for r in range(world):
        out = call(gen, method, inputs, kw, s, fdist.RayShard(r, world, collective=False))
        outs.append(out)
        if per_rank is not None:
            per_rank(r)
    return assemble(outs, kw['img_size'], world)


def grad_targets(gen, inputs):
    """What a render's backward reaches: the inputs that require grad and every parameter of the generator."""
    return [t for t in inputs if t.requires_grad] + [p for p in gen.parameters() if p.requires_grad]


def grads(gen, method, inputs, kw, s, world=None, shard_of=None):
    """Gradients of L = sum(pixels * W) w.r.t. grad_targets: unsharded (world None), or summed over the ranks of a
    virtual-rank run (each rank's window backward accumulates into the same .grad).  -> (pixels, [grad or None])."""
    targets = grad_targets(gen, inputs)
    for t in targets:
        t.grad = None
    ranks = [None] if world is None else [fdist.RayShard(r, world, collective=False) for r in range(world)]
    pixels = None
    for shard in ranks:
        px = call(gen, method, inputs, kw, s, shard)[0]
        w = _cases.loss_weights(px.shape).to(px.device)
        (px * w).sum().backward()
        pixels = px.detach() if pixels is None else pixels
    return pixels, [None if t.grad is None else t.grad.detach().clone() for t in targets]


def worst_rel(a, b):
    """max over tensors of max|a - b| / max|a| (None where neither has a gradient)."""
    worst = 0.0
    for x, y in zip(a, b):
        assert (x is None) == (y is None)
        if x is None:
            continue
        scale = x.abs().max().item()
        worst = max(worst, (x - y).abs().max().item() / max(scale, 1e-30))
    return worst
