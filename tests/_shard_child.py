"""Child processes of tests/test_shard_rays.py.

  _shard_child.py det <out_dir> 0     torch.use_deterministic_algorithms(True): two virtual-rank gradient sums per mode,
                                      bitwise equal (CUBLAS_WORKSPACE_CONFIG comes from the parent)
  _shard_child.py ranks <out_dir> r   rank r of WORLD_SIZE NCCL processes (MASTER_ADDR / MASTER_PORT from the parent),
                                      on cuda:r: the virtual-rank run's frames and gradients, then three Adam steps
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(HERE), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch                                        # noqa: E402
import torch.distributed as dist                    # noqa: E402

import _cases                                       # noqa: E402
import _shard_rays as sr                            # noqa: E402
from fenerf_b200 import dist as fdist               # noqa: E402


def det():
    torch.use_deterministic_algorithms(True)
    dev = "cuda:0"
    for model, precision, grad_precision in (("B", "exact", None), ("B", "split", "split"), ("B", "guard", None),
                                             ("P", "exact", None)):
        gen = _cases.build_mirror(_cases.Case("x", model, 1, 0), dev)
        zs = [z.requires_grad_(True) for z in sr.latents(model, 1, dev)]
        kw = sr.kwargs(128, num_steps=16, precision=precision, grad_precision=grad_precision, nerf_noise=0.5)
        _, a = sr.grads(gen, "forward", zs, kw, 31, world=3)
        _, b = sr.grads(gen, "forward", zs, kw, 31, world=3)
        n = 0
        for x, y in zip(a, b):
            assert (x is None) == (y is None)
            if x is not None:
                assert torch.equal(x, y), (model, precision)
                n += 1
        print("det %s %s %s: %d gradient tensors bitwise equal over two runs" % (model, precision, grad_precision, n))


def _same_on_every_rank(t, tag):
    ref = t.clone()
    dist.broadcast(ref, 0)
    assert torch.equal(ref, t), "%s differs from rank 0's on rank %d" % (tag, dist.get_rank())


def ranks(rank):
    world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = "cuda:%d" % rank
    dist.init_process_group("nccl", init_method="env://", rank=rank, world_size=world, device_id=torch.device(dev))
    try:
        gen = _cases.build_mirror(_cases.Case("x", "B", 1, 0), dev)
        film = [t.clone().requires_grad_(True) for t in sr.film_inputs(gen, sr.latents("B", 1, dev))]
        for img, kw in ((128, sr.kwargs(128, precision="guard", nerf_noise=0.5)),
                        (67, sr.kwargs(67, precision="exact")),
                        (64, sr.kwargs(64, precision="guard", fill_mode='seg_padding_background'))):
            staged = 'fill_mode' in kw
            method = "staged_forward_with_frequencies" if staged else "forward_with_frequencies"
            with torch.no_grad():
                want = sr.virtual_forward(gen, method, film, kw, world, 5)
                sr.seed(5)
                got = fdist.render_sharded_rays(gen, method, *film, **kw)
            for a, b in zip(want, got):
                assert torch.equal(a, b), (img, "frame")
            if staged:
                continue
            _, want_g = sr.grads(gen, method, film, kw, 6, world=world)
            targets = sr.grad_targets(gen, film)
            for t in targets:
                t.grad = None
            sr.seed(6)
            px = fdist.render_sharded_rays(gen, method, *film, **kw)[0]
            (px * _cases.loss_weights(px.shape).to(dev)).sum().backward()
            got_g = [None if t.grad is None else t.grad.clone() for t in targets]
            worst = sr.worst_rel(want_g, got_g)
            print("rank %d R %d: reduced gradients vs the virtual-rank sum %.2e" % (rank, img, worst))
            assert worst <= 1e-5, worst
            for i, g in enumerate(got_g):
                if g is not None:
                    _same_on_every_rank(g, "gradient %d" % i)
        # three Adam steps on the FiLM offsets, as inverse_render_double_semantic.py takes them
        for t in film:
            t.requires_grad_(False)
        offsets = [torch.zeros_like(t, requires_grad=True) for t in film]
        target = torch.zeros(1, 22 - 1, 64, 64, device=dev)
        opt = torch.optim.Adam(offsets, lr=1e-2, weight_decay=1e-2)
        kw = sr.kwargs(64, precision="guard")
        for step in range(3):
            opt.zero_grad()
            sr.seed(100 + step)
            px = fdist.render_sharded_rays(gen, "forward_with_frequencies", *[f + o for f, o in zip(film, offsets)],
                                           **kw)[0]
            ((px - target) ** 2).mean().backward()
            opt.step()
        for i, o in enumerate(offsets):
            assert o.detach().abs().max() > 0
            _same_on_every_rank(o.detach(), "offset %d" % i)
        print("rank %d of %d: frames, gradients and Adam offsets agree" % (rank, world))
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    mode, out_dir, rank = sys.argv[1], sys.argv[2], int(sys.argv[3])
    if mode == "det":
        det()
    else:
        ranks(rank)
