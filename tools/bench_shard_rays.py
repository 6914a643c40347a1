"""Ray-sharded renders (fenerf_b200.dist.render_sharded_rays) on 1, 2, 4 and 8 GPUs, as many as are present.

Two workloads, model B (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96), B = 1, 256²:
  invert  one inversion step: forward_with_frequencies on FiLM tables that require grad, 24 + 24 steps, guard, and the
          backward of an L2 loss against a fixed target (inverse_render_double_semantic.py's step)
  staged  one staged_forward at 48 + 48 steps (render_multiview_images_double_semantic.py's call)
One process per GPU (NCCL); world size w uses ranks [0, w) as its own group.  Every round runs each (workload, w) arm in
turn; each arm starts after the same idle settle as bench.py's (queue drained, then SETTLE_S of idle), then --warmup
steps, then --steps timed steps between CUDA events; the slowest rank's time counts.  Prints the card, its power limit
and SM clock, one line per arm with the median over rounds, and the time of the gather's reorder copy at w = 2, 4, 8.

    python tools/bench_shard_rays.py [--steps 10] [--warmup 2] [--rounds 3] [--max-gpus 8]"""
import argparse
import os
import socket
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import _cases  # noqa: E402
from fenerf_b200 import dist as fdist  # noqa: E402

SETTLE_S = 1.0      # bench.py's idle time in front of every timed arm
IMG = 256
CURRICULUM = dict(img_size=IMG, fov=12, ray_start=0.88, ray_end=1.12, h_stddev=0.3, v_stddev=0.155, h_mean=np.pi * 0.5,
                  v_mean=np.pi * 0.5, hierarchical_sample=True, sample_dist='gaussian', clamp_mode='relu', nerf_noise=0.0,
                  precision='guard')


def worlds(n):
    return [w for w in (1, 2, 4, 8) if w <= n]


def make_steps(gen, dev):
    g = torch.Generator(device=dev).manual_seed(5)
    zs = [torch.randn(1, 256, generator=g, device=dev) for _ in range(2)]
    with torch.no_grad():
        fg, pg = gen.siren.geo_mapping_network(zs[0])
        fa, pa = gen.siren.app_mapping_network(zs[1])
    film = [t.clone().requires_grad_(True) for t in (fg, fa, pg, pa)]
    target = torch.zeros(1, 21, IMG, IMG, device=dev)

    def invert(group):
        px = fdist.render_sharded_rays(gen, "forward_with_frequencies", *film, group=group, num_steps=24, **CURRICULUM)[0]
        ((px - target) ** 2).mean().backward()

    def staged(group):
        with torch.no_grad():
            fdist.render_sharded_rays(gen, "staged_forward", *zs, group=group, num_steps=48, psi=0.7, **CURRICULUM)

    return {"invert": invert, "staged": staged}


def reorder_ms(dev, reps=50):
    """The gather's reorder (one torch.cat of the gathered windows into NCHW) for model B's 21-channel 256² frame."""
    out = {}
    for w in (2, 4, 8):
        buf = torch.randn(w, 1, 21, IMG // w, IMG, device=dev)
        fn = lambda: torch.cat([buf[r] for r in range(w)], 2)   # noqa: E731
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[w] = e0.elapsed_time(e1) / reps
    return out


def child(rank, world, args):
    torch.cuda.set_device(rank)
    dev = "cuda:%d" % rank
    if world > 1:
        dist.init_process_group("nccl", init_method="env://", rank=rank, world_size=world, device_id=torch.device(dev))
        groups = {w: dist.new_group(list(range(w))) for w in worlds(world)}
    else:
        groups = {1: None}
    gen = _cases.build_mirror(_cases.Case("x", "B", 1, 0), dev)
    steps = make_steps(gen, dev)
    times = {}

    def barrier():
        if world > 1:
            dist.barrier()

    for rnd in range(args.rounds):
        for name, fn in steps.items():
            for w, group in groups.items():
                torch.cuda.synchronize()
                barrier()
                time.sleep(SETTLE_S)
                ms = 0.0
                if rank < w:
                    for _ in range(args.warmup):
                        fn(group)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.steps):
                        fn(group)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1) / args.steps
                if world > 1:
                    t = torch.tensor([ms], device=dev)
                    dist.all_reduce(t, op=dist.ReduceOp.MAX)
                    ms = t.item()
                times.setdefault((name, w), []).append(ms)
    if rank == 0:
        for (name, w), v in sorted(times.items()):
            base = statistics.median(times[(name, 1)])
            print("%-6s %d GPU%s: %8.2f ms per call (median of %d rounds: %s) | %.2fx of 1 GPU" % (
                name, w, "s" if w > 1 else " ", statistics.median(v), len(v), ", ".join("%.2f" % x for x in v),
                base / statistics.median(v)))
        print("gather reorder (torch.cat, 1 x 21 x 256 x 256): %s" % ", ".join(
            "w=%d %.3f ms" % (w, ms) for w, ms in reorder_ms(dev).items()))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-gpus", type=int, default=8)
    ap.add_argument("--child", type=int, default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child is not None:
        child(args.child, int(os.environ["WORLD_SIZE"]), args)
        return
    assert torch.cuda.is_available(), "bench_shard_rays needs CUDA devices"
    world = max(worlds(min(torch.cuda.device_count(), args.max_gpus)))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s x %d visible, %d used | nvidia-smi: %s" % (torch.cuda.get_device_name(0), torch.cuda.device_count(),
                                                                 world, q.replace("\n", " ; ")))
    sys.stdout.flush()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__)] + sys.argv[1:]
    procs = [subprocess.Popen(cmd + ["--child", str(r)], env=env) for r in range(world)]
    try:
        rcs = [p.wait() for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    sys.exit(max(rcs, key=abs))


if __name__ == "__main__":
    main()
