"""Cost of the pose gradient: render + backward of forward_with_frequencies with and without h_mean / v_mean requiring
grad, on one GPU.

Two workloads, precision 'guard', FiLM tables that require grad in both arms:
  invert  model B (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96), B = 1, 256², 24 steps, no hierarchical sampling:
          an inversion step with the camera pose fitted jointly (inverse_render_double_semantic.py's call)
  cfg2    model A (TALLSIREN), B = 4, 128², 24 + 24 steps, per-image (B, 1) means
Every round runs the two arms of a workload in turn (pose grad off, on), each after the same idle settle as bench.py's
(queue drained, then SETTLE_S of idle), --warmup steps, then --steps timed steps between CUDA events.  Prints the card,
its power limit and SM clock, and per arm the median over rounds.

    python tools/bench_pose_grad.py [--steps 10] [--warmup 2] [--rounds 5]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import _cases  # noqa: E402

SETTLE_S = 1.0
KW = dict(fov=12, ray_start=0.88, ray_end=1.12, h_stddev=0.3, v_stddev=0.155, sample_dist='gaussian', clamp_mode='relu',
          nerf_noise=0.0, precision='guard')
WORKLOADS = {"invert": dict(model="B", batch=1, img_size=256, num_steps=24, hierarchical_sample=False),
             "cfg2": dict(model="A", batch=4, img_size=128, num_steps=24, hierarchical_sample=True)}


def make_step(name, dev):
    w = dict(WORKLOADS[name])
    model, b = w.pop("model"), w.pop("batch")
    gen = _cases.build_mirror(_cases.Case("x", model, 1, 0), dev)
    g = torch.Generator(device=dev).manual_seed(5)
    zs = [torch.randn(b, 256, generator=g, device=dev) for _ in range(_cases.n_latents(model))]
    with torch.no_grad():
        if len(zs) == 1:
            film = list(gen.siren.mapping_network(zs[0]))
        else:
            fg, pg = gen.siren.geo_mapping_network(zs[0])
            fa, pa = gen.siren.app_mapping_network(zs[1])
            film = [fg, fa, pg, pa]
    film = [t.clone().requires_grad_(True) for t in film]
    shape = (b, 1) if b > 1 else ()

    def step(pose_grad):
        pose = dict(h_mean=torch.full(shape, math.pi / 2, device=dev), v_mean=torch.full(shape, math.pi / 2, device=dev))
        if pose_grad:
            for t in pose.values():
                t.requires_grad_(True)
        px, poses = gen.forward_with_frequencies(*film, **w, **KW, **pose)
        (px.square().mean() + poses.sum()).backward()

    return step


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pose_grad.py needs a CUDA device")
    dev = "cuda:0"
    print("card: %s" % card())
    results = {}
    for name in WORKLOADS:
        step = make_step(name, dev)
        times = {False: [], True: []}
        for _ in range(args.rounds):
            for pose_grad in (False, True):
                torch.cuda.synchronize()
                time.sleep(SETTLE_S)
                for _ in range(args.warmup):
                    step(pose_grad)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step(pose_grad)
                e1.record()
                torch.cuda.synchronize()
                times[pose_grad].append(e0.elapsed_time(e1) / args.steps)
        off, on = statistics.median(times[False]), statistics.median(times[True])
        results[name] = dict(off_ms=off, on_ms=on, overhead=on / off - 1, off_all=times[False], on_all=times[True])
        print("%-7s pose grad off %.2f ms  on %.2f ms  (%+.1f %%)" % (name, off, on, 100 * (on / off - 1)))
    print(json.dumps(results))


if __name__ == "__main__":
    main()
