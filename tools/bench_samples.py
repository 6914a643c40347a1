"""Times renders with more samples per pass: model B, 256², default (guard) precision, batch 1 and 4, at
num_steps 24 to 256 (+ as many fine samples), with the per-stage split of fenerf_debug_stage_times; one differentiable
model B step at 64², 96 + 96; and the compositing backward alone at n = 256 and 512 merged samples, where narrow fields
switch from staging their raw rows in shared memory to reading them from global memory.

    python tools/bench_samples.py [--steps 10] [--warmup 3] [--num-steps 24,48,64,72,96,128,256] [--batches 1,4]

Every timed call ends in a device synchronise (CUDA events around it); the median is reported.  no_grad for the renders,
as in rendering.  Prints one JSON line with the GPU's name and power limit, read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402
from fenerf_b200 import _lib, ops  # noqa: E402

STAGES = ["ray_setup", "field_coarse", "guard", "resample", "field_fine", "composite"]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers still stand; say why the card is unnamed
        out = "unknown (%s)" % e
    return out


def _med(v):
    return sorted(v)[len(v) // 2]


def _timed(fn, steps, warmup):
    """median ms of fn() over `steps` calls after `warmup`, CUDA events around each call."""
    out = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            out.append(e0.elapsed_time(e1))
    return _med(out)


def render_times(gen, s, batch, steps, warmup):
    """ms per call and per face, and the median in-step stage times (ms) of fenerf_render_forward."""
    lib = _lib.lib()
    md = dict(bench.metadata(256), num_steps=s)
    lat = [z.cuda() for z in bench.make_latents("B", 1, batch)[0]]
    with torch.no_grad():
        total = _timed(lambda: gen(*lat, **md), steps, warmup)
        acc = [[] for _ in STAGES]
        lib.fenerf_debug_stage_times(1, None)
        for _ in range(steps):
            gen(*lat, **md)
            out = (ctypes.c_float * len(STAGES))()
            lib.fenerf_debug_stage_times(1, out)
            torch.cuda.synchronize()
            for i in range(len(STAGES)):
                acc[i].append(out[i])
        lib.fenerf_debug_stage_times(0, None)
    return dict(ms=round(total, 3), ms_per_face=round(total / batch, 3),
                stages_ms={k: round(_med(v), 4) for k, v in zip(STAGES, acc)})


def train_step_ms(gen, steps, warmup, batch=4, img=64, s=96):
    """one differentiable step: forward with autograd, sum(pixels * W), backward to latents and weights."""
    md = dict(bench.metadata(img), num_steps=s)
    lat = [z.cuda().requires_grad_(True) for z in bench.make_latents("B", 1, batch)[0]]
    w = torch.randn(batch, 21, img, img, device="cuda")

    def step():
        px, _ = gen(*lat, **md)
        (px * w).sum().backward()
    return round(_timed(step, steps, warmup), 3)


def composite_backward_ms(c, steps_per_pass, steps, warmup, batch=4, img=128):
    """fenerf_composite_backward alone on random depths and outputs (hierarchical: n = 2 S merged samples)."""
    g = torch.Generator(device="cuda").manual_seed(c + steps_per_pass)
    n = img * img
    s = steps_per_pass
    z_c = 0.88 + 0.24 * torch.sort(torch.rand(batch, n, s, generator=g, device="cuda"), -1)[0]
    z_f = 0.88 + 0.24 * torch.sort(torch.rand(batch, n, s, generator=g, device="cuda"), -1)[0]
    raw_c = torch.randn(batch, n, s, c, generator=g, device="cuda") * 0.1
    raw_f = torch.randn(batch, n, s, c, generator=g, device="cuda") * 0.1
    d_px = torch.randn(batch, c - 1, img, img, generator=g, device="cuda")
    d_c, d_f = torch.empty_like(raw_c), torch.empty_like(raw_f)
    rd = ops.make_render_desc(batch=batch, img_size=img, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                              fov=12)
    lib = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream

    def run():
        _lib.check(lib.fenerf_composite_backward(ctypes.byref(rd), c, raw_c.data_ptr(), z_c.data_ptr(), raw_f.data_ptr(),
                                                 z_f.data_ptr(), 0, d_px.data_ptr(), d_c.data_ptr(), d_f.data_ptr(), st))
    ms = _timed(run, steps, warmup)
    # the plan composite.cu's composite_backward() picks: eight warps' staged raw blocks, or rows from global memory
    n_pad = (2 * s + 3) & ~3
    narrow = c <= 32 and 8 * ((7 * n_pad + 64 + 2 * s * c + 3) & ~3) * 4 <= 227 * 1024
    return dict(C=c, n=2 * s, rays=batch * n, ms=round(ms, 3), ns_per_ray=round(ms * 1e6 / (batch * n), 1),
                kernel="staged rows" if narrow else "rows from global memory")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--num-steps", default="24,48,64,72,96,128,256")
    ap.add_argument("--batches", default="1,4")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_samples needs a CUDA device"
    dev = torch.device("cuda:0")
    gen = bench.build_generator("B", dev)
    result = dict(gpu=gpu_info(), model="B", img_size=256, precision="guard", steps=args.steps, renders=[])
    for batch in [int(v) for v in args.batches.split(",")]:
        for s in [int(v) for v in args.num_steps.split(",")]:
            r = dict(batch=batch, num_steps=s, **render_times(gen, s, batch, args.steps, args.warmup))
            print(json.dumps(r), file=sys.stderr)
            result["renders"].append(r)
            torch.cuda.empty_cache()
    result["train_step_64px_96+96_B4_ms"] = train_step_ms(gen, args.steps, args.warmup)
    result["composite_backward"] = [composite_backward_ms(c, s, args.steps, args.warmup)
                                    for c in (4, 22) for s in (64, 128, 256)]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
