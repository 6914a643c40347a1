"""Mesh extraction (fenerf_b200.shapes.extract_mesh) at 256^3 and 512^3: the density grid, marching cubes (classify, the
two scans, emit) and the per-vertex attributes, for models A, B and L (whose density gathers the feature grid).
Prints the card, its power limit and SM clock, then one line per (model, N) with milliseconds per stage and V, F.

CUDA events time the stages over --reps runs after one warm-up; a separate torch.profiler run of the count splits it into
mc_classify_kernel and the scan kernels.

    python tools/bench_mesh.py [--models A,B,L] [--res 256,512] [--reps 5]"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import _cases  # noqa: E402
from fenerf_b200 import ops, shapes  # noqa: E402

CASE = {"A": "a_small", "B": "b_small", "L": "l_small"}
CUBE = 0.3


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def kernel_split(fn):
    """-> (mc_classify_kernel ms, every other kernel's ms) of one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    classify = other = 0.0
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        ms = ev.device_time / 1e3 if hasattr(ev, "device_time") else ev.cuda_time / 1e3
        if "mc_classify_kernel" in ev.name:
            classify += ms
        elif "memset" not in ev.name.lower() and "Memset" not in ev.name:
            other += ms
    return classify, other


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="A,B,L")
    ap.add_argument("--res", default="256,512")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q))
    for model in args.models.split(","):
        gen = _cases.build_mirror(_cases.CASE_BY_NAME[CASE[model]], "cuda:0")
        siren = gen.siren
        g = torch.Generator(device="cuda").manual_seed(5)
        with torch.no_grad():
            zs = [torch.randn(1, 256, generator=g, device="cuda") for _ in range(_cases.n_latents(model))]
            film = siren.film_from_latents(*zs)
            coarse = shapes.extract_mesh(gen, film=film, level=0.0, resolution=24, attributes=False)["sigma"]
            level = float(torch.quantile(coarse.flatten(), 0.7))
        for n in (int(r) for r in args.res.split(",")):
            voxel = CUBE / (n - 1)
            origin = (-CUBE / 2,) * 3
            with torch.no_grad():
                t_density, sigma = timed(lambda: shapes.density_grid(siren, film, n, origin, voxel), args.reps)
                t_count, (ws, counts) = timed(lambda: ops.mc_count(sigma, level), args.reps)
                nv, nf = (int(c) for c in counts.tolist())
                t_emit, (verts, _) = timed(lambda: ops.mc_emit(sigma, level, origin, voxel, ws, nv, nf), args.reps)
                t_attr, _ = timed(lambda: shapes.vertex_attributes(siren, verts, film), args.reps)
                classify, scan = kernel_split(lambda: ops.mc_count(sigma, level))
            print("model %s %d^3: density %.2f ms | count %.3f ms (classify %.3f, scan %.3f) | emit %.3f ms | attributes "
                  "%.2f ms | V %d F %d | level %.4g" % (model, n, t_density, t_count, classify, scan, t_emit, t_attr, nv, nf,
                                                      level))
            del sigma, ws, counts, verts
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
