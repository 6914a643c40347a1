"""precision='split' against 'exact' and 'guard' at cfg2 (B = 4, 128², 24 + 24 samples per ray, CUDA graph) for models A,
B and P (P: 'exact' and 'split' only; its fp16 colour path is refused), alternating the arms in one process, --rounds
rounds.  Per arm: the graphed step time, the point network's launch time (CUDA events around ops.siren_points on one
cfg2 pass, 4 x 128² x 24 points) and its achieved TFLOP/s, each GEMM counted once (SURVEY.md section 8d; the split
kernel issues three fp16 products per GEMM).  Prints the card, its power limit and SM clock limit first.

    python tools/bench_split.py [--rounds N] [--models A,B,P]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import _cases  # noqa: E402
from _fp64 import _film  # noqa: E402
from fenerf_b200 import ops  # noqa: E402
from fenerf_b200.graphs import GraphedRender  # noqa: E402

# FLOP per point, each GEMM once: A / B as tools/bench_configs.py; P: 14 hidden layers, the 288-wide first colour layer,
# the first layer and the heads (18 labels, sigma, rgb)
_W = 2 * 256 * 256
FLOP_PER_POINT = {"A": 1053696, "B": 1341440, "P": 14 * _W + 2 * 288 * 256 + 2 * 3 * 256 + 2 * 22 * 256}
CASE = {"A": "a_small", "B": "b_small", "P": "p_small"}
ARMS = {"A": ("split", "exact", "guard"), "B": ("split", "exact", "guard"), "P": ("split", "exact")}
BATCH, IMG, STEPS, REPS = 4, 128, 24, 10


def _timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", default="A,B,P")
    args = ap.parse_args()
    dev = "cuda:0"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device: %s (%s)" % (torch.cuda.get_device_name(dev), q.stdout.strip() or "nvidia-smi unavailable"))
    setups = {}
    for model in args.models.split(","):
        gen = _cases.build_mirror(_cases.CASE_BY_NAME[CASE[model]], dev)
        md = dict(_cases.BASE, img_size=IMG, num_steps=STEPS, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)
        g = torch.Generator().manual_seed(1)
        lat = [torch.randn(BATCH, 256, generator=g).to(dev) for _ in range(_cases.n_latents(model))]
        n = IMG * IMG * STEPS
        pts = ((torch.rand(BATCH, n, 3, generator=g) - 0.5) * 0.24).to(dev)
        dirs = torch.nn.functional.normalize(torch.randn(BATCH, IMG * IMG, 3, generator=g), dim=-1).to(dev)
        film = _film(gen.siren, BATCH, 1).contiguous()
        setups[model] = (gen, md, lat, pts, dirs, film)
    for r in range(args.rounds):
        for model in args.models.split(","):
            gen, md, lat, pts, dirs, film = setups[model]
            for arm in ARMS[model]:
                with torch.no_grad():
                    gr = GraphedRender(gen, lat, dict(md, precision=arm))
                    step = _timed(lambda: gr(*lat), REPS)
                    pn = _timed(lambda: ops.siren_points(gen.siren, pts, film, dirs, precision=arm), REPS)
                del gr
                flop = BATCH * IMG * IMG * STEPS * FLOP_PER_POINT[model]
                print("round %d  model %s  %-5s  cfg2 step %8.3f ms (graph)   point network %7.3f ms / pass  %6.1f TFLOP/s" % (
                    r, model, arm, step, pn, flop / pn / 1e9))
                sys.stdout.flush()


if __name__ == "__main__":
    main()
