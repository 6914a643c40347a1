"""Times DoubleImplicitGenerator3d.point_forward against forward on the same rays (cfg2: B = 4, 128², 24 + 24, model B).

    python tools/bench_point_forward.py [--steps 20] [--warmup 5] [--precisions guard,exact]

The rays are those of one camera render (its workspace views, render_forward_stages), handed to point_forward with one
direction per sample (B, N, S, 3), the layout the reference's callers pass.  The two calls alternate in one process,
each step ending in a device synchronise; ms per step is the median.  no_grad, as in rendering.  Prints one JSON line
with the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import _cases  # noqa: E402
from fenerf_b200 import ops  # noqa: E402
from fenerf_b200.generators import volumetric_rendering as vr  # noqa: E402

CFG = dict(img_size=128, num_steps=24, batch=4)
KW = dict(fov=12, ray_start=0.88, ray_end=1.12, h_stddev=0.3, v_stddev=0.155, h_mean=3.14159265 / 2, v_mean=3.14159265 / 2,
          hierarchical_sample=True, sample_dist='gaussian', clamp_mode='relu', nerf_noise=0.0, last_back=False)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers still stand; say why the card is unnamed
        out = "unknown (%s)" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precisions", default="guard,exact")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_point_forward needs a CUDA device"
    dev = torch.device("cuda:0")
    b, r, s = CFG["batch"], CFG["img_size"], CFG["num_steps"]
    n = r * r
    gen = _cases.build_mirror(_cases.Case("bench", "B", b, 0), dev)
    torch.manual_seed(1)
    z_geo, z_app = torch.randn(b, 256, device=dev), torch.randn(b, 256, device=dev)
    with torch.no_grad():
        film = gen.siren.film_from_latents(z_geo, z_app)
    result = dict(gpu=gpu_info(), model="B", batch=b, img_size=r, num_steps=s, steps=args.steps, modes={})
    for precision in args.precisions.split(","):
        # the rays of one camera render
        rng = vr.DeviceRng(dev)
        perturb = rng.rand(b, n, s, 1).contiguous()
        c2w, _, _ = ops.camera_poses(b, "gaussian", KW["h_stddev"], KW["v_stddev"], KW["h_mean"], KW["v_mean"], rng, dev)
        noise_c, u, noise_f = rng.randn(b, n, s, 1), rng.rand(b * n, s), rng.randn(b, n, 2 * s, 1)
        rd = ops.make_render_desc(batch=b, img_size=r, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                                  fov=12, precision=precision)
        with torch.no_grad():
            st = ops.render_forward_stages(gen.siren, rd, film, *ops.ray_tables(r, s, 0.88, 1.12, dev), c2w, perturb,
                                           noise_c, u, noise_f)
        points = st["points_c"].clone()
        dirs = st["dirs"].unsqueeze(2).expand(-1, -1, s, -1).contiguous()       # one direction per sample
        ray_dirs = st["dirs"].clone()
        origins = c2w[:, :3, 3].unsqueeze(1).expand(b, n, 3).contiguous()
        z_vals = st["z_c"].unsqueeze(-1).clone()
        del st

        def run_forward():
            gen(z_geo, z_app, img_size=r, num_steps=s, precision=precision, **KW)

        def run_points():
            gen.point_forward(points, dirs, origins, ray_dirs, z_vals, z_geo, z_app, s, True, clamp_mode="relu",
                              nerf_noise=0.0, precision=precision)

        times = {"forward": [], "point_forward": []}
        with torch.no_grad():
            for i in range(args.warmup + args.steps):
                for name, fn in (("forward", run_forward), ("point_forward", run_points)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    if i >= args.warmup:
                        times[name].append((time.perf_counter() - t0) * 1e3)
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        result["modes"][precision] = {"forward_ms": round(med["forward"], 3), "point_forward_ms": round(med["point_forward"], 3),
                                      "ratio": round(med["point_forward"] / med["forward"], 4),
                                      "forward_ms_min_max": [round(min(times["forward"]), 3), round(max(times["forward"]), 3)],
                                      "point_forward_ms_min_max": [round(min(times["point_forward"]), 3),
                                                                   round(max(times["point_forward"]), 3)]}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
