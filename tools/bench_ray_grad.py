"""Times point_forward's render + backward with and without ray_grad=True (cfg2: B = 4, 128², 24 + 24; models B and D).

    python tools/bench_ray_grad.py [--steps 10] [--warmup 3] [--models B,D] [--precisions guard,exact]

point_forward belongs to the double-latent generator, so the plain FiLM-SIREN field is model D's (model A's field in a
double-latent generator) beside model B's grid field.  The rays are those of one camera render (render_forward_stages) with per-sample directions varied along each ray, so the
fine pass's direction gradients go back through the draw slots.  The loss is a fixed projection of the pixels; the two
calls (latents only, and latents + points + directions with ray_grad=True) alternate in one process, each step ending in
a device synchronise; ms per step is the median.  The grid coordinate gradient (fenerf_grid_coord_grad, model B's
1 KB-per-point gather of 8 corners x 32 fp32 channels) is timed alone with CUDA events over the coarse pass's points,
and its bytes/s is that gather over the kernel time.  Prints one JSON line with the GPU's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import _cases  # noqa: E402
from bench_point_forward import CFG, KW, gpu_info  # noqa: E402
from fenerf_b200 import _lib, ops  # noqa: E402
from fenerf_b200.generators import volumetric_rendering as vr  # noqa: E402


def camera_rays(gen, film, b, r, s, precision, dev):
    rng = vr.DeviceRng(dev)
    n = r * r
    perturb = rng.rand(b, n, s, 1).contiguous()
    c2w, _, _ = ops.camera_poses(b, "gaussian", KW["h_stddev"], KW["v_stddev"], KW["h_mean"], KW["v_mean"], rng, dev)
    noise_c, u, noise_f = rng.randn(b, n, s, 1), rng.rand(b * n, s), rng.randn(b, n, 2 * s, 1)
    rd = ops.make_render_desc(batch=b, img_size=r, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                              fov=12, precision=precision)
    with torch.no_grad():
        st = ops.render_forward_stages(gen.siren, rd, film, *ops.ray_tables(r, s, 0.88, 1.12, dev), c2w, perturb,
                                       noise_c, u, noise_f)
    dirs = st["dirs"].unsqueeze(2).expand(-1, -1, s, -1)
    dirs = torch.nn.functional.normalize(dirs + 0.05 * torch.randn(dirs.shape, device=dev), dim=-1).contiguous()
    return dict(points=st["points_c"].clone(), dirs=dirs, origins=c2w[:, :3, 3].unsqueeze(1).expand(b, n, 3).contiguous(),
                ray_dirs=st["dirs"].clone(), z_vals=st["z_c"].unsqueeze(-1).clone())


def grid_kernel(gen, points, dev, reps=20):
    """ms per launch of fenerf_grid_coord_grad over `points` (B, P, 3) and the bytes/s of its 1 KB-per-point gather."""
    packed = gen.siren.packed()
    pts = points.reshape(-1, 3).contiguous()
    P = pts.shape[0]
    d_feat = torch.randn((P, 32), device=dev, dtype=torch.float16)
    out = torch.empty((P, 3), device=dev)

    def launch():
        _lib.check(_lib.lib().fenerf_grid_coord_grad(C.byref(packed.desc), packed.ptr, pts.data_ptr(), d_feat.data_ptr(), 32,
                                                     P, out.data_ptr(), 0, torch.cuda.current_stream(dev).cuda_stream))

    for _ in range(3):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return dict(points=P, ms=round(ms, 4), gather_GBps=round(P * 1024 / (ms * 1e-3) / 1e9, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", default="B,D")
    ap.add_argument("--precisions", default="guard,exact")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ray_grad needs a CUDA device"
    dev = torch.device("cuda:0")
    b, r, s = CFG["batch"], CFG["img_size"], CFG["num_steps"]
    result = dict(gpu=gpu_info(), batch=b, img_size=r, num_steps=s, steps=args.steps, runs={})
    for model in args.models.split(","):
        gen = _cases.build_mirror(_cases.Case("bench", model, b, 0), dev)
        torch.manual_seed(1)
        zs = [torch.randn(b, 256, device=dev) for _ in range(_cases.n_latents(model))]
        with torch.no_grad():
            film = gen.siren.film_from_latents(*zs)
        for precision in args.precisions.split(","):
            rays = camera_rays(gen, film, b, r, s, precision, dev)
            w = torch.randn((b, r * r, gen.siren.field_spec().out_dim - 1), device=dev)

            def step(ray_grad):
                z = [t.clone().requires_grad_(True) for t in zs]
                rr = dict(rays)
                if ray_grad:
                    rr["points"] = rays["points"].clone().requires_grad_(True)
                    rr["dirs"] = rays["dirs"].clone().requires_grad_(True)
                px = gen.point_forward(rr["points"], rr["dirs"], rr["origins"], rr["ray_dirs"], rr["z_vals"], *z, s, True,
                                       clamp_mode="relu", nerf_noise=0.0, precision=precision,
                                       **({"ray_grad": True} if ray_grad else {}))
                (px * w).sum().backward()

            times = {False: [], True: []}
            for i in range(args.warmup + args.steps):
                for rg in (False, True):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    step(rg)
                    torch.cuda.synchronize()
                    if i >= args.warmup:
                        times[rg].append((time.perf_counter() - t0) * 1e3)
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            result["runs"]["%s_%s" % (model, precision)] = {
                "render_backward_ms": round(med[False], 2), "with_ray_grad_ms": round(med[True], 2),
                "overhead_ms": round(med[True] - med[False], 2),
                "min_max_ms": [[round(min(times[k]), 2), round(max(times[k]), 2)] for k in (False, True)]}
            if gen.siren.field_spec().grid_channels and precision == args.precisions.split(",")[0]:
                result["grid_coord_grad_" + model] = grid_kernel(gen, rays["points"], dev)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
