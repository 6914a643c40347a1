"""Per-stage timing of the feature-head fields against SPATIALSIRENSEMANTIC, in one process, alternating:
    python tools/bench_hd.py [reps]

For SPATIALSIRENSEMANTIC (23 channels), SPATIALSIRENBASELINEHD (65) and SPATIALSIRENSEMANTICHD (129), at B = 4, 64² and
128², 24 + 24 samples, guard precision: the per-stage times of fenerf_render_forward (fenerf_debug_stage_times, CUDA
events), the point network's TFLOP/s (FLOP counts below, each GEMM counted once) and the compositor's GB/s (the bytes
the algorithm must move: S' (4 C + 4) in and 4 (C - 1 + 2) out per ray).  Prints the GPU's name and power limit."""
import ctypes
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from fenerf_b200 import _lib  # noqa: E402

#: FLOP per point (2 per multiply-add, each GEMM once): first layer 3 -> 256, 7 trunk + label + colour layers
#: 256 -> 256 (the colour layer's 3 direction inputs included), heads
def _flops(label_film, label_dim, rgb_dim):
    f = 2 * 3 * 256 + 7 * 2 * 256 * 256 + 2 * 256                    # trunk + sigma
    f += 2 * 259 * 256 + 2 * 256 * rgb_dim                           # colour layer + head
    if label_film:
        f += 2 * 256 * 256 + 2 * 256 * label_dim
    return f


FIELDS = [("SPATIALSIRENSEMANTIC", 23, _flops(True, 19, 3)), ("SPATIALSIRENBASELINEHD", 65, _flops(False, 0, 64)),
          ("SPATIALSIRENSEMANTICHD", 129, _flops(True, 64, 64))]
STAGES = ["ray_setup", "field_coarse", "guard", "resample", "field_fine", "composite"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    dev = torch.device("cuda:0")
    from fenerf_b200.generators import generators as G
    from fenerf_b200.siren import siren as S
    print("GPU:", card())
    gens = {}
    for name, c, _ in FIELDS:
        torch.manual_seed(0)
        gens[name] = G.ImplicitGenerator3d(getattr(S, name), 256, c).to(dev).eval()
        gens[name].set_device(dev)
    lib = _lib.lib()
    B, spr = 4, 24
    for img in (64, 128):
        md = dict(img_size=img, fov=12, ray_start=0.88, ray_end=1.12, num_steps=spr, h_stddev=0.3, v_stddev=0.155,
                  h_mean=math.pi * 0.5, v_mean=math.pi * 0.5, hierarchical_sample=True, sample_dist='gaussian',
                  clamp_mode='relu', nerf_noise=0.0, last_back=False, precision="guard")
        torch.manual_seed(1000)
        z = torch.randn(B, 256, device=dev)
        acc = {name: [[] for _ in STAGES] for name, _, _ in FIELDS}
        with torch.no_grad():
            for name, _, _ in FIELDS:
                for _ in range(3):
                    gens[name](z, **md)
            torch.cuda.synchronize()
            lib.fenerf_debug_stage_times(1, None)
            for _ in range(reps):
                for name, _, _ in FIELDS:            # alternating: every field sees the same device state
                    gens[name](z, **md)
                    out = (ctypes.c_float * 6)()
                    lib.fenerf_debug_stage_times(1, out)
                    for i in range(6):
                        acc[name][i].append(out[i])
            lib.fenerf_debug_stage_times(0, None)
        med = lambda v: sorted(v)[len(v) // 2]          # noqa: E731
        n_rays = B * img * img
        print("\nB=%d %dx%d %d+%d samples, guard, median of %d (ms)" % (B, img, img, spr, spr, reps))
        print("%-24s " % "field" + " ".join("%12s" % s for s in STAGES) + "  %10s %10s %12s" % ("net TFLOP/s", "us/Mpt", "comp GB/s"))
        for name, c, fl in FIELDS:
            t = [med(v) for v in acc[name]]
            pts = n_rays * spr
            net_ms = t[1] + t[4]
            tflops = fl * 2 * pts / (net_ms * 1e-3) / 1e12
            comp_bytes = n_rays * (2 * spr * (4 * c + 4) + 4 * (c - 1 + 2))
            gbs = comp_bytes / (t[5] * 1e-3) / 1e9
            print("%-24s " % name + " ".join("%12.4f" % x for x in t) + "  %10.1f %10.2f %12.0f" % (
                tflops, net_ms * 1e3 / (2 * pts / 1e6), gbs))
    print("\nFLOP per point:", {n: f for n, _, f in FIELDS})


if __name__ == "__main__":
    main()
