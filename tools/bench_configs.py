"""Forward-render throughput at the shapes of SURVEY.md section 8d (cfg1, cfg2, cfg5) for both benchmarked
fields, and at cfg2 for SPATIALSIRENBASELINE (C), the grid-trunk EmbeddingPiGAN256 (L) and the bridge fields AUG (M,
against H: 8 + 8 FiLM rows) and RES (N, against G), through the class API
(generator(z, **metadata)), latents resident.  One line per configuration.

    python tools/bench_configs.py [--models C,L] [--rounds N]     (--rounds: the chosen rows N times, alternating)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import _cases
import _grid_trunk  # (registers model L)
import _bridge_fields  # (registers models M, N: the bridge fields AUG and RES)

# C: A's layers; L: C's plus 32 more inputs of the first layer; G / H: 8 + 3 / 8 + 8 FiLM layers; M (AUG): H's trunk, 7
# wide colour layers and a 6-wide first one; N (RES): 7 + 5 wide layers, the narrow first layers and heads
_W = 2 * 256 * 256
FLOP_PER_POINT = {"A": 1053696, "B": 1341440, "C": 1053696, "L": 1053696 + 2 * 32 * 256,
                  "G": 10 * _W, "H": 15 * _W, "M": 14 * _W, "N": 12 * _W}
CASE = {"A": "a_small", "B": "b_small", "C": "c_small", "L": "l_small", "G": "g_small", "H": "h_small",
        "M": "m_small", "N": "n_small"}
ROWS = [("cfg1", "A", 1, 64, 12), ("cfg1x4", "A", 4, 64, 12), ("cfg2", "A", 4, 128, 24), ("cfg2", "B", 4, 128, 24),
        ("cfg2", "C", 4, 128, 24), ("cfg2", "L", 4, 128, 24), ("cfg2", "G", 4, 128, 24), ("cfg2", "H", 4, 128, 24),
        ("cfg2", "M", 4, 128, 24), ("cfg2", "N", 4, 128, 24),
        ("cfg5", "A", 1, 256, 48), ("cfg5", "B", 1, 256, 48), ("cfg5x8", "A", 8, 256, 48)]

def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="")
    ap.add_argument("--rounds", type=int, default=1)
    args = ap.parse_args()
    dev = "cuda:0"
    print("device: %s" % torch.cuda.get_device_name(dev))
    rows = [r for r in ROWS if not args.models or r[1] in args.models.split(",")]
    for label, model, batch, img, steps in rows * args.rounds:
        case = (_cases.CASE_BY_NAME.get(CASE[model]) or _grid_trunk.CASE_BY_NAME.get(CASE[model])
                or _bridge_fields.CASE_BY_NAME[CASE[model]])
        gen = _cases.build_mirror(case, dev)
        md = dict(_cases.BASE, img_size=img, num_steps=steps, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)
        lat = [torch.randn(batch, 256, device=dev) for _ in range(_cases.n_latents(model))]
        with torch.no_grad():
            for _ in range(3):
                gen(*lat, **md)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 10
            e0.record()
            for _ in range(reps):
                gen(*lat, **md)
            e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        # the same step captured as one CUDA graph (fenerf_b200/graphs.py): what a sampling loop would run
        from fenerf_b200.graphs import GraphedRender
        gr = GraphedRender(gen, lat, md)
        for _ in range(3):
            gr(*lat)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            gr(*lat)
        e1.record(); torch.cuda.synchronize()
        ms_g = e0.elapsed_time(e1) / reps
        pts = batch * img * img * steps * 2
        print("%-7s model %s  B=%d  %dx%d  %d+%d samples/ray: %8.3f ms/step eager, %8.3f as a CUDA graph  %8.1f faces/s (graph)  %6.1f Mpoints/step  %6.1f TFLOP/s (whole step, graph)" % (
            label, model, batch, img, img, steps, steps, ms, ms_g, batch / ms_g * 1e3, pts / 1e6, pts * FLOP_PER_POINT[model] / ms_g / 1e9))

main()
