"""256^3 density grid through the point network (extract_double_semantic_shapes.py:59-62 workload):
density-only entry vs the full evaluation, for both benchmarked models, SPATIALSIRENBASELINE (C) and the grid-trunk
EmbeddingPiGAN256 (L), whose density needs the grid, and the bridge fields AUG (M, against H) and RES (N, whose
density comes from v; against G).  Prints one line per run.

    python tools/bench_density.py [res] [--models C,L] [--rounds N]     (--rounds: the models N times, alternating)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import _cases
import _grid_trunk  # (registers model L)
import _bridge_fields  # (registers models M, N: the bridge fields AUG and RES)
from fenerf_b200 import ops

CASE = {"A": "a_small", "B": "b_small", "C": "c_small", "L": "l_small", "G": "g_small", "H": "h_small",
        "M": "m_small", "N": "n_small"}

def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("res", type=int, nargs="?", default=256)
    ap.add_argument("--models", default="A,B,C,L")
    ap.add_argument("--rounds", type=int, default=1)
    args = ap.parse_args()
    res = args.res
    print("device: %s" % torch.cuda.get_device_name("cuda:0"))
    for model in args.models.split(",") * args.rounds:
        case = (_cases.CASE_BY_NAME.get(CASE[model]) or _grid_trunk.CASE_BY_NAME.get(CASE[model])
                or _bridge_fields.CASE_BY_NAME[CASE[model]])
        gen = _cases.build_mirror(case, "cuda:0")
        lin = torch.linspace(-0.15, 0.15, res, device="cuda")
        pts = torch.stack(torch.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(1, -1, 3).contiguous()
        dirs = torch.zeros(1, 1, 3, device="cuda"); dirs[..., -1] = -1
        with torch.no_grad():
            if _cases.n_latents(model) == 1:
                film = gen.siren.film_table(*gen.siren.mapping_network(torch.randn(1, 256, device="cuda")))
            else:
                fg, pg = gen.siren.geo_mapping_network(torch.randn(1, 256, device="cuda"))
                fa, pa = gen.siren.app_mapping_network(torch.randn(1, 256, device="cuda"))
                film = gen.siren.film_table(fg, fa, pg, pa)
            for name, fn in (("density-only", lambda: ops.siren_sigma(gen.siren, pts, film, precision="fast")),
                             ("full", lambda: ops.siren_points(gen.siren, pts, film, dirs, precision="fast", dir_group=pts.shape[1]))):
                fn(); torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(3):
                    fn()
                e1.record(); torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / 3
                print("model %s  %d^3 = %d points  %-12s %.2f ms  %.1f Mpoints/s" % (model, res, pts.shape[1], name, ms, pts.shape[1] / ms / 1e3))

main()
