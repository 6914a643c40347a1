"""Timeline of the fast point network (siren_fast_kernel) from clock64 stamps of the traced instantiation.

    python tools/siren_timeline.py [--models A,B] [--ctas 8] [--json OUT]

Runs one cfg2 coarse launch (batch 4, 128^2 rays x 24 samples, bench.py's field and latents) of the traced production
kernel (every sine on the SFU) and of the traced kernel with one column pair in four on the software sine
(fenerf_debug_fast_variant 2 / 3), lane 0 of every warp of the first --ctas
CTAs recording {event, clock64} (csrc/siren_fast.cuh, TraceEvent).  Per variant it reports, over those CTAs:

  tensor idle   share of clocks between a CTA's first MMA issue and its last MMA completion in which no consumer
                warpgroup has an MMA group in flight (its turn taken, its wg_wait not yet returned)
  per group     MMA group duration (its completion minus the later of its turn and the other warpgroups' latest
                completion before it) and the epilogue after it (wg_wait returned -> FiLM epilogue done), median / p90
                clocks
  waits         consumer clocks in turn waits, weight-slot waits (acquire) and FiLM-entry waits, as shares of the
                window; the producers' empty-slot waits

Clock stamps cost a few instructions each; the traced kernels run slightly slower than the production ones.
"""
import argparse
import bisect
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from fenerf_b200 import _lib, ops  # noqa: E402
from fenerf_b200.generators import volumetric_rendering as vr  # noqa: E402

WARPS, CAP = 16, 1024
CONSUMER_WGS = 3                      # warps 0..11; warp 12 streams the weights, warps 13..15 fold the FiLM rows
WEIGHT_WARP = 4 * CONSUMER_WGS
(PAIR, TURN_WAIT, TURN_DONE, ACQ_WAIT, ACQ_DONE, COMMIT, MMA_DONE, EPI_DONE, FILM_WAIT, FILM_DONE, EMPTY_WAIT,
 EMPTY_DONE) = range(1, 13)
GROUPS = ["first", "hidden", "color0", "trunk_head", "label_layer", "label_head", "out_head"]
VARIANTS = {"production": 2, "soft_sine_split": 3}


def coarse_inputs(model, dev):
    gen = bench.build_generator(model, dev)
    lat = [z.to(dev) for z in bench.make_latents(model, 1, bench.BATCH_PER_GPU)[0]]
    md = bench.metadata()
    B, S, R = bench.BATCH_PER_GPU, md["num_steps"], md["img_size"]
    with torch.no_grad():
        if model == "A":
            film = gen.siren.film_table(*gen.siren.mapping_network(lat[0]))
        else:
            fg, pg = gen.siren.geo_mapping_network(lat[0]); fa, pa = gen.siren.app_mapping_network(lat[1])
            film = gen.siren.film_table(fg, fa, pg, pa)
        rd = ops.make_render_desc(batch=B, img_size=R, num_steps=S, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                                  fov=md["fov"], precision="fast")
        x_lin, y_lin, z_lin = vr.ray_tables(R, S, md["ray_start"], md["ray_end"], dev)
        c2w, _, _ = ops.camera_poses(B, "gaussian", 0.3, 0.155, md["h_mean"], md["v_mean"], vr.DeviceRng(dev), dev)
        pts, _, dirs, _ = ops.ray_setup(rd, x_lin, y_lin, z_lin, c2w, torch.rand(B, R * R, S, 1, device=dev))
    return gen.siren, pts.reshape(B, R * R * S, 3), film, dirs


def run_traced(siren, pts, film, dirs, variant, ctas):
    lib = _lib.lib()
    trace = torch.zeros(ctas * WARPS * CAP, dtype=torch.int64, device=pts.device)
    with torch.no_grad():
        ops.siren_points(siren, pts, film, dirs, precision="fast")            # warm
        _lib.check(lib.fenerf_debug_fast_variant(variant, ctypes.c_void_p(trace.data_ptr()), ctas))
        try:
            ops.siren_points(siren, pts, film, dirs, precision="fast")
            torch.cuda.synchronize()
        finally:
            _lib.check(lib.fenerf_debug_fast_variant(0, None, 0))
    return trace.cpu().numpy().view(np.uint64).reshape(ctas, WARPS, CAP)


def decode(words):
    words = words[words != 0]
    return [(int(w >> np.uint64(56)), int((w >> np.uint64(48)) & np.uint64(0xFF)), int(w & np.uint64((1 << 48) - 1)))
            for w in words]


def consumer_groups(ev):
    """[(group, issue, done, epilogue_done or None)] of one consumer warp, in order; a group's MMAs are issued from its
    turn on (the weight-slot acquires of the group come between its first wgmma and the commit)."""
    out, cur, turn = [], None, None
    for kind, grp, t in ev:
        if kind == TURN_DONE:
            turn = t
        elif kind == COMMIT:
            cur = [grp, turn if turn is not None else t, None, None]
        elif kind == MMA_DONE and cur is not None:
            cur[2] = t
            out.append(cur)
        elif kind == EPI_DONE and out and out[-1][3] is None:
            out[-1][3] = t
        elif kind in (TURN_WAIT, PAIR):
            cur, turn = None, None
    return out


def wait_clocks(ev, begin, end):
    total, t0 = 0, None
    for kind, _, t in ev:
        if kind == begin:
            t0 = t
        elif kind == end and t0 is not None:
            total += t - t0
            t0 = None
    return total


def analyse(buf):
    idle, window = 0, 0
    mma, epi = {}, {}
    waits = {"turn": 0, "weight_slot": 0, "film_entry": 0}
    consumer_clocks = 0
    producer = {"weight_empty": 0, "film_empty": 0}
    producer_clocks = 0
    for cta in range(buf.shape[0]):
        evs = [decode(buf[cta, w]) for w in range(WARPS)]
        if any(not evs[4 * g] for g in range(CONSUMER_WGS)):
            continue
        # warp 4 g stands for warpgroup g (all four warps of a warpgroup wait for the same MMA group)
        wgs = [consumer_groups(evs[4 * g]) for g in range(CONSUMER_WGS)]
        ivs = sorted([(c, d) for groups in wgs for _, c, d, _ in groups])
        lo, hi = ivs[0][0], max(d for _, d in ivs)
        busy, cur_s, cur_e = 0, None, None
        for s, e in ivs:
            if cur_e is None or s > cur_e:
                if cur_e is not None:
                    busy += cur_e - cur_s
                cur_s, cur_e = s, e
            else:
                cur_e = max(cur_e, e)
        busy += cur_e - cur_s
        idle += (hi - lo) - busy
        window += hi - lo
        for wg, groups in enumerate(wgs):
            done_other = sorted(d for o, other in enumerate(wgs) if o != wg for _, _, d, _ in other)
            for grp, c, d, e in groups:
                i = bisect.bisect_right(done_other, d)
                start = max(c, done_other[i - 1]) if i else c
                mma.setdefault(GROUPS[grp], []).append(d - start)
                if e is not None:
                    epi.setdefault(GROUPS[grp], []).append(e - d)
        for w in range(WEIGHT_WARP):
            ev = evs[w]
            if not ev:
                continue
            consumer_clocks += ev[-1][2] - ev[0][2]
            waits["turn"] += wait_clocks(ev, TURN_WAIT, TURN_DONE)
            waits["weight_slot"] += wait_clocks(ev, ACQ_WAIT, ACQ_DONE)
            waits["film_entry"] += wait_clocks(ev, FILM_WAIT, FILM_DONE)
        for w, key in [(WEIGHT_WARP, "weight_empty")] + [(WEIGHT_WARP + 1 + g, "film_empty") for g in range(CONSUMER_WGS)]:
            ev = evs[w]
            if ev:
                producer_clocks += ev[-1][2] - ev[0][2]
                producer[key] += wait_clocks(ev, EMPTY_WAIT, EMPTY_DONE)
    q = lambda v, p: float(np.percentile(v, p)) if v else None
    return {
        "tensor_idle_share": idle / window if window else None,
        "window_clocks_per_cta": window / max(1, buf.shape[0]),
        "groups": {g: {"n": len(mma[g]), "mma_median": q(mma[g], 50), "mma_p90": q(mma[g], 90),
                       "epilogue_median": q(epi.get(g, []), 50), "epilogue_p90": q(epi.get(g, []), 90)} for g in mma},
        "consumer_wait_share": {k: v / consumer_clocks for k, v in waits.items()} if consumer_clocks else None,
        "producer_wait_share": {k: v / producer_clocks for k, v in producer.items()} if producer_clocks else None,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="A,B")
    ap.add_argument("--ctas", type=int, default=8)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    report = {"device": torch.cuda.get_device_name(dev)}
    for model in args.models.split(","):
        siren, pts, film, dirs = coarse_inputs(model, dev)
        for name, variant in VARIANTS.items():
            r = analyse(run_traced(siren, pts, film, dirs, variant, args.ctas))
            report["%s/%s" % (model, name)] = r
            print("model %s, %s kernel: tensor idle %.1f %% of %.0f clocks per CTA" % (
                model, name, 100 * r["tensor_idle_share"], r["window_clocks_per_cta"]))
            for g, s in r["groups"].items():
                print("  %-12s n %5d  MMA median %6.0f p90 %6.0f   epilogue median %s p90 %s" % (
                    g, s["n"], s["mma_median"], s["mma_p90"],
                    "%6.0f" % s["epilogue_median"] if s["epilogue_median"] is not None else "     -",
                    "%6.0f" % s["epilogue_p90"] if s["epilogue_p90"] is not None else "     -"))
            print("  consumer waits: " + ", ".join("%s %.1f %%" % (k, 100 * v) for k, v in r["consumer_wait_share"].items()))
            print("  producer waits: " + ", ".join("%s %.1f %%" % (k, 100 * v) for k, v in r["producer_wait_share"].items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
