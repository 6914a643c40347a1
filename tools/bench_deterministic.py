"""The cost of torch.use_deterministic_algorithms(True) in the render backward: one differentiable render + backward at cfg2
(B = 4, 128², 24 + 24 samples per ray), gradients to the latents and every parameter, with the flag off and on.
Arms per model: B, L and D in the default precision, B also in precision='split' + grad_precision='split'.  The flag
arms alternate in one process, --rounds rounds of --reps timed steps each after one warm-up step.  Per arm: the median
step, the median backward, and the two stages the flag changes, summed over the step (CUDA events around each call of
_FieldBackward._gate, the column sums, and _FieldBackward._grid_grad, the grid gradient's d feat product and scatter).
Prints the card, its power limit and SM clock limit first.  Set CUBLAS_WORKSPACE_CONFIG=:4096:8 before starting it, as
torch requires for deterministic cuBLAS (it is set here when missing, before any cuBLAS handle exists).

    python tools/bench_deterministic.py [--rounds N] [--reps N] [--models B,L,D]"""
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import _cases  # noqa: E402
from fenerf_b200 import backward  # noqa: E402

CASE = {"B": "b_small", "L": "l_small", "D": "d_small"}
BATCH, IMG, STEPS = 4, 128, 24
_STAGE_EVENTS = {"gate": [], "grid": []}


def _timed(name, fn):
    def wrapper(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*a, **k)
        e1.record()
        _STAGE_EVENTS[name].append((e0, e1))
        return out
    return wrapper


backward._FieldBackward._gate = _timed("gate", backward._FieldBackward._gate)
backward._FieldBackward._grid_grad = _timed("grid", backward._FieldBackward._grid_grad)


def _step(gen, md, lat, arm, mode):
    det = mode != "off"
    kw = dict(md)
    if arm == "split":
        kw.update(precision="split", grad_precision="split")
    for v in _STAGE_EVENTS.values():
        v.clear()
    torch.use_deterministic_algorithms(det)
    torch.utils.deterministic.fill_uninitialized_memory = mode != "on-nofill"
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    for z in lat:
        z.grad = None
    gen.zero_grad(set_to_none=True)
    e0.record()
    pixels, _ = gen(*lat, **kw)
    loss = pixels.square().mean()
    e1.record()
    loss.backward()
    e2.record()
    torch.cuda.synchronize()
    torch.use_deterministic_algorithms(False)
    torch.utils.deterministic.fill_uninitialized_memory = True
    stages = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in _STAGE_EVENTS.items()}
    return e0.elapsed_time(e2), e1.elapsed_time(e2), stages["gate"], stages["grid"]


def _median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--models", default="B,L,D")
    args = ap.parse_args()
    dev = "cuda:0"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device: %s (%s)" % (torch.cuda.get_device_name(dev), q.stdout.strip() or "nvidia-smi unavailable"))
    arms = []
    setups = {}
    for model in args.models.split(","):
        gen = _cases.build_mirror(_cases.CASE_BY_NAME[CASE[model]], dev)
        md = dict(_cases.BASE, img_size=IMG, num_steps=STEPS, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)
        g = torch.Generator().manual_seed(1)
        lat = [torch.randn(BATCH, 256, generator=g).to(dev).requires_grad_(True) for _ in range(_cases.n_latents(model))]
        setups[model] = (gen, md, lat)
        arms += [(model, "default")] + ([(model, "split")] if model == "B" else [])
    for r in range(args.rounds):
        for model, arm in arms:
            gen, md, lat = setups[model]
            res = {}
            modes = ("off", "on", "on-nofill")
            for mode in modes:
                _step(gen, md, lat, arm, mode)                                 # warm-up
            runs = {m: [] for m in modes}
            for _ in range(args.reps):                                        # the flag arms alternating
                for mode in modes:
                    runs[mode].append(_step(gen, md, lat, arm, mode))
            for mode in modes:
                t = runs[mode]
                res[mode] = [_median([x[i] for x in t]) for i in range(4)]
                print("round %d  model %s  %-7s  flag %-9s  cfg2 step %8.2f ms  backward %8.2f ms  column sums %6.2f ms  "
                      "grid gradient %6.2f ms  (medians of %d)" % (r, model, arm, mode, *res[mode], args.reps))
            for mode in modes[1:]:
                print("round %d  model %s  %-7s  %-9s - off: step %+7.2f ms (%+.1f %%)" % (
                    r, model, arm, mode, res[mode][0] - res["off"][0], 100.0 * (res[mode][0] / res["off"][0] - 1)))
            sys.stdout.flush()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
