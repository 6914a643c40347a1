"""grad_precision='split' against the exact backward and guard's fp16 backward: one differentiable render + backward at cfg2
(B = 4, 128², 24 + 24 samples per ray) for models A, B and P, gradients to the latents and every field parameter.  Arms:
  split+split   forward precision='split', grad_precision='split'
  split+exact   forward precision='split', the exact backward (what a differentiable split render runs without the keyword)
  guard         forward and backward of precision='guard' (fp16 streams; refused for P)
The arms alternate in one process, --rounds rounds, --reps timed steps each after one warm-up step.  Per arm: ms per step
and the backward's share of it (CUDA events around the forward and around the whole step).  Prints the card, its power
limit and SM clock limit first.

    python tools/bench_split_backward.py [--rounds N] [--reps N] [--models A,B,P]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import _cases  # noqa: E402

CASE = {"A": "a_small", "B": "b_small", "P": "p_small"}
ARMS = {"A": ("split+split", "split+exact", "guard"), "B": ("split+split", "split+exact", "guard"),
        "P": ("split+split", "split+exact")}
BATCH, IMG, STEPS = 4, 128, 24


def _step(gen, md, lat, arm):
    fwd, grad = arm.split("+") if "+" in arm else (arm, None)
    kw = dict(md, precision=fwd)
    if grad == "split":
        kw["grad_precision"] = "split"
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
    return e0.elapsed_time(e2), e1.elapsed_time(e2)


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
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
        lat = [torch.randn(BATCH, 256, generator=g).to(dev).requires_grad_(True) for _ in range(_cases.n_latents(model))]
        setups[model] = (gen, md, lat)
    for r in range(args.rounds):
        for model in args.models.split(","):
            gen, md, lat = setups[model]
            for arm in ARMS[model]:
                _step(gen, md, lat, arm)                                  # warm-up
                times = [_step(gen, md, lat, arm) for _ in range(args.reps)]
                step = sorted(t for t, _ in times)[len(times) // 2]
                bwd = sorted(b for _, b in times)[len(times) // 2]
                print("round %d  model %s  %-12s  cfg2 step %9.2f ms (median of %d)   backward %9.2f ms  (%4.1f %%)" % (
                    r, model, arm, step, args.reps, bwd, 100.0 * bwd / step))
                sys.stdout.flush()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
