"""One process of the ray-gradient reproducibility check (tests/test_ray_grads.py).

Run as ``python tests/_ray_grad_det_child.py OUT.pt`` with CUBLAS_WORKSPACE_CONFIG=:4096:8 in the environment;
torch.use_deterministic_algorithms(True) is switched on before the first render.  Writes the ray gradients of
point_forward(..., ray_grad=True) for a few golden cases and precisions to OUT.pt (CPU tensors).
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import _cases  # noqa: E402
import _point_forward as pf  # noqa: E402
import _ray_grads as rg  # noqa: E402
from fenerf_b200.generators import volumetric_rendering as vr  # noqa: E402

DEV = "cuda:0"
RUNS = [("pf_b_vardirs", "guard"), ("pf_b_vardirs", "exact"), ("pf_b_nohier_lastback", "guard"), ("rg_n_vardirs", "guard"),
        ("rg_b_expand", "guard")]


def main(path):
    torch.use_deterministic_algorithms(True)
    out = {}
    for name, precision in RUNS:
        case, _ = rg.CASES[name]
        rays, _, _ = rg.load_golden(name)
        run = pf.oracle_run(case, {k: v.contiguous() for k, v in rays.items()})
        gen = _cases.build_mirror(pf.base_case(case), DEV)
        leaves, call = rg.leaf_rays(rays, device=DEV)
        px = gen.point_forward(call["points"], call["dirs"], call["origins"], call["ray_dirs"], call["z_vals"],
                               *[z.to(DEV) for z in run["latents"]], ray_grad=True,
                               **dict(pf.call_kwargs(case), precision=precision, _rng=vr.ReplayRng(run["draws"], DEV)))
        (px * _cases.loss_weights(px.shape).to(DEV)).sum().backward()
        for k in rg.RAY_KEYS:
            if leaves[k].grad is not None:
                out["%s/%s/%s" % (name, precision, k)] = leaves[k].grad.cpu()
    torch.save(out, path)


if __name__ == "__main__":
    main(sys.argv[1])
