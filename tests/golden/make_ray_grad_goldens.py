"""Generates tests/golden/grad_rays_*.npz by differentiating the UNMODIFIED reference's
DoubleImplicitGenerator3d.point_forward (generators/generators.py:800-856) w.r.t. its ray tensors, from a checkout named
by $FENERF_REFERENCE_ROOT.

    python tests/golden/make_ray_grad_goldens.py [case names]

Seed protocol: make_point_forward_goldens.py's.  Every ray tensor (points, directions -- the per-ray leaf of an expand()
--, origins, ray directions, z_vals) and every latent requires grad; the loss is sum(pixels * _cases.loss_weights).  Each
file stores the rays, the loss, each ray tensor's gradient or its absence ('none_<name>': the reference left .grad None),
the latents' gradients and a probe of every parameter gradient.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import ref_shim  # noqa: E402
import _cases  # noqa: E402
import _point_forward as pf  # noqa: E402
import _ray_grads as rg  # noqa: E402
from make_goldens import _RecordDraws, build_reference  # noqa: E402


def main(only):
    ref_generators, ref_siren, _ = ref_shim.load()
    for name, (case, expand) in rg.CASES.items():
        if only and name not in only:
            continue
        gen, _ = build_reference(pf.base_case(case), ref_generators, ref_siren)
        latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(pf.base_case(case)))
        rays = rg.make_rays(name)
        leaves, call = rg.leaf_rays(rays)
        torch.manual_seed(case.seed)
        with _RecordDraws() as rec:
            pixels = gen.point_forward(call["points"], call["dirs"], call["origins"], call["ray_dirs"], call["z_vals"],
                                       *latents, **pf.call_kwargs(case))
        draws = pf.oracle_run(case, {k: v.contiguous() for k, v in rays.items()})["draws"]
        assert len(draws) == len(rec.log) and all(k == kr and torch.equal(t, tr) for (k, t), (kr, tr) in zip(draws, rec.log)), \
            "%s: the oracle's draws are not the reference's" % name
        loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
        loss.backward()
        out = {"loss": np.array(loss.item()), "expand": np.array(expand)}
        for k in rg.RAY_KEYS:
            out["ray_" + k] = (rays["ray_dirs"] if (k == "dirs" and expand) else rays[k]).detach().contiguous().numpy()
            if leaves[k].grad is None:
                out["none_" + k] = np.array(True)
            else:
                out["grad_" + k] = leaves[k].grad.numpy()
        for i, z in enumerate(latents):
            out["latent%d" % i] = z.grad.numpy()
        for pname, prm in gen.named_parameters():
            if prm.grad is not None:
                out["param_" + pname] = rg.probe(prm.grad).numpy()
        path = rg.golden_path(name)
        np.savez_compressed(path, **out)
        print("%-22s loss %.6f  ray grads: %s -> %s (%.1f KB)" % (
            name, loss.item(), " ".join(k for k in rg.RAY_KEYS if leaves[k].grad is not None), os.path.basename(path),
            os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main(set(sys.argv[1:]))
