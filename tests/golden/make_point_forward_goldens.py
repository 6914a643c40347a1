"""Generates tests/golden/pf_*.npz and grad_pf_*.npz by running the UNMODIFIED reference's
DoubleImplicitGenerator3d.point_forward (generators/generators.py:800-856) from a checkout named by
$FENERF_REFERENCE_ROOT.

    python tests/golden/make_point_forward_goldens.py [case names]

Seed protocol: make_goldens.py's for the generator and the latents; the rays of tests/_point_forward.py under
manual_seed(case.seed + 5000); point_forward under manual_seed(case.seed).  Each file stores the rays it was made from
and the reference's pixels; the draws the reference made are checked against the oracle's restatement here, so the
tests replay the oracle's.
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
from make_goldens import _RecordDraws, build_reference  # noqa: E402


def _reference_call(gen, case, rays, latents):
    return gen.point_forward(rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"], rays["z_vals"], *latents,
                             **pf.call_kwargs(case))


def _check_draws(case, rays, log):
    draws = pf.oracle_run(case, rays)["draws"]
    assert len(draws) == len(log) and all(k == kr and torch.equal(t, tr) for (k, t), (kr, tr) in zip(draws, log)), \
        "%s: the oracle's draws are not the reference's" % case.name


def forward_goldens(only):
    ref_generators, ref_siren, _ = ref_shim.load()
    for case in pf.CASES:
        if only and case.name not in only:
            continue
        gen, digest = build_reference(pf.base_case(case), ref_generators, ref_siren)
        latents = _cases.make_latents(pf.base_case(case))
        rays = pf.make_rays(case)
        torch.manual_seed(case.seed)
        with torch.no_grad(), _RecordDraws() as rec:
            pixels = _reference_call(gen, case, rays, latents)
        _check_draws(case, rays, rec.log)
        path = pf.golden_path(case)
        np.savez_compressed(path, pixels=pixels.numpy(), state_digest=np.array(digest),
                            **{k: v.numpy() for k, v in rays.items()})
        print("%-24s pixels %s  %d draws -> %s (%.1f KB)" % (case.name, tuple(pixels.shape), len(rec.log),
                                                              os.path.basename(path), os.path.getsize(path) / 1024))


def grad_golden():
    ref_generators, ref_siren, _ = ref_shim.load()
    case = pf.CASE_BY_NAME[pf.GRAD_CASE]
    gen, _ = build_reference(pf.base_case(case), ref_generators, ref_siren)
    latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(pf.base_case(case)))
    rays = pf.load_rays(case)
    torch.manual_seed(case.seed)
    pixels = _reference_call(gen, case, rays, latents)
    loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
    loss.backward()
    out = {"loss": np.array(loss.item())}
    out.update({k: v.numpy() for k, v in pf.grad_record(latents, dict(gen.named_parameters())).items()})
    path = pf.grad_golden_path()
    np.savez_compressed(path, **out)
    print("%-24s loss %.6f  %d gradient tensors -> %s (%.1f KB)" % (
        "grad_" + case.name, loss.item(), len(out) - 1, os.path.basename(path), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    only = set(sys.argv[1:])
    forward_goldens(only)
    if not only or pf.GRAD_CASE in only:
        grad_golden()
