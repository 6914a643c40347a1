"""Generates the goldens of renders with more than 64 samples per pass (tests/_many_samples.py) by running the UNMODIFIED
reference (a checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_many_samples_goldens.py

  ms_*.npz              forward / staged_forward outputs (make_goldens.py's seed protocol)
  pf_b_vardirs_96.npz   DoubleImplicitGenerator3d.point_forward with the rays it was made from (the draws the reference
                        made are checked against the oracle's restatement, as make_point_forward_goldens.py does)
  grad_ms_b_96.npz      d L / d (latents, _point_forward.GRAD_PARAMS) of forward(); tensors above 8192 entries and the
                        grid as fixed 4096-entry probes
"""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens  # noqa: E402  (puts the repository root and tests/ on sys.path)
import make_point_forward_goldens as mpf  # noqa: E402
import _cases  # noqa: E402
import _many_samples as ms  # noqa: E402
import _point_forward as pf  # noqa: E402
from oracle import ref_shim  # noqa: E402


def forward_goldens(ref_generators, ref_siren):
    for case in ms.CASES:
        gen, digest = make_goldens.build_reference(case, ref_generators, ref_siren)
        latents = _cases.make_latents(case)
        kw = _cases.reference_kwargs(case)
        torch.manual_seed(case.seed)
        random.seed(case.seed)
        with torch.no_grad():
            if case.method == "forward":
                pixels, poses = gen(*latents, **kw)
                extra = {"poses": poses.numpy()}
            else:
                res = gen.staged_forward(*latents, **kw)
                pixels = res[0]
                extra = {"depth_map": res[1].numpy()}
        path = _cases.golden_path(case)
        np.savez_compressed(path, pixels=pixels.numpy(), state_digest=np.array(digest), **extra)
        print("%-26s pixels %s -> %s (%.1f KB)" % (case.name, tuple(pixels.shape), os.path.basename(path),
                                                 os.path.getsize(path) / 1024))


def point_forward_goldens(ref_generators, ref_siren):
    for case in ms.POINT_CASES:
        gen, digest = make_goldens.build_reference(pf.base_case(case), ref_generators, ref_siren)
        latents = _cases.make_latents(pf.base_case(case))
        rays = pf.make_rays(case)
        torch.manual_seed(case.seed)
        with torch.no_grad(), make_goldens._RecordDraws() as rec:
            pixels = mpf._reference_call(gen, case, rays, latents)
        mpf._check_draws(case, rays, rec.log)
        path = pf.golden_path(case)
        np.savez_compressed(path, pixels=pixels.numpy(), state_digest=np.array(digest),
                            **{k: v.numpy() for k, v in rays.items()})
        print("%-26s pixels %s  %d draws -> %s (%.1f KB)" % (case.name, tuple(pixels.shape), len(rec.log),
                                                              os.path.basename(path), os.path.getsize(path) / 1024))


def grad_golden(ref_generators, ref_siren):
    case = ms.CASE_BY_NAME[ms.GRAD_CASE]
    gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
    torch.manual_seed(case.seed)
    pixels, _ = gen(*latents, **case.cfg)
    loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
    loss.backward()
    out = {"loss": np.array(loss.item())}
    out.update({k: v.numpy() for k, v in pf.grad_record(latents, dict(gen.named_parameters())).items()})
    path = ms.grad_golden_path()
    np.savez_compressed(path, **out)
    print("%-26s loss %.6f  %d gradient tensors -> %s (%.1f KB)" % (
        "grad_" + case.name, loss.item(), len(out) - 1, os.path.basename(path), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    ref_generators, ref_siren, _ = ref_shim.load()
    forward_goldens(ref_generators, ref_siren)
    point_forward_goldens(ref_generators, ref_siren)
    grad_golden(ref_generators, ref_siren)
