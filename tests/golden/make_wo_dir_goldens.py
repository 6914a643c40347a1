"""Generates the goldens of the direction-free texture-grid field (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96)
by running the UNMODIFIED reference (a checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_wo_dir_goldens.py [--init | --forward | --grads]      (no flag: all three)

Same seed protocol as tests/golden/make_goldens.py, whose helpers it uses; the cases are tests/_wo_dir_fields.py's.
  <case>.npz         forward / staged_forward outputs (p_cfg2: a fixed probe of the pixels and their abs-sum)
  grad_p_small_opaque.npz      d L / d (latents, _wo_dir_fields.GRAD_PARAMS) of forward()
  gradfreq_p_small_opaque.npz  d L / d (frequencies, phase shifts) through forward_with_frequencies
  wo_dir_init.json   per class, built under torch.manual_seed(0) with the arguments of tests/_wo_dir_fields.py: the
                     state digest (tests/_harness.py), parameter names, state-dict keys and shapes, child names, and the
                     first draw of the RNG after the constructor (the init consumed exactly the reference's draws)
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens  # noqa: E402,F401  (puts the repository root and tests/ on sys.path)
import make_bridge_goldens as MB  # noqa: E402
import _wo_dir_fields as WF  # noqa: E402
from oracle import ref_shim  # noqa: E402

import torch  # noqa: E402


def init_goldens(ref_siren):
    out = {}
    for name in WF.CLASSES:
        torch.manual_seed(0)
        out[name] = MB.describe(getattr(ref_siren, name)(**WF.KWARGS))
    with open(os.path.join(HERE, "wo_dir_init.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print({k: v["digest"][:12] for k, v in out.items()})


class _Cases:
    """The shape make_bridge_goldens' forward / gradient writers read (CASES, PROBED, GRAD_CASES, GRAD_PARAMS)."""
    CASES = WF.CASES
    PROBED = WF.PROBED
    GRAD_CASES = (WF.GRAD_CASE,)
    GRAD_PARAMS = {"P": WF.GRAD_PARAMS}


if __name__ == "__main__":
    ref_generators, ref_siren, _ = ref_shim.load()
    which = sys.argv[1:2]
    MB.BF = _Cases
    if which in ([], ["--init"]):
        init_goldens(ref_siren)
    if which in ([], ["--forward"]):
        MB.forward_goldens(ref_generators, ref_siren)
    if which in ([], ["--grads"]):
        MB.grad_goldens(ref_generators, ref_siren)
