"""The oracle against the unmodified reference on the same inputs.  With a reference checkout
($FENERF_REFERENCE_ROOT) the reference runs live and the match must be bit-exact; without one the
reference's stored outputs (tests/golden/*.npz, made by tests/golden/make_goldens.py) stand in for it, at
the cross-host tolerance of test_oracle.py (the goldens' host may round sgemm / vectorised sums differently).
That fallback overlaps test_oracle.py::test_oracle_matches_reference_golden on these cases; the bit-exact
comparison needs the live reference."""
import numpy as np
import pytest
import torch

import _cases
import _harness
from oracle import ref_shim

TOL = 2e-5


@pytest.mark.parametrize("name", ["a_small", "a_small_noise", "a_nohier_softplus", "a_lockview_uniform", "b_small", "c_small", "d_small",
                                  "a_hier_softplus", "b_noise_b2", "a_cam_hybrid", "a_cam_hybrid2", "a_cam_truncgauss",
                                  "a_cam_spherical", "s_small", "f_small", "g_small", "h_small"])
def test_oracle_is_bit_exact_with_reference(name):
    import sys
    sys.path.insert(0, _cases.GOLDEN_DIR)
    import make_goldens
    case = _cases.CASE_BY_NAME[name]
    run = _harness.oracle_run(case, keep_stages=False)
    if not ref_shim.available():
        gold = np.load(_cases.golden_path(case))
        assert np.abs(run["out"]["pixels"].numpy() - gold["pixels"]).max() <= TOL
        assert np.abs(run["out"]["poses"].numpy() - gold["poses"]).max() <= 1e-6
        return
    ref_generators, ref_siren, _ = ref_shim.load()
    gen_ref, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    latents = _cases.make_latents(case)
    torch.manual_seed(case.seed)
    import random
    random.seed(case.seed)
    with torch.no_grad():
        px_ref, poses_ref = gen_ref(*latents, **_cases.reference_kwargs(case))
    assert torch.equal(run["out"]["pixels"], px_ref), float((run["out"]["pixels"] - px_ref).abs().max())
    assert torch.equal(run["out"]["poses"], poses_ref)
