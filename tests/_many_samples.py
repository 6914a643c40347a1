"""Cases of renders with more than 64 samples per pass (up to the library's 256): their goldens, made by
tests/golden/make_many_samples_goldens.py from the unmodified reference, and their tests (tests/test_many_samples.py).

Same seed protocol as tests/golden/make_goldens.py (camera renders) and tests/_point_forward.py (the rays-in render).
Small images (8² to 16²) keep the reference's CPU run short while every per-ray stage sees the large S.
"""
import os

import _cases
import _point_forward as pf

_cfg = _cases._cfg

CASES = [
    # --ray_step_multiplier 3 and 4 on the production curriculum's 24 steps
    _cases.Case("ms_b_72", "B", 1, 601, _cfg(img_size=12, num_steps=72, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("ms_b_96", "B", 1, 602, _cfg(img_size=10, num_steps=96, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("ms_a_softplus_noise_80", "A", 2, 603, _cfg(img_size=12, num_steps=80, h_stddev=0.3, v_stddev=0.155,
                                                            nerf_noise=0.4, clamp_mode='softplus')),
    _cases.Case("ms_d_staged_softmax_128", "D", 1, 604, _cfg(img_size=10, num_steps=128, h_stddev=0.0, v_stddev=0.0,
                                                             nerf_noise=0.0, softmax_label=True, fill_mode='weight'),
                method="staged_forward", psi=0.7),
    # a feature-head field: 129 channels through the wide compositor, forward and backward
    _cases.Case("ms_k_96", "K", 1, 605, _cfg(img_size=8, num_steps=96, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("ms_a_nohier_256", "A", 1, 606, _cfg(img_size=10, num_steps=256, h_stddev=0.3, v_stddev=0.155,
                                                     nerf_noise=0.0, hierarchical_sample=False, last_back=True)),
    _cases.Case("ms_a_256", "A", 1, 607, _cfg(img_size=8, num_steps=256, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
]
CASE_BY_NAME = {c.name: c for c in CASES}
#: the gradient golden: d L / d (latents, pf.GRAD_PARAMS, grid probe) of forward()
GRAD_CASE = "ms_b_96"

#: the rays-in render at 96 steps, directions varying along each ray
POINT_CASES = [pf.PointCase("pf_b_vardirs_96", "B", 1, 608, img_size=10, num_steps=96, vary_dirs=1.0, cfg=pf._kw())]


def grad_golden_path():
    return os.path.join(_cases.GOLDEN_DIR, "grad_%s.npz" % GRAD_CASE)
