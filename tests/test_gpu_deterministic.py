"""torch.use_deterministic_algorithms(True) in the render backward: bitwise-reproducible gradients.

Every check runs in child processes (tests/_det_child.py) started with CUBLAS_WORKSPACE_CONFIG=:4096:8 and the flag set,
so the cuBLAS setting is in force before any handle exists and "run to run" means two fresh processes:
  - models A, B, D, L, P in the default, exact and split + grad_precision='split' modes, the cfg2 shape and two more
    chunk layouts of the backward, point_forward and part_forward: every gradient (latents, d film, every parameter, the
    grid included) equal between two processes
  - three Adam steps of model B at a training shape under autocast with GradScaler: the same parameters twice
  - in one process: the camera render's gradients equal those of its own rays fed back; a loss scaled by 2^k gives
    gradients exactly 2^k times; the flag-off path launches none of the deterministic kernels and differs from the
    flag-on path by no more than 2e-6 of each tensor's largest entry (its atomics' run-to-run spread is printed); an inf
    or a NaN upstream makes the same grid entries and the same gradients non-finite as the flag-off path
"""
import os
import subprocess
import sys

import pytest
import torch

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _child(out_dir, suite, tag):
    out = os.path.join(str(out_dir), "%s_%s.pt" % (suite, tag))
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(HERE, "_det_child.py"), out, suite]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, "%s child failed:\n%s\n%s" % (suite, r.stdout[-4000:], r.stderr[-8000:])
    return torch.load(out, weights_only=False)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("det")
    return {"repro": (_child(d, "repro", "a"), _child(d, "repro", "b")),
            "train": (_child(d, "train", "a"), _child(d, "train", "b")),
            "checks": _child(d, "checks", "a")}


@gpu
def test_gradients_are_equal_between_two_processes(runs):
    a, b = runs["repro"]
    assert sorted(a) == sorted(b) and len(a) >= 20
    for name in a:
        assert len(a[name]) == len(b[name]), name
        assert any(t.abs().max().item() > 0 for t in a[name][:3]), name       # latents / d film carry a gradient
        for i, (x, y) in enumerate(zip(a[name], b[name])):
            assert torch.equal(x, y), "%s: tensor %d of %d differs by %g" % (name, i, len(a[name]), (x - y).abs().max().item())


@gpu
def test_three_training_steps_give_the_same_parameters(runs):
    a, b = runs["train"]
    assert len(a["params"]) == len(b["params"]) > 10
    for i, (x, y) in enumerate(zip(a["params"], b["params"])):
        assert torch.equal(x, y), "parameter %d differs by %g" % (i, (x - y).abs().max().item())


def _checks(runs, prefix):
    got = {k[len(prefix):]: v for k, v in runs["checks"].items() if k.startswith(prefix)}
    assert got, prefix
    return got


@gpu
def test_camera_render_gradients_equal_its_rays_bit_for_bit(runs):
    for precision, equal in _checks(runs, "camera_vs_rays/").items():
        assert equal is True, precision


@gpu
def test_power_of_two_loss_scales_give_exactly_scaled_gradients(runs):
    for case, exact in _checks(runs, "pow2/").items():
        assert exact is True, case


@gpu
def test_flag_off_launches_no_deterministic_kernel(runs):
    off = _checks(runs, "off_det_launches/")
    on = _checks(runs, "on_det_launches/")
    assert all(n == 0 for n in off.values()), off
    assert all(n > 0 for n in on.values()), on


@gpu
def test_deterministic_gradients_are_within_the_atomics_spread_of_the_flag_off_path(runs):
    """Largest difference relative to each tensor's largest entry; the flag-off path's own run-to-run spread is printed
    beside it.  Measured on an H100 80GB HBM3 (700 W): 5.8e-10 (L) ... 1.24e-6 (P exact), against a flag-off spread of up
    to 1.36e-6 (B split) in the same run."""
    for case, (worst, spread) in _checks(runs, "vs_off/").items():
        print("%s: %.2e of each tensor's largest entry (flag off against itself: %.2e)" % (case, worst, spread))
        assert worst <= 2e-6, (case, worst, spread)


@gpu
def test_non_finite_upstream_gradients_reach_the_same_entries(runs):
    for case, same in _checks(runs, "nonfinite_same/").items():
        assert same is True, case
    for case, (same_tensors, grid, film, n_bad, n) in _checks(runs, "nonfinite_reaches/").items():
        print("%s: %d of %d gradients non-finite" % (case, n_bad, n))
        assert same_tensors and grid and film, case
