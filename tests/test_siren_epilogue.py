"""The FiLM epilogue of the fast point network: the software sine and the folded FiLM entries.

  - soft_sinf (csrc/siren_fast.cuh), restated in float32 on the CPU and evaluated on the device, against float64 sin
    over every argument range the epilogue sees: |a| up to 4096 rad, dense near multiples of pi / 2 and near the points
    where the rounding of n = rint(a / 2pi) changes;
  - the folded FiLM entries {f, f b + p} of the production kernel (every sine on the SFU) give the same bits as the
    kernel that evaluated f b + p in its epilogue: the SHA-256 of its outputs, fixture fast_fold_sha256.json (models A,
    B, I, J, K, recorded on an H100 80GB HBM3);
  - the kernel with one column pair in four on soft_sinf (fenerf_debug_fast_variant 1) stays within the fast bound
    against float64.
"""
import ctypes
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

import _cases
from _fp64 import _film, _siren, field_ref
from test_gpu_fp64_reference import FWD_BOUND, _forward_inputs, _per_point

DEV = "cuda:0"
gpu = pytest.mark.gpu
SINE_BOUND = 2.0 ** -20
FOLD_MODELS = ("A", "B", "I", "J", "K")
FOLD_GOLDEN = os.path.join(_cases.GOLDEN_DIR, "fast_fold_sha256.json")
# Measured on an H100 80GB HBM3: max |soft_sinf(a) - sin(a)| over the sweep 4.83e-7, the float32 restatement and the
# device bit-equal.

# the constants of soft_sinf, in its order of evaluation
_INV_2PI, _MAGIC, _TWO_PI_HI, _TWO_PI_LO = 0.159154943, 12582912.0, 6.28318548, -1.74845553e-7
_POLY = (-2.041572245e-08, 2.701100129e-06, -1.980991656e-04, 8.332454599e-03, -1.666656137e-01, 9.999996424e-01)


def _fma(a, b, c):
    """float32 fused multiply-add: the float64 product of two float32 values is exact; one rounding to float32 after
    the add (a float64 rounding in between only matters at exact float32 ties)."""
    f64 = lambda x: np.asarray(x, np.float32).astype(np.float64)
    return (f64(a) * f64(b) + f64(c)).astype(np.float32)


def soft_sin_f32(a):
    a = np.asarray(a, np.float32)
    k = _fma(a, np.float32(_INV_2PI), np.float32(_MAGIC))
    n = (k - np.float32(_MAGIC)).astype(np.float32)
    r = _fma(-n, np.float32(_TWO_PI_HI), a)
    r = _fma(-n, np.float32(_TWO_PI_LO), r)
    r2 = (r * r).astype(np.float32)
    p = np.full_like(r, np.float32(_POLY[0]))
    for c in _POLY[1:]:
        p = _fma(p, r2, np.float32(c))
    return (r * p).astype(np.float32)


def sine_sweep():
    """float32 arguments: uniform over |a| <= 4096, dense around k pi / 2 and around (m + 1/2) 2 pi (where n steps) for
    |a| up to 4096, and the float32 neighbours of each such point."""
    g = np.random.default_rng(7)
    parts = [g.uniform(-4096, 4096, 400_000), np.linspace(-8 * math.pi, 8 * math.pi, 200_001)]
    k = np.arange(-2608, 2609)                               # k pi / 2 up to 4096
    parts.append((k[:, None] * (math.pi / 2) + np.linspace(-1e-3, 1e-3, 21)[None, :]).ravel())
    m = np.arange(-652, 652)                                 # (m + 1/2) 2 pi up to 4096
    parts.append(((m[:, None] + 0.5) * (2 * math.pi) + np.linspace(-1e-3, 1e-3, 21)[None, :]).ravel())
    a = np.concatenate(parts).astype(np.float32)
    ups = np.nextafter(a, np.float32(np.inf)).astype(np.float32)
    downs = np.nextafter(a, np.float32(-np.inf)).astype(np.float32)
    return np.concatenate([a, ups, downs])


def _sine_error(got, a):
    return float(np.abs(got.astype(np.float64) - np.sin(a.astype(np.float64))).max())


def test_soft_sine_f32_within_bound():
    a = sine_sweep()
    err = _sine_error(soft_sin_f32(a), a)
    print("soft_sinf, float32 restatement: max |err| %.3g over %d arguments" % (err, a.size))
    assert err <= SINE_BOUND


def test_soft_sine_sweep_reaches_the_rounding_boundaries():
    """The sweep puts arguments on both sides of each step of n (the reduced argument sits at +-pi there)."""
    a = sine_sweep().astype(np.float64)
    n = np.rint(a / (2 * math.pi))
    r = a - n * 2 * math.pi
    assert np.abs(r).max() >= math.pi - 1e-6
    assert np.abs(a).max() >= 4090


# --------------------------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------------------------
def _lib():
    from fenerf_b200 import _lib as L
    return L


class _Variant:
    """fenerf_debug_fast_variant for the body of a with block; always back to the production kernel."""

    def __init__(self, variant, trace=None, ctas=0):
        self.args = (variant, ctypes.c_void_p(trace.data_ptr() if trace is not None else 0), ctas)

    def __enter__(self):
        L = _lib()
        L.check(L.lib().fenerf_debug_fast_variant(*self.args))

    def __exit__(self, *exc):
        L = _lib()
        L.check(L.lib().fenerf_debug_fast_variant(0, None, 0))


def fold_inputs(model, points=256):
    """A fixed small forward of the fast point network: 1 image, `points` points, one direction each."""
    siren = _siren(model, DEV)
    g = torch.Generator().manual_seed(500 + FOLD_MODELS.index(model))
    pts = ((torch.rand(1, points, 3, generator=g) - 0.5) * 0.24).to(DEV)
    dirs = torch.nn.functional.normalize(torch.randn(1, points, 3, generator=g), dim=-1).to(DEV)
    return siren, pts, dirs, _film(siren, 1, 600 + FOLD_MODELS.index(model))


def fold_outputs(model):
    from fenerf_b200 import ops
    siren, pts, dirs, film = fold_inputs(model)
    with torch.no_grad():
        return ops.siren_points(siren, pts, film, dirs, precision="fast")


@gpu
def test_soft_sine_device_within_bound():
    L = _lib()
    a = sine_sweep()
    ta = torch.from_numpy(a).to(DEV)
    out = torch.empty_like(ta)
    L.check(L.lib().fenerf_debug_soft_sine(ctypes.c_void_p(ta.data_ptr()), ctypes.c_void_p(out.data_ptr()), a.size, None))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    err = _sine_error(got, a)
    print("soft_sinf, device: max |err| %.3g; max |device - float32 restatement| %.3g" % (
        err, float(np.abs(got - soft_sin_f32(a)).max())))
    assert err <= SINE_BOUND


@gpu
@pytest.mark.parametrize("model", FOLD_MODELS)
def test_film_fold_is_bit_identical(model):
    """The folded entries {f, f b + p} give exactly the outputs of the unfolded epilogue."""
    with open(FOLD_GOLDEN) as f:
        want = json.load(f)[model]
    got = np.ascontiguousarray(fold_outputs(model).cpu().numpy(), np.float32)
    assert list(got.shape) == want["shape"]
    assert hashlib.sha256(got.tobytes()).hexdigest() == want["sha256"]


@gpu
@pytest.mark.parametrize("layout", _cases.TILE_LAYOUTS)
@pytest.mark.parametrize("model", ("A", "B", "C", "D", "H"))
def test_soft_sine_split_within_fast_bound(model, layout):
    """One column pair in four on soft_sinf (variant 1) and the production kernel against float64, per output channel."""
    from fenerf_b200 import ops
    siren = _siren(model, DEV)
    pts, dirs, film = _forward_inputs(siren, layout, 2000 + ("A", "B", "C", "D", "E", "F", "G", "H", "D32").index(model))
    with torch.no_grad():
        sfu = ops.siren_points(siren, pts, film, dirs, precision="fast")
        with _Variant(1):
            fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
    want = field_ref(siren, pts, _per_point(dirs, pts.shape[1], False), film)[0]
    err = (fast.double() - want).abs().amax((0, 1)).max().item()
    err_sfu = (sfu.double() - want).abs().amax((0, 1)).max().item()
    print("split %s %s: soft split %.3g, all-SFU %.3g, max |split - all-SFU| %.3g" % (
        model, layout, err, err_sfu, (fast - sfu).abs().max().item()))
    assert torch.isfinite(fast).all()
    assert err <= FWD_BOUND["fast"]
