"""The deterministic backward's fixed-point grid scatter restated on the CPU, and the C-ABI's refusals of its entries.

The restatement follows csrc/backward_det.cu: per point set of P points, s = 62 - ceil(log2(amax P)) with amax the
largest finite |d feat|; each trilinear contribution w d (exact in float64) rounded to the nearest integer at 2^s and
summed in int64; NaN / +inf / -inf contributions recorded as flags.  Checked: the integers do not depend on the point
order, every entry is within n_v 2^-(s+1) of the exact sum (n_v: the contributions it receives) and that bound is below
the error of an fp32 scatter of the same data in a shuffled order, the non-finite rules, and no int64 overflow at the
largest |d feat| a point set can hold.
"""
import ctypes as C
import math

import numpy as np
import pytest

from fenerf_b200 import _lib

R = 6
NAN, POS, NEG = 1, 2, 4


def _trilinear(points, r):
    """Corner voxels (P, 8) (-1 outside) and weights (P, 8) float32, rounded as csrc/siren_common.cuh's trilinear()."""
    f32 = np.float32
    half = f32(r - 1)
    i = ((points.astype(f32) + f32(1)) * f32(0.5)) * half
    i0 = np.floor(i)
    w1 = (i - i0).astype(f32)
    w0 = ((i0 + f32(1)) - i).astype(f32)
    base = i0.astype(np.int64)
    vox, wts = [], []
    for k in range(8):
        d = np.array([k & 1, (k >> 1) & 1, k >> 2])
        c = base + d
        inside = np.all((c >= 0) & (c < r), axis=1)
        w = (np.where(d[0], w1[:, 0], w0[:, 0]) * np.where(d[1], w1[:, 1], w0[:, 1])).astype(f32)
        w = (w * np.where(d[2], w1[:, 2], w0[:, 2])).astype(f32)
        vox.append(np.where(inside, (c[:, 2] * r + c[:, 1]) * r + c[:, 0], -1))
        wts.append(w)
    return np.stack(vox, 1), np.stack(wts, 1)


def _contributions(points, d_feat, r):
    """(entry index, w d in float64) of every contribution, in point order."""
    vox, w = _trilinear(points, r)
    g = d_feat.shape[1]
    ent = (vox[:, :, None] * g + np.arange(g)[None, None, :])                      # (P, 8, G)
    val = w.astype(np.float64)[:, :, None] * d_feat.astype(np.float64)[:, None, :]
    keep = np.broadcast_to(vox[:, :, None] >= 0, ent.shape)
    return ent[keep], val[keep]


def fixed_exponent(amax, n_points):
    if not amax > 0:
        return 0
    m, e = math.frexp(float(amax) * float(n_points))
    return int(min(960, max(-960, 62 - (e - 1 if m == 0.5 else e))))


def fixed_scatter(points, d_feat, r, order=None):
    """int64 sums (R^3 * G), flags and s of one point set; `order` permutes the contributions before they are added."""
    d = d_feat.astype(np.float32)
    fin = np.isfinite(d)
    amax = float(np.abs(d[fin]).max()) if fin.any() else 0.0
    s = fixed_exponent(amax, len(points))
    ent, val = _contributions(points, d, r)
    if order is not None:
        p = order(len(ent))
        ent, val = ent[p], val[p]
    n = r ** 3 * d.shape[1]
    acc = np.zeros(n, dtype=np.int64)
    flags = np.zeros(n, dtype=np.int64)
    ok = np.isfinite(val)
    q = np.rint(np.ldexp(val[ok], s)).astype(np.int64)                               # round half to even, as __double2ll_rn
    np.add.at(acc, ent[ok], q)
    bad = ~ok
    code = np.where(np.isnan(val[bad]), NAN, np.where(val[bad] > 0, POS, NEG))
    np.bitwise_or.at(flags, ent[bad], code)
    return acc, flags, s


def convert(acc, flags, s):
    """The convert pass: the float each entry adds to the fp32 accumulator."""
    v = np.ldexp(acc.astype(np.float64), -s).astype(np.float32)
    both = (flags & (POS | NEG)) == (POS | NEG)
    v = np.where((flags & NAN) != 0, np.nan, v)
    v = np.where(both, np.nan, v)
    v = np.where(~both & ((flags & NAN) == 0) & ((flags & POS) != 0), np.inf, v)
    v = np.where(~both & ((flags & NAN) == 0) & ((flags & NEG) != 0), -np.inf, v)
    return v.astype(np.float32)


def _data(seed, n=3000, g=32, spread=1.0):
    rng = np.random.default_rng(seed)
    # rays' samples crowd a few voxels, as a render's do; a few points outside the grid
    centre = rng.uniform(-0.7, 0.7, size=(n // 30, 3)).repeat(30, axis=0)
    pts = (centre + rng.normal(scale=0.05, size=centre.shape)).astype(np.float32)
    pts[:10] = 1.3
    d = (rng.standard_normal((len(pts), g)) * np.exp(rng.uniform(-spread, spread, size=(len(pts), 1)))).astype(np.float16)
    return pts, d.astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_fixed_point_sums_do_not_depend_on_the_point_order(seed):
    pts, d = _data(seed)
    acc, flags, s = fixed_scatter(pts, d, R)
    rng = np.random.default_rng(100 + seed)
    for _ in range(3):
        acc2, flags2, s2 = fixed_scatter(pts, d, R, order=rng.permutation)
        assert s2 == s and np.array_equal(acc2, acc) and np.array_equal(flags2, flags)
    perm = rng.permutation(len(pts))                                                  # the points themselves reordered
    acc3, _, _ = fixed_scatter(pts[perm], d[perm], R)
    assert np.array_equal(acc3, acc)


@pytest.mark.parametrize("seed,spread", [(0, 1.0), (3, 6.0)])
def test_fixed_point_error_is_within_its_bound_and_below_the_fp32_scatter(seed, spread):
    pts, d = _data(seed, spread=spread)
    acc, _, s = fixed_scatter(pts, d, R)
    ent, val = _contributions(pts, d, R)
    n = R ** 3 * d.shape[1]
    n_v = np.bincount(ent, minlength=n)
    order = np.argsort(ent, kind="stable")
    groups = np.split(val[order], np.cumsum(n_v)[:-1])
    exact = np.array([math.fsum(g) for g in groups])                                 # correctly rounded float64 sums
    got = np.ldexp(acc.astype(np.float64), -s)
    err = np.abs(got - exact)
    bound = n_v * 2.0 ** -(s + 1) + 2.0 ** -52 * np.abs(exact)
    assert np.all(err <= bound), float(np.max(err - bound))
    # fp32 atomics of the same data: each w d rounded to fp32 and added in a shuffled order
    rng = np.random.default_rng(7)
    p = rng.permutation(len(ent))
    acc32 = np.zeros(n, dtype=np.float32)
    np.add.at(acc32, ent[p], val[p].astype(np.float32))
    err32 = np.abs(acc32.astype(np.float64) - exact)
    assert float(np.max(n_v * 2.0 ** -(s + 1))) < float(np.max(err32))
    # ... and after the convert pass's single fp32 rounding, no worse than fp32's own rounding of the exact sum
    conv = convert(acc, np.zeros(n, dtype=np.int64), s).astype(np.float64)
    assert np.all(np.abs(conv - exact) <= np.abs(exact.astype(np.float32).astype(np.float64) - exact) + 2 * bound +
                  np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64))


def test_no_overflow_at_the_largest_point_set_values():
    """P points at one voxel corner with weight 1 and |d| = amax: the entry's sum stays inside int64."""
    n = 4096
    pts = np.full((n, 3), -1.0, dtype=np.float32)                                     # exactly on voxel 0: weight 1
    d = np.full((n, 32), 65504.0, dtype=np.float32)                                  # fp16's largest finite value
    d[:, 1] = -65504.0
    acc, _, s = fixed_scatter(pts, d, R)
    assert acc[0] == round(n * 65504.0 * 2.0 ** s) and acc[0] <= 2 ** 62 < 2 ** 63 - 1
    assert acc[1] == -acc[0]
    assert np.ldexp(float(acc[0]), -s) == n * 65504.0


def test_non_finite_contributions_follow_the_float_scatter():
    """NaN -> NaN; one infinity -> that infinity; both infinities -> NaN; an infinity at weight 0 is a NaN (0 * inf, as the
    float scatter's product); the finite contributions of other entries keep their fixed-point sums."""
    pts = np.full((5, 3), -1.0, dtype=np.float32)          # on voxel 0 with weight 1; the x + 1 corner with weight 0
    d = np.zeros((5, 32), dtype=np.float32)
    d[:, 6] = 1.0
    d[0, 0] = np.nan
    d[0, 1], d[1, 1] = np.inf, 2.0
    d[0, 2], d[1, 2] = -np.inf, 3.0
    d[0, 3], d[1, 3] = np.inf, -np.inf
    d[2, 4] = -np.inf
    with np.errstate(invalid="ignore"):
        acc, flags, s = fixed_scatter(pts, d, R)
    out = convert(acc, flags, s)
    assert np.isnan(out[0]) and out[1] == np.inf and out[2] == -np.inf and np.isnan(out[3]) and out[4] == -np.inf
    assert out[6] == 5.0                                                                # finite channel of voxel 0
    vox, w = _trilinear(pts[:1], R)
    assert w[0, 0] == 1.0 and vox[0, 1] == 1 and w[0, 1] == 0.0
    x1 = 32                                                                             # voxel 1 = (x 1, y 0, z 0)
    assert all(np.isnan(out[x1 + c]) for c in range(5)) and out[x1 + 6] == 0.0 and acc[x1 + 6] == 0
    # amax is over the finite entries only
    assert s == fixed_exponent(3.0, 5)


# ---------------------------------------------------------------------------------------------------------------------
# C-ABI: argument checks run on the host (no GPU is touched by a refused call)
# ---------------------------------------------------------------------------------------------------------------------
def _grid_desc(grid=32):
    """Model B's field description (its 32 x 96^3 grid), or model A's (no grid)."""
    import _cases
    from fenerf_b200 import packing
    gen = _cases.build_mirror(_cases.CASE_BY_NAME["b_small" if grid else "a_small"])
    return packing.field_desc(gen.siren.field_spec())


FAKE = 1 << 20          # a non-NULL, aligned address the refused calls never dereference


def _err(lib):
    return lib.fenerf_last_error().decode()


def test_workspace_query_of_the_fixed_point_scatter():
    lib = _lib.lib()
    n = 96 ** 3 * 32
    assert lib.fenerf_grid_scatter_det_workspace_bytes(C.byref(_grid_desc())) == n * 8 + n // 8 * 4 + 256
    assert lib.fenerf_grid_scatter_det_workspace_bytes(C.byref(_grid_desc(0))) == 0


@pytest.mark.parametrize("args,code,message", [
    (dict(dA=0), -1, "bad argument"),
    (dict(partial=0), -1, "bad argument"),
    (dict(n_points=0), -1, "bad argument"),
    (dict(n_points=1000, ppb=300), -1, "whole number of images"),
    (dict(dtype=5), -1, "dtype"),
    (dict(partial_bytes=4 * 256 * 2 - 4), -4, "partial buffer too small"),
])
def test_gate_backward_det_refuses(args, code, message):
    lib = _lib.lib()
    a = dict(dA=FAKE, gate=FAKE, n_points=1024, ppb=1024, partial=FAKE, partial_bytes=0, colsum=FAKE, dtype=0)
    a.update(args)
    rc = lib.fenerf_gate_backward_det(a["dA"], a["gate"], a["n_points"], a["ppb"], a["partial"], a["partial_bytes"],
                                      a["colsum"], a["dtype"], None)
    assert rc == code and message in _err(lib), (rc, _err(lib))


@pytest.mark.parametrize("args,code,message", [
    (dict(field=0), -1, "field has no grid"),
    (dict(points=0), -1, "bad argument"),
    (dict(n_points=0), -1, "bad argument"),
    (dict(ld=16), -1, "bad argument"),
    (dict(workspace=FAKE + 4), -1, "8-byte aligned"),
    (dict(dtype=2), -1, "dtype"),
    (dict(workspace_bytes=1 << 20), -4, "workspace too small"),
])
def test_grid_scatter_add_det_refuses(args, code, message):
    lib = _lib.lib()
    a = dict(field=32, points=FAKE, d_feat=FAKE, ld=32, n_points=100, workspace=FAKE, workspace_bytes=0, grad=FAKE, dtype=0)
    a.update(args)
    desc = _grid_desc(a["field"])
    rc = lib.fenerf_grid_scatter_add_det(C.byref(desc), a["points"], a["d_feat"], a["ld"], a["n_points"], a["workspace"],
                                         a["workspace_bytes"], a["grad"], a["dtype"], None)
    assert rc == code and message in _err(lib), (rc, _err(lib))


@pytest.mark.parametrize("args,message", [
    (dict(x=0), "bad argument"), (dict(amax=0), "bad argument"), (dict(rows=-1), "bad argument"),
    (dict(ld=16), "bad argument"), (dict(dtype=3), "dtype"),
])
def test_absmax_finite_refuses(args, message):
    lib = _lib.lib()
    a = dict(x=FAKE, rows=10, cols=32, ld=32, dtype=0, amax=FAKE)
    a.update(args)
    rc = lib.fenerf_absmax_finite(a["x"], a["rows"], a["cols"], a["ld"], a["dtype"], a["amax"], None)
    assert rc == -1 and message in _err(lib), (rc, _err(lib))
