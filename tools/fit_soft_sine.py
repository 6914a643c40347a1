"""Derives the coefficients of the software sine of the point network's FiLM epilogue (soft_sinf, siren_fast.cuh).

soft_sinf reduces its argument to r = a - n 2pi with n = rint(a / 2pi), so |r| <= pi (1 + 1e-4) for |a| up to a few
thousand, and evaluates sin(r) = r P(r^2) with an odd polynomial of degree 11.  The coefficients are the minimax fit of
sin on [-pi (1 + 5e-4), pi (1 + 5e-4)] in absolute error, solved as a linear program on a dense grid (scipy's HiGHS),
then rounded to float32.  The script prints the coefficients, the fit's own error and the error of the float32 Horner
evaluation against float64 sin.

    python tools/fit_soft_sine.py
"""
import numpy as np
from scipy.optimize import linprog

HALF = np.pi * (1 + 5e-4)
DEGREE = 11


def fit(half=HALF, degree=DEGREE, n=6000):
    x = np.concatenate([half * np.cos(np.linspace(0, np.pi, n)), np.linspace(-half, half, n)])
    k = (degree + 1) // 2
    u = x / half                                              # scaled basis: a well-conditioned program
    A = np.stack([u ** (2 * i + 1) for i in range(k)], 1)
    y = np.sin(x)
    ones = np.ones((len(x), 1))
    res = linprog(np.r_[np.zeros(k), 1.0], A_ub=np.vstack([np.hstack([A, -ones]), np.hstack([-A, -ones])]),
                  b_ub=np.r_[y, -y], bounds=[(None, None)] * (k + 1), method="highs")
    assert res.success, res.message
    return res.x[:k] / half ** (2 * np.arange(k) + 1), res.x[k]


def horner_f32(c, r):
    """r P(r^2) in float32, each step one fused multiply-add (float64 product and sum, rounded once to float32)."""
    c = np.asarray(c, np.float32)
    r = np.asarray(r, np.float32)
    r2 = (r * r).astype(np.float32)
    p = np.full_like(r, c[-1])
    for ci in c[-2::-1]:
        p = (p.astype(np.float64) * r2 + np.float64(ci)).astype(np.float32)
    return (r * p).astype(np.float32)


if __name__ == "__main__":
    c, e = fit()
    c32 = c.astype(np.float32)
    xs = np.linspace(-HALF, HALF, 400001).astype(np.float32)
    err = np.abs(horner_f32(c32, xs).astype(np.float64) - np.sin(xs.astype(np.float64))).max()
    print("minimax error %.3e, float32 evaluation %.3e (2^-20 = %.3e)" % (e, err, 2.0 ** -20))
    for i, v in enumerate(c32):
        print("c%d = %.9ef" % (2 * i + 1, v))
