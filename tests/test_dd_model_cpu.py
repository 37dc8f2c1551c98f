"""The numpy double-double model of tests/dd_model.py, the GPU tests' reference for fx128 / cx128: its operations against mpmath at
300 bits (error within a few units of 2^-104 of the result), and its products and LU against exact rational arithmetic."""
import os
import sys
from fractions import Fraction as F

import mpmath
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dd_model as M  # noqa: E402

mpmath.mp.prec = 300
U = 2.0 ** -104


def _rand(rng, n, spread=30):
    hi = rng.standard_normal(n) * 10.0 ** rng.integers(-spread, spread, n)
    lo = hi * 2.0 ** -53 * rng.uniform(-0.5, 0.5, n)
    return hi + 0.0, lo


def _mp(h, l):
    return mpmath.mpf(float(h)) + mpmath.mpf(float(l))


def test_operations_against_mpmath():
    rng = np.random.default_rng(1)
    x, y = _rand(rng, 400), _rand(rng, 400)
    ax = (np.abs(x[0]), np.where(x[0] < 0, -x[1], x[1]))
    for name, got, ref, rel in (
        ("add", M.add(x, y), lambda a, b: a + b, None),
        ("mul", M.mul(x, y), lambda a, b: a * b, 4),
        ("div", M.div(x, y), lambda a, b: a / b, 8),
    ):
        for i in range(400):
            a, b = _mp(x[0][i], x[1][i]), _mp(y[0][i], y[1][i])
            r, g = ref(a, b), _mp(got[0][i], got[1][i])
            bound = (4 * (abs(a) + abs(b)) if rel is None else rel * abs(r)) * U
            assert abs(g - r) <= bound, (name, i)
    s = M.sqrt(ax)
    for i in range(400):
        r = mpmath.sqrt(_mp(ax[0][i], ax[1][i]))
        assert abs(_mp(s[0][i], s[1][i]) - r) <= 8 * U * r


def test_matmul_and_lu_against_fractions():
    rng = np.random.default_rng(2)
    for n in (1, 5, 12):
        A = (rng.standard_normal((n, n)), rng.standard_normal((n, n)) * 2.0 ** -60)
        B = (rng.standard_normal((n, n)), rng.standard_normal((n, n)) * 2.0 ** -60)
        C = M.matmul(A, B, False)
        fa = [[F(A[0][i, j]) + F(A[1][i, j]) for j in range(n)] for i in range(n)]
        fb = [[F(B[0][i, j]) + F(B[1][i, j]) for j in range(n)] for i in range(n)]
        for i in range(n):
            for j in range(n):
                exact = sum(fa[i][t] * fb[t][j] for t in range(n))
                mag = sum(abs(fa[i][t] * fb[t][j]) for t in range(n))
                assert abs(F(C[0][i, j]) + F(C[1][i, j]) - exact) <= 4 * n * F(U) * mag
        LU, perm, _ = M.lu(A)
        # exact elimination with the same pivots: the model's factors agree to a few n 2^-104
        P = [fa[p][:] for p in perm]
        for j in range(n):
            for i in range(j + 1, n):
                P[i][j] = P[i][j] / P[j][j]
                for c in range(j + 1, n):
                    P[i][c] -= P[i][j] * P[j][c]
        scale = max(abs(v) for row in P for v in row)
        for i in range(n):
            for j in range(n):
                assert abs(F(LU[0][i, j]) + F(LU[1][i, j]) - P[i][j]) <= F(1, 10 ** 24) * scale
