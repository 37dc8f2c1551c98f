"""Pins the numpy restatement of faer's Bunch-Kaufman LBL^H (tests/lblt_model.py), the model the GPU tests compare with:

* the reference's own tests, restated with seeded inputs: bunch_kaufman/mod.rs `test_real` / `test_cplx` (every strategy,
  block_size 4, n in {2, 3, 6, 19, 100, 421}, solve residual < 1e-9) and reconstruct.rs `test_reconstruct`;
* exact small cases: identity, zero matrix, a column that becomes exactly zero inside a block, the 2 x 2-forcing [[0, 1], [1, 0]],
  repeated diagonal values (first maximum);
* LAPACK ?sytrf (scipy.linalg.ldl) for the P A P^T = L B L^H identity only: its pivot rule is not faer's."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lblt_model as M  # noqa: E402

STRATS = [M.PARTIAL, M.PARTIAL_DIAG, M.ROOK, M.ROOK_DIAG, M.FULL]


def sym(rng, n, cx):
    X = rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0)
    return X + np.conj(X.T)


def full(R):
    return np.tril(R) + np.conj(np.tril(R, -1)).T


@pytest.mark.parametrize("cx", [False, True])
@pytest.mark.parametrize("strat", STRATS)
def test_reference_solve_tests(cx, strat):
    rng = np.random.default_rng(0)
    for n in (2, 3, 6, 19, 100, 421):
        A = sym(rng, n, cx)
        LB, sub, p, pi, cnt, _ = M.factor(A if strat == M.FULL else np.tril(A), np.zeros(n, A.dtype), strat, 4)
        rhs = rng.standard_normal((n, 2)) + (1j * rng.standard_normal((n, 2)) if cx else 0)
        # residual relative to |A| |x| (the reference's approximate equality scales with the operands)
        x = M.solve(np.tril(LB), sub, p, pi, rhs)
        assert np.abs(A @ x - rhs).max() < 1e-9 * np.abs(A).max() * np.abs(x).max()
        xc = M.solve(np.tril(LB), sub, p, pi, rhs, conj=True)
        assert np.abs(np.conj(A) @ xc - rhs).max() < 1e-9 * np.abs(A).max() * np.abs(xc).max()
        assert np.array_equal(np.sort(p), np.arange(n)) and np.array_equal(pi[p], np.arange(n)) and 0 <= cnt < n


def test_reference_reconstruct():
    rng = np.random.default_rng(0)
    n = 50
    A = sym(rng, n, True)
    LB, sub, p, pi, _, _ = M.factor(np.tril(A), np.zeros(n, complex))
    R = M.reconstruct(np.tril(LB), sub, pi)
    assert np.abs(full(R) - A).max() < 1e-12 * n * np.abs(A).max()


@pytest.mark.parametrize("strat", STRATS)
def test_exact_small_cases(strat):
    for bs in (0, 2, 64):
        LB, sub, p, pi, cnt, _ = M.factor(np.eye(5), np.zeros(5), strat, bs)
        assert cnt == 0 and np.array_equal(np.tril(LB), np.eye(5))
        sub0 = np.full(4, 7.0)
        LB, sub, p, pi, cnt, _ = M.factor(np.zeros((4, 4)), sub0, strat, bs)
        if strat != M.FULL:
            assert np.array_equal(sub, sub0) and cnt == 0  # nothing to do: subdiag left as given
        else:
            assert np.all(np.isnan(np.diag(LB)))  # 1 / norm_max of a zero matrix
        LB, sub, p, pi, cnt, _ = M.factor(np.array([[0.0, 1.0], [1.0, 0.0]]), np.zeros(2), strat, bs)
        assert sub[0] == 1 and sub[1] == 0 and LB[1, 0] == 0
        # a column that becomes exactly zero after the first pivot: the second column is a multiple of the first
        A = np.array([[4.0, 2, 0], [2, 1, 0], [0, 0, 3]])
        LB, sub, p, pi, cnt, _ = M.factor(A, np.full(3, np.nan), strat, bs)
        assert np.abs(full(M.reconstruct(np.tril(LB), np.nan_to_num(sub), pi)) - A).max() < 1e-14
        # repeated diagonal values: the first maximum is kept
        D = np.diag([2.0, 3.0, 3.0, 1.0])
        LB, sub, p, pi, cnt, _ = M.factor(D, np.zeros(4), strat, bs)
        if strat in (M.PARTIAL_DIAG, M.ROOK_DIAG, M.FULL):
            assert p[0] == 1


@pytest.mark.parametrize("n", [5, 40, 200])
def test_identity_against_lapack_sytrf(n):
    rng = np.random.default_rng(n)
    A = sym(rng, n, False)
    lu, d, perm = scipy.linalg.ldl(A, lower=True)
    assert np.abs(lu @ d @ lu.T - A).max() < 1e-10 * n
    for strat in STRATS:
        LB, sub, p, pi, _, _ = M.factor(A if strat == M.FULL else np.tril(A), np.zeros(n), strat, 8)
        assert np.abs(full(M.reconstruct(np.tril(LB), sub, pi)) - A).max() < 1e-10 * n
