"""The numpy restatement of faer's pivoted Cholesky (tests/piv_llt_model.py), which the GPU tests check the library against,
pinned on the reference's own tests (llt_pivoting/{solve,inverse,reconstruct}.rs, restated with seeded inputs), on LAPACK's
?pstrf and on exact edge cases."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg.lapack as lapack

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import piv_llt_model as M  # noqa: E402

DTYPES = [np.float64, np.float32, np.complex128, np.complex64]
PSTRF = {np.float64: lapack.dpstrf, np.float32: lapack.spstrf, np.complex128: lapack.zpstrf, np.complex64: lapack.cpstrf}


def randn(rng, shape, dtype):
    x = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.standard_normal(shape)
    return x


def approx_eq(a, b, tol):
    """faer's ApproxEq (utils/approx.rs): |a - b| <= abs_tol or <= rel_tol * max(|a|, |b|)."""
    d = np.abs(a - b)
    return bool(np.all((d <= tol) | (d <= tol * np.maximum(np.abs(a), np.abs(b)))))


def c64_aah(rng, n):
    A = randn(rng, (n, n), np.complex128)
    return A @ np.conj(A.T)


def test_reference_solve():
    """solve.rs:72-140: n = 50, k = 3, c64 A A^H; A X ~ B and conj(A) X ~ B at 128 * 8 n eps (ApproxEq::eps() * 8 n)."""
    rng = np.random.default_rng(0)
    n, k = 50, 3
    A = c64_aah(rng, n)
    B = randn(rng, (n, k), np.complex128)
    L = A.copy(order="F")
    ok, rank, _, p, pi = M.piv_llt(L)
    assert ok and rank == n
    tol = 128 * np.finfo(np.float64).eps * 8 * n
    assert approx_eq(A @ M.solve(L, p, pi, B), B, tol)
    assert approx_eq(np.conj(A) @ M.solve(L, p, pi, B, conj=True), B, tol)


def test_reference_inverse():
    """inverse.rs:64-110: A_inv A ~ I at ApproxEq::eps() * n."""
    rng = np.random.default_rng(1)
    n = 50
    A = c64_aah(rng, n)
    L = A.copy(order="F")
    ok, rank, _, p, pi = M.piv_llt(L)
    assert ok and rank == n
    A_inv = M.mirror(M.inverse(L, pi))
    assert approx_eq(A_inv @ A, np.eye(n), 128 * np.finfo(np.float64).eps * n * np.linalg.cond(A))


def test_reference_reconstruct():
    """reconstruct.rs:62-107: the reconstruction ~ A at ApproxEq::eps() * n."""
    rng = np.random.default_rng(2)
    n = 50
    A = c64_aah(rng, n)
    L = A.copy(order="F")
    ok, rank, _, p, pi = M.piv_llt(L)
    assert ok and rank == n
    assert approx_eq(M.mirror(M.reconstruct(L, pi)), A, 128 * np.finfo(np.float64).eps * n)


def gram(rng, n, dtype, m):
    G = randn(rng, (n, m), dtype)
    return (G @ np.conj(G.T)).astype(dtype)


def graded(rng, n, dtype):
    """D G D with D over six decades (two in single precision, where six would leave most of the diagonal below tol)."""
    half = 3 if np.finfo(dtype).eps < 1e-10 else 1
    D = np.diag(10.0 ** rng.uniform(-half, half, n))
    return (D @ gram(rng, n, np.complex128 if np.issubdtype(dtype, np.complexfloating) else np.float64, 2 * n) @ D).astype(dtype)


def pstrf(A):
    c, piv, rank, info = PSTRF[A.dtype.type](np.asfortranarray(A), lower=1)
    return np.tril(c), piv - 1, int(rank)


@pytest.mark.parametrize("dtype", DTYPES)
def test_pivots_match_lapack_pstrf(dtype):
    rng = np.random.default_rng(3)
    for n, bs in [(30, 128), (97, 7), (200, 16)]:
        for A in (gram(rng, n, dtype, 2 * n), graded(rng, n, dtype)):
            L = A.copy(order="F")
            ok, rank, _, p, _ = M.piv_llt(L, bs)
            c, piv, rank_l = pstrf(A)
            assert ok and rank == rank_l == n
            assert np.array_equal(p, piv), (n, bs)
            if dtype == np.float64:
                assert np.all(np.abs(np.tril(L) - c) <= 1e-12 * np.abs(c).max())


@pytest.mark.parametrize("dtype", DTYPES)
def test_rank_matches_lapack_pstrf(dtype):
    """Rank-r Gram inputs: the residual at step r is far below both tolerances (checked), so both stop at r."""
    rng = np.random.default_rng(4)
    eps = np.finfo(dtype).eps
    for n, r, bs in [(200, 3, 128), (400, 5, 7), (600, 8, 64)]:
        A = gram(rng, n, dtype, r)
        L = A.copy(order="F")
        ok, rank, _, p, _ = M.piv_llt(L, bs)
        assert ok and rank == r
        tol = eps * n * np.real(np.diagonal(A)).max()
        assert abs(L[r, r]) <= tol / 100, (n, r, abs(L[r, r]), tol)
        c, piv, rank_l = pstrf(A)
        assert rank_l == r and np.array_equal(p[:r], piv[:r])


def test_edge_cases_exact():
    for dtype in DTYPES:
        ok, rank, tc, p, pi = M.piv_llt(np.zeros((0, 0), dtype=dtype))
        assert (ok, rank, tc) == (True, 0, 0) and p.size == 0
        A = np.full((1, 1), 0.0, dtype=dtype)
        assert M.piv_llt(A)[:3] == (True, 1, 0) and A[0, 0] == 0
        A = np.eye(7, dtype=dtype)
        ok, rank, tc, p, _ = M.piv_llt(A)
        assert (ok, rank, tc) == (True, 7, 0) and np.array_equal(p, np.arange(7))
        for bs in (1, 2, 128):
            d = np.array([1, 3, 2, 3, 5, 5, 0.5, 5, 2])
            ok, rank, tc, p, pi = M.piv_llt(np.diag(d).astype(dtype), bs)
            assert (ok, rank, tc) == (True, 9, 6) and list(p) == [4, 5, 7, 3, 1, 2, 8, 0, 6]
            assert np.array_equal(pi[p], np.arange(9))
        # a negative or NaN diagonal entry: index 0, A untouched
        for bad in (-1e-30, np.nan):
            A = np.eye(5, dtype=dtype)
            A[3, 3] = bad
            B = A.copy()
            assert M.piv_llt(B)[:2] == (False, 0) and np.array_equal(A, B, equal_nan=True)
        # NaN off the diagonal: reached at column 3 (the pivots are the identity here)
        A = np.diag(np.arange(10, 0, -1)).astype(dtype)
        A[6, 2] = np.nan
        assert M.piv_llt(A, 128)[:2] == (False, 3)
        # zero matrix, n >= 2: column 0 divides by sqrt(0) and the NaN shows up at column 1
        for n in (2, 5):
            assert M.piv_llt(np.zeros((n, n), dtype=dtype))[:2] == (False, 1)
