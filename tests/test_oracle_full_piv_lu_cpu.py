"""The numpy restatement of faer's full-pivoting LU (tests/full_piv_lu_model.py), which the GPU tests check the library against,
pinned on the reference's own tests (full_pivoting/{factor,solve,reconstruct,inverse}.rs, restated with seeded inputs), on
LAPACK's ?getc2 (real types, tie-free inputs) and on exact edge cases."""
import json
import os
import sys

import numpy as np
import pytest
import scipy.linalg.lapack as lapack

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_piv_lu_model as M  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def randn(rng, shape, dtype=np.complex128):
    x = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.standard_normal(shape)
    return np.asfortranarray(x.astype(dtype))


def approx_eq(a, b, tol):
    """faer's ApproxEq (utils/approx.rs): |a - b| <= abs_tol or <= rel_tol * max(|a|, |b|)."""
    d = np.abs(a - b)
    return bool(np.all((d <= tol) | (d <= tol * np.maximum(np.abs(a), np.abs(b)))))


def factor(A, row_major=False):
    LU = A.copy()
    rf, rb, cf, cb, cnt = M.lu_in_place(LU, row_major)
    L, U = M.split(LU)
    return LU, L, U, rf, rb, cf, cb, cnt


@pytest.mark.parametrize("m", [8, 16, 24, 32, 128, 255, 256, 257])
def test_reference_flu_c64_tall(m):
    """factor.rs:547-603: c64 m x 8, P^-1 L U Q^-1 ~ A at 1e-10."""
    A = randn(np.random.default_rng(m), (m, 8))
    _, L, U, rf, rb, cf, cb, _ = factor(A)
    assert approx_eq(M.reconstruct(L, U, rb, cb), A, 1e-10)


@pytest.mark.parametrize("n", [16, 24, 32, 128, 255, 256, 257])
def test_reference_flu_f64_square(n):
    """factor.rs:604-652: f64 n x n."""
    A = randn(np.random.default_rng(n), (n, n), np.float64)
    _, L, U, rf, rb, cf, cb, _ = factor(A)
    assert approx_eq(M.reconstruct(L, U, rb, cb), A, 1e-10)


def _gh238():
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "full_piv_lu_gh238.json")))
    n = d["n"]
    return np.asfortranarray(np.array(d["A_row_major"]).reshape(n, n)), np.array(d["b"]).reshape(n, 1)


def test_reference_gh238_solve_is_finite():
    """factor.rs:656-854: the solve of this 28 x 28 system must be all finite."""
    A, b = _gh238()
    _, L, U, rf, rb, cf, cb, _ = factor(A)
    assert np.all(np.isfinite(M.solve(L, U, rf, rb, cf, cb, b)))


def test_reference_solve():
    """solve.rs:152-252: c64 n = 50, k = 3: A X ~ B, A^T X ~ B, conj(A) X ~ B, A^H X ~ B at eps * n."""
    rng = np.random.default_rng(0)
    n, k = 50, 3
    A, B = randn(rng, (n, n)), randn(rng, (n, k))
    _, L, U, rf, rb, cf, cb, _ = factor(A)
    tol = np.finfo(float).eps * n * 100
    assert approx_eq(A @ M.solve(L, U, rf, rb, cf, cb, B), B, tol)
    assert approx_eq(A.T @ M.solve_transpose(L, U, rf, rb, cf, cb, B), B, tol)
    assert approx_eq(np.conj(A) @ M.solve(L, U, rf, rb, cf, cb, B, conj=True), B, tol)
    assert approx_eq(np.conj(A).T @ M.solve_transpose(L, U, rf, rb, cf, cb, B, conj=True), B, tol)


@pytest.mark.parametrize("shape", [(100, 50), (50, 100)])
def test_reference_reconstruct(shape):
    """reconstruct.rs:91-142."""
    A = randn(np.random.default_rng(0), shape)
    _, L, U, rf, rb, cf, cb, _ = factor(A)
    assert approx_eq(M.reconstruct(L, U, rb, cb), A, np.finfo(float).eps * max(shape) * 100)


def test_reference_inverse():
    """inverse.rs:72-119: A^-1 A ~ I."""
    n = 50
    A = randn(np.random.default_rng(0), (n, n))
    _, L, U, rf, rb, cf, cb, _ = factor(A)
    assert approx_eq(M.inverse(L, U, rb, cb) @ A, np.eye(n), np.finfo(float).eps * n * 100)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(6, 6), (40, 40), (120, 120)])
def test_lapack_getc2_pivots(dtype, shape):
    """?getc2 on tie-free Gaussian inputs: the same row and column transpositions, L and U to tolerance."""
    n = shape[0]
    A = randn(np.random.default_rng(n), shape, dtype)
    getc2 = lapack.dgetc2 if dtype == np.float64 else lapack.sgetc2
    lu, ipiv, jpiv, info = getc2(A.copy())
    LU = A.copy()
    rt, ct, _ = M.lu_in_place_unblocked(LU, False)
    # scipy returns LAPACK's 1-based IPIV / JPIV converted to 0-based; ?getc2 stops one step early (its last pivot is the
    # remaining entry), so the first n - 1 transpositions are compared
    assert [int(x) for x in ipiv[: n - 1]] == rt[: n - 1]
    assert [int(x) for x in jpiv[: n - 1]] == ct[: n - 1]
    eps = np.finfo(dtype).eps
    assert np.max(np.abs(lu - LU)) <= 50 * n * eps * np.max(np.abs(A))


@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_zero_matrix_exits_at_step_0(dtype):
    A = np.zeros((5, 4), dtype=dtype, order="F")
    LU, L, U, rf, rb, cf, cb, cnt = factor(A)
    assert cnt == 0 and np.array_equal(LU, A)
    assert np.array_equal(rf, np.arange(5)) and np.array_equal(cf, np.arange(4))


def test_ones_matrix_exits_after_step_0():
    A = np.ones((5, 4), order="F")
    X = A.copy()
    rt, ct, cnt = M.lu_in_place_unblocked(X, False)
    assert cnt == 0 and rt == [0, 1, 2, 3] and ct == [0, 1, 2, 3]
    assert np.array_equal(X[1:, 1:], np.zeros((4, 3))) and np.array_equal(X[:, 0], np.ones(5))


def test_subnormal_only_input_exits_at_step_0():
    A = np.full((3, 3), 1e-310, order="F")
    X = A.copy()
    rt, ct, cnt = M.lu_in_place_unblocked(X, False)
    assert cnt == 0 and np.array_equal(X, A)


def test_nan_next_to_zero_column_is_never_chosen():
    A = np.asfortranarray(np.array([[0.0, np.nan, 0.5], [0.0, 1.0, 0.25], [0.0, 2.0, 0.0]]))
    X = A.copy()
    rt, ct, cnt = M.lu_in_place_unblocked(X, False)
    assert (rt[0], ct[0]) == (2, 1)  # the 2.0, not the NaN above it nor the zero column


def test_inf_entry_is_chosen_first():
    A = np.asfortranarray(np.array([[1.0, 2.0], [np.inf, 3.0]]))
    X = A.copy()
    rt, ct, _ = M.lu_in_place_unblocked(X, False)
    assert (rt[0], ct[0]) == (1, 0)


@pytest.mark.parametrize("shape", [(0, 4), (4, 0), (1, 1), (1, 6), (6, 1)])
def test_degenerate_shapes(shape):
    A = randn(np.random.default_rng(1), shape, np.float64)
    LU, L, U, rf, rb, cf, cb, cnt = factor(A, row_major=shape[0] == 1)
    assert len(rf) == shape[0] and len(cf) == shape[1]
    if A.size:
        assert approx_eq(M.reconstruct(L, U, rb, cb), A, 1e-14)


def test_first_maximum_tie_rule_in_both_branches():
    """Exact ties: the first maximum in the working matrix's column-major order, i.e. A's column-major order for a column-major
    A and A's row-major order for a row-major one (the transposed branch)."""
    A = np.asfortranarray(np.array([[1.0, 2.0], [2.0, 1.0]]))
    X = A.copy()
    rt, ct, _ = M.lu_in_place_unblocked(X, False)
    assert (rt[0], ct[0]) == (1, 0)
    rf, rb, cf, cb, _ = M.lu_in_place(A.copy(), row_major=True)
    assert rf[0] == 0 and cf[0] == 1
    assert M.takes_transposed_branch(2, 1) and not M.takes_transposed_branch(1, 2) and M.takes_transposed_branch(1, 1)


def test_transposed_branch_scales_the_row():
    A = randn(np.random.default_rng(3), (30, 20), np.float64)
    X = np.ascontiguousarray(A)
    rf, rb, cf, cb, _ = M.lu_in_place(X, row_major=True)
    L, U = M.split(X)
    assert approx_eq(M.reconstruct(L, U, rb, cb), A, 1e-12)
    assert np.max(np.abs(np.tril(X, -1))) <= 1 + 1e-15
