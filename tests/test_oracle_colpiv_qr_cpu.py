"""The numpy restatement of faer's column-pivoted QR (tests/colpiv_qr_model.py), which the GPU tests check the library against,
pinned on the reference's own tests (col_pivoting/{factor,solve,reconstruct,inverse}.rs, restated with seeded inputs), on
LAPACK's ?geqp3 (scipy `qr(pivoting=True)`) and on exact edge cases."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg as sl

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import colpiv_qr_model as M  # noqa: E402


def randn(rng, shape, dtype=np.complex128):
    x = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.standard_normal(shape)
    return x.astype(dtype)


def graded(rng, m, n, dtype=np.float64):
    """Gaussian columns scaled by a random permutation of a geometric sequence from 1 to 1e3: pivot gaps far above rounding."""
    g = np.geomspace(1.0, 1e3, n)
    rng.shuffle(g)
    return (randn(rng, (m, n), dtype) * g).astype(dtype)


def approx_eq(a, b, tol):
    """faer's ApproxEq (utils/approx.rs): |a - b| <= abs_tol or <= rel_tol * max(|a|, |b|)."""
    d = np.abs(a - b)
    return bool(np.all((d <= tol) | (d <= tol * np.maximum(np.abs(a), np.abs(b)))))


@pytest.mark.parametrize("shape", [(n, n) for n in (2, 3, 4, 8, 16, 24, 32, 128, 255)] + [(m, 20) for m in (2, 3, 4, 8, 16, 24, 32, 128, 255)])
def test_reference_unblocked_qr(shape):
    """factor.rs:396-525: c64, bs = 15, Q R P ~ A at 1e-10."""
    rng = np.random.default_rng(0)
    A = randn(rng, shape)
    QR = A.copy()
    tau, perm, _ = M.factor_unblocked(QR)
    H = M.t_blocks(QR, tau, 15)
    assert np.array_equal(np.real(H[np.arange(len(tau)) % 15, np.arange(len(tau))]), tau)  # taus on the block diagonals
    assert approx_eq(M.reconstruct(QR, tau, perm), A, 1e-10)


def test_reference_reconstruct_and_inverse():
    """reconstruct.rs:54-100 ((100, 50), (50, 100)) and inverse.rs:59-110 (n = 50), c64."""
    rng = np.random.default_rng(0)
    for m, n in ((100, 50), (50, 100)):
        A = randn(rng, (m, n))
        QR = A.copy()
        tau, perm, _ = M.factor_unblocked(QR)
        assert approx_eq(M.reconstruct(QR, tau, perm), A, 50 * 128 * np.finfo(float).eps * max(m, n))
    n = 50
    A = randn(rng, (n, n))
    QR = A.copy()
    tau, perm, _ = M.factor_unblocked(QR)
    Q = M.q_matrix(QR, tau)
    R = M.r_matrix(QR)
    X = np.empty((n, n), dtype=A.dtype)
    X[perm] = np.linalg.solve(R, Q.conj().T)
    assert approx_eq(A @ X, np.eye(n), 128 * np.finfo(float).eps * n)


def test_reference_lstsq_and_solve():
    """solve.rs:219-416: lstsq (100 x 50, k = 3) with and without conjugation; square solve (n = 50)."""
    rng = np.random.default_rng(0)
    m, n, k = 100, 50, 3
    A, B = randn(rng, (m, n)), randn(rng, (m, k))
    QR = A.copy()
    tau, perm, _ = M.factor_unblocked(QR)
    tol = 128 * np.finfo(float).eps * n
    X = M.solve_lstsq(QR, tau, perm, B)
    assert approx_eq(A.conj().T @ A @ X, A.conj().T @ B, tol)
    X = M.solve_lstsq(QR, tau, perm, B, conj=True)
    assert approx_eq(A.T @ A.conj() @ X, A.T @ B, tol)
    A, B = randn(rng, (n, n)), randn(rng, (n, k))
    QR = A.copy()
    tau, perm, _ = M.factor_unblocked(QR)
    assert approx_eq(A @ M.solve_lstsq(QR, tau, perm, B), B, tol)


@pytest.mark.parametrize("shape", [(50, 50), (128, 128), (200, 200), (255, 255), (300, 40), (40, 300)])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_permutation_matches_geqp3(shape, seed):
    """Graded inputs: the same first min(m, n) pivots as LAPACK ?geqp3, |diag R| to 1e-10 of |R_00|."""
    rng = np.random.default_rng(seed)
    m, n = shape
    A = graded(rng, m, n)
    QR, _, perm, _, _ = M.factor(A, 15)
    _, R, P = sl.qr(A, pivoting=True, mode="economic")
    s = min(m, n)
    assert (P[:s] == perm[:s]).all()
    assert np.max(np.abs(np.abs(np.diag(R)) - np.abs(np.diag(QR)[:s]))) <= 1e-10 * abs(R[0, 0])


def test_row_stride_flag_takes_the_recompute_branch():
    """row_stride != 1: every step recomputes the norms; the pivots still match ?geqp3 on graded input."""
    rng = np.random.default_rng(3)
    A = graded(rng, 120, 90)
    QR1, _, p1, _, c1 = M.factor(A, 8, row_stride_one=True)
    QR2, _, p2, _, c2 = M.factor(A, 8, row_stride_one=False)
    assert (p1 == p2).all() and c1 == c2
    assert np.max(np.abs(QR1 - QR2)) <= 1e-10 * np.max(np.abs(QR1))


def test_edge_cases():
    for m, n in ((0, 0), (0, 5), (5, 0)):
        QR, H, p, pi, c = M.factor(np.zeros((m, n)), 4)
        assert (p == np.arange(n)).all() and c == 0
    # n = 1: no pivoting; R_00 = -|a| sign(a_0)
    a = np.array([[3.0], [4.0]])
    QR, H, p, _, c = M.factor(a, 4)
    assert c == 0 and abs(QR[0, 0]) == pytest.approx(5.0)
    # all zero: NaN factors, identity permutation, count 0 (recip(0) = inf)
    QR, H, p, _, c = M.factor(np.zeros((6, 5)), 4)
    assert (p == np.arange(5)).all() and c == 0 and np.isnan(QR).all()
    # zero column: pivoted last
    rng = np.random.default_rng(5)
    A = graded(rng, 10, 6)
    A[:, 2] = 0
    QR, H, p, _, c = M.factor(A, 4)
    assert p[-1] == 2
    # a NaN column next to a zero column: nothing qualifies at k = 1, the pivot stays at k
    A = np.array([[1.0, np.nan, 0.0], [2.0, np.nan, 0.0], [3.0, np.nan, 0.0]])
    QR, H, p, _, c = M.factor(A, 4)
    assert (p == np.arange(3)).all() and c == 0
    # NaN column: never chosen as a pivot while others qualify
    A = graded(rng, 10, 6)
    A[:, 1] = np.nan
    QR, H, p, _, c = M.factor(A, 4)
    assert 1 not in list(p[:1])
