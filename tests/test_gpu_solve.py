"""GPU tests of the solves on top of the factors (SURVEY.md §8f rank 1), through the C ABI.

reference tests: cholesky/llt/solve.rs:55-... (n in {50, 200, 400}: A X ~ B, tolerance eps*128*8n) and the LU analogue
(lu/partial_pivoting/solve.rs tests): restated with our seeded inputs; the expected X also comes from the oracle's
factor + triangular solves (same composition, CPU).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


def test_llt_solve(fb, oracle, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(31)
    for n, k in [(1, 1), (50, 3), (200, 7), (400, 130), (1000, 16)]:
        G = rng.standard_normal((n, n)); A = np.asfortranarray(G @ G.T + n * np.eye(n))
        B = np.asfortranarray(rng.standard_normal((n, k)))
        L = A.copy(order="F"); la.cholesky_in_place(L)
        X = B.copy(order="F"); la.llt_solve_in_place(L, X)
        tol = EPS * 128 * 8 * n * np.abs(A).max() * max(1.0, np.abs(X).max())
        assert np.all(np.abs(A @ X - B) <= tol), (n, k)
        # oracle composition: L y = b, L^T x = y
        Lo = A.copy(order="F"); assert oracle.llt(Lo)[0] == -1
        Xo = B.copy(order="F")
        oracle.solve_triangular(Lo, Xo, lower=True, unit=False)
        oracle.solve_triangular(np.asfortranarray(Lo.T), Xo, lower=False, unit=False)
        assert np.allclose(X, Xo, rtol=1e-9, atol=1e-12), (n, k)


@pytest.mark.parametrize("idx", [np.uint64, np.uint32])
def test_lu_solve(fb, oracle, cuda_dev, idx):
    import torch
    la = fb.linalg
    rng = np.random.default_rng(32)
    for n, k in [(1, 1), (50, 3), (200, 7), (400, 130), (1000, 16), (3, 65537)]:
        A = np.asfortranarray(rng.standard_normal((n, n)))
        B = np.asfortranarray(rng.standard_normal((n, k)))
        LU = A.copy(order="F"); p = np.zeros(n, idx); pi = np.zeros(n, idx)
        la.lu_in_place(LU, p, pi)
        X = B.copy(order="F"); la.lu_solve_in_place(LU, p, pi, X)
        cond = np.linalg.cond(A)
        assert np.all(np.abs(A @ X - B) <= EPS * 128 * 8 * n * cond * max(1.0, np.abs(B).max())), (n, k)
        assert np.allclose(X, np.linalg.solve(A, B), rtol=1e-7 * max(1, cond / 1e4), atol=1e-9), (n, k)
    # device-resident factors, rhs and permutation
    n, k = 600, 9
    A = np.asfortranarray(rng.standard_normal((n, n))); B = np.asfortranarray(rng.standard_normal((n, k)))
    dA = torch.from_numpy(np.ascontiguousarray(A.T)).to(cuda_dev).T
    dB = torch.from_numpy(np.ascontiguousarray(B.T)).to(cuda_dev).T
    tdt = torch.int64 if idx == np.uint64 else torch.int32
    dp = torch.zeros(n, dtype=tdt, device=cuda_dev); dpi = torch.zeros(n, dtype=tdt, device=cuda_dev)
    la.lu_in_place(dA, dp, dpi)
    la.lu_solve_in_place(dA, dp, dpi, dB)
    assert np.allclose(dB.cpu().numpy(), np.linalg.solve(A, B), rtol=1e-8, atol=1e-9)

