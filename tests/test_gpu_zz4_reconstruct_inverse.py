"""`*_reconstruct` / `*_inverse` on the factors through the C ABI (csrc/reconstruct_types.cu; compositions of validated kernels).
Reference tests restated for f64:
llt/reconstruct.rs and inverse.rs tests (n = 50, eps * n), lu/partial_pivoting/reconstruct.rs and inverse.rs tests,
qr/no_pivoting/reconstruct.rs tests ((100, 50) and (50, 100)) and inverse.rs tests."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
U = np.finfo(np.float64).eps


def _close(a, b, n, scale):
    return np.abs(a - b).max() <= 128 * n * U * scale


def test_llt_reconstruct_and_inverse(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(141)
    for n in [1, 50, 200, 513]:
        G = rng.standard_normal((n, n)); A = np.asfortranarray(G @ G.T + n * np.eye(n))
        L = A.copy(order="F"); la.cholesky_in_place(L)
        out = np.full((n, n), np.nan, order="F"); out[np.tril_indices(n)] = 7.0
        la.llt_reconstruct(out, L)          # L's strict upper part still holds A's entries: it must not be read
        assert np.all(np.isnan(out[np.triu_indices(n, 1)]))                   # only the lower triangle is written
        assert _close(np.tril(out), np.tril(A), n, np.abs(A).max())
        inv = np.full((n, n), np.nan, order="F"); inv[np.tril_indices(n)] = 7.0
        la.llt_inverse(inv, L)
        assert np.all(np.isnan(inv[np.triu_indices(n, 1)]))
        full = np.tril(inv) + np.tril(inv, -1).T
        assert _close(full @ A, np.eye(n), n, np.linalg.cond(A))


@pytest.mark.parametrize("idx", [np.uint64, np.uint32])
def test_lu_reconstruct_and_inverse(fb, cuda_dev, idx):
    la = fb.linalg
    rng = np.random.default_rng(142)
    for (m, n) in [(50, 50), (100, 40), (40, 100), (300, 300)]:
        A = np.asfortranarray(rng.standard_normal((m, n)))
        LU = A.copy(order="F"); p = np.zeros(m, idx); pi = np.zeros(m, idx)
        la.lu_in_place(LU, p, pi)
        out = np.full((m, n), np.nan, order="F")
        la.lu_reconstruct(out, LU, LU, p, pi)                                  # packed factors passed twice
        assert _close(out, A, max(m, n), np.abs(A).max() * max(1.0, np.abs(np.triu(LU)).max()))
        L, Uf = fb.solvers.split_LU(LU.copy(order="F"))                        # split factors give the same answer
        out2 = np.full((m, n), np.nan, order="F")
        la.lu_reconstruct(out2, L, Uf, p, pi)
        assert np.allclose(out2, out, rtol=1e-12, atol=1e-13)
        if m == n:
            inv = np.full((n, n), np.nan, order="F")
            la.lu_inverse(inv, LU, LU, p, pi)
            assert _close(inv @ A, np.eye(n), n, np.linalg.cond(A))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_qr_reconstruct_and_inverse(fb, cuda_dev, dtype):
    la = fb.linalg
    rng = np.random.default_rng(143)
    u = np.finfo(dtype).eps
    for (m, n) in [(100, 50), (50, 100), (64, 64), (300, 129)]:
        A = np.asfortranarray(rng.standard_normal((m, n)).astype(dtype))
        size = min(m, n)
        QR = A.copy(order="F"); H = np.zeros((la.qr_recommended_block_size(m, n), size), dtype=dtype, order="F")
        la.qr_in_place(QR, H)
        out = np.full((m, n), np.nan, dtype=dtype, order="F")
        la.qr_reconstruct(out, QR[:, :size], H, QR[:size, :])                   # R = the leading rows of the packed matrix
        assert np.abs(out - A).max() <= 128 * max(m, n) * u * np.abs(A).max(), (m, n)
        if m == n and dtype == np.float64:
            inv = np.full((n, n), np.nan, order="F")
            la.qr_inverse(inv, QR, H, QR)
            assert _close(inv @ A, np.eye(n), n, np.linalg.cond(A))
