"""`*_reconstruct` / `*_inverse` on the factors for f64 / f32 / c64 / c32 through the C ABI (csrc/reconstruct_types.cu: one
composition over the products, solves and Householder sequences of each scalar kind).
The reference's own tests restated per dtype (they draw complex matrices):
  cholesky/llt/reconstruct.rs + inverse.rs tests (n = 50), lu/partial_pivoting/reconstruct.rs tests ((100, 50), (50, 100),
  (50, 50)) + inverse.rs tests (n = 50), qr/no_pivoting/reconstruct.rs tests ((100, 50), (50, 100)) + inverse.rs tests (n = 50),
plus sizes that cross the block boundaries of the kernels underneath. The f64 entry points are also covered by
test_gpu_zz4_reconstruct_inverse.py; here the f64 results also serve as the cross-check of the f32 ones."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32, np.complex128, np.complex64]


def _rand(rng, shape, dtype):
    a = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        a = a + 1j * rng.standard_normal(shape)
    return np.asfortranarray(a.astype(dtype))


def _u(dtype):
    return float(np.finfo(dtype).eps)


def _wide(x):
    return x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)


@pytest.mark.parametrize("dtype", DTYPES)
def test_llt_reconstruct_and_inverse_types(fb, cuda_dev, dtype):
    la = fb.linalg
    rng = np.random.default_rng(241)
    u = _u(dtype)
    for n in [1, 50, 200, 513]:
        G = _wide(_rand(rng, (n, n), dtype))
        A = np.asfortranarray((G @ G.conj().T + n * np.eye(n)).astype(dtype))
        L = A.copy(order="F"); la.cholesky_in_place(L)
        fill = dtype(7.0)
        out = np.full((n, n), np.nan, dtype=dtype, order="F"); out[np.tril_indices(n)] = fill
        la.llt_reconstruct(out, L)          # L's strict upper part still holds A's entries: it must not be read
        assert np.all(np.isnan(out[np.triu_indices(n, 1)])), n               # only the lower triangle is written
        assert np.abs(np.tril(_wide(out)) - np.tril(_wide(A))).max() <= 128 * n * u * np.abs(A).max(), n
        inv = np.full((n, n), np.nan, dtype=dtype, order="F"); inv[np.tril_indices(n)] = fill
        la.llt_inverse(inv, L)
        assert np.all(np.isnan(inv[np.triu_indices(n, 1)])), n
        lo = np.tril(_wide(inv))
        full = lo + np.tril(lo, -1).conj().T                                  # the inverse is self-adjoint
        assert np.abs(full @ _wide(A) - np.eye(n)).max() <= 128 * n * u * np.linalg.cond(_wide(A)), n


@pytest.mark.parametrize("idx", [np.uint64, np.uint32])
@pytest.mark.parametrize("dtype", DTYPES)
def test_lu_reconstruct_and_inverse_types(fb, cuda_dev, dtype, idx):
    la = fb.linalg
    rng = np.random.default_rng(242)
    u = _u(dtype)
    for (m, n) in [(50, 50), (100, 50), (50, 100), (300, 300), (1, 1), (130, 257)]:
        A = _rand(rng, (m, n), dtype)
        LU = A.copy(order="F"); p = np.zeros(m, idx); pi = np.zeros(m, idx)
        la.lu_in_place(LU, p, pi)
        out = np.full((m, n), np.nan, dtype=dtype, order="F")
        la.lu_reconstruct(out, LU, LU, p, pi)                                  # packed factors passed twice
        scale = np.abs(A).max() * max(1.0, float(np.abs(np.triu(LU)).max()))
        assert np.abs(_wide(out) - _wide(A)).max() <= 128 * max(m, n) * u * scale, (m, n)
        if m == n:
            inv = np.full((n, n), np.nan, dtype=dtype, order="F")
            la.lu_inverse(inv, LU, LU, p, pi)
            assert np.abs(_wide(inv) @ _wide(A) - np.eye(n)).max() <= 128 * n * u * np.linalg.cond(_wide(A)), n


@pytest.mark.parametrize("dtype", DTYPES)
def test_qr_reconstruct_and_inverse_types(fb, cuda_dev, dtype):
    la = fb.linalg
    rng = np.random.default_rng(243)
    u = _u(dtype)
    for (m, n) in [(100, 50), (50, 100), (50, 50), (64, 64), (300, 129), (1, 1)]:
        A = _rand(rng, (m, n), dtype)
        size = min(m, n)
        for bs in sorted({la.qr_recommended_block_size(m, n), min(7, size)}):
            QR = A.copy(order="F"); H = np.zeros((bs, size), dtype=dtype, order="F")
            assert la.qr_in_place(QR, H).rank == size
            out = np.full((m, n), np.nan, dtype=dtype, order="F")
            la.qr_reconstruct(out, QR[:, :size], H, QR[:size, :])               # R = the leading rows of the packed matrix
            assert np.abs(_wide(out) - _wide(A)).max() <= 128 * max(m, n) * u * np.abs(A).max(), (m, n, bs)
            if m == n:
                inv = np.full((n, n), np.nan, dtype=dtype, order="F")
                la.qr_inverse(inv, QR, H, QR)
                assert np.abs(_wide(inv) @ _wide(A) - np.eye(n)).max() <= 128 * n * u * np.linalg.cond(_wide(A)), (n, bs)


def test_f32_reconstruct_matches_f64(fb, cuda_dev):
    """The f32 entry points against the (already validated) f64 ones on the same f32-representable matrix."""
    la = fb.linalg
    rng = np.random.default_rng(244)
    n = 96
    G = rng.standard_normal((n, n)).astype(np.float32)
    A32 = np.asfortranarray((G.astype(np.float64) @ G.astype(np.float64).T + n * np.eye(n)).astype(np.float32))
    A64 = np.asfortranarray(A32.astype(np.float64))
    L32 = A32.copy(order="F"); la.cholesky_in_place(L32)
    L64 = A64.copy(order="F"); la.cholesky_in_place(L64)
    i32 = np.zeros((n, n), np.float32, order="F"); la.llt_inverse(i32, L32)
    i64 = np.zeros((n, n), np.float64, order="F"); la.llt_inverse(i64, L64)
    assert np.abs(np.tril(i32) - np.tril(i64)).max() <= 64 * n * _u(np.float32) * np.linalg.cond(A64) * np.abs(i64).max()
