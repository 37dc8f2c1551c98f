"""The compositions of csrc/reconstruct_types.cu (`*_reconstruct` / `*_inverse` on the factors), restated call
for call on the oracle's building blocks with the SAME structure codes and conjugation flags the CUDA file passes to the GPU's
products, solves and Householder sequences (which are tested against these very oracle functions on hardware). Pins the one
non-mechanical part of that file — which operand is conjugated, which sequence is applied — on the CPU:
  llt/reconstruct.rs:12-33, llt/inverse.rs:10-39, lu/partial_pivoting/reconstruct.rs:12-80, inverse.rs,
  qr/no_pivoting/reconstruct.rs:13-39, inverse.rs (reference tests: n = 50, (100, 50), (50, 100))."""
import numpy as np
import pytest

RECT, TRI_LOWER, TRI_UPPER, UNIT_LOWER = 0, 1, 2, 5
DTYPES = [np.float32, np.complex128, np.complex64]


def rand(rng, shape, dtype):
    a = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        a = a + 1j * rng.standard_normal(shape)
    return np.asfortranarray(a.astype(dtype))


def wide(x):
    return x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)


def tol(dtype, n):
    return 256 * n * float(np.finfo(dtype).eps)


# ---- the compositions, as reconstruct_types.cu issues them ----
def llt_reconstruct(orc, out, L):
    orc.matmul_triangular(out, TRI_LOWER, False, L, TRI_LOWER, L.T, TRI_UPPER, 1.0, conj_lhs=False, conj_rhs=True)


def llt_inverse(orc, out, L):
    n = L.shape[0]
    Li = np.asfortranarray(np.eye(n, dtype=L.dtype))
    orc.solve_triangular(L, Li, lower=True, unit=False, conj=False)
    orc.matmul_triangular(out, TRI_LOWER, False, Li.T, TRI_UPPER, Li, TRI_LOWER, 1.0, conj_lhs=True, conj_rhs=False)


def permute_rows(M, perm):
    M[...] = M[perm, :]


def lu_reconstruct(orc, out, L, U, perm_bwd):
    m, n = L.shape[0], U.shape[1]
    s = min(m, n)
    orc.matmul_triangular(out[:s, :s], RECT, False, L[:s, :s], UNIT_LOWER, U[:s, :s], TRI_UPPER, 1.0)
    if m > n:
        orc.matmul_triangular(out[s:, :s], RECT, False, L[s:, :s], RECT, U[:s, :s], TRI_UPPER, 1.0)
    if m < n:
        orc.matmul_triangular(out[:s, s:], RECT, False, L[:s, :s], UNIT_LOWER, U[:s, s:], RECT, 1.0)
    permute_rows(out, perm_bwd)


def lu_inverse(orc, out, L, U, perm_fwd):
    n = out.shape[0]
    out[...] = np.eye(n, dtype=out.dtype)
    permute_rows(out, perm_fwd)
    orc.solve_triangular(L, out, lower=True, unit=True, conj=False)
    orc.solve_triangular(U, out, lower=False, unit=False, conj=False)


def qr_reconstruct(orc, out, Qb, Qc, R):
    m, n = out.shape
    s = min(m, n)
    out[...] = 0
    out[:s, :] = np.triu(R[:s, :])
    orc.apply_q_sequence(Qb, Qc, out, conj_lhs=False)


def qr_inverse(orc, out, Qb, Qc, R):
    n = out.shape[0]
    out[...] = np.eye(n, dtype=out.dtype)
    orc.apply_q_transpose_sequence(Qb, Qc, out, conj_lhs=True)   # householder_sequence_t with conj = transpose = true
    orc.solve_triangular(R, out, lower=False, unit=False, conj=False)


@pytest.mark.parametrize("dtype", DTYPES)
def test_llt_compositions(oracle, dtype):
    rng = np.random.default_rng(1500)
    for n in [1, 50, 131]:
        G = wide(rand(rng, (n, n), dtype))
        A = np.asfortranarray((G @ G.conj().T + n * np.eye(n)).astype(dtype))
        L = A.copy(order="F")
        assert oracle.llt(L)[0] == -1
        out = np.full((n, n), np.nan, dtype=dtype, order="F"); out[np.tril_indices(n)] = 7
        llt_reconstruct(oracle, out, L)
        assert np.all(np.isnan(out[np.triu_indices(n, 1)]))
        assert np.abs(np.tril(wide(out)) - np.tril(wide(A))).max() <= tol(dtype, n) * np.abs(A).max()
        inv = np.full((n, n), np.nan, dtype=dtype, order="F"); inv[np.tril_indices(n)] = 7
        llt_inverse(oracle, inv, L)
        assert np.all(np.isnan(inv[np.triu_indices(n, 1)]))
        lo = np.tril(wide(inv)); full = lo + np.tril(lo, -1).conj().T
        assert np.abs(full @ wide(A) - np.eye(n)).max() <= tol(dtype, n) * np.linalg.cond(wide(A))


@pytest.mark.parametrize("dtype", DTYPES)
def test_lu_compositions(oracle, dtype):
    rng = np.random.default_rng(1501)
    for (m, n) in [(50, 50), (100, 50), (50, 100), (1, 1)]:
        A = rand(rng, (m, n), dtype)
        LU = A.copy(order="F")
        perm, perm_inv, _ = oracle.lu(LU)
        out = np.full((m, n), np.nan, dtype=dtype, order="F")
        lu_reconstruct(oracle, out, LU, LU, perm_inv)
        scale = np.abs(A).max() * max(1.0, float(np.abs(np.triu(LU)).max()))
        assert np.abs(wide(out) - wide(A)).max() <= tol(dtype, max(m, n)) * scale, (m, n)
        if m == n:
            inv = np.full((n, n), np.nan, dtype=dtype, order="F")
            lu_inverse(oracle, inv, LU, LU, perm)
            assert np.abs(wide(inv) @ wide(A) - np.eye(n)).max() <= tol(dtype, n) * np.linalg.cond(wide(A))


@pytest.mark.parametrize("dtype", DTYPES)
def test_qr_compositions(oracle, dtype):
    rng = np.random.default_rng(1502)
    for (m, n) in [(100, 50), (50, 100), (50, 50), (1, 1)]:
        A = rand(rng, (m, n), dtype)
        s = min(m, n)
        for bs in sorted({oracle.qr_recommended_block_size(m, n), min(7, s)}):
            QR = A.copy(order="F")
            H, rank = oracle.qr(QR, block_size=bs)
            assert rank == s
            out = np.full((m, n), np.nan, dtype=dtype, order="F")
            qr_reconstruct(oracle, out, np.asfortranarray(QR[:, :s]), H, QR[:s, :])
            assert np.abs(wide(out) - wide(A)).max() <= tol(dtype, max(m, n)) * np.abs(A).max(), (m, n, bs)
            if m == n:
                inv = np.full((n, n), np.nan, dtype=dtype, order="F")
                qr_inverse(oracle, inv, QR, H, QR)
                assert np.abs(wide(inv) @ wide(A) - np.eye(n)).max() <= tol(dtype, n) * np.linalg.cond(wide(A)), (n, bs)
