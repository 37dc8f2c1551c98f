"""numpy restatement of faer's pivoted Cholesky (faer/src/linalg/cholesky/llt_pivoting/factor.rs:47-199), the model the tests
check the library against, plus the solve / reconstruct / inverse compositions (solve.rs:13-41, reconstruct.rs:12-52,
inverse.rs:12-54).

The factorization follows the reference's operation order: the residual diagonal is `dot + |x|^2` then `Re a_ii - dot`, each a
separately rounded numpy operation (unfused, as the reference's Rust), the pivot is the first maximum with strict `>` from
(pvt = j, ajj = 0), the left-looking GEMV and the trailing update are numpy products. Integer outputs (status, rank,
transposition count, permutation) are therefore the reference's; the GEMV and the trailing update round differently from the
reference's kernels, which moves a pivot only at a near-tie."""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla


def _real_dtype(dt):
    return np.float32 if np.dtype(dt) in (np.dtype(np.float32), np.dtype(np.complex64)) else np.float64


def _abs2(x):
    if np.iscomplexobj(x):
        return x.real * x.real + x.imag * x.imag
    return x * x


def _scale(col, r):
    if np.iscomplexobj(col):
        col.real *= r
        col.imag *= r
    else:
        col *= r


def piv_llt(A, block_size=128):
    """In-place pivoted LLT of the lower triangle of A (2-D numpy array, any strides). Returns
    (ok, index, transposition_count, perm, perm_inv): ok = True -> index is the rank; ok = False -> NonPositivePivot { index }
    (perm_inv is then None, perm the identity with the swaps made so far)."""
    n = A.shape[0]
    assert A.shape == (n, n) and block_size > 0
    R = _real_dtype(A.dtype)
    perm = np.arange(n, dtype=np.int64)
    if n == 0:
        return True, 0, 0, perm, perm.copy()
    d0 = np.real(np.diagonal(A)).astype(R)
    if np.any(d0 < 0) or np.any(np.isnan(d0)):
        return False, 0, 0, perm, None
    m = d0.max()
    pvt, ajj = (int(np.argmax(d0)), R(m)) if m > 0 else (0, R(0))
    tol = R(np.finfo(R).eps) * R(n) * ajj
    dot = np.zeros(n, dtype=R)
    diag = np.zeros(n, dtype=R)
    rank, tc = n, 0
    with np.errstate(all="ignore"):
        k = 0
        while k < n and rank == n:
            bs = min(n - k, block_size)
            dot[k:] = 0
            for j in range(k, k + bs):
                ad = np.real(np.diagonal(A)[j:]).astype(R)
                if j == k:
                    diag[j:] = ad
                else:
                    dot[j:] = dot[j:] + _abs2(A[j:, j - 1]).astype(R)
                    diag[j:] = ad - dot[j:]
                if j > 0:
                    seg = diag[j:]
                    if np.any(np.isnan(seg)):
                        return False, j, tc, perm, None
                    m = seg.max()
                    pvt, ajj = (j + int(np.argmax(seg)), R(m)) if m > 0 else (j, R(0))
                    if ajj < tol:
                        A[j, j] = ajj
                        rank = j
                        break
                if pvt != j:
                    tc += 1
                    A[pvt, pvt] = A[j, j]
                    A[[j, pvt], :j] = A[[pvt, j], :j]
                    A[pvt + 1:, [j, pvt]] = A[pvt + 1:, [pvt, j]]
                    a = A[j + 1:pvt, j].copy()
                    b = A[pvt, j + 1:pvt].copy()
                    A[j + 1:pvt, j] = np.conj(b)
                    A[pvt, j + 1:pvt] = np.conj(a)
                    A[pvt, j] = np.conj(A[pvt, j])
                    dot[j], dot[pvt] = dot[pvt], dot[j]
                    perm[j], perm[pvt] = perm[pvt], perm[j]
                ajj = np.sqrt(ajj)
                A[j, j] = ajj
                if j > k:
                    A[j + 1:, j] -= A[j + 1:, k:j] @ np.conj(A[j, k:j])
                _scale(A[j + 1:, j], R(1) / ajj)
            if rank == n and k + bs < n:
                P = A[k + bs:, k:k + bs]
                D = P @ np.conj(P.T)
                A[k + bs:, k + bs:] -= np.tril(D)  # the strict upper triangle loses exact zeros: unchanged
            k += bs
    perm_inv = np.empty(n, dtype=np.int64)
    perm_inv[perm] = np.arange(n)
    return True, rank, tc, perm, perm_inv


def sym_gather(tmp, p):
    """out(i, j), i >= j: tmp(p[i], p[j]) if p[i] >= p[j] else conj(tmp(p[j], p[i])) (reconstruct.rs:40-51); returns the lower
    triangle (zeros above it)."""
    p = np.asarray(p, dtype=np.int64)
    ii, jj = p[:, None], p[None, :]
    return np.tril(np.where(ii >= jj, tmp[ii, jj], np.conj(tmp[jj, ii])))


def reconstruct(L, perm_inv):
    Lt = np.tril(L)
    return sym_gather(np.tril(Lt @ np.conj(Lt.T)), perm_inv)


def inverse(L, perm_inv):
    Li = sla.solve_triangular(np.tril(L), np.eye(L.shape[0], dtype=L.dtype), lower=True)
    return sym_gather(np.tril(np.conj(Li.T) @ Li), perm_inv)


def solve(L, perm, perm_inv, rhs, conj=False):
    """solve.rs:13-41: permute by perm, L (conj?) solve, L^H (conj?) solve, permute back by perm_inv."""
    Lc = np.conj(np.tril(L)) if conj else np.tril(L)
    x = rhs[perm]
    x = sla.solve_triangular(Lc, x, lower=True)
    x = sla.solve_triangular(np.conj(Lc.T), x, lower=False)
    return x[perm_inv]


def mirror(lower):
    """Hermitian matrix from its lower triangle."""
    return np.tril(lower) + np.conj(np.tril(lower, -1).T)
