"""Componentwise backward-error checks for f64 LLT and partial-pivoting LU, and NaN sentinels around a matrix.

The bounds hold for any correct f64 implementation, whatever its blocking or summation order, so they carry no tuning to
observed errors (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Theorems 9.3 and 10.3):

  LLT   |tril(A0 - L L^T)|  <=  2 gamma_{n+2} |L| |L|^T + u |A0|        (lower triangle, entry by entry)
  LU    |P A0 - L U|        <=  2 gamma_{n+2} |L| |U|   + u |P A0|

with gamma_m = m u / (1 - m u). One gamma term is the factorization's, the other the error of evaluating the residual in
f64; the +2 absorbs the reciprocal-multiply scaling of a column, which rounds twice; u |A0| covers the final subtraction.
Everything runs in torch on whichever device holds the tensors. The ratio functions return the largest error-to-bound
ratio (a pass is <= 1; a NaN residual counts as infinite), so a test can report how much margin a kernel leaves.

Sentinels: a matrix is placed inside a larger buffer whose other elements (padding rows between n and ld, a leading
offset, optionally the strict upper triangle) hold a quiet NaN with a recognisable payload; `changed_outside` counts the
elements a call was not allowed to write whose bits differ afterwards.
"""
import torch

U = 2.0 ** -53
SENTINEL = 0x7FF8_5E47_1AE1_0BAD  # quiet NaN, payload recognisable in a hex dump


def gamma(m: int) -> float:
    return m * U / (1.0 - m * U)


def _max_ratio(err, bound) -> float:
    r = err / bound  # 0 / 0 -> NaN (exact entry under a zero bound: ratio 0), e / 0 -> inf
    r.masked_fill_((err == 0) & (bound == 0), 0.0)
    r = torch.nan_to_num(r, nan=float("inf"), posinf=float("inf"))  # a NaN residual fails
    return float(r.max()) if r.numel() else 0.0


def llt_residual(A0, L):
    """(|tril(A0 - L L^T)|, 2 gamma_{n+2} tril(|L||L|^T) + u |tril(A0)|). Only the lower triangles of A0 and L are read
    (the strict upper parts may hold anything, NaN included)."""
    n = A0.shape[0]
    A0 = torch.tril(A0)
    L = torch.tril(L)
    err = (A0 - torch.tril(L @ L.T)).abs_()
    La = L.abs_()
    bound = torch.tril(La @ La.T).mul_(2.0 * gamma(n + 2)).add_(A0.abs_(), alpha=U)
    return err, bound


def llt_ratio(A0, L) -> float:
    """Largest entry of |tril(A0 - L L^T)| / (2 gamma_{n+2} |L||L|^T + u |A0|); <= 1 passes."""
    return _max_ratio(*llt_residual(A0, L))


def lu_residual(A0, LU, perm):
    """(|A0[perm] - L U|, 2 gamma_{n+2} |L||U| + u |A0[perm]|) for a square packed factor (unit-lower L strictly below the
    diagonal, U on and above it); (P A0)[i, :] = A0[perm[i], :]."""
    n = A0.shape[0]
    PA = A0[torch.as_tensor(perm, device=A0.device, dtype=torch.int64), :]
    L = torch.tril(LU, -1)
    L.diagonal().fill_(1.0)
    Um = torch.triu(LU)
    err = (PA - L @ Um).abs_()
    bound = (L.abs_() @ Um.abs_()).mul_(2.0 * gamma(n + 2)).add_(PA.abs_(), alpha=U)
    return err, bound


def lu_ratio(A0, LU, perm) -> float:
    """Largest entry of |P A0 - L U| / (2 gamma_{n+2} |L||U| + u |P A0|); <= 1 passes."""
    return _max_ratio(*lu_residual(A0, LU, perm))


def sentinel_buffer(numel: int, device) -> torch.Tensor:
    """1-D float64 buffer with every element set to the sentinel NaN."""
    return torch.full((numel,), SENTINEL, dtype=torch.int64, device=device).view(torch.float64)


def matrix_in(buf, n: int, ld: int, offset: int = 0, row_major: bool = False):
    """n x n view of `buf` starting at element `offset`: column-major (strides (1, ld)) or row-major (strides (ld, 1))."""
    M = buf[offset:offset + ld * n].view(n, ld)[:, :n]
    return M if row_major else M.T


def changed_outside(buf, before, writable) -> int:
    """Number of elements of `buf` outside the boolean mask `writable` (same shape) whose bits differ from `before`."""
    diff = buf.view(torch.int64) != before.view(torch.int64)
    return int((diff & ~writable).sum())
