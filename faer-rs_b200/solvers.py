"""High-level decompositions over the C ABI: the ergonomic surface of faer (`A.llt(Side::Lower)?.solve(&b)`,
`A.partial_piv_lu()`, `A.qr().solve_lstsq(&b)`, `&A * &B`) for the factorizations on the hot path (SURVEY.md §8f rank 2).

Reference: faer/src/linalg/solvers.rs
    Llt::new / new_imp / L                      770-816   (copy the chosen triangle, factor, zero the strict upper part)
    split_LU                                    955-980   (packed factors -> unit-lower L and upper U, both owned)
    PartialPivLu::new / L / U / P               981-1034
    Qr::new / Q_basis / Q_coeff / R / thin_R / compute_Q / compute_thin_Q   1106-1205
    ColPivQr::new / Q_basis / Q_coeff / R / thin_R / P / compute_Q / compute_thin_Q   1206-1260
    Solve / SolveLstsq extension traits         93-282, 639-690  (solve, solve_conjugate, solve_transpose, solve_adjoint and
                                                                   the rsolve_* family through the transposed system)
    SolveCore impls                             1861-1905 (Llt), 2147-2196 (PartialPivLu), 2339-2418 (Qr), 2462-2530 (ColPivQr)
    DenseSolveCore::reconstruct / inverse       1917-1936 (Llt), 2198-2217 (PartialPivLu), 2420-2440 (Qr), 2532-2560 (ColPivQr)
and faer/src/mat/mat_ops.rs:869-897 (`Mul` for matrices -> `mul`).

Every flop runs in libfaer_b200.so through `linalg.py`; this module only owns buffers, splits the packed factors and
orders the calls the way the reference does. Operands are numpy arrays (host; staged by the library) or torch CUDA
tensors (device; used in place); results are of the same kind, column-major. Llt, PartialPivLu and Qr take real (f64; Qr and Llt
also f32) and complex (c64 / c32) matrices — the reference's own `test_all_solvers` runs on c64 —, with the `Conj` argument of
the C ABI carrying the conjugate / adjoint variants; Ldlt, Svd and SelfAdjointEigen are real-only (their kernels are).
`inverse` is `solve` applied to the identity (the reference has dedicated kernels: `*/inverse.rs`); same result up
to rounding.
"""
from __future__ import annotations

import numpy as np

from . import capi
from . import linalg as la
from .linalg import LdltError, LltError  # noqa: F401  (re-exported: Llt.new / Ldlt.new raise them)


class Side:
    Lower = 0
    Upper = 1


# ---- buffer helpers: numpy (host) or torch (device), always column-major ------------------------------------------
def _t(x) -> bool:
    return capi._is_torch(x)


def _owned(A):
    """Column-major owned copy (Mat::to_owned)."""
    if _t(A):
        import torch
        return A.t().clone(memory_format=torch.contiguous_format).t()
    return np.array(A, order="F", copy=True)


def _zeros(like, m, n):
    if _t(like):
        import torch
        return torch.zeros((n, m), dtype=like.dtype, device=like.device).t()
    return np.zeros((m, n), dtype=like.dtype, order="F")


def _identity(like, m, n):
    out = _zeros(like, m, n)
    if _t(out):
        out.diagonal().fill_(1)
    else:
        np.fill_diagonal(out, 1)
    return out


def _is_cplx(x) -> bool:
    if _t(x):
        return x.is_complex()
    return np.iscomplexobj(x)


def _conj(x):
    """Element-wise conjugate as an owned value (the identity for real scalars)."""
    if not _is_cplx(x):
        return x
    if _t(x):
        return x.conj().resolve_conj()
    return np.conj(x)


def _adjoint(x):
    return _conj(x).T


def _zero_strict_upper(A):
    if _t(A):
        A.tril_()
    else:
        A[np.triu_indices(A.shape[0], 1, A.shape[1])] = 0


def _zero_strict_lower(A):
    if _t(A):
        A.triu_()
    else:
        A[np.tril_indices(A.shape[0], -1, A.shape[1])] = 0


def _fill_diag_one(A):
    if _t(A):
        A.diagonal().fill_(1)
    else:
        np.fill_diagonal(A, 1)


def _tri(A, lower: bool, k: int = 0):
    if _t(A):
        import torch
        return torch.tril(A, k) if lower else torch.triu(A, k)
    return np.tril(A, k) if lower else np.triu(A, k)


def _assign(dst, src):
    if _t(dst):
        dst.copy_(src)
    else:
        dst[...] = src


def _as_2d(x):
    """Vectors are n x 1 matrices (the reference's `AsMatMut` for `Col`)."""
    if x.ndim == 1:
        return x.reshape(-1, 1) if not _t(x) else x.unsqueeze(1)
    return x


def split_LU(LU):
    """solvers.rs:955-980. Consumes LU. m >= n: (LU with its strict upper part zeroed and a unit diagonal, upper
    triangle copied out as size x size); m < n: (unit-lower size x size copy, LU with its strict lower part zeroed)."""
    m, n = LU.shape
    size = min(m, n)
    if m >= n:
        L = LU
        U = _zeros(LU, size, size)
        _assign(U, _tri(L[:size, :size], lower=False))
        _zero_strict_upper(L)
        _fill_diag_one(L)
    else:
        U = LU
        L = _zeros(LU, size, size)
        _assign(L, _tri(U[:size, :size], lower=True, k=-1))
        _zero_strict_lower(U)
        _fill_diag_one(L)
    return L, U


def mul(A, B):
    """`&A * &B` (mat_ops.rs:869-897): owned product through matmul (Accum::Replace, alpha = 1)."""
    assert A.shape[1] == B.shape[0]
    out = _zeros(A, A.shape[0], B.shape[1])
    la.matmul(out, la.Accum.Replace, A, B, 1.0)
    return out


class _Solve:
    """The `Solve` extension trait (solvers.rs:93-282) over the two core operations of a decomposition."""

    def nrows(self) -> int:
        raise NotImplementedError

    def ncols(self) -> int:
        raise NotImplementedError

    def _solve_core(self, rhs, conj: int) -> None:  # SolveCore::solve_in_place_with_conj: rhs <- conj?(A)^-1 rhs
        raise NotImplementedError

    def _solve_transpose_core(self, rhs, conj: int) -> None:  # SolveCore::solve_transpose_in_place_with_conj: conj?(A)^-T rhs
        raise NotImplementedError

    def _sq(self, rhs):
        r = _as_2d(rhs)
        assert self.nrows() == self.ncols() == r.shape[0]
        return r

    # in place (solvers.rs:93-185)
    def solve_in_place(self, rhs) -> None:
        self._solve_core(self._sq(rhs), la.CONJ_NO)

    def solve_conjugate_in_place(self, rhs) -> None:
        self._solve_core(self._sq(rhs), la.CONJ_YES)

    def solve_transpose_in_place(self, rhs) -> None:
        self._solve_transpose_core(self._sq(rhs), la.CONJ_NO)

    def solve_adjoint_in_place(self, rhs) -> None:
        self._solve_transpose_core(self._sq(rhs), la.CONJ_YES)

    # owned results
    def _owned_solve(self, rhs, f):
        out = _owned(_as_2d(rhs))
        f(out)
        return out

    def solve(self, rhs):
        return self._owned_solve(rhs, self.solve_in_place)

    def solve_conjugate(self, rhs):
        return self._owned_solve(rhs, self.solve_conjugate_in_place)

    def solve_transpose(self, rhs):
        return self._owned_solve(rhs, self.solve_transpose_in_place)

    def solve_adjoint(self, rhs):
        return self._owned_solve(rhs, self.solve_adjoint_in_place)

    # X op(A) = lhs  <=>  op(A)^T X^T = lhs^T   (solvers.rs:186-282)
    def rsolve(self, lhs):
        return _owned(self.solve_transpose(_as_2d(lhs).T).T)

    def rsolve_conjugate(self, lhs):
        return _owned(self.solve_adjoint(_as_2d(lhs).T).T)

    def rsolve_transpose(self, lhs):
        return _owned(self.solve(_as_2d(lhs).T).T)

    def rsolve_adjoint(self, lhs):
        return _owned(self.solve_conjugate(_as_2d(lhs).T).T)

    def rsolve_in_place(self, lhs) -> None:
        _assign(lhs, self.rsolve(lhs))

    def rsolve_transpose_in_place(self, lhs) -> None:
        _assign(lhs, self.rsolve_transpose(lhs))

    def inverse(self):
        assert self.nrows() == self.ncols()
        out = _identity(self._like(), self.nrows(), self.nrows())
        self._solve_core(out, la.CONJ_NO)
        return out

    def _like(self):
        raise NotImplementedError


class Llt(_Solve):
    """A = L L^H (solvers.rs:770-816). `Llt.new(A, side)` raises LltError(index) on a non-positive pivot."""

    def __init__(self, L):
        self._L = L

    @classmethod
    def new(cls, A, side: int = Side.Lower) -> "Llt":
        assert A.ndim == 2 and A.shape[0] == A.shape[1]
        n = A.shape[0]
        L = _zeros(A, n, n)
        # copy_from_triangular_lower(A) / (A.adjoint()): only the chosen triangle of A is read
        _assign(L, _tri(A if side == Side.Lower else _adjoint(A), lower=True))
        la.cholesky_in_place(L)  # default regularization and params; LltError propagates
        _zero_strict_upper(L)
        return cls(L)

    def L(self):
        return self._L

    def nrows(self) -> int:
        return self._L.shape[0]

    ncols = nrows

    def _like(self):
        return self._L

    def _solve_core(self, rhs, conj: int) -> None:
        la.llt_solve_in_place(self._L, rhs, conj)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        # A^T = conj(A) for a self-adjoint A: conj composed with Yes (solvers.rs:1883-1904)
        la.llt_solve_in_place(self._L, rhs, la.CONJ_NO if conj == la.CONJ_YES else la.CONJ_YES)

    def reconstruct(self):
        """llt/reconstruct.rs: lower triangle of L L^H through the triangular product, then mirrored
        (make_self_adjoint, solvers.rs:1906-1915)."""
        n = self.nrows()
        out = _zeros(self._L, n, n)
        la.matmul_triangular(out, la.BlockStructure.TriangularLower, la.Accum.Replace, self._L,
                             la.BlockStructure.TriangularLower, _adjoint(self._L), la.BlockStructure.TriangularUpper, 1.0)
        _assign(out, _tri(out, lower=True) + _adjoint(_tri(out, lower=True, k=-1)))
        return out


class Ldlt(_Solve):
    """A = L D L^H without pivoting (solvers.rs:818-872): unit-lower L (explicit unit diagonal, zero strict upper part) and
    the diagonal D as a vector. `Ldlt.new(A, side)` raises LdltError(index) on a zero pivot."""

    def __init__(self, L, D):
        self._L, self._D = L, D

    @classmethod
    def new(cls, A, side: int = Side.Lower) -> "Ldlt":
        assert A.ndim == 2 and A.shape[0] == A.shape[1]
        n = A.shape[0]
        L = _zeros(A, n, n)
        _assign(L, _tri(A if side == Side.Lower else _adjoint(A), lower=True))  # Upper: the lower triangle of the adjoint
        la.ldlt_in_place(L)  # default regularization and params; LdltError propagates
        if _t(L):
            D = L.diagonal().clone()
        else:
            D = np.ascontiguousarray(np.diagonal(L).copy())
        _fill_diag_one(L)
        _zero_strict_upper(L)
        return cls(L, D)

    def L(self):
        return self._L

    def D(self):
        return self._D

    def nrows(self) -> int:
        return self._L.shape[0]

    ncols = nrows

    def _like(self):
        return self._L

    def _solve_core(self, rhs, conj: int) -> None:
        la.ldlt_solve_in_place(self._L, rhs, conj, D=self._D)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        # A^T = conj(A) for a self-adjoint A: conj composed with Yes (as Llt above)
        la.ldlt_solve_in_place(self._L, rhs, la.CONJ_NO if conj == la.CONJ_YES else la.CONJ_YES, D=self._D)

    def reconstruct(self):
        """ldlt/reconstruct.rs: L D L^H."""
        LDm = _owned(self._L)
        if _t(LDm):
            LDm.mul_(self._D.unsqueeze(0))
        else:
            LDm *= self._D[None, :]
        return mul(LDm, _adjoint(self._L))


class Lblt(_Solve):
    """P A P^T = L B L^H, Bunch-Kaufman pivoting (solvers.rs Lblt): the factored matrix holds L strictly below the diagonal and
    B's diagonal on it, `subdiag()` B's subdiagonal (zeroed before the factorization, as the reference does). Factors the
    indefinite self-adjoint matrices that Ldlt cannot, such as saddle-point systems. `P()` returns (perm_fwd, perm_bwd)."""

    def __init__(self, LB, sub, fwd, bwd):
        self._LB, self._sub, self._fwd, self._bwd = LB, sub, fwd, bwd

    @classmethod
    def new(cls, A, side: int = Side.Lower, params=None) -> "Lblt":
        assert A.ndim == 2 and A.shape[0] == A.shape[1]
        n = A.shape[0]
        LB = _zeros(A, n, n)
        _assign(LB, _tri(A if side == Side.Lower else _adjoint(A), lower=True))
        if _t(LB):
            import torch
            sub = torch.zeros(n, dtype=LB.dtype, device=LB.device)
            fwd, bwd = (torch.zeros(n, dtype=torch.int64, device=LB.device) for _ in range(2))
        else:
            sub = np.zeros(n, dtype=LB.dtype)
            fwd, bwd = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
        la.lblt_in_place(LB, sub, fwd, bwd, params=params)
        return cls(LB, sub, fwd, bwd)

    def LB(self):
        return self._LB

    def subdiag(self):
        return self._sub

    def P(self):
        return self._fwd, self._bwd

    def nrows(self) -> int:
        return self._LB.shape[0]

    ncols = nrows

    def _like(self):
        return self._LB

    def _solve_core(self, rhs, conj: int) -> None:
        la.lblt_solve_in_place(self._LB, self._sub, self._fwd, self._bwd, rhs, conj)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        # A^T = conj(A) for a self-adjoint A: conj composed with Yes (as Llt above)
        la.lblt_solve_in_place(self._LB, self._sub, self._fwd, self._bwd, rhs, la.CONJ_NO if conj == la.CONJ_YES else la.CONJ_YES)

    def reconstruct(self):
        """bunch_kaufman/reconstruct.rs: the lower triangle of A, mirrored (make_self_adjoint)."""
        n = self.nrows()
        out = _zeros(self._LB, n, n)
        la.lblt_reconstruct(out, self._LB, self._sub, self._fwd, self._bwd)
        _assign(out, _tri(out, lower=True) + _adjoint(_tri(out, lower=True, k=-1)))
        return out

    def inverse(self):
        """bunch_kaufman/inverse.rs."""
        n = self.nrows()
        out = _zeros(self._LB, n, n)
        la.lblt_inverse(out, self._LB, self._sub, self._fwd, self._bwd)
        return out


class PartialPivLu(_Solve):
    """P A = L U (solvers.rs:981-1034). `P()` returns (perm_fwd, perm_bwd): (P A)[i, :] = A[perm_fwd[i], :]."""

    def __init__(self, L, U, fwd, bwd, m, n):
        self._L, self._U, self._fwd, self._bwd, self._m, self._n = L, U, fwd, bwd, m, n

    @classmethod
    def new(cls, A) -> "PartialPivLu":
        assert A.ndim == 2
        LU = _owned(A)
        m, n = LU.shape
        if _t(LU):
            import torch
            fwd = torch.zeros(m, dtype=torch.int64, device=LU.device)
            bwd = torch.zeros(m, dtype=torch.int64, device=LU.device)
        else:
            fwd = np.zeros(m, dtype=np.uint64)
            bwd = np.zeros(m, dtype=np.uint64)
        la.lu_in_place(LU, fwd, bwd)
        L, U = split_LU(LU)
        return cls(L, U, fwd, bwd, m, n)

    def L(self):
        return self._L

    def U(self):
        return self._U

    def P(self):
        return self._fwd, self._bwd

    def nrows(self) -> int:
        return self._m

    def ncols(self) -> int:
        return self._n

    def _like(self):
        return self._L

    def _solve_core(self, rhs, conj: int) -> None:
        la.lu_solve_in_place(self._L, self._fwd, self._bwd, rhs, conj, U=self._U)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        la.lu_solve_transpose_in_place(self._L, self._fwd, self._bwd, rhs, conj, U=self._U)

    def reconstruct(self):
        """lu/partial_pivoting/reconstruct.rs: tmp = L U by structured products, then out[perm_fwd[i], :] = tmp[i, :]."""
        m, n = self._m, self._n
        size = min(m, n)
        BS = la.BlockStructure
        tmp = _zeros(self._L, m, n)
        la.matmul_triangular(tmp[:size, :size], BS.Rectangular, la.Accum.Replace, self._L[:size, :size],
                             BS.UnitTriangularLower, self._U[:size, :size], BS.TriangularUpper, 1.0)
        if m > n:
            la.matmul_triangular(tmp[size:, :size], BS.Rectangular, la.Accum.Replace, self._L[size:, :size], BS.Rectangular,
                                 self._U[:size, :size], BS.TriangularUpper, 1.0)
        if m < n:
            la.matmul_triangular(tmp[:size, size:], BS.Rectangular, la.Accum.Replace, self._L[:size, :size],
                                 BS.UnitTriangularLower, self._U[:size, size:], BS.Rectangular, 1.0)
        out = _zeros(self._L, m, n)
        if _t(out):
            out[self._fwd.long()] = tmp
        else:
            out[self._fwd.astype(np.int64)] = tmp
        return out


class FullPivLu(_Solve):
    """P A Q = L U with full pivoting (solvers.rs:1036-1105; SolveCore 2241-2292, DenseSolveCore 2294-2330). `P()` / `Q()`
    return (perm_fwd, perm_bwd): (P A Q)[i, j] = A[P_fwd[i], Q_fwd[j]]."""

    def __init__(self, L, U, row, col, m, n):
        self._L, self._U, self._row, self._col, self._m, self._n = L, U, row, col, m, n

    @classmethod
    def new(cls, A) -> "FullPivLu":
        assert A.ndim == 2
        LU = _owned(A)
        m, n = LU.shape

        def perm(k):
            if _t(LU):
                import torch
                return torch.zeros(k, dtype=torch.int64, device=LU.device)
            return np.zeros(k, dtype=np.uint64)

        row = (perm(m), perm(m))
        col = (perm(n), perm(n))
        la.full_piv_lu_in_place(LU, row[0], row[1], col[0], col[1])
        L, U = split_LU(LU)
        return cls(L, U, row, col, m, n)

    def L(self):
        return self._L

    def U(self):
        return self._U

    def P(self):
        return self._row

    def Q(self):
        return self._col

    def nrows(self) -> int:
        return self._m

    def ncols(self) -> int:
        return self._n

    def _like(self):
        return self._L

    def _solve_core(self, rhs, conj: int) -> None:
        la.full_piv_lu_solve_in_place(self._L, self._U, *self._row, *self._col, rhs, conj)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        la.full_piv_lu_solve_transpose_in_place(self._L, self._U, *self._row, *self._col, rhs, conj)

    def reconstruct(self):
        """full_pivoting/reconstruct.rs:13-82: A from the factors."""
        out = _zeros(self._L, self._m, self._n)
        la.full_piv_lu_reconstruct(out, self._L, self._U, *self._row, *self._col)
        return out

    def inverse(self):
        """full_pivoting/inverse.rs:12-63."""
        assert self._m == self._n
        out = _zeros(self._L, self._m, self._m)
        la.full_piv_lu_inverse(out, self._L, self._U, *self._row, *self._col)
        return out


class Qr(_Solve):
    """A = Q R, Householder QR without pivoting (solvers.rs:1106-1205). Q is kept as the Householder basis (unit-lower
    trapezoid) and the block coefficients; `compute_Q` / `compute_thin_Q` form it."""

    def __init__(self, Q_basis, Q_coeff, R, m, n):
        self._Qb, self._Qc, self._R, self._m, self._n = Q_basis, Q_coeff, R, m, n

    @classmethod
    def new(cls, A) -> "Qr":
        assert A.ndim == 2
        QR = _owned(A)
        m, n = QR.shape
        size = min(m, n)
        bs = la.qr_recommended_block_size(m, n)
        Q_coeff = _zeros(QR, bs, size)
        la.qr_in_place(QR, Q_coeff)
        Q_basis, R = split_LU(QR)
        return cls(Q_basis, Q_coeff, R, m, n)

    def Q_basis(self):
        return self._Qb

    def Q_coeff(self):
        return self._Qc

    def R(self):
        return self._R

    def thin_R(self):
        return self._R[:min(self._m, self._n), :]

    def nrows(self) -> int:
        return self._m

    def ncols(self) -> int:
        return self._n

    def _like(self):
        return self._R

    def compute_Q(self):
        Q = _identity(self._R, self._m, self._m)
        la.apply_block_householder_sequence_on_the_left_in_place(self._Qb, self._Qc, Q)
        return Q

    def compute_thin_Q(self):
        Q = _identity(self._R, self._m, min(self._m, self._n))
        la.apply_block_householder_sequence_on_the_left_in_place(self._Qb, self._Qc, Q)
        return Q

    def _solve_core(self, rhs, conj: int) -> None:
        la.qr_solve_in_place(self._Qb, self._Qc, self._R, rhs, conj)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        la.qr_solve_transpose_in_place(self._Qb, self._Qc, self._R, rhs, conj)

    # SolveLstsq (solvers.rs:639-690)
    def _lstsq(self, rhs, conj: int) -> None:
        r = _as_2d(rhs)
        assert self._m == r.shape[0] and self._m >= self._n
        la.qr_solve_lstsq_in_place(self._Qb, self._Qc, self._R, r, conj)

    def solve_lstsq_in_place(self, rhs) -> None:
        self._lstsq(rhs, la.CONJ_NO)

    def solve_conjugate_lstsq_in_place(self, rhs) -> None:
        self._lstsq(rhs, la.CONJ_YES)

    def solve_lstsq(self, rhs):
        out = _owned(_as_2d(rhs))
        self.solve_lstsq_in_place(out)
        return _owned(out[:self._n, :])  # truncate(ncols, rhs_ncols)

    def solve_conjugate_lstsq(self, rhs):
        out = _owned(_as_2d(rhs))
        self.solve_conjugate_lstsq_in_place(out)
        return _owned(out[:self._n, :])

    def reconstruct(self):
        """qr/no_pivoting/reconstruct.rs: out = R padded to m rows, then out <- Q out."""
        m, n = self._m, self._n
        size = min(m, n)
        out = _zeros(self._R, m, n)
        _assign(out[:size, :], self.thin_R())
        la.apply_block_householder_sequence_on_the_left_in_place(self._Qb, self._Qc, out)
        return out


class ColPivQr(Qr):
    """A P = Q R, column-pivoted Householder QR (solvers.rs:738, 1206-1260, 2462-2560). `P()` returns (perm_fwd, perm_bwd):
    (A P)[:, j] = A[:, perm_fwd[j]]. Q is kept as for `Qr`; solves, reconstruct and inverse go through the library's
    `colpiv_qr_*` entry points, which apply the permutation."""

    def __init__(self, Q_basis, Q_coeff, R, fwd, bwd, m, n):
        super().__init__(Q_basis, Q_coeff, R, m, n)
        self._fwd, self._bwd = fwd, bwd

    @classmethod
    def new(cls, A) -> "ColPivQr":
        assert A.ndim == 2
        QR = _owned(A)
        m, n = QR.shape
        size = min(m, n)
        bs = la.qr_recommended_block_size(m, n)
        Q_coeff = _zeros(QR, bs, size)
        if _t(QR):
            import torch
            fwd = torch.zeros(n, dtype=torch.int64, device=QR.device)
            bwd = torch.zeros(n, dtype=torch.int64, device=QR.device)
        else:
            fwd = np.zeros(n, dtype=np.uint64)
            bwd = np.zeros(n, dtype=np.uint64)
        la.colpiv_qr_in_place(QR, Q_coeff, fwd, bwd)
        Q_basis, R = split_LU(QR)
        return cls(Q_basis, Q_coeff, R, fwd, bwd, m, n)

    def P(self):
        return self._fwd, self._bwd

    def _solve_core(self, rhs, conj: int) -> None:
        la.colpiv_qr_solve_in_place(self._Qb, self._Qc, self._R, self._fwd, self._bwd, rhs, conj)

    def _solve_transpose_core(self, rhs, conj: int) -> None:
        la.colpiv_qr_solve_transpose_in_place(self._Qb, self._Qc, self._R, self._fwd, self._bwd, rhs, conj)

    def _lstsq(self, rhs, conj: int) -> None:
        r = _as_2d(rhs)
        assert self._m == r.shape[0] and self._m >= self._n
        la.colpiv_qr_solve_lstsq_in_place(self._Qb, self._Qc, self._R, self._fwd, self._bwd, r, conj)

    def reconstruct(self):
        """col_pivoting/reconstruct.rs: Q R P^T."""
        out = _zeros(self._R, self._m, self._n)
        la.colpiv_qr_reconstruct(out, self._Qb, self._Qc, self.thin_R(), self._fwd, self._bwd)
        return out

    def inverse(self):
        """col_pivoting/inverse.rs: P R^-1 Q^H (square A)."""
        assert self._m == self._n
        out = _zeros(self._R, self._n, self._n)
        la.colpiv_qr_inverse(out, self._Qb, self._Qc, self._R, self._fwd, self._bwd)
        return out


class Svd:
    """`Svd<T>` (solvers.rs:1324-1400): `new` = full U and V, `new_thin` = the first min(nrows, ncols) columns of each;
    A = U diag(S) V^H, S non-increasing. Accessors U(), V(), S() as in the reference; pseudoinverse() = V S^+ U^H
    (solvers.rs:1390-1400 / svd::pseudoinverse_from_svd)."""

    def __init__(self, U, S, V):
        self._U, self._S, self._V = U, S, V

    @classmethod
    def _new(cls, A, thin: bool):
        m, n = A.shape
        size = min(m, n)
        U = la._new_mat(A, m, size if thin else m)
        V = la._new_mat(A, n, size if thin else n)
        if capi._is_torch(A):
            import torch
            S = torch.zeros(size, dtype=A.dtype, device=A.device)
        else:
            S = np.zeros(size, dtype=A.dtype)
        la.svd(A, S, U, V)
        return cls(U, la._real_values(S), V)  # the ABI's S is T-typed; the singular values are kept real

    @classmethod
    def new(cls, A):
        return cls._new(A, False)

    @classmethod
    def new_thin(cls, A):
        return cls._new(A, True)

    def U(self):
        return self._U

    def V(self):
        return self._V

    def S(self):
        return self._S

    def pseudoinverse(self):
        """V diag(1 / s_i for s_i above eps * max(nrows, ncols) * s_max, else 0) U^H (svd/mod.rs pseudoinverse_from_svd)."""
        S = self._S
        size = S.shape[0]
        if size == 0:
            return la._new_mat(self._U, self._V.shape[0], self._U.shape[0])
        xp_abs = abs
        smax = float(S[0])
        eps = float(np.finfo(np.float64 if str(S.dtype).endswith("64") else np.float32).eps)
        tol = eps * max(self._U.shape[0], self._V.shape[0]) * smax
        inv = S.clone() if capi._is_torch(S) else S.copy()
        mask = S > tol
        inv[mask] = 1.0 / S[mask]
        inv[~mask] = 0
        Vt = self._V[:, :size] * inv[None, :]
        out = la._new_mat(self._U, self._V.shape[0], self._U.shape[0])
        la.matmul(out, la.Accum.Replace, Vt, _conj(self._U[:, :size]).T, 1.0)
        return out


class SelfAdjointEigen:
    """`SelfAdjointEigen<T>` (solvers.rs:1459-1520): A = U diag(S) U^H from the chosen triangle, S nondecreasing."""

    def __init__(self, U, S):
        self._U, self._S = U, S

    @classmethod
    def new(cls, A, side: int = Side.Lower):
        n = A.shape[0]
        U = la._new_mat(A, n, n)
        if capi._is_torch(A):
            import torch
            S = torch.zeros(n, dtype=A.dtype, device=A.device)
        else:
            S = np.zeros(n, dtype=A.dtype)
        la.self_adjoint_evd(A if side == Side.Lower else _conj(A).T, S, U)  # Upper: the lower triangle of the adjoint
        return cls(U, la._real_values(S))

    def U(self):
        return self._U

    def S(self):
        return self._S


class Eigen:
    """`Eigen<T>` (solvers.rs: `Eigen::new`, `new_from_real`, `new_from_complex`): A U = U diag(S) for a general square A, with U
    and S complex also for real A (a real conjugate pair's packed columns k, k + 1 become column k +- i column k + 1)."""

    def __init__(self, U, S):
        self._U, self._S = U, S

    @classmethod
    def new(cls, A):
        n = A.shape[0]
        UR = la._new_mat(A, n, n)
        if capi._is_torch(A):
            import torch
            S, S_im = (torch.zeros(n, dtype=A.dtype, device=A.device) for _ in range(2))
            cx = A.dtype.is_complex
        else:
            S, S_im = np.zeros(n, dtype=A.dtype), np.zeros(n, dtype=A.dtype)
            cx = np.iscomplexobj(A)
        la.evd(A, S, None if cx else S_im, None, UR)
        if cx:
            return cls(UR, S)
        U = UR + 0j * UR
        first = S_im > 0
        second = S_im < 0
        im = UR[:, 1:][:, first[:-1]]
        U[:, first] = UR[:, first] + 1j * im
        U[:, second] = UR[:, first] - 1j * im
        return cls(U, S + 1j * S_im)

    def U(self):
        return self._U

    def S(self):
        return self._S


def svd(A) -> Svd:
    return Svd.new(A)


def thin_svd(A) -> Svd:
    return Svd.new_thin(A)


def self_adjoint_eigen(A, side: int = Side.Lower) -> SelfAdjointEigen:
    return SelfAdjointEigen.new(A, side)


# `A.llt(side)`, `A.partial_piv_lu()`, `A.qr()` (solvers.rs:346-392) as free functions
def llt(A, side: int = Side.Lower) -> Llt:
    return Llt.new(A, side)


def ldlt(A, side: int = Side.Lower) -> Ldlt:
    return Ldlt.new(A, side)


def lblt(A, side: int = Side.Lower) -> Lblt:
    return Lblt.new(A, side)


def partial_piv_lu(A) -> PartialPivLu:
    return PartialPivLu.new(A)


def full_piv_lu(A) -> FullPivLu:
    return FullPivLu.new(A)


def qr(A) -> Qr:
    return Qr.new(A)


def colpiv_qr(A) -> ColPivQr:
    return ColPivQr.new(A)


def singular_values(A):
    """`A.singular_values()` (solvers.rs:457-487): non-increasing, through `svd` with no vectors."""
    return la.singular_values(A)


def eigen(A) -> Eigen:
    return Eigen.new(A)


def eigenvalues(A):
    """`A.eigenvalues()` (solvers.rs): complex, through `evd` with no vectors."""
    n = A.shape[0]
    if capi._is_torch(A):
        import torch
        S, S_im = (torch.zeros(n, dtype=A.dtype, device=A.device) for _ in range(2))
        cx = A.dtype.is_complex
    else:
        S, S_im = np.zeros(n, dtype=A.dtype), np.zeros(n, dtype=A.dtype)
        cx = np.iscomplexobj(A)
    la.evd(A, S, None if cx else S_im)
    return S if cx else S + 1j * S_im


def self_adjoint_eigenvalues(A, side: int = Side.Lower):
    """`A.self_adjoint_eigenvalues(side)` (solvers.rs:417-456): nondecreasing; only the chosen triangle of A is read."""
    return la.self_adjoint_eigenvalues(A if side == Side.Lower else A.T)
