"""Host-side mirror of faer::linalg for the hot path, over the C ABI (capi.py).

Function names, argument order and error behaviour follow the reference's Rust surface so the parity tests
read like faer's own tests:
  matmul::matmul                      faer/src/linalg/matmul/mod.rs:1617-1660
  matmul::triangular::matmul          faer/src/linalg/matmul/triangular.rs:1193-1245
  triangular_solve::solve_*_in_place  faer/src/linalg/triangular_solve.rs:220-419
  cholesky::llt::factor::cholesky_in_place   faer/src/linalg/cholesky/llt/factor.rs:68-97
  lu::partial_pivoting::factor::lu_in_place  faer/src/linalg/lu/partial_pivoting/factor.rs:234-295
Arguments are numpy arrays (host, staged by the library) or torch CUDA tensors (device, in place).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import capi
from .capi import (ACCUM_ADD, ACCUM_REPLACE, BLOCK_LOWER, BLOCK_RECT, BLOCK_STRICT_LOWER, BLOCK_STRICT_UPPER,  # noqa: F401
                   BLOCK_UNIT_LOWER, BLOCK_UNIT_UPPER, BLOCK_UPPER, CONJ_NO, CONJ_YES, PIVOTING_FULL, PIVOTING_PARTIAL,
                   PIVOTING_PARTIAL_DIAG, PIVOTING_ROOK, PIVOTING_ROOK_DIAG)


class Accum:
    Replace = ACCUM_REPLACE
    Add = ACCUM_ADD


class BlockStructure:
    Rectangular = BLOCK_RECT
    TriangularLower = BLOCK_LOWER
    TriangularUpper = BLOCK_UPPER
    StrictTriangularLower = BLOCK_STRICT_LOWER
    StrictTriangularUpper = BLOCK_STRICT_UPPER
    UnitTriangularLower = BLOCK_UNIT_LOWER
    UnitTriangularUpper = BLOCK_UNIT_UPPER


def _check_f64(*xs):
    for x in xs:
        if capi._is_torch(x):
            import torch
            assert x.dtype == torch.float64, "f64 entry point needs float64 tensors"
        else:
            assert x.dtype == np.float64, "f64 entry point needs float64 arrays"


def _is_c64(x) -> bool:
    if capi._is_torch(x):
        import torch
        return x.dtype == torch.complex128
    return x.dtype == np.complex128


def _is_c32(x) -> bool:
    if capi._is_torch(x):
        import torch
        return x.dtype == torch.complex64
    return x.dtype == np.complex64


def _scalar_c32(v):
    buf = (C.c_float * 2)(complex(v).real, complex(v).imag)
    return C.cast(buf, C.c_void_p), buf


def _scalar_c64(v):
    buf = (C.c_double * 2)(complex(v).real, complex(v).imag)
    return C.cast(buf, C.c_void_p), buf


def _is_f32(x) -> bool:
    if capi._is_torch(x):
        import torch
        return x.dtype == torch.float32
    return x.dtype == np.float32


def matmul(dst, accum: int, lhs, rhs, alpha, par=None) -> None:
    """dst = [dst +] alpha * lhs * rhs  (Accum.Replace never reads dst). f64, f32, c64 (complex128) or c32 (complex64)."""
    lib = capi.load()
    if _is_c32(dst):
        assert _is_c32(lhs) and _is_c32(rhs)
        p, keep = _scalar_c32(alpha)
        lib.libfaer_v0_23_matmul_c32(capi.mat_mut(dst), accum, capi.mat_ref(lhs), capi.mat_ref(rhs), p,
                                     par or capi.par_default())
        del keep
        return
    if _is_f32(dst):
        assert _is_f32(lhs) and _is_f32(rhs)
        a = C.c_float(float(alpha))
        lib.libfaer_v0_23_matmul_f32(capi.mat_mut(dst), accum, capi.mat_ref(lhs), capi.mat_ref(rhs), C.byref(a),
                                     par or capi.par_default())
        return
    if _is_c64(dst):
        assert _is_c64(lhs) and _is_c64(rhs)
        p, keep = _scalar_c64(alpha)
        lib.libfaer_v0_23_matmul_c64(capi.mat_mut(dst), accum, capi.mat_ref(lhs), capi.mat_ref(rhs), p,
                                     par or capi.par_default())
        del keep
        return
    _check_f64(dst, lhs, rhs)
    lib.libfaer_v0_23_matmul_f64(capi.mat_mut(dst), accum, capi.mat_ref(lhs), capi.mat_ref(rhs),
                                 capi._scalar_f64(alpha), par or capi.par_default())


def matmul_triangular(dst, dst_structure: int, accum: int, lhs, lhs_structure: int, rhs, rhs_structure: int,
                      alpha: float, par=None) -> None:
    lib = capi.load()
    if _is_c32(dst):
        assert _is_c32(lhs) and _is_c32(rhs)
        p, keep = _scalar_c32(alpha)
        lib.libfaer_v0_23_matmul_triangular_c32(capi.mat_mut(dst), dst_structure, accum, capi.mat_ref(lhs), lhs_structure,
                                                capi.mat_ref(rhs), rhs_structure, p, par or capi.par_default())
        del keep
        return
    if _is_f32(dst):
        assert _is_f32(lhs) and _is_f32(rhs)
        a = C.c_float(float(alpha))
        lib.libfaer_v0_23_matmul_triangular_f32(capi.mat_mut(dst), dst_structure, accum, capi.mat_ref(lhs), lhs_structure,
                                                capi.mat_ref(rhs), rhs_structure, C.byref(a), par or capi.par_default())
        return
    if _is_c64(dst):
        assert _is_c64(lhs) and _is_c64(rhs)
        p, keep = _scalar_c64(alpha)
        lib.libfaer_v0_23_matmul_triangular_c64(capi.mat_mut(dst), dst_structure, accum, capi.mat_ref(lhs), lhs_structure,
                                                capi.mat_ref(rhs), rhs_structure, p, par or capi.par_default())
        del keep
        return
    _check_f64(dst, lhs, rhs)
    lib.libfaer_v0_23_matmul_triangular_f64(capi.mat_mut(dst), dst_structure, accum, capi.mat_ref(lhs), lhs_structure,
                                            capi.mat_ref(rhs), rhs_structure, capi._scalar_f64(alpha),
                                            par or capi.par_default())


def _solve(name, tri, rhs, conj, par):
    """triangular_solve.rs:220-419; f64, f32, c64 (complex128) or c32 (complex64); `conj` solves with conj(tri)."""
    if _is_c64(rhs):
        assert _is_c64(tri), "c64 entry point needs complex128 operands"
        suf = "c64"
    elif _is_c32(rhs):
        assert _is_c32(tri), "c32 entry point needs complex64 operands"
        suf = "c32"
    elif _is_f32(rhs):
        assert _is_f32(tri), "f32 entry point needs float32 operands"
        suf = "f32"
    else:
        _check_f64(tri, rhs)
        suf = "f64"
    lib = capi.load()
    getattr(lib, f"libfaer_v0_23_{name}_in_place_{suf}")(capi.mat_ref(tri), conj, capi.mat_mut(rhs),
                                                         par or capi.par_default())


def solve_lower_triangular_in_place(tril, rhs, conj: int = CONJ_NO, par=None) -> None:
    _solve("solve_triangular_lower", tril, rhs, conj, par)


def solve_upper_triangular_in_place(triu, rhs, conj: int = CONJ_NO, par=None) -> None:
    _solve("solve_triangular_upper", triu, rhs, conj, par)


def solve_unit_lower_triangular_in_place(tril, rhs, conj: int = CONJ_NO, par=None) -> None:
    _solve("solve_unit_triangular_lower", tril, rhs, conj, par)


def solve_unit_upper_triangular_in_place(triu, rhs, conj: int = CONJ_NO, par=None) -> None:
    _solve("solve_unit_triangular_upper", triu, rhs, conj, par)


# ---- LLT ------------------------------------------------------------------------------------------
@dataclass
class LltInfo:
    dynamic_regularization_count: int


class LltError(Exception):
    """NonPositivePivot { index } (faer/src/linalg/cholesky/llt/factor.rs:21-24)."""

    def __init__(self, index: int):
        super().__init__(f"NonPositivePivot {{ index: {index} }}")
        self.index = index


def llt_params_default():
    return capi.load().libfaer_v0_23_LltParams_f64()


def cholesky_in_place(A, regularization=(0.0, 0.0), par=None, params=None) -> LltInfo:
    """In-place LLT of the lower triangle of A (f64; f32, c64 and c32 on the recursive drivers). regularization = (delta,
    epsilon). Raises LltError."""
    lib = capi.load()
    if _is_c64(A):
        suf, real = "c64", C.c_double
    elif _is_c32(A):
        suf, real = "c32", C.c_float
    elif _is_f32(A):
        suf, real = "f32", C.c_float
    else:
        _check_f64(A)
        suf, real = "f64", C.c_double
    params = params or getattr(lib, f"libfaer_v0_23_LltParams_{suf}")()
    par = par or capi.par_default()
    n = A.shape[0]
    lay = getattr(lib, f"libfaer_v0_23_llt_factor_in_place_scratch_{suf}")(n, par, params)
    scratch = np.empty(lay.len_bytes + lay.align_bytes, dtype=np.uint8)
    delta = real(float(regularization[0]))
    eps = real(float(regularization[1]))
    reg = capi.LltRegularization(C.cast(C.pointer(delta), C.c_void_p), C.cast(C.pointer(eps), C.c_void_p))
    st = getattr(lib, f"libfaer_v0_23_llt_factor_in_place_{suf}")(capi.mat_mut(A), reg, par,
                                                                 capi.MemAlloc(scratch.ctypes.data, scratch.size), params)
    if st.tag == 0:
        return LltInfo(int(st.value))
    if st.tag == 1:
        raise LltError(int(st.value))
    raise RuntimeError("LltStatus::Unknown")


# ---- LDLT (no pivoting) ---------------------------------------------------------------------------
@dataclass
class LdltInfo:
    dynamic_regularization_count: int


class LdltError(Exception):
    """ZeroPivot { index } (faer/src/linalg/cholesky/ldlt/factor.rs:689-692)."""

    def __init__(self, index: int):
        super().__init__(f"ZeroPivot {{ index: {index} }}")
        self.index = index


def ldlt_in_place(A, regularization=(0.0, 0.0), signs=None, par=None, params=None) -> LdltInfo:
    """cholesky::ldlt::factor::cholesky_in_place (ldlt/factor.rs:725-767): in-place LDLT of the lower triangle, D on the
    diagonal and the unit-lower L strictly below it. regularization = (delta, epsilon); signs: optional int8 array (numpy)
    or int8 CUDA tensor of expected pivot signs. f64 (tuned kernels), f32 / c64 / c32 (the functional path of ldlt_types.cu).
    Raises LdltError."""
    suf = _suf_lu(A)
    real = C.c_double if suf in ("f64", "c64") else C.c_float
    lib = capi.load()
    params = params or getattr(lib, f"libfaer_v0_23_LdltParams_{suf}")()
    par = par or capi.par_default()
    delta = real(float(regularization[0]))
    eps = real(float(regularization[1]))
    sl = capi.SliceMut(None, 0)
    if signs is not None:
        if not capi._is_torch(signs):
            signs = np.ascontiguousarray(signs, dtype=np.int8)
        sl = capi.slice_mut(signs)
        assert sl.len == A.shape[0]
    reg = capi.LdltRegularization(C.cast(C.pointer(delta), C.c_void_p), C.cast(C.pointer(eps), C.c_void_p), sl)
    st = getattr(lib, f"libfaer_v0_23_ldlt_factor_in_place_{suf}")(capi.mat_mut(A), reg, par, capi.MemAlloc(None, 0), params)
    if st.tag == 0:
        return LdltInfo(int(st.value))
    if st.tag == 1:
        raise LdltError(int(st.value))
    raise RuntimeError("LdltStatus::Unknown")


def _ldlt_diag(LD, D):
    """The `D: VecRef` argument: the diagonal of LD as a strided vector over the same storage (`L.diagonal()` in the reference), or a
    separate contiguous vector of LD's dtype (`Ldlt::D()`)."""
    p, m, n, rs, cs = capi._fields(LD)
    assert m == n
    if D is None:
        return capi.VecMut(p, n, rs + cs)
    if capi._is_torch(D):
        assert D.dim() == 1 and D.numel() == n and D.is_contiguous() and D.dtype == LD.dtype
        return capi.VecMut(D.data_ptr(), n, 1)
    assert D.ndim == 1 and D.size == n and D.dtype == LD.dtype and D.flags.c_contiguous
    return capi.VecMut(D.ctypes.data, n, 1)


def ldlt_solve_in_place(LD, rhs, conj: int = CONJ_NO, par=None, D=None) -> None:
    """cholesky::ldlt::solve::solve_in_place_with_conj (ldlt/solve.rs:11-49): rhs <- conj?(L D L^H)^-1 rhs with L the unit-lower
    part of LD. D defaults to the diagonal of LD; a separate contiguous vector of LD's dtype can be given instead. f64 / f32 /
    c64 / c32."""
    suf = _same_suffix(LD, rhs)
    getattr(capi.load(), f"libfaer_v0_23_ldlt_solve_in_place_{suf}")(capi.mat_ref(LD), _ldlt_diag(LD, D), conj, capi.mat_mut(rhs),
                                                                     par or capi.par_default(), capi.MemAlloc(None, 0))


def ldlt_reconstruct(out, LD, par=None, D=None) -> None:
    """cholesky::ldlt::reconstruct (ldlt/reconstruct.rs:9-55): the LOWER triangle of out <- L D L^H."""
    suf = _same_suffix(out, LD)
    getattr(capi.load(), f"libfaer_v0_23_ldlt_reconstruct_{suf}")(capi.mat_mut(out), capi.mat_ref(LD), _ldlt_diag(LD, D),
                                                                  par or capi.par_default(), capi.MemAlloc(None, 0))


def ldlt_inverse(out, LD, par=None, D=None) -> None:
    """cholesky::ldlt::inverse (ldlt/inverse.rs:9-60): the LOWER triangle of out <- (L D L^H)^-1."""
    suf = _same_suffix(out, LD)
    getattr(capi.load(), f"libfaer_v0_23_ldlt_inverse_{suf}")(capi.mat_mut(out), capi.mat_ref(LD), _ldlt_diag(LD, D),
                                                              par or capi.par_default(), capi.MemAlloc(None, 0))


def llt_solve_in_place(L, rhs, conj: int = CONJ_NO, par=None) -> None:
    """cholesky::llt::solve::solve_in_place_with_conj (llt/solve.rs:12-35): rhs <- (L L^H)^-1 rhs. f64, f32, c64 or c32."""
    lib = capi.load()
    if _is_c64(rhs):
        assert _is_c64(L)
        suf = "c64"
    elif _is_c32(rhs):
        assert _is_c32(L)
        suf = "c32"
    elif _is_f32(rhs):
        assert _is_f32(L)
        suf = "f32"
    else:
        _check_f64(L, rhs)
        suf = "f64"
    getattr(lib, f"libfaer_v0_23_llt_solve_in_place_{suf}")(capi.mat_ref(L), conj, capi.mat_mut(rhs),
                                                            par or capi.par_default(), capi.MemAlloc(None, 0))


def lu_solve_in_place(LU, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None, U=None) -> None:
    """lu::partial_pivoting::solve::solve_in_place_with_conj (lu/partial_pivoting/solve.rs:21-54):
    rhs <- A^-1 rhs from the packed factors (L unit-lower below the diagonal, U on/above) and the row permutation.
    With `U` given, `LU` is read as L only (its strict lower part) and `U` as the upper factor, as the reference's
    separate `L`, `U` arguments."""
    lib = capi.load()
    suf = _suf_lu(LU)
    assert _suf_lu(rhs) == suf
    isz = perm.element_size() if capi._is_torch(perm) else perm.itemsize
    it = {4: "u32", 8: "u64"}[isz]
    getattr(lib, f"libfaer_v0_23_partial_piv_lu_solve_in_place_{it}_{suf}")(
        capi.mat_ref(LU), capi.mat_ref(LU if U is None else U), conj, capi.slice_mut(perm), capi.slice_mut(perm_inv), capi.mat_mut(rhs),
        par or capi.par_default(), capi.MemAlloc(None, 0))


def lu_solve_transpose_in_place(LU, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None, U=None) -> None:
    """lu::partial_pivoting::solve::solve_transpose_in_place_with_conj (lu/partial_pivoting/solve.rs:55-86):
    rhs <- A^-T rhs from the packed factors and the row permutation (its inverse array is the one used)."""
    lib = capi.load()
    suf = _suf_lu(LU)
    assert _suf_lu(rhs) == suf
    isz = perm.element_size() if capi._is_torch(perm) else perm.itemsize
    it = {4: "u32", 8: "u64"}[isz]
    getattr(lib, f"libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_{it}_{suf}")(
        capi.mat_ref(LU), capi.mat_ref(LU if U is None else U), conj, capi.slice_mut(perm), capi.slice_mut(perm_inv), capi.mat_mut(rhs),
        par or capi.par_default(), capi.MemAlloc(None, 0))


# ---- Householder QR (no pivoting) -----------------------------------------------------------------
@dataclass
class QrInfo:
    rank: int


def _suf(x) -> str:
    return "f32" if _is_f32(x) else "f64"


def _suf_lu(x) -> str:
    return "c64" if _is_c64(x) else "c32" if _is_c32(x) else _suf(x)


def qr_recommended_block_size(nrows: int, ncols: int) -> int:
    """qr::no_pivoting::factor::recommended_block_size (qr/no_pivoting/factor.rs:91-116)."""
    return int(capi.load().libfaer_v0_23_qr_recommended_block_size_f64(nrows, ncols))


def qr_in_place(A, Q_coeff, par=None, params=None) -> QrInfo:
    """qr::no_pivoting::factor::qr_in_place (qr/no_pivoting/factor.rs:258-301). Q_coeff: block_size x min(m, n).
    f64, f32, c64 or c32. Returns QrInfo(rank): dependent columns are skipped and the reflectors compacted exactly as the reference
    does (factor.rs:40-83); Q_coeff's columns >= rank are zero with +inf on their block diagonals (287-299)."""
    lib = capi.load()
    suf = _suf_lu(A)
    assert _suf_lu(Q_coeff) == suf
    params = params or getattr(lib, f"libfaer_v0_23_QrParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{suf}")(capi.mat_mut(A), capi.mat_mut(Q_coeff),
                                                               par or capi.par_default(), capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("QrStatus::Unknown")
    return QrInfo(int(st.value))


def apply_block_householder_sequence_on_the_left_in_place(basis, factor, rhs, conj: int = CONJ_NO, par=None) -> None:
    """householder.rs:724-765: rhs <- Q rhs."""
    lib = capi.load()
    getattr(lib, f"libfaer_v0_23_apply_householder_on_the_left_{_suf_lu(rhs)}")(
        capi.mat_ref(basis), capi.mat_ref(factor), conj, capi.mat_mut(rhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def apply_block_householder_sequence_transpose_on_the_left_in_place(basis, factor, rhs, conj: int = CONJ_YES, par=None) -> None:
    """householder.rs:768-808: rhs <- Q^H rhs."""
    lib = capi.load()
    getattr(lib, f"libfaer_v0_23_apply_householder_transpose_on_the_left_{_suf_lu(rhs)}")(
        capi.mat_ref(basis), capi.mat_ref(factor), conj, capi.mat_mut(rhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def apply_block_householder_sequence_on_the_right_in_place(basis, factor, lhs, conj: int = CONJ_NO, par=None) -> None:
    """householder.rs:813-831: lhs <- lhs Q."""
    lib = capi.load()
    getattr(lib, f"libfaer_v0_23_apply_householder_on_the_right_{_suf_lu(lhs)}")(
        capi.mat_ref(basis), capi.mat_ref(factor), conj, capi.mat_mut(lhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def apply_block_householder_sequence_transpose_on_the_right_in_place(basis, factor, lhs, conj: int = CONJ_YES, par=None) -> None:
    """householder.rs:836-854: lhs <- lhs Q^H."""
    lib = capi.load()
    getattr(lib, f"libfaer_v0_23_apply_householder_transpose_on_the_right_{_suf_lu(lhs)}")(
        capi.mat_ref(basis), capi.mat_ref(factor), conj, capi.mat_mut(lhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def _qr_solve(name, Q_basis, Q_coeff, R, rhs, conj, par):
    lib = capi.load()
    suf = _suf_lu(rhs)
    assert _suf_lu(Q_basis) == suf and _suf_lu(Q_coeff) == suf and _suf_lu(R) == suf
    getattr(lib, f"libfaer_v0_23_{name}_{suf}")(capi.mat_ref(Q_basis), capi.mat_ref(Q_coeff), capi.mat_ref(R), conj,
                                               capi.mat_mut(rhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def qr_solve_lstsq_in_place(Q_basis, Q_coeff, R, rhs, conj: int = CONJ_NO, par=None) -> None:
    """qr::no_pivoting::solve::solve_lstsq_in_place_with_conj (qr/no_pivoting/solve.rs:38-76): least-squares solution of
    A x = rhs from the packed factors (Q_basis and R are normally the same matrix). rhs is m x k; the solution is
    left in rhs[:ncols, :], the rest of rhs holds the residual's components along the orthogonal complement."""
    _qr_solve("qr_solve_lstsq_in_place", Q_basis, Q_coeff, R, rhs, conj, par)


def qr_solve_in_place(Q_basis, Q_coeff, R, rhs, conj: int = CONJ_NO, par=None) -> None:
    """qr::no_pivoting::solve::solve_in_place_with_conj (solve.rs:96-119): rhs <- A^-1 rhs, square A."""
    _qr_solve("qr_solve_in_place", Q_basis, Q_coeff, R, rhs, conj, par)


def qr_solve_transpose_in_place(Q_basis, Q_coeff, R, rhs, conj: int = CONJ_NO, par=None) -> None:
    """qr::no_pivoting::solve::solve_transpose_in_place_with_conj (solve.rs:140-176): rhs <- A^-T rhs, square A."""
    _qr_solve("qr_solve_transpose_in_place", Q_basis, Q_coeff, R, rhs, conj, par)


# ---- reconstruct / inverse on the factors (f64 / f32 / c64 / c32) ---------------------------------------
def _same_suffix(*xs) -> str:
    sufs = {_suf_lu(x) for x in xs}
    if len(sufs) != 1:
        raise TypeError(f"mixed scalar types: {sorted(sufs)}")
    return sufs.pop()


def invert_triangular(dst, src, lower: bool, unit: bool = False, par=None) -> None:
    """linalg::triangular_inverse::invert_[unit_]{lower,upper}_triangular (triangular_inverse.rs): the chosen triangle of dst <- the
    inverse of the same triangle of src; nothing else of dst is written (not its diagonal for the unit variants)."""
    suf = _same_suffix(dst, src)
    name = f"inverse_{'unit_' if unit else ''}triangular_{'lower' if lower else 'upper'}_in_place"
    getattr(capi.load(), f"libfaer_v0_23_{name}_{suf}")(capi.mat_mut(dst), capi.mat_ref(src), par or capi.par_default())


def llt_reconstruct(out, L, par=None) -> None:
    """cholesky::llt::reconstruct (llt/reconstruct.rs:12-33): the LOWER triangle of out <- L L^H."""
    suf = _same_suffix(out, L)
    getattr(capi.load(), f"libfaer_v0_23_llt_reconstruct_{suf}")(capi.mat_mut(out), capi.mat_ref(L), par or capi.par_default(),
                                                                 capi.MemAlloc(None, 0))


def llt_inverse(out, L, par=None) -> None:
    """cholesky::llt::inverse (llt/inverse.rs:10-39): the LOWER triangle of out <- (L L^H)^-1."""
    suf = _same_suffix(out, L)
    getattr(capi.load(), f"libfaer_v0_23_llt_inverse_{suf}")(capi.mat_mut(out), capi.mat_ref(L), par or capi.par_default(),
                                                             capi.MemAlloc(None, 0))


def _lu_recon(name, out, L, U, perm, perm_inv, par):
    suf = _same_suffix(out, L, U)
    isz = perm.element_size() if capi._is_torch(perm) else perm.itemsize
    it = {4: "u32", 8: "u64"}[isz]
    getattr(capi.load(), f"libfaer_v0_23_{name}_{it}_{suf}")(capi.mat_mut(out), capi.mat_ref(L), capi.mat_ref(U),
                                                            capi.slice_mut(perm), capi.slice_mut(perm_inv),
                                                            par or capi.par_default(), capi.MemAlloc(None, 0))


def lu_reconstruct(out, L, U, perm, perm_inv, par=None) -> None:
    """lu::partial_pivoting::reconstruct: out <- P^-1 L U. L / U: the packed LU matrix (twice) or the split factors."""
    _lu_recon("partial_piv_lu_reconstruct", out, L, U, perm, perm_inv, par)


def lu_inverse(out, L, U, perm, perm_inv, par=None) -> None:
    """lu::partial_pivoting::inverse: out <- A^-1 from the factors (square)."""
    _lu_recon("partial_piv_lu_inverse", out, L, U, perm, perm_inv, par)


def qr_reconstruct(out, Q_basis, Q_coeff, R, par=None) -> None:
    """qr::no_pivoting::reconstruct (reconstruct.rs:13-39): out <- Q [R; 0]. R: min(m, n) x n (its strict lower part is not
    read)."""
    suf = _same_suffix(out, Q_basis, Q_coeff, R)
    getattr(capi.load(), f"libfaer_v0_23_qr_reconstruct_{suf}")(capi.mat_mut(out), capi.mat_ref(Q_basis), capi.mat_ref(Q_coeff),
                                                                capi.mat_ref(R), par or capi.par_default(), capi.MemAlloc(None, 0))


def qr_inverse(out, Q_basis, Q_coeff, R, par=None) -> None:
    """qr::no_pivoting::inverse: out <- A^-1 = R^-1 Q^H (square)."""
    suf = _same_suffix(out, Q_basis, Q_coeff, R)
    getattr(capi.load(), f"libfaer_v0_23_qr_inverse_{suf}")(capi.mat_mut(out), capi.mat_ref(Q_basis), capi.mat_ref(Q_coeff),
                                                            capi.mat_ref(R), par or capi.par_default(), capi.MemAlloc(None, 0))


def _real_values(S):
    """The ABI's S is T-typed: for complex T the values come back as (value, 0) pairs; the mirror returns them real."""
    if capi._is_torch(S):
        return S.real.contiguous() if S.is_complex() else S
    return np.ascontiguousarray(S.real) if np.iscomplexobj(S) else S


def singular_values(A, par=None, params=None):
    """`svd` with u = v = None (svd/mod.rs:530-648), as `MatRef::singular_values` (solvers.rs:457-487): the
    min(nrows, ncols) singular values of A in non-increasing order, as a numpy vector (host input) or a CUDA tensor (device
    input). f64 / f32 / c64 / c32 (real values for complex A)."""
    lib = capi.load()
    suf = _suf_lu(A)
    m, n = A.shape
    size = min(m, n)
    if capi._is_torch(A):
        import torch
        S = torch.zeros(size, dtype=A.dtype, device=A.device)
        sv = capi.VecMut(S.data_ptr(), size, 1)
    else:
        S = np.zeros(size, dtype=A.dtype)
        sv = capi.VecMut(S.ctypes.data, size, 1)
    params = params or getattr(lib, f"libfaer_v0_23_SvdParams_{suf}")()
    none = capi.MatMut(None, 0, 0, 0, 0)
    st = getattr(lib, f"libfaer_v0_23_svd_{suf}")(capi.mat_ref(A), none, sv, none, par or capi.par_default(),
                                                  capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("SvdError::NoConvergence")
    return _real_values(S)


def self_adjoint_eigenvalues(A, par=None, params=None):
    """`self_adjoint_evd` with u = None (evd/mod.rs:270-353), as `MatRef::self_adjoint_eigenvalues(Side::Lower)`
    (solvers.rs:417-456): the eigenvalues of the self-adjoint matrix whose LOWER triangle is in A, nondecreasing, as a numpy
    vector (host input) or a CUDA tensor (device input). f64 / f32 / c64 / c32 (real values for complex A)."""
    lib = capi.load()
    suf = _suf_lu(A)
    n = A.shape[0]
    assert A.shape[1] == n
    if capi._is_torch(A):
        import torch
        S = torch.zeros(n, dtype=A.dtype, device=A.device)
        sv = capi.VecMut(S.data_ptr(), n, 1)
    else:
        S = np.zeros(n, dtype=A.dtype)
        sv = capi.VecMut(S.ctypes.data, n, 1)
    params = params or getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_{suf}")(capi.mat_ref(A), capi.MatMut(None, 0, 0, 0, 0), sv,
                                                               par or capi.par_default(), capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("EvdError::NoConvergence")
    return _real_values(S)


def spicy_matmul(C, C_block: int, row_idx, col_idx, accum: int, A, B, D, alpha: float) -> None:
    """linalg::matmul::internal::spicy_matmul (matmul/internal/mod.rs:45-379), real f64:
    C[row_idx[i], col_idx[j]] (+)= alpha * (A diag(D) B)[i, j] for the (i, j) that `C_block` (block structure of the product)
    keeps. row_idx / col_idx: None or uint64 numpy arrays; D: None or a float64 numpy vector of length A.ncols."""
    lib = capi.load()
    _check_f64(C, A, B)
    ri = None if row_idx is None else np.ascontiguousarray(row_idx, dtype=np.uint64)
    ci = None if col_idx is None else np.ascontiguousarray(col_idx, dtype=np.uint64)
    dv = None if D is None else np.ascontiguousarray(D, dtype=np.float64)
    a = np.array([alpha], dtype=np.float64)
    lib.faer_b200_spicy_matmul_f64(capi.mat_mut(C), int(C_block), None if ri is None else ri.ctypes.data, 0 if ri is None else ri.size,
                                   None if ci is None else ci.ctypes.data, 0 if ci is None else ci.size, int(accum), capi.mat_ref(A),
                                   capi.mat_ref(B), None if dv is None else dv.ctypes.data, a.ctypes.data)


class GemmDstKind:
    """DstKind of the inner seam (include/faer_b200.h: FaerB200_GemmDstKind)"""
    Lower, Upper, Full = 0, 1, 2


_GEMM_DTYPE = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.complex64): 2, np.dtype(np.complex128): 3}


def gemm(dst, row_idx, col_idx, dst_kind: int, accum: int, lhs, conj_lhs: bool, diag, rhs, conj_rhs: bool, alpha, n_threads: int = 1) -> None:
    """The inner seam `faer_b200_gemm` = the argument list of `private_gemm_x86::gemm` at faer's three call sites
    (matmul/mod.rs:1373-1411, matmul/triangular.rs:641-680, matmul/internal/mod.rs:143-201), numpy arrays only (host pointers;
    any strides): dst[row_idx[i], col_idx[j]] (+)= alpha * sum_k lhs[i, k] diag[k] rhs[k, j] over the (i, j) `dst_kind` keeps.
    row_idx / col_idx: None or uint32 / uint64 arrays (same type); diag: None or a 1-D array (any stride)."""
    lib = capi.load()
    dt = np.dtype(dst.dtype)
    assert lhs.dtype == dt and rhs.dtype == dt
    m, k = lhs.shape
    n = rhs.shape[1]
    it = 1
    for ix in (row_idx, col_idx):
        if ix is not None:
            it = 0 if ix.dtype == np.uint32 else 1
    es = dt.itemsize
    a = np.array([alpha], dtype=dt)
    lib.faer_b200_gemm(_GEMM_DTYPE[dt], it, 0, m, n, k, dst.ctypes.data, dst.strides[0] // es, dst.strides[1] // es,
                       None if row_idx is None else row_idx.ctypes.data, None if col_idx is None else col_idx.ctypes.data, int(dst_kind),
                       int(accum), lhs.ctypes.data, lhs.strides[0] // es, lhs.strides[1] // es, bool(conj_lhs),
                       None if diag is None else diag.ctypes.data, 0 if diag is None else diag.strides[0] // es, rhs.ctypes.data,
                       rhs.strides[0] // es, rhs.strides[1] // es, bool(conj_rhs), a.ctypes.data, n_threads)


class ComputeSvdVectors:
    """svd/mod.rs:21-28 (faer-ffi/src/lib.rs:462-477)"""
    No, Thin, Full = 0, 1, 2


def _new_mat(like, nrows, ncols):
    """column-major matrix of the same kind (numpy / torch device) and dtype as `like`"""
    if capi._is_torch(like):
        import torch
        return torch.zeros((ncols, nrows), dtype=like.dtype, device=like.device).T
    return np.zeros((nrows, ncols), dtype=like.dtype, order="F")


def _values_vec(A, S, n):
    """The VecMut for the values of `svd` / `self_adjoint_evd`. The reference's S holds T-typed entries; for complex A a REAL numpy
    S is accepted too (filled through a complex temporary). Returns (VecMut, temporary or None)."""
    if capi._is_torch(S):
        assert S.dtype == A.dtype, "device S must have A's dtype (complex for complex A: the ABI's S is T-typed)"
        return capi.VecMut(S.data_ptr(), n, 1), None
    if np.iscomplexobj(A) and not np.iscomplexobj(S):
        tmp = np.zeros(n, dtype=A.dtype)
        return capi.VecMut(tmp.ctypes.data, n, 1), tmp
    assert S.dtype == A.dtype
    return capi.VecMut(S.ctypes.data, n, 1), None


def svd(A, S, U=None, V=None, par=None, params=None) -> None:
    """svd::svd (svd/mod.rs:530-672) through `libfaer_v0_23_svd_<T>` (faer-ffi/src/lib.rs:2345-2366): A = U diag(S) V^H with S
    (length min(nrows, ncols)) non-increasing. U: None, nrows x size (thin) or nrows x nrows (full); V likewise with ncols.
    f64 / f32 (f32 computes in f64), c64 / c32 (c32 computes in c64; S: A's dtype as in the ABI, or a real array).
    Raises RuntimeError("SvdError::NoConvergence") on non-finite input."""
    lib = capi.load()
    suf = _suf_lu(A)
    size = min(A.shape)
    assert S.shape == (size,)
    sv, tmp = _values_vec(A, S, size)
    none = capi.MatMut(None, 0, 0, 0, 0)
    params = params or getattr(lib, f"libfaer_v0_23_SvdParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_svd_{suf}")(capi.mat_ref(A), capi.mat_mut(U) if U is not None else none, sv,
                                                  capi.mat_mut(V) if V is not None else none, par or capi.par_default(),
                                                  capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("SvdError::NoConvergence")
    if tmp is not None:
        S[...] = tmp.real


def self_adjoint_evd(A, S, U=None, par=None, params=None) -> None:
    """evd::self_adjoint_evd (evd/mod.rs:270-418) through `libfaer_v0_23_self_adjoint_evd_<T>`: the LOWER triangle of A is
    read; S nondecreasing; U (n x n or None) the eigenvectors. f64 / f32 / c64 / c32 (S: A's dtype as in the ABI, or a real array
    for complex A). Raises RuntimeError("EvdError::NoConvergence") on non-finite input."""
    lib = capi.load()
    suf = _suf_lu(A)
    n = A.shape[0]
    assert A.shape[1] == n and S.shape == (n,)
    sv, tmp = _values_vec(A, S, n)
    params = params or getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_{suf}")(capi.mat_ref(A), capi.mat_mut(U) if U is not None else
                                                               capi.MatMut(None, 0, 0, 0, 0), sv, par or capi.par_default(),
                                                               capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("EvdError::NoConvergence")
    if tmp is not None:
        S[...] = tmp.real


def evd(A, S, S_im=None, UL=None, UR=None, par=None, params=None) -> None:
    """evd::evd_real / evd_cplx (evd/mod.rs:1180-1246) through `libfaer_v0_23_evd_<T>`: the eigenvalues of a general square A and,
    when given, its left (UL) and right (UR) eigenvectors, n x n each. Real A: eigenvalue k is S[k] + i S_im[k]; a conjugate pair
    sits at k, k + 1 with S_im[k] > 0 and its eigenvectors are column k +- i column k + 1. Complex A: S only (A's dtype).
    f64 / f32 / c64 / c32 (f32 / c32 compute in f64 / c64). Raises RuntimeError("EvdError::NoConvergence") on non-finite input
    or when the sweep cap is reached; the outputs are then as they were."""
    lib = capi.load()
    suf = _suf_lu(A)
    n = A.shape[0]
    cx = suf in ("c64", "c32")
    assert A.shape[1] == n and S.shape == (n,) and S.dtype == A.dtype
    if not cx:
        assert S_im is not None and S_im.shape == (n,) and S_im.dtype == A.dtype

    def vec(v):
        return capi.VecMut(v.data_ptr() if capi._is_torch(v) else v.ctypes.data, n, 1)

    none = capi.MatMut(None, 0, 0, 0, 0)
    params = params or getattr(lib, f"libfaer_v0_23_EvdParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_evd_{suf}")(capi.mat_ref(A), capi.mat_mut(UL) if UL is not None else none,
                                                  capi.mat_mut(UR) if UR is not None else none, vec(S),
                                                  vec(S_im) if not cx else capi.VecMut(None, 0, 1), par or capi.par_default(),
                                                  capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("EvdError::NoConvergence")


def bidiag_in_place(A, H_left, H_right, par=None, params=None) -> None:
    """svd::bidiag::bidiag_in_place (svd/bidiag.rs:47-256): A = U B V^H for nrows >= ncols, f64 / f32 (HBM-bound kernels) or c64 / c32 (functional). B ends up on A's
    diagonal / superdiagonal, the left reflectors below the diagonal (T blocks in H_left, bl x ncols), the right
    reflectors to the right of the superdiagonal (T blocks in H_right, br x (ncols - 1))."""
    lib = capi.load()
    suf = _same_suffix(A, H_left, H_right)
    getattr(lib, f"faer_b200_bidiag_in_place_{suf}")(capi.mat_mut(A), capi.mat_mut(H_left), capi.mat_mut(H_right))


def hessenberg_in_place(A, householder, par=None, params=None) -> None:
    """evd::hessenberg::hessenberg_in_place (evd/hessenberg.rs:549-567): A = Q H Q^H for a general square A; H ends up in the entries
    (i, j) with i <= j + 1, the reflectors of Q below the subdiagonal, their T blocks in `householder` (b x (n - 1)).
    f64 / f32 / c64 / c32; functional (unblocked)."""
    suf = _same_suffix(A, householder)
    getattr(capi.load(), f"faer_b200_hessenberg_in_place_{suf}")(capi.mat_mut(A), capi.mat_mut(householder))


def tridiag_in_place(A, householder, par=None, params=None) -> None:
    """evd::tridiag::tridiag_in_place (evd/tridiag.rs:274-529): A = Q T Q^H for a self-adjoint A (only the lower triangle
    is read / written), f64 / f32 (HBM-bound kernel) or c64 / c32 (functional). T ends up on A's diagonal / subdiagonal, the
    reflectors below the subdiagonal, their T blocks in `householder` (b x (n - 1))."""
    lib = capi.load()
    suf = _same_suffix(A, householder)
    getattr(lib, f"faer_b200_tridiag_in_place_{suf}")(capi.mat_mut(A), capi.mat_mut(householder))


# ---- partial-pivoting LU ---------------------------------------------------------------------------
@dataclass
class PartialPivLuInfo:
    transposition_count: int


def lu_in_place(A, perm, perm_inv, par=None, params=None) -> PartialPivLuInfo:
    """In-place P A = L U. `perm`/`perm_inv`: uint32/uint64 arrays (numpy) or int32/int64 CUDA tensors of
    length nrows; (P A)[i, :] = A[perm[i], :]. f64, c64, c32, or f32 (computed in f64 on the device and rounded back)."""
    lib = capi.load()
    suf = _suf_lu(A)
    params = params or getattr(lib, f"libfaer_v0_23_PartialPivLuParams_{suf}")()
    par = par or capi.par_default()
    isz = perm.element_size() if capi._is_torch(perm) else perm.itemsize
    it = {4: "u32", 8: "u64"}[isz]
    m, n = A.shape
    lay = getattr(lib, f"libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_{it}_{suf}")(m, n, par, params)
    scratch = np.empty(lay.len_bytes + lay.align_bytes, dtype=np.uint8)
    st = getattr(lib, f"libfaer_v0_23_partial_piv_lu_factor_in_place_{it}_{suf}")(
        capi.mat_mut(A), capi.slice_mut(perm), capi.slice_mut(perm_inv), par,
        capi.MemAlloc(scratch.ctypes.data, scratch.size), params)
    if st.tag != 0:
        raise RuntimeError("PartialPivLuStatus::Unknown")
    return PartialPivLuInfo(int(st.value))


# ---- pivoted Cholesky (llt_pivoting) ---------------------------------------------------------------
@dataclass
class PivLltInfo:
    rank: int
    transposition_count: int


def piv_llt_params_default():
    return capi.load().libfaer_v0_23_PivLltParams_f64()


def _perm_width(perm) -> str:
    isz = perm.element_size() if capi._is_torch(perm) else perm.itemsize
    return {4: "u32", 8: "u64"}[isz]


def piv_llt_in_place(A, perm, perm_inv, par=None, params=None) -> PivLltInfo:
    """cholesky::llt_pivoting::factor::cholesky_in_place (llt_pivoting/factor.rs:47-199): P A P^T = L L^H of the lower triangle
    of a positive semi-definite A, in place. `perm`/`perm_inv`: uint32/uint64 arrays (numpy) or int32/int64 CUDA tensors of
    length n; (P A P^T)[i, j] = A[perm[i], perm[j]]. Returns the numerical rank: columns 0..rank of L are the factor. Raises
    LltError(index) for a negative or NaN diagonal (index 0, A untouched) or a NaN residual (its column)."""
    lib = capi.load()
    suf = _suf_lu(A)
    params = params or getattr(lib, f"libfaer_v0_23_PivLltParams_{suf}")()
    par = par or capi.par_default()
    it = _perm_width(perm)
    lay = getattr(lib, f"libfaer_v0_23_piv_llt_factor_in_place_scratch_{it}_{suf}")(A.shape[0], par, params)
    scratch = np.empty(lay.len_bytes + lay.align_bytes, dtype=np.uint8)
    st = getattr(lib, f"libfaer_v0_23_piv_llt_factor_in_place_{it}_{suf}")(
        capi.mat_mut(A), capi.slice_mut(perm), capi.slice_mut(perm_inv), par,
        capi.MemAlloc(scratch.ctypes.data, scratch.size), params)
    if st.tag == 0:
        return PivLltInfo(int(st.ok.rank), int(st.ok.transposition_count))
    if st.tag == 1:
        raise LltError(int(st.index))
    raise RuntimeError("PivLltStatus::Unknown")


def piv_llt_solve_in_place(L, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None) -> None:
    """cholesky::llt_pivoting::solve::solve_in_place_with_conj (llt_pivoting/solve.rs:13-41): rhs <- A^-1 rhs (conj(A)^-1 rhs
    with CONJ_YES) from the factor and its permutation."""
    suf = _same_suffix(L, rhs)
    getattr(capi.load(), f"libfaer_v0_23_piv_llt_solve_in_place_{_perm_width(perm)}_{suf}")(
        capi.mat_ref(L), capi.slice_mut(perm), capi.slice_mut(perm_inv), conj, capi.mat_mut(rhs), par or capi.par_default(),
        capi.MemAlloc(None, 0))


def piv_llt_reconstruct(out, L, perm, perm_inv, par=None) -> None:
    """cholesky::llt_pivoting::reconstruct (reconstruct.rs:12-52): the LOWER triangle of out <- A from the factor."""
    suf = _same_suffix(out, L)
    getattr(capi.load(), f"libfaer_v0_23_piv_llt_reconstruct_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(L), capi.slice_mut(perm), capi.slice_mut(perm_inv), par or capi.par_default(),
        capi.MemAlloc(None, 0))


def piv_llt_inverse(out, L, perm, perm_inv, par=None) -> None:
    """cholesky::llt_pivoting::inverse (inverse.rs:12-54): the LOWER triangle of out <- A^-1 from the factor."""
    suf = _same_suffix(out, L)
    getattr(capi.load(), f"libfaer_v0_23_piv_llt_inverse_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(L), capi.slice_mut(perm), capi.slice_mut(perm_inv), par or capi.par_default(),
        capi.MemAlloc(None, 0))


# ---- Bunch-Kaufman LBLT (cholesky::lblt) -----------------------------------------------------------
@dataclass
class LbltInfo:
    transposition_count: int


def lblt_params_default():
    """LbltParams { pivoting: PartialDiag, par_threshold: 128 * 128, block_size: 64 } (bunch_kaufman/factor.rs:903-910)."""
    return capi.load().libfaer_v0_23_LbltParams_f64()


def _vec(x, n, like):
    """A VecRef / VecMut over a 1-D numpy array or torch tensor of `like`'s dtype, or (x a 2-D matrix) over its diagonal."""
    if capi._is_torch(x):
        if x.dim() == 2:
            return capi.VecMut(x.data_ptr(), n, x.stride(0) + x.stride(1))
        assert x.dim() == 1 and x.numel() == n and x.dtype == like.dtype
        return capi.VecMut(x.data_ptr(), n, x.stride(0))
    if x.ndim == 2:
        return capi.VecMut(x.ctypes.data, n, (x.strides[0] + x.strides[1]) // x.itemsize)
    assert x.ndim == 1 and x.size == n and x.dtype == like.dtype
    return capi.VecMut(x.ctypes.data, n, x.strides[0] // x.itemsize)


def lblt_in_place(A, subdiag, perm, perm_inv, params=None, par=None) -> LbltInfo:
    """cholesky::lblt::factor::cholesky_in_place (bunch_kaufman/factor.rs:1161-1234): P A P^T = L B L^H of the self-adjoint A
    (lower triangle), in place: L strictly below the diagonal, B's diagonal on it, B's subdiagonal in `subdiag` (a 1-D array or
    tensor of A's dtype; pass it zeroed: entries of 1 x 1 blocks with a zero column are left as given). `perm`/`perm_inv`:
    uint32/uint64 arrays (numpy) or int32/int64 CUDA tensors; (P A P^T)[i, j] = A[perm[i], perm[j]]. PIVOTING_FULL also
    scales the strict upper triangle (see include/faer_b200_lblt.h)."""
    lib = capi.load()
    suf = _suf_lu(A)
    params = params or getattr(lib, f"libfaer_v0_23_LbltParams_{suf}")()
    par = par or capi.par_default()
    it = _perm_width(perm)
    n = A.shape[0]
    lay = getattr(lib, f"libfaer_v0_23_lblt_factor_in_place_scratch_{it}_{suf}")(n, par, params)
    scratch = np.empty(lay.len_bytes + lay.align_bytes, dtype=np.uint8)
    st = getattr(lib, f"libfaer_v0_23_lblt_factor_in_place_{it}_{suf}")(
        capi.mat_mut(A), _vec(subdiag, n, A), capi.slice_mut(perm), capi.slice_mut(perm_inv), par,
        capi.MemAlloc(scratch.ctypes.data, scratch.size), params)
    if st.tag != 0:
        raise RuntimeError("LbltStatus::Unknown")
    return LbltInfo(int(st.ok.transposition_count))


def lblt_solve_in_place(L, subdiag, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None, diag=None) -> None:
    """cholesky::lblt::solve::solve_in_place_with_conj (bunch_kaufman/solve.rs:35-104): rhs <- A^-1 rhs (conj(A)^-1 rhs with
    CONJ_YES). `diag` defaults to L's diagonal."""
    suf = _same_suffix(L, rhs)
    n = L.shape[0]
    getattr(capi.load(), f"libfaer_v0_23_lblt_solve_in_place_{_perm_width(perm)}_{suf}")(
        capi.mat_ref(L), _vec(L if diag is None else diag, n, L), _vec(subdiag, n, L), conj, capi.slice_mut(perm),
        capi.slice_mut(perm_inv), capi.mat_mut(rhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def lblt_reconstruct(out, L, subdiag, perm, perm_inv, par=None, diag=None) -> None:
    """cholesky::lblt::reconstruct (bunch_kaufman/reconstruct.rs:12-87): every entry of out is written; its LOWER triangle is A."""
    suf = _same_suffix(out, L)
    n = L.shape[0]
    getattr(capi.load(), f"libfaer_v0_23_lblt_reconstruct_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(L), _vec(L if diag is None else diag, n, L), _vec(subdiag, n, L), capi.slice_mut(perm),
        capi.slice_mut(perm_inv), par or capi.par_default(), capi.MemAlloc(None, 0))


def lblt_inverse(out, L, subdiag, perm, perm_inv, par=None, diag=None) -> None:
    """cholesky::lblt::inverse (bunch_kaufman/inverse.rs:11-42): out <- A^-1 (all n^2 entries)."""
    suf = _same_suffix(out, L)
    n = L.shape[0]
    getattr(capi.load(), f"libfaer_v0_23_lblt_inverse_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(L), _vec(L if diag is None else diag, n, L), _vec(subdiag, n, L), capi.slice_mut(perm),
        capi.slice_mut(perm_inv), par or capi.par_default(), capi.MemAlloc(None, 0))


# ---- column-pivoted QR (qr::col_pivoting) ----------------------------------------------------------
@dataclass
class ColPivQrInfo:
    transposition_count: int


def colpiv_qr_params_default():
    return capi.load().libfaer_v0_23_ColPivQrParams_f64()


def colpiv_qr_in_place(A, Q_coeff, perm, perm_inv, par=None, params=None) -> ColPivQrInfo:
    """qr::col_pivoting::factor::qr_in_place (col_pivoting/factor.rs:345-388): A P = Q R in place. Q_coeff: block_size x
    min(m, n) (T blocks as qr_in_place); `perm`/`perm_inv`: uint32/uint64 arrays (numpy) or int32/int64 CUDA tensors of length
    n, (A P)[:, j] = A[:, perm[j]]. f64, f32, c64 or c32."""
    lib = capi.load()
    suf = _same_suffix(A, Q_coeff)
    params = params or getattr(lib, f"libfaer_v0_23_ColPivQrParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_colpiv_qr_factor_in_place_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(A), capi.mat_mut(Q_coeff), capi.slice_mut(perm), capi.slice_mut(perm_inv), par or capi.par_default(),
        capi.MemAlloc(None, 0), params)
    if st.tag != 0:
        raise RuntimeError("ColPivQrStatus::Unknown")
    return ColPivQrInfo(int(st.ok.transposition_count))


def _colpiv_solve(name, Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj, par):
    suf = _same_suffix(Q_basis, Q_coeff, R, rhs)
    getattr(capi.load(), f"libfaer_v0_23_colpiv_qr_{name}_in_place_{_perm_width(perm)}_{suf}")(
        capi.mat_ref(Q_basis), capi.mat_ref(Q_coeff), capi.mat_ref(R), conj, capi.slice_mut(perm), capi.slice_mut(perm_inv),
        capi.mat_mut(rhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def colpiv_qr_solve_in_place(Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None) -> None:
    """col_pivoting/solve.rs:107-131: rhs <- A^-1 rhs (conj(A)^-1 rhs with CONJ_YES), square A."""
    _colpiv_solve("solve", Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj, par)


def colpiv_qr_solve_transpose_in_place(Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None) -> None:
    """col_pivoting/solve.rs:158-184: rhs <- A^-T rhs (A^-H with CONJ_YES), square A."""
    _colpiv_solve("solve_transpose", Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj, par)


def colpiv_qr_solve_lstsq_in_place(Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj: int = CONJ_NO, par=None) -> None:
    """col_pivoting/solve.rs:52-80: least-squares solution (m >= n) left in rhs[:ncols, :]."""
    _colpiv_solve("solve_lstsq", Q_basis, Q_coeff, R, perm, perm_inv, rhs, conj, par)


def colpiv_qr_reconstruct(out, Q_basis, Q_coeff, R, perm, perm_inv, par=None) -> None:
    """col_pivoting/reconstruct.rs:16-45: out <- Q R P^T."""
    suf = _same_suffix(out, Q_basis, Q_coeff, R)
    getattr(capi.load(), f"libfaer_v0_23_colpiv_qr_reconstruct_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(Q_basis), capi.mat_ref(Q_coeff), capi.mat_ref(R), capi.slice_mut(perm),
        capi.slice_mut(perm_inv), par or capi.par_default(), capi.MemAlloc(None, 0))


def colpiv_qr_inverse(out, Q_basis, Q_coeff, R, perm, perm_inv, par=None) -> None:
    """col_pivoting/inverse.rs:16-50: out <- A^-1 = P R^-1 Q^H, square A."""
    suf = _same_suffix(out, Q_basis, Q_coeff, R)
    getattr(capi.load(), f"libfaer_v0_23_colpiv_qr_inverse_{_perm_width(perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(Q_basis), capi.mat_ref(Q_coeff), capi.mat_ref(R), capi.slice_mut(perm),
        capi.slice_mut(perm_inv), par or capi.par_default(), capi.MemAlloc(None, 0))


# ---- full-pivoting LU (lu::full_pivoting) ----------------------------------------------------------
@dataclass
class FullPivLuInfo:
    transposition_count: int


def full_piv_lu_params_default():
    return capi.load().libfaer_v0_23_FullPivLuParams_f64()


def full_piv_lu_in_place(A, row_perm, row_perm_inv, col_perm, col_perm_inv, par=None, params=None) -> FullPivLuInfo:
    """lu::full_pivoting::factor::lu_in_place (full_pivoting/factor.rs:466-538): P A Q = L U in place (L unit-lower below the
    diagonal, U on and above it). `row_perm`/`row_perm_inv` (length m) and `col_perm`/`col_perm_inv` (length n): uint32/uint64
    arrays (numpy) or int32/int64 CUDA tensors of one width; (P A Q)[i, j] = A[row_perm[i], col_perm[j]]. f64, f32, c64 or c32."""
    lib = capi.load()
    suf = _suf_lu(A)
    params = params or getattr(lib, f"libfaer_v0_23_FullPivLuParams_{suf}")()
    par = par or capi.par_default()
    it = _perm_width(row_perm)
    assert _perm_width(col_perm) == it
    m, n = A.shape
    lay = getattr(lib, f"libfaer_v0_23_full_piv_lu_factor_in_place_scratch_{it}_{suf}")(m, n, par, params)
    scratch = np.empty(lay.len_bytes + lay.align_bytes, dtype=np.uint8)
    st = getattr(lib, f"libfaer_v0_23_full_piv_lu_factor_in_place_{it}_{suf}")(
        capi.mat_mut(A), capi.slice_mut(row_perm), capi.slice_mut(row_perm_inv), capi.slice_mut(col_perm),
        capi.slice_mut(col_perm_inv), par, capi.MemAlloc(scratch.ctypes.data, scratch.size), params)
    if st.tag != 0:
        raise RuntimeError("FullPivLuStatus::Unknown")
    return FullPivLuInfo(int(st.ok.transposition_count))


def _full_piv_lu_solve(name, L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, rhs, conj, par):
    suf = _same_suffix(L, U, rhs)
    getattr(capi.load(), f"libfaer_v0_23_full_piv_lu_{name}_in_place_{_perm_width(row_perm)}_{suf}")(
        capi.mat_ref(L), capi.mat_ref(U), conj, capi.slice_mut(row_perm), capi.slice_mut(row_perm_inv), capi.slice_mut(col_perm),
        capi.slice_mut(col_perm_inv), capi.mat_mut(rhs), par or capi.par_default(), capi.MemAlloc(None, 0))


def full_piv_lu_solve_in_place(L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, rhs, conj: int = CONJ_NO, par=None) -> None:
    """full_pivoting/solve.rs:21-56: rhs <- A^-1 rhs (conj(A)^-1 rhs with CONJ_YES), square A. L and U may be the packed factor."""
    _full_piv_lu_solve("solve", L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, rhs, conj, par)


def full_piv_lu_solve_transpose_in_place(L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, rhs, conj: int = CONJ_NO,
                                         par=None) -> None:
    """full_pivoting/solve.rs:58-93: rhs <- A^-T rhs (A^-H with CONJ_YES), square A."""
    _full_piv_lu_solve("solve_transpose", L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, rhs, conj, par)


def full_piv_lu_reconstruct(out, L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, par=None) -> None:
    """full_pivoting/reconstruct.rs:13-82: out (m x n) <- P^-1 L U Q^-1."""
    suf = _same_suffix(out, L, U)
    getattr(capi.load(), f"libfaer_v0_23_full_piv_lu_reconstruct_{_perm_width(row_perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(L), capi.mat_ref(U), capi.slice_mut(row_perm), capi.slice_mut(row_perm_inv),
        capi.slice_mut(col_perm), capi.slice_mut(col_perm_inv), par or capi.par_default(), capi.MemAlloc(None, 0))


def full_piv_lu_inverse(out, L, U, row_perm, row_perm_inv, col_perm, col_perm_inv, par=None) -> None:
    """full_pivoting/inverse.rs:12-63: out <- A^-1 = Q U^-1 L^-1 P, square A."""
    suf = _same_suffix(out, L, U)
    getattr(capi.load(), f"libfaer_v0_23_full_piv_lu_inverse_{_perm_width(row_perm)}_{suf}")(
        capi.mat_mut(out), capi.mat_ref(L), capi.mat_ref(U), capi.slice_mut(row_perm), capi.slice_mut(row_perm_inv),
        capi.slice_mut(col_perm), capi.slice_mut(col_perm_inv), par or capi.par_default(), capi.MemAlloc(None, 0))
