"""ctypes binding of libfaer_b200.so — the binding a faer-ffi user would write against faer.h.

Struct layouts and symbol names follow include/faer_b200.h (== /root/reference/faer-ffi/faer.h for these
entry points; Rust bodies in faer-ffi/src/lib.rs:855-1010, 1952-1983). Arguments may be numpy arrays (host
memory: staged by the library) or torch CUDA tensors (device memory: used in place); views with arbitrary
strides are passed as-is (strides in elements, any sign).

There is no CPU fallback here: `load()` raises if the shared library is missing, and the library itself
aborts if no CUDA device is present when a compute entry point is called.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Any

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfaer_b200.so")

# ---- PODs (faer-ffi/src/lib.rs:12-128) -----------------------------------------------------------


class MatRef(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("nrows", C.c_size_t), ("ncols", C.c_size_t),
                ("row_stride", C.c_ssize_t), ("col_stride", C.c_ssize_t)]


class MatMut(C.Structure):
    _fields_ = MatRef._fields_


class VecMut(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("len", C.c_size_t), ("stride", C.c_ssize_t)]


class SliceMut(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("len", C.c_size_t)]


class Par(C.Structure):
    _fields_ = [("tag", C.c_int), ("nthreads", C.c_size_t)]


class Layout(C.Structure):
    _fields_ = [("len_bytes", C.c_size_t), ("align_bytes", C.c_size_t)]


class MemAlloc(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("len_bytes", C.c_size_t)]


class LltParams(C.Structure):
    _fields_ = [("recursion_threshold", C.c_size_t), ("block_size", C.c_size_t)]


class PartialPivLuParams(C.Structure):
    _fields_ = [("recursion_threshold", C.c_size_t), ("block_size", C.c_size_t), ("par_threshold", C.c_size_t)]


class QrParams(C.Structure):
    _fields_ = [("blocking_threshold", C.c_size_t), ("par_threshold", C.c_size_t)]


class LltRegularization(C.Structure):
    _fields_ = [("dynamic_regularization_delta", C.c_void_p), ("dynamic_regularization_epsilon", C.c_void_p)]


class _StatusBody(C.Union):
    _fields_ = [("value", C.c_size_t)]


class LltStatus(C.Structure):
    """tag: 0 Ok{dynamic_regularization_count}, 1 NonPositivePivot{index}, 2 Unknown (faer.h:383-403)."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _StatusBody)]


class TridiagParams(C.Structure):
    _fields_ = [("par_threshold", C.c_size_t)]


class SelfAdjointEvdParams(C.Structure):
    """faer.h:191-194."""
    _fields_ = [("tridiag", TridiagParams), ("recursion_threshold", C.c_size_t)]


class EvdStatus(C.Structure):
    """tag: 0 Ok, 1 NoConvergence (faer.h:260-279)."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _StatusBody)]


class HessenbergParams(C.Structure):
    """faer.h:110-113."""
    _fields_ = [("par_threshold", C.c_size_t), ("blocking_threshold", C.c_size_t)]


SHIFT_COUNT_FN = C.CFUNCTYPE(C.c_size_t, C.c_size_t, C.c_size_t)


class SchurParams(C.Structure):
    """faer.h:115-120; the two callbacks run on the host."""
    _fields_ = [("recommended_shift_count", SHIFT_COUNT_FN), ("recommended_deflation_window", SHIFT_COUNT_FN),
                ("blocking_threshold", C.c_size_t), ("nibble_threshold", C.c_size_t)]


class EvdFromSchurParams(C.Structure):
    """faer.h:106-108."""
    _fields_ = [("recursion_threshold", C.c_size_t)]


class EvdParams(C.Structure):
    """faer.h:122-126."""
    _fields_ = [("hessenberg", HessenbergParams), ("schur", SchurParams), ("evd_from_schur", EvdFromSchurParams)]


class BidiagParams(C.Structure):
    _fields_ = [("par_threshold", C.c_size_t)]


class SvdParams(C.Structure):
    """faer.h:196-201."""
    _fields_ = [("bidiag", BidiagParams), ("qr", QrParams), ("recursion_threshold", C.c_size_t),
                ("qr_ratio_threshold", C.c_double)]


class SvdStatus(C.Structure):
    """tag: 0 Ok, 1 NoConvergence (faer.h:471-490)."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _StatusBody)]


class LdltParams(C.Structure):
    _fields_ = [("recursion_threshold", C.c_size_t), ("block_size", C.c_size_t)]


class LdltRegularization(C.Structure):
    """faer.h:368-381; dynamic_regularization_signs: i8 slice, null ptr = none."""
    _fields_ = [("dynamic_regularization_delta", C.c_void_p), ("dynamic_regularization_epsilon", C.c_void_p),
                ("dynamic_regularization_signs", SliceMut)]


class LdltStatus(C.Structure):
    """tag: 0 Ok{dynamic_regularization_count}, 1 ZeroPivot{index}, 2 Unknown (faer.h:346-366)."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _StatusBody)]


class PartialPivLuStatus(C.Structure):
    """tag: 0 Ok{transposition_count}, 1 Unknown (faer.h:412-427)."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _StatusBody)]


class QrStatus(C.Structure):
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _StatusBody)]


class PivLltParams(C.Structure):
    """faer.h:178-180."""
    _fields_ = [("block_size", C.c_size_t)]


class _PivLltOkBody(C.Structure):
    _fields_ = [("rank", C.c_size_t), ("transposition_count", C.c_size_t)]


class _PivLltBody(C.Union):
    _fields_ = [("ok", _PivLltOkBody), ("index", C.c_size_t)]


class PivLltStatus(C.Structure):
    """tag: 0 Ok{rank, transposition_count}, 1 NonPositivePivot{index}, 2 Unknown (faer.h:432-453); 24 bytes, body at 8."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _PivLltBody)]


class ColPivQrParams(C.Structure):
    """faer.h:101-104."""
    _fields_ = [("blocking_threshold", C.c_size_t), ("par_threshold", C.c_size_t)]


class _ColPivQrOkBody(C.Structure):
    _fields_ = [("transposition_count", C.c_size_t)]


class _ColPivQrBody(C.Union):
    _fields_ = [("ok", _ColPivQrOkBody)]


class ColPivQrStatus(C.Structure):
    """tag: 0 Ok{transposition_count}, 1 Unknown (faer.h:234-248); 16 bytes, body at 8."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _ColPivQrBody)]


class FullPivLuParams(C.Structure):
    """faer.h:128-130."""
    _fields_ = [("par_threshold", C.c_size_t)]


class _FullPivLuOkBody(C.Structure):
    _fields_ = [("transposition_count", C.c_size_t)]


class _FullPivLuBody(C.Union):
    _fields_ = [("ok", _FullPivLuOkBody)]


class FullPivLuStatus(C.Structure):
    """tag: 0 Ok{transposition_count}, 1 Unknown (faer.h:287-301); 16 bytes, body at 8."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _FullPivLuBody)]


class LbltParams(C.Structure):
    """faer.h:156-160; `pivoting` is a PIVOTING_* value."""
    _fields_ = [("pivoting", C.c_int), ("par_threshold", C.c_size_t), ("block_size", C.c_size_t)]


class _LbltOkBody(C.Structure):
    _fields_ = [("transposition_count", C.c_size_t)]


class _LbltBody(C.Union):
    _fields_ = [("ok", _LbltOkBody)]


class LbltStatus(C.Structure):
    """tag: 0 Ok{transposition_count}, 1 Unknown (faer.h:324-338); 16 bytes, body at 8."""
    _anonymous_ = ("body",)
    _fields_ = [("tag", C.c_int), ("body", _LbltBody)]


# faer-ffi `PivotingStrategy` discriminants (faer-ffi/src/lib.rs:492-508)
PIVOTING_PARTIAL, PIVOTING_PARTIAL_DIAG, PIVOTING_ROOK, PIVOTING_ROOK_DIAG, PIVOTING_FULL = range(5)

ACCUM_REPLACE, ACCUM_ADD = 0, 1
CONJ_NO, CONJ_YES = 0, 1
PAR_SEQ, PAR_RAYON = 0, 1
# faer-ffi `Block` discriminants (faer-ffi/src/lib.rs:86-97)
BLOCK_RECT, BLOCK_LOWER, BLOCK_UPPER, BLOCK_STRICT_LOWER, BLOCK_STRICT_UPPER, BLOCK_UNIT_LOWER, BLOCK_UNIT_UPPER = range(7)

_lib = None


def load() -> C.CDLL:
    """Load libfaer_b200.so (raises if it has not been built: there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). This backend has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    P = Par
    lib.libfaer_v0_23_matmul_f64.argtypes = [MatMut, C.c_int, MatRef, MatRef, C.c_void_p, P]
    lib.libfaer_v0_23_matmul_f64.restype = None
    lib.libfaer_v0_23_matmul_triangular_f64.argtypes = [MatMut, C.c_int, C.c_int, MatRef, C.c_int, MatRef, C.c_int,
                                                        C.c_void_p, P]
    lib.libfaer_v0_23_matmul_triangular_f64.restype = None
    lib.libfaer_v0_23_matmul_f32.argtypes = [MatMut, C.c_int, MatRef, MatRef, C.c_void_p, P]
    lib.libfaer_v0_23_matmul_f32.restype = None
    lib.libfaer_v0_23_matmul_triangular_f32.argtypes = [MatMut, C.c_int, C.c_int, MatRef, C.c_int, MatRef, C.c_int,
                                                        C.c_void_p, P]
    lib.libfaer_v0_23_matmul_triangular_f32.restype = None
    lib.libfaer_v0_23_matmul_c64.argtypes = [MatMut, C.c_int, MatRef, MatRef, C.c_void_p, P]
    lib.libfaer_v0_23_matmul_c64.restype = None
    lib.libfaer_v0_23_matmul_triangular_c64.argtypes = [MatMut, C.c_int, C.c_int, MatRef, C.c_int, MatRef, C.c_int,
                                                        C.c_void_p, P]
    lib.libfaer_v0_23_matmul_triangular_c64.restype = None
    lib.libfaer_v0_23_matmul_c32.argtypes = [MatMut, C.c_int, MatRef, MatRef, C.c_void_p, P]
    lib.libfaer_v0_23_matmul_c32.restype = None
    lib.libfaer_v0_23_matmul_triangular_c32.argtypes = [MatMut, C.c_int, C.c_int, MatRef, C.c_int, MatRef, C.c_int,
                                                        C.c_void_p, P]
    lib.libfaer_v0_23_matmul_triangular_c32.restype = None
    for name in ("solve_triangular_lower", "solve_triangular_upper", "solve_unit_triangular_lower",
                 "solve_unit_triangular_upper"):
        for suf in ("f64", "f32", "c64", "c32"):
            f = getattr(lib, f"libfaer_v0_23_{name}_in_place_{suf}")
            f.argtypes = [MatRef, C.c_int, MatMut, P]
            f.restype = None
    lib.libfaer_v0_23_LltParams_f64.argtypes = []
    lib.libfaer_v0_23_LltParams_f64.restype = LltParams
    lib.libfaer_v0_23_llt_factor_in_place_scratch_f64.argtypes = [C.c_size_t, P, LltParams]
    lib.libfaer_v0_23_llt_factor_in_place_scratch_f64.restype = Layout
    lib.libfaer_v0_23_llt_factor_in_place_f64.argtypes = [MatMut, LltRegularization, P, MemAlloc, LltParams]
    lib.libfaer_v0_23_llt_factor_in_place_f64.restype = LltStatus
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_PartialPivLuParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_PartialPivLuParams_{suf}").restype = PartialPivLuParams
        for it in ("u32", "u64"):
            f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P, PartialPivLuParams]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_factor_in_place_{it}_{suf}")
            f.argtypes = [MatMut, SliceMut, SliceMut, P, MemAlloc, PartialPivLuParams]
            f.restype = PartialPivLuStatus
    for suf in ("f64", "f32", "c64", "c32", "fx128", "cx128"):
        getattr(lib, f"libfaer_v0_23_QrParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_QrParams_{suf}").restype = QrParams
        f = getattr(lib, f"libfaer_v0_23_qr_recommended_block_size_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t]
        f.restype = C.c_size_t
        f = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, P, QrParams]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{suf}")
        f.argtypes = [MatMut, MatMut, P, MemAlloc, QrParams]
        f.restype = QrStatus
        for name in ("apply_householder_on_the_left", "apply_householder_transpose_on_the_left",
                     "apply_householder_on_the_right", "apply_householder_transpose_on_the_right"):
            f = getattr(lib, f"libfaer_v0_23_{name}_scratch_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_{name}_{suf}")
            f.argtypes = [MatRef, MatRef, C.c_int, MatMut, P, MemAlloc]
            f.restype = None
        f = getattr(lib, f"libfaer_v0_23_qr_solve_lstsq_in_place_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, P]
        f.restype = Layout
        for name in ("qr_solve_in_place", "qr_solve_transpose_in_place"):
            f = getattr(lib, f"libfaer_v0_23_{name}_scratch_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, P]
            f.restype = Layout
        for name in ("qr_solve_lstsq_in_place", "qr_solve_in_place", "qr_solve_transpose_in_place"):
            f = getattr(lib, f"libfaer_v0_23_{name}_{suf}")
            f.argtypes = [MatRef, MatRef, MatRef, C.c_int, MatMut, P, MemAlloc]
            f.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_BidiagParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_BidiagParams_{suf}").restype = BidiagParams
        getattr(lib, f"libfaer_v0_23_SvdParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_SvdParams_{suf}").restype = SvdParams
        f = getattr(lib, f"libfaer_v0_23_svd_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, C.c_int, C.c_int, P, SvdParams]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_svd_{suf}")
        f.argtypes = [MatRef, MatMut, VecMut, MatMut, P, MemAlloc, SvdParams]
        f.restype = SvdStatus
    for suf in ("f64", "f32", "c64", "c32", "fx128", "cx128"):
        getattr(lib, f"libfaer_v0_23_TridiagParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_TridiagParams_{suf}").restype = TridiagParams
        getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}").restype = SelfAdjointEvdParams
        f = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_int, P, SelfAdjointEvdParams]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_{suf}")
        f.argtypes = [MatRef, MatMut, VecMut, P, MemAlloc, SelfAdjointEvdParams]
        f.restype = EvdStatus
    for suf in ("f64", "f32", "c64", "c32"):
        for name, ty in (("EvdFromSchurParams", EvdFromSchurParams), ("SchurParams", SchurParams), ("EvdParams", EvdParams)):
            getattr(lib, f"libfaer_v0_23_{name}_{suf}").argtypes = []
            getattr(lib, f"libfaer_v0_23_{name}_{suf}").restype = ty
        f = getattr(lib, f"libfaer_v0_23_evd_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_int, C.c_int, P, EvdParams]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_evd_{suf}")
        f.argtypes = [MatRef, MatMut, MatMut, VecMut, VecMut, P, MemAlloc, EvdParams]
        f.restype = EvdStatus
    lib.faer_b200_evd_last_sweep_counts.argtypes = [C.POINTER(C.c_longlong)]
    lib.faer_b200_evd_last_sweep_counts.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        for name in ("inverse_triangular_lower", "inverse_triangular_upper", "inverse_unit_triangular_lower", "inverse_unit_triangular_upper"):
            f = getattr(lib, f"libfaer_v0_23_{name}_in_place_{suf}")
            f.argtypes = [MatMut, MatRef, P]
            f.restype = None
        for name in ("llt_reconstruct", "llt_inverse"):
            f = getattr(lib, f"libfaer_v0_23_{name}_scratch_{suf}")
            f.argtypes = [C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_{name}_{suf}")
            f.argtypes = [MatMut, MatRef, P, MemAlloc]
            f.restype = None
        for it in ("u32", "u64"):
            f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_reconstruct_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_inverse_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, P]
            f.restype = Layout
            for name in ("partial_piv_lu_reconstruct", "partial_piv_lu_inverse"):
                f = getattr(lib, f"libfaer_v0_23_{name}_{it}_{suf}")
                f.argtypes = [MatMut, MatRef, MatRef, SliceMut, SliceMut, P, MemAlloc]
                f.restype = None
        f = getattr(lib, f"libfaer_v0_23_qr_reconstruct_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, P]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_qr_reconstruct_{suf}")
        f.argtypes = [MatMut, MatRef, MatRef, MatRef, P, MemAlloc]
        f.restype = None
        f = getattr(lib, f"libfaer_v0_23_qr_inverse_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, P]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_qr_inverse_{suf}")
        f.argtypes = [MatMut, MatRef, MatRef, MatRef, P, MemAlloc]
        f.restype = None
    for suf in ("f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_LltParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_LltParams_{suf}").restype = LltParams
        getattr(lib, f"libfaer_v0_23_llt_factor_in_place_scratch_{suf}").argtypes = [C.c_size_t, P, LltParams]
        getattr(lib, f"libfaer_v0_23_llt_factor_in_place_scratch_{suf}").restype = Layout
        getattr(lib, f"libfaer_v0_23_llt_factor_in_place_{suf}").argtypes = [MatMut, LltRegularization, P, MemAlloc, LltParams]
        getattr(lib, f"libfaer_v0_23_llt_factor_in_place_{suf}").restype = LltStatus
        getattr(lib, f"libfaer_v0_23_llt_solve_in_place_scratch_{suf}").argtypes = [C.c_size_t, C.c_size_t, P]
        getattr(lib, f"libfaer_v0_23_llt_solve_in_place_scratch_{suf}").restype = Layout
        getattr(lib, f"libfaer_v0_23_llt_solve_in_place_{suf}").argtypes = [MatRef, C.c_int, MatMut, P, MemAlloc]
        getattr(lib, f"libfaer_v0_23_llt_solve_in_place_{suf}").restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_LdltParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_LdltParams_{suf}").restype = LdltParams
        f = getattr(lib, f"libfaer_v0_23_ldlt_factor_in_place_scratch_{suf}")
        f.argtypes = [C.c_size_t, P, LdltParams]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_ldlt_factor_in_place_{suf}")
        f.argtypes = [MatMut, LdltRegularization, P, MemAlloc, LdltParams]
        f.restype = LdltStatus
        f = getattr(lib, f"libfaer_v0_23_ldlt_solve_in_place_scratch_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, P]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_ldlt_solve_in_place_{suf}")
        f.argtypes = [MatRef, VecMut, C.c_int, MatMut, P, MemAlloc]
        f.restype = None
        for name in ("ldlt_reconstruct", "ldlt_inverse"):
            f = getattr(lib, f"libfaer_v0_23_{name}_scratch_{suf}")
            f.argtypes = [C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_{name}_{suf}")
            f.argtypes = [MatMut, MatRef, VecMut, P, MemAlloc]
            f.restype = None
    lib.libfaer_v0_23_llt_solve_in_place_scratch_f64.argtypes = [C.c_size_t, C.c_size_t, P]
    lib.libfaer_v0_23_llt_solve_in_place_scratch_f64.restype = Layout
    lib.libfaer_v0_23_llt_solve_in_place_f64.argtypes = [MatRef, C.c_int, MatMut, P, MemAlloc]
    lib.libfaer_v0_23_llt_solve_in_place_f64.restype = None
    for it, suf in [(i, s_) for i in ("u32", "u64") for s_ in ("f64", "f32", "c64", "c32")]:
        f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_{it}_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, P]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_solve_in_place_{it}_{suf}")
        f.argtypes = [MatRef, MatRef, C.c_int, SliceMut, SliceMut, MatMut, P, MemAlloc]
        f.restype = None
        f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_{it}_{suf}")
        f.argtypes = [C.c_size_t, C.c_size_t, P]
        f.restype = Layout
        f = getattr(lib, f"libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_{it}_{suf}")
        f.argtypes = [MatRef, MatRef, C.c_int, SliceMut, SliceMut, MatMut, P, MemAlloc]
        f.restype = None
    lib.libfaer_v0_23_get_global_par.argtypes = []
    lib.libfaer_v0_23_get_global_par.restype = Par
    lib.libfaer_v0_23_set_global_par.argtypes = [Par]
    lib.libfaer_v0_23_set_global_par.restype = None
    lib.libfaer_v0_23_alloc.argtypes = [C.c_size_t, C.c_size_t]
    lib.libfaer_v0_23_alloc.restype = C.c_void_p
    lib.libfaer_v0_23_dealloc.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t]
    lib.libfaer_v0_23_dealloc.restype = None
    lib.faer_b200_device_count.argtypes = []
    lib.faer_b200_device_count.restype = C.c_int
    lib.faer_b200_set_stream.argtypes = [C.c_void_p]
    lib.faer_b200_set_stream.restype = None
    lib.faer_b200_launch_count.argtypes = []
    lib.faer_b200_launch_count.restype = C.c_ulonglong
    lib.faer_b200_launch_log_begin.argtypes = [C.c_void_p, C.c_size_t]
    lib.faer_b200_launch_log_begin.restype = None
    lib.faer_b200_launch_log_end.argtypes = []
    lib.faer_b200_launch_log_end.restype = C.c_size_t
    lib.faer_b200_release_workspace.argtypes = []
    lib.faer_b200_release_workspace.restype = None
    lib.faer_b200_profile_begin.argtypes = []
    lib.faer_b200_profile_begin.restype = None
    lib.faer_b200_profile_end.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_ulonglong)]
    lib.faer_b200_profile_end.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        f = getattr(lib, f"faer_b200_bidiag_in_place_{suf}")
        f.argtypes = [MatMut, MatMut, MatMut]
        f.restype = None
        f = getattr(lib, f"faer_b200_tridiag_in_place_{suf}")
        f.argtypes = [MatMut, MatMut]
        f.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        f = getattr(lib, f"faer_b200_hessenberg_in_place_{suf}")
        f.argtypes = [MatMut, MatMut]
        f.restype = None
    lib.faer_b200_spicy_matmul_f64.argtypes = [MatMut, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, MatRef,
                                               MatRef, C.c_void_p, C.c_void_p]
    lib.faer_b200_spicy_matmul_f64.restype = None
    lib.faer_b200_gemm.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_ssize_t, C.c_ssize_t,
                                   C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_bool, C.c_void_p,
                                   C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_bool, C.c_void_p, C.c_size_t]
    lib.faer_b200_gemm.restype = None
    lib.faer_b200_set_option.argtypes = [C.c_char_p, C.c_longlong]
    lib.faer_b200_set_option.restype = C.c_int
    lib.faer_b200_get_option.argtypes = [C.c_char_p]
    lib.faer_b200_get_option.restype = C.c_longlong
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_PivLltParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_PivLltParams_{suf}").restype = PivLltParams
        for it in ("u32", "u64"):
            f = getattr(lib, f"libfaer_v0_23_piv_llt_factor_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, P, PivLltParams]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_piv_llt_factor_in_place_{it}_{suf}")
            f.argtypes = [MatMut, SliceMut, SliceMut, P, MemAlloc, PivLltParams]
            f.restype = PivLltStatus
            f = getattr(lib, f"libfaer_v0_23_piv_llt_solve_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"libfaer_v0_23_piv_llt_solve_in_place_{it}_{suf}")
            f.argtypes = [MatRef, SliceMut, SliceMut, C.c_int, MatMut, P, MemAlloc]
            f.restype = None
            for name in ("reconstruct", "inverse"):
                f = getattr(lib, f"libfaer_v0_23_piv_llt_{name}_scratch_{it}_{suf}")
                f.argtypes = [C.c_size_t, P]
                f.restype = Layout
                f = getattr(lib, f"libfaer_v0_23_piv_llt_{name}_{it}_{suf}")
                f.argtypes = [MatMut, MatRef, SliceMut, SliceMut, P, MemAlloc]
                f.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_LbltParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_LbltParams_{suf}").restype = LbltParams
        for it in ("u32", "u64"):
            pre = "libfaer_v0_23_lblt_"
            f = getattr(lib, f"{pre}factor_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, P, LbltParams]
            f.restype = Layout
            f = getattr(lib, f"{pre}factor_in_place_{it}_{suf}")
            f.argtypes = [MatMut, VecMut, SliceMut, SliceMut, P, MemAlloc, LbltParams]
            f.restype = LbltStatus
            f = getattr(lib, f"{pre}solve_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"{pre}solve_in_place_{it}_{suf}")
            f.argtypes = [MatRef, VecMut, VecMut, C.c_int, SliceMut, SliceMut, MatMut, P, MemAlloc]
            f.restype = None
            for name in ("reconstruct", "inverse"):
                f = getattr(lib, f"{pre}{name}_scratch_{it}_{suf}")
                f.argtypes = [C.c_size_t, P]
                f.restype = Layout
                f = getattr(lib, f"{pre}{name}_{it}_{suf}")
                f.argtypes = [MatMut, MatRef, VecMut, VecMut, SliceMut, SliceMut, P, MemAlloc]
                f.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_ColPivQrParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_ColPivQrParams_{suf}").restype = ColPivQrParams
        for it in ("u32", "u64"):
            pre = f"libfaer_v0_23_colpiv_qr_"
            f = getattr(lib, f"{pre}factor_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, P, ColPivQrParams]
            f.restype = Layout
            f = getattr(lib, f"{pre}factor_in_place_{it}_{suf}")
            f.argtypes = [MatMut, MatMut, SliceMut, SliceMut, P, MemAlloc, ColPivQrParams]
            f.restype = ColPivQrStatus
            for name in ("solve", "solve_transpose"):
                f = getattr(lib, f"{pre}{name}_in_place_scratch_{it}_{suf}")
                f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, P]
                f.restype = Layout
            f = getattr(lib, f"{pre}solve_lstsq_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            for name in ("solve", "solve_transpose", "solve_lstsq"):
                f = getattr(lib, f"{pre}{name}_in_place_{it}_{suf}")
                f.argtypes = [MatRef, MatRef, MatRef, C.c_int, SliceMut, SliceMut, MatMut, P, MemAlloc]
                f.restype = None
            f = getattr(lib, f"{pre}reconstruct_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"{pre}inverse_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            for name in ("reconstruct", "inverse"):
                f = getattr(lib, f"{pre}{name}_{it}_{suf}")
                f.argtypes = [MatMut, MatRef, MatRef, MatRef, SliceMut, SliceMut, P, MemAlloc]
                f.restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"libfaer_v0_23_FullPivLuParams_{suf}").argtypes = []
        getattr(lib, f"libfaer_v0_23_FullPivLuParams_{suf}").restype = FullPivLuParams
        for it in ("u32", "u64"):
            pre = "libfaer_v0_23_full_piv_lu_"
            f = getattr(lib, f"{pre}factor_in_place_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P, FullPivLuParams]
            f.restype = Layout
            f = getattr(lib, f"{pre}factor_in_place_{it}_{suf}")
            f.argtypes = [MatMut, SliceMut, SliceMut, SliceMut, SliceMut, P, MemAlloc, FullPivLuParams]
            f.restype = FullPivLuStatus
            for name in ("solve", "solve_transpose"):
                f = getattr(lib, f"{pre}{name}_in_place_scratch_{it}_{suf}")
                f.argtypes = [C.c_size_t, C.c_size_t, P]
                f.restype = Layout
                f = getattr(lib, f"{pre}{name}_in_place_{it}_{suf}")
                f.argtypes = [MatRef, MatRef, C.c_int, SliceMut, SliceMut, SliceMut, SliceMut, MatMut, P, MemAlloc]
                f.restype = None
            f = getattr(lib, f"{pre}reconstruct_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, C.c_size_t, P]
            f.restype = Layout
            f = getattr(lib, f"{pre}inverse_scratch_{it}_{suf}")
            f.argtypes = [C.c_size_t, P]
            f.restype = Layout
            for name in ("reconstruct", "inverse"):
                f = getattr(lib, f"{pre}{name}_{it}_{suf}")
                f.argtypes = [MatMut, MatRef, MatRef, SliceMut, SliceMut, SliceMut, SliceMut, P, MemAlloc]
                f.restype = None
    # double-double kinds (include/faer_b200_fx128.h)
    for suf in ("fx128", "cx128"):
        sig = {
            "matmul": ([MatMut, C.c_int, MatRef, MatRef, C.c_void_p, P], None),
            "matmul_triangular": ([MatMut, C.c_int, C.c_int, MatRef, C.c_int, MatRef, C.c_int, C.c_void_p, P], None),
            "LltParams": ([], LltParams),
            "llt_factor_in_place_scratch": ([C.c_size_t, P, LltParams], Layout),
            "llt_factor_in_place": ([MatMut, LltRegularization, P, MemAlloc, LltParams], LltStatus),
            "llt_solve_in_place_scratch": ([C.c_size_t, C.c_size_t, P], Layout),
            "llt_solve_in_place": ([MatRef, C.c_int, MatMut, P, MemAlloc], None),
            "llt_reconstruct_scratch": ([C.c_size_t, P], Layout),
            "llt_reconstruct": ([MatMut, MatRef, P, MemAlloc], None),
            "llt_inverse_scratch": ([C.c_size_t, P], Layout),
            "llt_inverse": ([MatMut, MatRef, P, MemAlloc], None),
            "PartialPivLuParams": ([], PartialPivLuParams),
            # the rest of the QR family is in the QrParams loop above (include/faer_b200_fx128_qr.h)
            "qr_reconstruct_scratch": ([C.c_size_t, C.c_size_t, C.c_size_t, P], Layout),
            "qr_reconstruct": ([MatMut, MatRef, MatRef, MatRef, P, MemAlloc], None),
            "qr_inverse_scratch": ([C.c_size_t, C.c_size_t, P], Layout),
            "qr_inverse": ([MatMut, MatRef, MatRef, MatRef, P, MemAlloc], None),
            # include/faer_b200_fx128_svd.h
            "BidiagParams": ([], BidiagParams),
            "SvdParams": ([], SvdParams),
            "svd_scratch": ([C.c_size_t, C.c_size_t, C.c_int, C.c_int, P, SvdParams], Layout),
            "svd": ([MatRef, MatMut, VecMut, MatMut, P, MemAlloc, SvdParams], SvdStatus),
        }
        for name in ("solve_triangular_lower", "solve_triangular_upper", "solve_unit_triangular_lower",
                     "solve_unit_triangular_upper"):
            sig[f"{name}_in_place"] = ([MatRef, C.c_int, MatMut, P], None)
        for name in ("inverse_triangular_lower", "inverse_triangular_upper", "inverse_unit_triangular_lower",
                     "inverse_unit_triangular_upper"):
            sig[f"{name}_in_place"] = ([MatMut, MatRef, P], None)
        for it in ("u32", "u64"):
            sig[f"partial_piv_lu_factor_in_place_scratch_{it}"] = ([C.c_size_t, C.c_size_t, P, PartialPivLuParams], Layout)
            sig[f"partial_piv_lu_factor_in_place_{it}"] = ([MatMut, SliceMut, SliceMut, P, MemAlloc, PartialPivLuParams],
                                                           PartialPivLuStatus)
            for name in ("solve", "solve_transpose"):
                sig[f"partial_piv_lu_{name}_in_place_scratch_{it}"] = ([C.c_size_t, C.c_size_t, P], Layout)
                sig[f"partial_piv_lu_{name}_in_place_{it}"] = ([MatRef, MatRef, C.c_int, SliceMut, SliceMut, MatMut, P,
                                                                MemAlloc], None)
            sig[f"partial_piv_lu_reconstruct_scratch_{it}"] = ([C.c_size_t, C.c_size_t, P], Layout)
            sig[f"partial_piv_lu_inverse_scratch_{it}"] = ([C.c_size_t, P], Layout)
            for name in ("reconstruct", "inverse"):
                sig[f"partial_piv_lu_{name}_{it}"] = ([MatMut, MatRef, MatRef, SliceMut, SliceMut, P, MemAlloc], None)
        for name, (args, res) in sig.items():
            f = getattr(lib, f"libfaer_v0_23_{name}_{suf}")
            f.argtypes = args
            f.restype = res
    lib.faer_b200_version.argtypes = []
    lib.faer_b200_version.restype = C.c_char_p
    _lib = lib
    return lib


# ---- view construction ----------------------------------------------------------------------------

def _is_torch(x: Any) -> bool:
    return type(x).__module__.startswith("torch")


# Double-double element types. On the host: numpy structured dtypes, {hi, lo} per fx128 and {re.hi, re.lo, im.hi, im.lo} per cx128.
FX128 = np.dtype([("hi", "<f8"), ("lo", "<f8")])
CX128 = np.dtype([("re_hi", "<f8"), ("re_lo", "<f8"), ("im_hi", "<f8"), ("im_lo", "<f8")])


class DDTensor:
    """A CUDA (or CPU) float64 tensor seen as a matrix of fx128 (trailing limb axis of 2: [..., (hi, lo)]) or cx128 (trailing
    axes 2 x 2: [..., (re, im), (hi, lo)]) elements; the limb axes must be contiguous. _fields turns it into element strides."""

    def __init__(self, t, complex: bool = False):
        limbs = 4 if complex else 2
        assert t.dtype.is_floating_point and t.element_size() == 8, "double-double tensors are float64"
        assert t.dim() == (4 if complex else 3) and t.shape[2:] == ((2, 2) if complex else (2,)), "bad limb axes"
        inner = (2, 1) if complex else (1,)
        assert tuple(t.stride()[2:]) == inner, "the limb axes must be contiguous"
        assert t.stride(0) % limbs == 0 and t.stride(1) % limbs == 0, "element strides must be whole elements"
        self.t, self.complex = t, complex

    @property
    def shape(self):
        return tuple(self.t.shape[:2])


def _fields(x: Any, itemsize_expected: int | None = None):
    """(ptr, nrows, ncols, row_stride, col_stride) of a 2-D numpy array, torch tensor or DDTensor (strides in elements)."""
    if isinstance(x, DDTensor):
        limbs = 4 if x.complex else 2
        if itemsize_expected is not None:
            assert 8 * limbs == itemsize_expected
        t = x.t
        return t.data_ptr(), t.shape[0], t.shape[1], t.stride(0) // limbs, t.stride(1) // limbs
    if _is_torch(x):
        assert x.dim() == 2, "expected a 2-D tensor"
        if itemsize_expected is not None:
            assert x.element_size() == itemsize_expected
        return x.data_ptr(), x.shape[0], x.shape[1], x.stride(0), x.stride(1)
    a = x
    assert isinstance(a, np.ndarray) and a.ndim == 2, "expected a 2-D array"
    if itemsize_expected is not None:
        assert a.itemsize == itemsize_expected
    return a.ctypes.data, a.shape[0], a.shape[1], a.strides[0] // a.itemsize, a.strides[1] // a.itemsize


def mat_ref(x: Any) -> MatRef:
    p, m, n, rs, cs = _fields(x)
    return MatRef(p, m, n, rs, cs)


def mat_mut(x: Any) -> MatMut:
    p, m, n, rs, cs = _fields(x)
    if isinstance(x, np.ndarray):
        assert x.flags.writeable
    return MatMut(p, m, n, rs, cs)


def slice_mut(x: Any) -> SliceMut:
    if _is_torch(x):
        return SliceMut(x.data_ptr(), x.numel())
    return SliceMut(x.ctypes.data, x.size)


def par_default() -> Par:
    return Par(PAR_RAYON, 0)


def _scalar_f64(v: float):
    return C.byref(C.c_double(float(v)))
