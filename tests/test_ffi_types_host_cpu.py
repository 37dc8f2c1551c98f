"""The C-ABI entry points of csrc/ffi_types.cu (`*_reconstruct` / `*_inverse`, LDLT, complex `svd` / `self_adjoint_evd`) run on
the CPU through the real Python binding: tools/emul/ffi_types_host.cpp builds csrc/ffi_types.cu + runtime.cu (entry lock, workspace
pool, StagedMat staging) + the three flat-map drivers, as they are, against a host stand-in of <cuda_runtime.h>; `capi.load()` is
pointed at that library and THE GPU TESTS' OWN FUNCTIONS are executed — same arrays, same views, same assertions as on the GPU.
Only the layers below are stand-ins: the building blocks (products, solves, Householder sequences, real condensed solvers) come
back through a callback and run on the oracle / LAPACK, and the factorizations the tests start from (LLT, LU, QR, f64 LDLT — GPU
code validated on hardware, not part of this library) are the oracle's."""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

from test_drivers_host_cpu import CB, MockCall, view

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory, fb, oracle):
    capi = fb.capi
    out = str(tmp_path_factory.mktemp("ffih") / "libffih.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    emul = os.path.join(ROOT, "tools", "emul")
    subprocess.check_call([cxx, "-O1", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(emul, "hostcuda"), "-o", out,
                           os.path.join(emul, "ffi_types_host.cpp")])
    lib = C.CDLL(out)

    def callback(cp):
        c = cp.contents
        if c.op == 1:
            alpha = complex(c.d[0], c.d[1]) if c.m[0].is_complex else c.d[0]
            oracle.matmul_triangular(view(c.m[0]), int(c.i[0]), bool(c.i[1]), view(c.m[1]), int(c.i[2]), view(c.m[2]), int(c.i[4]), alpha,
                                     conj_lhs=bool(c.i[3]), conj_rhs=bool(c.i[5]))
        elif c.op == 2:
            oracle.solve_triangular(view(c.m[0]), view(c.m[1]), lower=bool(c.i[0]), unit=bool(c.i[1]), conj=bool(c.i[2]))
        elif c.op == 3:
            f = oracle.apply_q_transpose_sequence if c.i[1] else oracle.apply_q_sequence
            f(view(c.m[0]), view(c.m[1]), view(c.m[2]), conj_lhs=bool(c.i[0]))
        elif c.op == 4:
            d, e, lam, Q = (view(c.m[k]) for k in range(4))
            n = d.shape[0]
            w, q = np.linalg.eigh(np.diag(d[:, 0]) + np.diag(e[:n - 1, 0], 1) + np.diag(e[:n - 1, 0], -1))
            lam[:, 0] = w; Q[...] = q; c.ret = 1
        elif c.op == 5:
            d, e, S, UB, VB = (view(c.m[k]) for k in range(5))
            n = d.shape[0]
            u, s, vt = np.linalg.svd(np.diag(d[:, 0]) + np.diag(e[:n - 1, 0], 1))
            S[:, 0] = s; UB[...] = u; VB[...] = vt.T; c.ret = 1
        elif c.op == 6:
            A, Hl, Hr = view(c.m[0]), view(c.m[1]), view(c.m[2])
            hl, hr = oracle.bidiag(A, Hl.shape[0], Hr.shape[0])
            Hl[...] = hl; Hr[...] = hr
        elif c.op == 7:
            A, H = view(c.m[0]), view(c.m[1])
            H[...] = oracle.tridiag(A, H.shape[0])

    cb = CB(callback)
    lib.drivers_set_callback(cb)
    lib._keep = cb
    lib.drivers_guard_errors.restype = C.c_longlong
    lib.drivers_live_blocks.restype = C.c_longlong
    # argument types of the subset, as capi.py sets them on the product library
    P, Layout, MatRef, MatMut, VecMut, SliceMut, MemAlloc = capi.Par, capi.Layout, capi.MatRef, capi.MatMut, capi.VecMut, capi.SliceMut, capi.MemAlloc
    g = lambda name: getattr(lib, "libfaer_v0_23_" + name)
    for suf in ("f64", "f32", "c64", "c32"):
        for name in ("ldlt_reconstruct", "ldlt_inverse"):
            g(f"{name}_{suf}").argtypes = [MatMut, MatRef, VecMut, P, MemAlloc]; g(f"{name}_{suf}").restype = None
        for name in ("llt_reconstruct", "llt_inverse"):
            g(f"{name}_{suf}").argtypes = [MatMut, MatRef, P, MemAlloc]; g(f"{name}_{suf}").restype = None
        for it in ("u32", "u64"):
            for name in ("partial_piv_lu_reconstruct", "partial_piv_lu_inverse"):
                g(f"{name}_{it}_{suf}").argtypes = [MatMut, MatRef, MatRef, SliceMut, SliceMut, P, MemAlloc]; g(f"{name}_{it}_{suf}").restype = None
        for name in ("qr_reconstruct", "qr_inverse"):
            g(f"{name}_{suf}").argtypes = [MatMut, MatRef, MatRef, MatRef, P, MemAlloc]; g(f"{name}_{suf}").restype = None
        if suf in ("c64", "c32"):
            g(f"SvdParams_{suf}").argtypes = []; g(f"SvdParams_{suf}").restype = capi.SvdParams
            g(f"svd_{suf}").argtypes = [MatRef, MatMut, VecMut, MatMut, P, MemAlloc, capi.SvdParams]; g(f"svd_{suf}").restype = capi.SvdStatus
            g(f"SelfAdjointEvdParams_{suf}").argtypes = []; g(f"SelfAdjointEvdParams_{suf}").restype = capi.SelfAdjointEvdParams
            g(f"self_adjoint_evd_{suf}").argtypes = [MatRef, MatMut, VecMut, P, MemAlloc, capi.SelfAdjointEvdParams]
            g(f"self_adjoint_evd_{suf}").restype = capi.EvdStatus
        if suf == "f64":
            continue                                                      # the f64 LDLT factorization is ldlt_f64.cu, not in this library
        g(f"LdltParams_{suf}").argtypes = []; g(f"LdltParams_{suf}").restype = capi.LdltParams
        g(f"ldlt_factor_in_place_{suf}").argtypes = [MatMut, capi.LdltRegularization, P, MemAlloc, capi.LdltParams]
        g(f"ldlt_factor_in_place_{suf}").restype = capi.LdltStatus
        g(f"ldlt_solve_in_place_{suf}").argtypes = [MatRef, VecMut, C.c_int, MatMut, P, MemAlloc]; g(f"ldlt_solve_in_place_{suf}").restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        for name in ("inverse_triangular_lower", "inverse_triangular_upper", "inverse_unit_triangular_lower", "inverse_unit_triangular_upper"):
            g(f"{name}_in_place_{suf}").argtypes = [MatMut, MatRef, P]; g(f"{name}_in_place_{suf}").restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"faer_b200_hessenberg_in_place_{suf}").argtypes = [MatMut, MatMut]; getattr(lib, f"faer_b200_hessenberg_in_place_{suf}").restype = None
    for suf in ("f64", "f32", "c64", "c32"):
        getattr(lib, f"faer_b200_bidiag_in_place_{suf}").argtypes = [MatMut, MatMut, MatMut]; getattr(lib, f"faer_b200_bidiag_in_place_{suf}").restype = None
        getattr(lib, f"faer_b200_tridiag_in_place_{suf}").argtypes = [MatMut, MatMut]; getattr(lib, f"faer_b200_tridiag_in_place_{suf}").restype = None
    yield lib
    assert lib.drivers_guard_errors() == 0 and lib.drivers_live_blocks() == 0


@pytest.fixture()
def host_fb(fb, oracle, hostlib, monkeypatch):
    """The real package with `capi.load()` pointed at the host library and the starting factorizations on the oracle."""
    la = fb.linalg
    monkeypatch.setattr(fb.capi, "load", lambda: hostlib)

    def cholesky_in_place(A, regularization=(0.0, 0.0), par=None, params=None):
        fail, count = oracle.llt(A, regularization[0], regularization[1])
        if fail >= 0:
            raise la.LltError(fail)
        return la.LltInfo(count)

    def lu_in_place(A, perm, perm_inv, par=None, params=None):
        p, pi, cnt = oracle.lu(A)
        perm[...] = p; perm_inv[...] = pi
        return la.PartialPivLuInfo(cnt)

    def qr_in_place(A, Q_coeff, par=None, params=None):
        H, rank = oracle.qr(A, block_size=Q_coeff.shape[0])
        Q_coeff[...] = H
        return la.QrInfo(rank)

    real_ldlt = la.ldlt_in_place

    def ldlt_in_place(A, regularization=(0.0, 0.0), signs=None, par=None, params=None):
        if A.dtype != np.float64:
            return real_ldlt(A, regularization, signs, par, params)       # the host library's own entry point
        fail, count = oracle.ldlt(A, regularization[0], regularization[1], None if signs is None else np.asarray(signs, dtype=np.int8))
        if fail >= 0:
            raise la.LdltError(fail)
        return la.LdltInfo(count)

    def matmul(dst, accum, lhs, rhs, alpha, par=None):
        oracle.matmul(dst, accum == la.Accum.Add, np.asarray(lhs), np.asarray(rhs), alpha)

    for name, f in (("cholesky_in_place", cholesky_in_place), ("lu_in_place", lu_in_place), ("qr_in_place", qr_in_place),
                    ("ldlt_in_place", ldlt_in_place), ("matmul", matmul),
                    ("qr_recommended_block_size", oracle.qr_recommended_block_size)):
        monkeypatch.setattr(la, name, f)
    return fb


def test_reconstruct_types_through_the_abi(host_fb):
    T = importlib.import_module("test_gpu_zzzzzzzzz_2_reconstruct_types")
    for dtype in T.DTYPES:
        T.test_llt_reconstruct_and_inverse_types(host_fb, None, dtype)
        T.test_qr_reconstruct_and_inverse_types(host_fb, None, dtype)
        for idx in (np.uint64, np.uint32):
            T.test_lu_reconstruct_and_inverse_types(host_fb, None, dtype, idx)


def test_ldlt_types_through_the_abi(host_fb, oracle):
    T = importlib.import_module("test_gpu_zzzzzzzzz_3_ldlt_types")
    for dtype in T.FS_DTYPES:
        T.test_ldlt_types_vs_oracle(host_fb, oracle, None, dtype)
        T.test_ldlt_types_zero_pivot_and_regularisation(host_fb, oracle, None, dtype)
    for dtype in T.ALL_DTYPES:
        T.test_ldlt_reconstruct_and_inverse(host_fb, None, dtype)
    for dtype in (np.complex128, np.float32):
        T.test_ldlt_solver_class_other_dtypes(host_fb, None, dtype)


def test_cplx_svd_evd_through_the_abi(host_fb):
    T = importlib.import_module("test_gpu_zzzzzzzzzz_cplx_svd_evd")
    for dtype in T.CDTYPES:
        T.test_cplx_svd_reference_shapes(host_fb, None, dtype)
        T.test_cplx_self_adjoint_evd(host_fb, None, dtype)
    T.test_cplx_non_finite_input_is_no_convergence(host_fb, None)
    T.test_cplx_solvers_svd_and_eigen(host_fb, None)


def test_condensed_extension_layouts_through_the_abi(host_fb):
    T = importlib.import_module("test_gpu_zzzzzzzzz_4_condensed_layouts")
    for dtype in (np.float64, np.float32):
        T.test_bidiag_row_major_and_strided_host_views(host_fb, None, dtype)
        T.test_tridiag_row_major_and_strided_host_views(host_fb, None, dtype)


def test_invert_triangular_through_the_abi(host_fb):
    T = importlib.import_module("test_gpu_zzzzzzzzz_1_inverse_triangular")
    for dtype in T.DTYPES:
        T.test_invert_triangular(host_fb, None, dtype)


def test_hessenberg_through_the_abi(host_fb, oracle):
    T = importlib.import_module("test_gpu_zzzzzzzzz_5_hessenberg")
    for dtype in T.DTYPES:
        T.test_hessenberg(host_fb, oracle, None, dtype)


def test_cplx_condensed_forms_through_the_abi(host_fb, oracle):
    T = importlib.import_module("test_gpu_zzzzzzzzz_6_cplx_condensed_forms")
    for dtype in T.CDTYPES:
        T.test_cplx_bidiag_vs_oracle(host_fb, oracle, None, dtype)
        T.test_cplx_tridiag_vs_oracle(host_fb, oracle, None, dtype)
