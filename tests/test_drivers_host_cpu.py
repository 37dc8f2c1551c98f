"""The flat-map DRIVERS themselves — csrc/cplx_condensed.cu, ldlt_types.cu, reconstruct_types.cu, as they are — compiled for the
host (tools/emul/drivers_host.cpp against tools/emul/hostcuda/cuda_runtime.h) and run end to end on the CPU: control flow, view
arithmetic, workspace sizes (a checking allocator with guard words; fresh workspace is NaN-filled) and the structure codes /
conjugation flags they hand to the building blocks. The building blocks (structured products, triangular solves, Householder
sequences, the real tridiagonal / bidiagonal solvers) arrive here through a callback and are executed with the oracle / LAPACK —
the functions the GPU's own building blocks are tested against on hardware. What this does NOT cover: the C-ABI staging layer
(ffi.cu) and the GPU building blocks themselves."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64 = C.c_longlong
U = np.finfo(np.float64).eps
KIND = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.complex64): 2, np.dtype(np.complex128): 3}


class MockMat(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("nrows", I64), ("ncols", I64), ("rs", I64), ("cs", I64), ("is_double", C.c_int), ("is_complex", C.c_int)]


class MockCall(C.Structure):
    _fields_ = [("op", C.c_int), ("m", MockMat * 5), ("i", I64 * 8), ("d", C.c_double * 4), ("ret", I64)]


CB = C.CFUNCTYPE(None, C.POINTER(MockCall))


def mat(a):
    """MockMat of a 2-D numpy array (None: the `not wanted` view)"""
    if a is None:
        return MockMat(None, 0, 0, 1, 1, 1, 1)
    dt = np.dtype(a.dtype)
    it = dt.itemsize
    return MockMat(a.ctypes.data, a.shape[0], a.shape[1], a.strides[0] // it, a.strides[1] // it,
                   1 if dt in (np.dtype(np.float64), np.dtype(np.complex128)) else 0, 1 if dt.kind == "c" else 0)


def view(m):
    dt = {(1, 0): np.float64, (0, 0): np.float32, (1, 1): np.complex128, (0, 1): np.complex64}[(m.is_double, m.is_complex)]
    it = np.dtype(dt).itemsize
    if m.nrows == 0 or m.ncols == 0:
        return np.zeros((m.nrows, m.ncols), dtype=dt)
    assert m.rs >= 0 and m.cs >= 0
    span = (m.nrows - 1) * m.rs + (m.ncols - 1) * m.cs + 1
    base = np.frombuffer((C.c_char * (span * it)).from_address(m.ptr), dtype=dt)
    return np.lib.stride_tricks.as_strided(base, shape=(m.nrows, m.ncols), strides=(m.rs * it, m.cs * it))


@pytest.fixture(scope="module")
def drv(tmp_path_factory, oracle):
    out = str(tmp_path_factory.mktemp("drv") / "libdrv.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    emul = os.path.join(ROOT, "tools", "emul")
    subprocess.check_call([cxx, "-O1", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(emul, "hostcuda"), "-o", out,
                           os.path.join(emul, "drivers_host.cpp")])
    lib = C.CDLL(out)
    log = []

    def callback(cp):
        c = cp.contents
        if c.op == 1:
            dst, lhs, rhs = view(c.m[0]), view(c.m[1]), view(c.m[2])
            alpha = complex(c.d[0], c.d[1]) if c.m[0].is_complex else c.d[0]
            log.append(("gemm", c.i[0], c.i[2], c.i[3], c.i[4], c.i[5]))
            oracle.matmul_triangular(dst, int(c.i[0]), bool(c.i[1]), lhs, int(c.i[2]), rhs, int(c.i[4]), alpha,
                                     conj_lhs=bool(c.i[3]), conj_rhs=bool(c.i[5]))
        elif c.op == 2:
            oracle.solve_triangular(view(c.m[0]), view(c.m[1]), lower=bool(c.i[0]), unit=bool(c.i[1]), conj=bool(c.i[2]))
        elif c.op == 3:
            basis, factor, rhs = view(c.m[0]), view(c.m[1]), view(c.m[2])
            # the GPU's complex sequence (cplx.cu) and the real ones (householder.cu) are the reference's
            # apply_block_householder_sequence_[transpose_]on_the_left_in_place_with_conj (householder.rs:724-808)
            if c.i[1]:
                oracle.apply_q_transpose_sequence(basis, factor, rhs, conj_lhs=bool(c.i[0]))
            else:
                oracle.apply_q_sequence(basis, factor, rhs, conj_lhs=bool(c.i[0]))
        elif c.op == 4:
            d, e, lam, Q = (view(c.m[k]) for k in range(4))
            n = d.shape[0]
            T = np.diag(d[:, 0]) + np.diag(e[:n - 1, 0], 1) + np.diag(e[:n - 1, 0], -1)
            w, q = np.linalg.eigh(T)
            lam[:, 0] = w
            Q[...] = q
            c.ret = 1
        elif c.op == 5:
            d, e, S, UB, VB = (view(c.m[k]) for k in range(5))
            n = d.shape[0]
            u, s, vt = np.linalg.svd(np.diag(d[:, 0]) + np.diag(e[:n - 1, 0], 1))
            S[:, 0] = s
            UB[...] = u
            VB[...] = vt.T
            c.ret = 1
        else:  # pragma: no cover
            raise AssertionError(c.op)

    cb = CB(callback)
    lib.drivers_set_callback(cb)
    lib.drv_svd.argtypes = [C.c_int, MockMat, MockMat, C.c_void_p, I64, MockMat]
    lib.drv_evd.argtypes = [C.c_int, MockMat, MockMat, C.c_void_p, I64]
    lib.drv_recon.argtypes = [C.c_int, C.c_int, MockMat, MockMat, MockMat, MockMat, C.c_void_p]
    lib.drv_ldlt.argtypes = [C.c_int, C.c_int, MockMat, MockMat, C.c_void_p, I64, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_void_p]
    lib.drv_ldlt_f64.argtypes = [C.c_int, MockMat, MockMat, C.c_void_p, I64]
    lib.drivers_guard_errors.restype = I64
    lib.drivers_live_blocks.restype = I64
    lib._keep = cb
    lib._log = log
    yield lib
    assert lib.drivers_guard_errors() == 0 and lib.drivers_live_blocks() == 0      # no overrun, no leak, in the whole module


def crandn(rng, shape, dtype):
    a = rng.standard_normal(shape)
    if np.dtype(dtype).kind == "c":
        a = a + 1j * rng.standard_normal(shape)
    return np.asfortranarray(a.astype(dtype))


def rdt(dtype):
    return np.float32 if np.dtype(dtype) in (np.dtype(np.float32), np.dtype(np.complex64)) else np.float64


def wide(x):
    return x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)


# ---- cplx_condensed.cu ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_svd_driver(drv, dtype):
    rng = np.random.default_rng(1700)
    eps = np.finfo(rdt(dtype)).eps
    for (m, n) in [(1, 1), (3, 2), (10, 10), (40, 17), (17, 40), (1, 7), (7, 1), (64, 64)]:
        size = min(m, n)
        for rev in (0, 1):
            drv.drivers_set_reverse(rev)
            A = crandn(rng, (m, n), dtype)
            ref = np.linalg.svd(wide(A), compute_uv=False)
            tol = eps * 128 * np.sqrt(8 * max(m, n)) * max(1.0, np.abs(A).max())
            for kind in ("full", "thin", "u_only", "v_only", "none"):
                S = np.full(2 * size, np.nan, dtype=dtype)                    # stride 2: every other entry must stay NaN
                U_ = None if kind in ("v_only", "none") else np.full((m, m if kind == "full" else size), np.nan, dtype=dtype, order="F")
                V_ = None if kind in ("u_only", "none") else np.full((n, n if kind == "full" else size), np.nan, dtype=dtype, order="C")  # row-major V
                ok = drv.drv_svd(1 if dtype == np.complex128 else 0, mat(A), mat(U_), S.ctypes.data, 2, mat(V_))
                assert ok == 1
                assert np.all(np.isnan(S[1::2])) and np.all(S[::2].imag == 0)
                s = S[::2].real
                assert np.abs(s - ref).max() <= tol and np.all(np.diff(s) <= 0)
                if U_ is not None:
                    assert np.abs(wide(U_).conj().T @ wide(U_) - np.eye(U_.shape[1])).max() <= tol, (m, n, kind)
                if V_ is not None:
                    assert np.abs(wide(V_).conj().T @ wide(V_) - np.eye(V_.shape[1])).max() <= tol, (m, n, kind)
                if U_ is not None and V_ is not None:
                    assert np.abs((wide(U_)[:, :size] * s[None, :]) @ wide(V_)[:, :size].conj().T - wide(A)).max() <= tol, (m, n, kind)
    drv.drivers_set_reverse(0)
    # non-finite input: false, nothing else required
    A = crandn(rng, (12, 9), np.complex128); A[4, 2] = np.nan
    S = np.zeros(9, dtype=np.complex128); U_ = np.zeros((12, 9), dtype=np.complex128, order="F"); V_ = np.zeros((9, 9), dtype=np.complex128, order="F")
    assert drv.drv_svd(1, mat(A), mat(U_), S.ctypes.data, 1, mat(V_)) == 0
    # an empty dimension with a full left factor: the identity
    A = np.zeros((5, 0), dtype=np.complex128, order="F"); U_ = np.full((5, 5), np.nan, dtype=np.complex128, order="F")
    assert drv.drv_svd(1, mat(A), mat(U_), None, 1, mat(None)) == 1 and np.array_equal(U_, np.eye(5))


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_self_adjoint_evd_driver(drv, dtype):
    rng = np.random.default_rng(1701)
    eps = np.finfo(rdt(dtype)).eps
    for n in [1, 2, 3, 17, 64]:
        G = crandn(rng, (n, n), np.complex128)
        A = np.asfortranarray(((G + G.conj().T) / 2).astype(dtype))
        poisoned = A.copy(order="F"); poisoned[np.triu_indices(n, 1)] = np.nan
        row_major = np.ascontiguousarray(poisoned)
        for src in (poisoned, row_major):
            S = np.full(n, np.nan, dtype=dtype); U_ = np.full((n, n), np.nan, dtype=dtype, order="F")
            assert drv.drv_evd(1 if dtype == np.complex128 else 0, mat(src), mat(U_), S.ctypes.data, 1) == 1
            tol = eps * 128 * np.sqrt(8 * n) * max(1.0, np.abs(A).max())
            s = S.real
            assert np.all(S.imag == 0) and np.all(np.diff(s) >= 0)
            assert np.abs(wide(U_).conj().T @ wide(U_) - np.eye(n)).max() <= tol
            assert np.abs((wide(U_) * s[None, :]) @ wide(U_).conj().T - wide(A)).max() <= tol
            S2 = np.full(n, np.nan, dtype=dtype)
            assert drv.drv_evd(1 if dtype == np.complex128 else 0, mat(src), mat(None), S2.ctypes.data, 1) == 1
            assert np.abs(S2.real - s).max() <= tol


# ---- reconstruct_types.cu --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.complex128, np.complex64])
def test_reconstruct_types_drivers(drv, oracle, dtype):
    rng = np.random.default_rng(1702)
    u = float(np.finfo(rdt(dtype)).eps)
    kind = KIND[np.dtype(dtype)]
    none = mat(None)
    for n in [1, 50, 97]:
        G = wide(crandn(rng, (n, n), dtype))
        A = np.asfortranarray((G @ G.conj().T + n * np.eye(n)).astype(dtype))
        L = A.copy(order="F"); assert oracle.llt(L)[0] == -1
        out = np.full((n, n), np.nan, dtype=dtype, order="F"); out[np.tril_indices(n)] = 7
        drv.drv_recon(kind, 0, mat(out), mat(L), none, none, None)
        assert np.all(np.isnan(out[np.triu_indices(n, 1)]))
        assert np.abs(np.tril(wide(out)) - np.tril(wide(A))).max() <= 256 * n * u * np.abs(A).max()
        inv = np.full((n, n), np.nan, dtype=dtype, order="C"); inv[np.tril_indices(n)] = 7          # row-major output
        drv.drv_recon(kind, 1, mat(inv), mat(L), none, none, None)
        assert np.all(np.isnan(inv[np.triu_indices(n, 1)]))
        lo = np.tril(wide(inv)); full = lo + np.tril(lo, -1).conj().T
        assert np.abs(full @ wide(A) - np.eye(n)).max() <= 256 * n * u * np.linalg.cond(wide(A))
    for (m, n) in [(50, 50), (100, 50), (50, 100), (1, 1)]:
        A = crandn(rng, (m, n), dtype)
        LU = A.copy(order="F"); perm, perm_inv, _ = oracle.lu(LU)
        out = np.full((m, n), np.nan, dtype=dtype, order="F")
        drv.drv_recon(kind, 2, mat(out), mat(LU), mat(LU), none, perm_inv.ctypes.data)
        scale = np.abs(A).max() * max(1.0, float(np.abs(np.triu(LU)).max()))
        assert np.abs(wide(out) - wide(A)).max() <= 256 * max(m, n) * u * scale, (m, n)
        if m == n:
            inv = np.full((n, n), np.nan, dtype=dtype, order="F")
            drv.drv_recon(kind, 3, mat(inv), mat(LU), mat(LU), none, perm.ctypes.data)
            assert np.abs(wide(inv) @ wide(A) - np.eye(n)).max() <= 256 * n * u * np.linalg.cond(wide(A))
        s = min(m, n)
        for bs in sorted({oracle.qr_recommended_block_size(m, n), min(7, s)}):
            QR = A.copy(order="F"); H, rank = oracle.qr(QR, block_size=bs); assert rank == s
            out = np.full((m, n), np.nan, dtype=dtype, order="F")
            drv.drv_recon(kind, 4, mat(out), mat(QR[:, :s]), mat(H), mat(QR[:s, :]), None)
            assert np.abs(wide(out) - wide(A)).max() <= 256 * max(m, n) * u * np.abs(A).max(), (m, n, bs)
            if m == n:
                inv = np.full((n, n), np.nan, dtype=dtype, order="F")
                drv.drv_recon(kind, 5, mat(inv), mat(QR), mat(H), mat(QR), None)
                assert np.abs(wide(inv) @ wide(A) - np.eye(n)).max() <= 256 * n * u * np.linalg.cond(wide(A)), (n, bs)


# ---- ldlt_types.cu ---------------------------------------------------------------------------------------------------------------------
def indefinite(rng, n, dtype):
    G = rng.standard_normal((n, n))
    if np.dtype(dtype).kind == "c":
        G = G + 1j * rng.standard_normal((n, n))
    s = np.where(rng.random(n) < 0.4, -1.0, 1.0)
    A = (G + G.conj().T) / np.sqrt(max(n, 1)) + np.diag(4.0 * s)
    A[np.diag_indices(n)] = A[np.diag_indices(n)].real
    return np.asfortranarray(A.astype(dtype))


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex128, np.complex64])
def test_ldlt_types_drivers(drv, oracle, dtype):
    rng = np.random.default_rng(1703)
    u = float(np.finfo(rdt(dtype)).eps)
    kind = KIND[np.dtype(dtype)]
    it = np.dtype(dtype).itemsize
    for n in [1, 33, 80]:
        A = indefinite(rng, n, dtype)
        want = A.copy(order="F"); assert oracle.ldlt(want) == (-1, 0)
        if dtype == np.float64:
            LD = want                                        # the f64 factorization is not in this file
        else:
            LD = A.copy(order="F"); LD[np.triu_indices(n, 1)] = np.nan
            info = np.zeros(2, dtype=np.int64)
            drv.drv_ldlt(kind, 0, mat(LD), mat(None), None, 0, None, 0.0, 0.0, 0, info.ctypes.data)
            assert tuple(info) == (-1, 0) and np.all(np.isnan(LD[np.triu_indices(n, 1)]))
            assert np.allclose(np.tril(LD), np.tril(want), rtol=2e3 * u, atol=2e3 * u)
            LD[np.triu_indices(n, 1)] = A[np.triu_indices(n, 1)]
            # ZeroPivot and the regularisation count through the driver's status plumbing
            bad = A.copy(order="F"); bad[:4, :4] = np.diag([2.0, 4.0, 8.0, 0.0]) if n >= 4 else bad[:4, :4]
            if n >= 4:
                bad[3, :3] = bad[:3, 3] = [2.0, 4.0, 8.0]; bad[3, 3] = 14.0
                drv.drv_ldlt(kind, 0, mat(bad), mat(None), None, 0, None, 0.0, 0.0, 0, info.ctypes.data)
                assert tuple(info) == (3, 0)
                reg = np.asfortranarray(np.diag(np.array([1.0, -2.0, 1e-20, -1e-20, 3.0])).astype(dtype))
                sg = np.array([1, 1, 1, -1, -1], dtype=np.int8)
                drv.drv_ldlt(kind, 0, mat(reg), mat(None), None, 0, sg.ctypes.data, 1e-3, 1e-10, 0, info.ctypes.data)
                assert tuple(info) == (-1, 2)
        Aw = wide(A)
        D = LD.ctypes.data
        dstride = (LD.strides[0] + LD.strides[1]) // it       # the diagonal as a strided vector over the same storage
        if dtype != np.float64:
            for conj in (0, 1):
                B = crandn(rng, (n, 4), dtype)
                X = np.array(B, order="C", copy=True)         # row-major right-hand side
                drv.drv_ldlt(kind, 1, mat(LD), mat(X), D, dstride, None, 0.0, 0.0, conj, None)
                Ae = Aw.conj() if conj else Aw
                assert np.abs(Ae @ wide(X) - wide(B)).max() <= 256 * n * u * np.linalg.cond(Aw) * np.abs(B).max(), (n, conj)
        run = (lambda which, out: drv.drv_ldlt_f64(which, mat(LD), mat(out), D, dstride)) if dtype == np.float64 else \
              (lambda which, out: drv.drv_ldlt(kind, which, mat(LD), mat(out), D, dstride, None, 0.0, 0.0, 0, None))
        out = np.full((n, n), np.nan, dtype=dtype, order="F"); out[np.tril_indices(n)] = 7
        run(2, out)
        assert np.all(np.isnan(out[np.triu_indices(n, 1)]))
        assert np.abs(np.tril(wide(out)) - np.tril(Aw)).max() <= 256 * n * u * np.abs(A).max()
        inv = np.full((n, n), np.nan, dtype=dtype, order="F"); inv[np.tril_indices(n)] = 7
        run(3, inv)
        assert np.all(np.isnan(inv[np.triu_indices(n, 1)]))
        lo = np.tril(wide(inv)); full = lo + np.tril(lo, -1).conj().T
        assert np.abs(full @ Aw - np.eye(n)).max() <= 256 * n * u * np.linalg.cond(Aw)
