"""The general eigensolver's Hessenberg -> Schur stage and its eigenvectors of the Schur form, run on the CPU from the very
header the GPU kernels are built from (faer-rs_b200/csrc/schur_core.cuh through tools/emul/schur_host.cpp): sweep driver, window
QR, small-bulge chase, deflation scan, shift selection, back substitution. The Hessenberg reduction in front is scipy's.

Checked against the definitions, not against another implementation's output: Z^H A Z = T with Z unitary, T (quasi-)triangular
with standardised 2 x 2 blocks, A X = X Lambda and Y^H A = Lambda Y^H column by column, and the eigenvalue multiset against
scipy.linalg.eigvals. Sizes sit below, at and above the window (96 real, 64 complex) and reach several windows per sweep."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg as sla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [1, 2, 3, 4, 5, 17, 33, 95, 96, 97, 130, 200, 300]
EPS = np.finfo(np.float64).eps


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("schur") / "libschur_host.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, os.path.join(ROOT, "tools", "emul", "schur_host.cpp")])
    return C.CDLL(out)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def run(lib, A, ns_limit=1 << 30):
    """-> (status, T, Z, lam, XR, XL, info) for a square real or complex A"""
    A = np.asarray(A)
    n = A.shape[0]
    cx = np.iscomplexobj(A)
    dt = np.complex128 if cx else np.float64
    Hh, Q = sla.hessenberg(A.astype(dt), calc_q=True)
    H = np.asfortranarray(np.triu(Hh, -1).astype(dt))
    Z = np.asfortranarray(Q.astype(dt))
    XR = np.zeros((n, n), dt, order="F")
    XL = np.zeros((n, n), dt, order="F")
    info = (C.c_longlong * 2)()
    if cx:
        s = np.zeros(n, dt)
        st = lib.schur_host_c64(n, _ptr(H), _ptr(Z), _ptr(s), _ptr(XR), _ptr(XL), C.c_int(min(ns_limit, 1 << 20)), info)
        lam = s
    else:
        sr, si = np.zeros(n), np.zeros(n)
        st = lib.schur_host_f64(n, _ptr(H), _ptr(Z), _ptr(sr), _ptr(si), _ptr(XR), _ptr(XL), C.c_int(min(ns_limit, 1 << 20)), info)
        lam = sr + 1j * si
    return st, H, Z, lam, XR, XL, list(info)


def unpack(X, lam, left=False):
    """the packed real convention -> complex eigenvector columns"""
    if np.iscomplexobj(X):
        return X
    V = X.astype(np.complex128)
    k = 0
    while k < len(lam):
        if lam[k].imag > 0:
            V[:, k] = X[:, k] + 1j * X[:, k + 1]
            V[:, k + 1] = X[:, k] - 1j * X[:, k + 1]
            k += 2
        else:
            k += 1
    return V


def check(A, st, T, Z, lam, XR, XL, c=40.0):
    n = A.shape[0]
    assert st == 0
    nA = max(np.linalg.norm(A), np.finfo(float).tiny)
    tol = c * max(n, 4) * EPS
    assert np.linalg.norm(Z.conj().T @ Z - np.eye(n)) <= tol
    assert np.linalg.norm(Z.conj().T @ A @ Z - T) <= tol * nA
    assert np.all(np.tril(T, -2) == 0)
    sub = np.diag(T, -1)
    if np.iscomplexobj(T):
        assert np.all(sub == 0)
    else:
        assert not np.any((sub[:-1] != 0) & (sub[1:] != 0))
        for k in np.nonzero(sub)[0]:
            assert T[k, k] == T[k + 1, k + 1] and T[k, k + 1] * T[k + 1, k] < 0
            assert lam[k].imag > 0 and lam[k + 1] == np.conj(lam[k])
    ref = sla.eigvals(A)
    # every computed eigenvalue near a reference one and the other way round (robust to the ordering of close values)
    d = np.abs(lam[:, None] - ref[None, :])
    vtol = 1e3 * n * EPS * nA if n < 40 else None
    if vtol is not None and np.linalg.cond(sla.eig(A)[1]) < 1e6:
        assert d.min(axis=0).max() <= vtol * 1e3 and d.min(axis=1).max() <= vtol * 1e3
    assert abs(lam.sum() - np.trace(A)) <= tol * nA * np.sqrt(n) * 10
    VR = Z @ unpack(XR, lam)
    VL = Z @ unpack(XL, lam, left=True)
    for k in range(n):
        x, y = VR[:, k], VL[:, k]
        assert np.linalg.norm(x) > 0 and np.linalg.norm(y) > 0
        assert np.linalg.norm(A @ x - lam[k] * x) <= 10 * tol * nA * np.linalg.norm(x), k
        assert np.linalg.norm(y.conj() @ A - lam[k] * y.conj()) <= 10 * tol * nA * np.linalg.norm(y), k


@pytest.mark.parametrize("cx", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_random(lib, n, cx):
    rng = np.random.default_rng(1000 + n + (7 if cx else 0))
    A = rng.standard_normal((n, n))
    if cx:
        A = A + 1j * rng.standard_normal((n, n))
    out = run(lib, A)
    check(A, *out[:6])
    W = 64 if cx else 96
    if n > W:
        assert out[6][0] > 0 and out[6][1] >= out[6][0]  # sweeps ran, at least one window each


@pytest.mark.parametrize("cx", [False, True])
def test_several_windows_per_sweep_and_a_small_shift_count(lib, cx):
    rng = np.random.default_rng(5)
    A = rng.standard_normal((300, 300)) + (1j * rng.standard_normal((300, 300)) if cx else 0)
    out = run(lib, A)
    check(A, *out[:6])
    assert out[6][1] >= 3 * out[6][0]
    out = run(lib, A[:150, :150], ns_limit=4)  # the caller's shift count is an upper bound
    check(A[:150, :150], *out[:6])


def _special(name, n, rng):
    if name == "zeros":
        return np.zeros((n, n))
    if name == "identity":
        return np.eye(n)
    if name == "ones":
        return np.ones((n, n))
    if name == "triangular":
        return np.triu(rng.standard_normal((n, n)))
    if name == "companion":
        return sla.companion(np.r_[1.0, rng.standard_normal(n)])
    if name == "repeated":
        Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
        return Q @ np.diag(np.r_[np.full(n // 2, 2.0), np.arange(n - n // 2)]) @ Q.T
    if name == "rotation":
        A = np.zeros((n, n))
        for k in range(0, n - 1, 2):
            A[k, k + 1], A[k + 1, k] = -(k + 1.0), k + 1.0
        return A
    if name == "graded":
        return rng.standard_normal((n, n))
    raise KeyError(name)


@pytest.mark.parametrize("n", [6, 40, 120])
@pytest.mark.parametrize("name", ["zeros", "identity", "ones", "triangular", "companion", "repeated", "rotation"])
def test_special_inputs(lib, name, n):
    A = _special(name, n, np.random.default_rng(n))
    st, T, Z, lam, XR, XL, _ = run(lib, A)
    assert st == 0
    nA = max(np.linalg.norm(A), 1e-300)
    tol = 40 * n * EPS
    assert np.linalg.norm(Z.T @ Z - np.eye(n)) <= tol
    assert np.linalg.norm(Z.T @ A @ Z - T) <= tol * nA
    VR = Z @ unpack(XR, lam)
    VL = Z @ unpack(XL, lam)
    assert np.all(np.isfinite(VR)) and np.all(np.isfinite(VL))
    # defective / derogatory inputs: the residual identity still holds column by column
    for k in range(n):
        assert np.linalg.norm(A @ VR[:, k] - lam[k] * VR[:, k]) <= 400 * tol * max(nA, 1e-300) * np.linalg.norm(VR[:, k])
        assert np.linalg.norm(VL[:, k].conj() @ A - lam[k] * VL[:, k].conj()) <= 400 * tol * max(nA, 1e-300) * np.linalg.norm(VL[:, k])
    if name == "rotation":
        assert np.allclose(lam.real, 0, atol=tol * nA) and np.count_nonzero(lam.imag) == n


@pytest.mark.parametrize("scale", [1e150, 1e-150])
@pytest.mark.parametrize("cx", [False, True])
def test_scaled_inputs(lib, scale, cx):
    rng = np.random.default_rng(3)
    A = rng.standard_normal((50, 50)) + (1j * rng.standard_normal((50, 50)) if cx else 0)
    st, T, Z, lam, XR, XL, _ = run(lib, A * scale)
    st1, T1, Z1, lam1, *_ = run(lib, A)
    assert st == 0 and st1 == 0
    assert np.linalg.norm(Z.conj().T @ (A * scale) @ Z - T) <= 40 * 50 * EPS * np.linalg.norm(A) * scale
    assert np.allclose(np.sort_complex(lam / scale), np.sort_complex(lam1), rtol=1e-9, atol=1e-9)
