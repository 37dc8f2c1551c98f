"""Double-double self-adjoint EVD (fx128 / cx128) through the C ABI (csrc/evd_dd.cu, csrc/ffi_dd.cu) against matrices whose
spectra need more than 53 bits (tests/dd_spectral_exact.py: clusters 2^60 + j, exact in dd).

Every case checks, with vectors: the eigenvalues against the exact integers, the residual max_j ||A u_j - lambda_j u_j|| and the
orthogonality max |U^H U - I| evaluated with the dd GEMM (matmul_fx128 / cx128), and the angle of each exact eigenspace; and the
values-only path (bisection) against the same spectrum. Every bound is 8 N 2^-104 ||A|| (angles: over the gap), not tuned.
Sizes cross the divide-and-conquer leaf / merge boundaries (32 / 33 ... 128 / 129) and reach 4096; cx128 at 64, 65 and 1024.
Also: eigenvalues 2^-80 apart across a double boundary against mpmath, a NaN strict upper triangle, non-finite input, n = 0 and 1,
device operands, row-major and strided views (fx128 and cx128), determinism, and the hi limbs of the values against the f64 entry
point."""
import time

import numpy as np
import pytest

import dd_spectral_exact as dse

pytestmark = pytest.mark.gpu
NOCONV = 1


def _capi():
    import faer_b200
    return faer_b200.capi


def _lib():
    return _capi().load()


def _to_dd(ex, order="F"):
    capi = _capi()
    n = ex.n
    if ex.cplx:
        A = np.zeros((n, n), dtype=capi.CX128, order=order)
        A["re_hi"], A["re_lo"], A["im_hi"], A["im_lo"] = ex.hr, ex.lr, ex.hi_, ex.li_
    else:
        A = np.zeros((n, n), dtype=capi.FX128, order=order)
        A["hi"], A["lo"] = ex.hr, ex.lr
    return A


def _evd(A, cplx, vectors=True, U=None, S=None):
    capi, lib = _capi(), _lib()
    suf = "cx128" if cplx else "fx128"
    n = A.shape[0]
    dt = capi.CX128 if cplx else capi.FX128
    if S is None:
        S = np.zeros(n, dtype=dt)
    if vectors and U is None:
        U = np.zeros((n, n), dtype=dt, order="F")
    p = getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}")()
    uv = capi.mat_mut(U) if vectors else capi.MatMut(None, 0, 0, 0, 0)
    sv = capi.VecMut(S.ctypes.data, n, S.strides[0] // S.itemsize)
    st = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_{suf}")(capi.mat_ref(A), uv, sv, capi.par_default(), capi.MemAlloc(None, 0), p)
    return st.tag, U, S


def _limbs(S, cplx):
    return (S["re_hi"], S["re_lo"]) if cplx else (S["hi"], S["lo"])


def _matmul(lib, cplx, C, A, B):
    capi = _capi()
    suf = "cx128" if cplx else "fx128"
    one = np.zeros(1, dtype=capi.CX128 if cplx else capi.FX128)
    one[0][0] = 1.0
    getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(C), 0, capi.mat_ref(A), capi.mat_ref(B), C_void(one), capi.par_default())
    return C


def C_void(a):
    import ctypes
    return ctypes.c_void_p(a.ctypes.data)


def _val(X, cplx):
    """(value, error-free) as complex128 / float64 hi + lo (for norms of small differences)"""
    if cplx:
        return (X["re_hi"] + X["re_lo"]) + 1j * (X["im_hi"] + X["im_lo"])
    return X["hi"] + X["lo"]


def _diff(X, Y, cplx):
    if cplx:
        return ((X["re_hi"] - Y["re_hi"]) + (X["re_lo"] - Y["re_lo"])) + 1j * ((X["im_hi"] - Y["im_hi"]) + (X["im_lo"] - Y["im_lo"]))
    return (X["hi"] - Y["hi"]) + (X["lo"] - Y["lo"])


def _check(ex, A, U, S, tag):
    capi, lib = _capi(), _lib()
    n, cplx = ex.n, ex.cplx
    bound = dse.P_FACTOR * n * dse.U * ex.norm()
    hi, lo = _limbs(S, cplx)
    r_val = dse.value_ratio(ex, hi, lo)
    # residual: A U - U diag(S), both products in dd
    D = np.zeros((n, n), dtype=A.dtype, order="F")
    if cplx:
        D["re_hi"][np.diag_indices(n)], D["re_lo"][np.diag_indices(n)] = hi, lo
    else:
        D["hi"][np.diag_indices(n)], D["lo"][np.diag_indices(n)] = hi, lo
    AU = _matmul(lib, cplx, np.zeros((n, n), dtype=A.dtype, order="F"), A, U)
    UL = _matmul(lib, cplx, np.zeros((n, n), dtype=A.dtype, order="F"), U, D)
    r_res = float(np.linalg.norm(_diff(AU, UL, cplx), axis=0).max() / bound)
    # orthogonality: U^H U - I (conjugate transpose as a view: conj through the imaginary limbs)
    Uh = U.T.copy(order="F")
    if cplx:
        Uh["im_hi"], Uh["im_lo"] = -Uh["im_hi"], -Uh["im_lo"]
    G = _matmul(lib, cplx, np.zeros((n, n), dtype=A.dtype, order="F"), Uh, U)
    I = np.zeros((n, n), dtype=A.dtype, order="F")
    (I["re_hi"] if cplx else I["hi"])[np.diag_indices(n)] = 1.0
    r_orth = float(np.abs(_diff(G, I, cplx)).max() / (dse.P_FACTOR * n * dse.U))
    r_ang = dse.angle_ratio(ex, (U["re_hi"] + 1j * U["im_hi"]) if cplx else U["hi"])
    ratios = {"values": r_val, "residual": r_res, "orth": r_orth, "angle": r_ang}
    print(f"[zz25] {tag}: {({k: float(f'{v:.3g}') for k, v in ratios.items()})}")
    for k, v in ratios.items():
        assert v <= 1.0, (tag, k, v)


def _spectrum(n, rng, kind):
    if kind == "cluster":  # 2^60 + j, a few repeated, plus a negative and a zero group
        a = np.ones(n, dtype=np.int64)
        b = rng.integers(-n, n, size=n)
        a[: n // 8] = -1
        a[n // 8: n // 8 + n // 16] = 0
        return a, b
    a = rng.integers(-1, 2, size=n)
    b = rng.integers(-3, 4, size=n)  # heavy ties
    return a, b


SIZES = [32, 33, 64, 65, 128, 129, 1000, 2048, 4096]


@pytest.mark.parametrize("n", SIZES)
def test_fx128_exact_spectrum(n):
    rng = np.random.default_rng(n)
    ex = dse.build(*_spectrum(n, rng, "cluster" if n % 2 == 0 else "ties"), rng)
    A = _to_dd(ex)
    t0 = time.time()
    tag, U, S = _evd(A, False)
    t1 = time.time()
    assert tag == 0
    _check(ex, A, U, S, f"fx128 n={n} ({t1 - t0:.2f} s)")
    tag, _, S2 = _evd(A, False, vectors=False)
    assert tag == 0
    r = dse.value_ratio(ex, *_limbs(S2, False))
    print(f"[zz25] fx128 n={n} values only: {r:.3g} ({time.time() - t1:.2f} s)")
    assert r <= 1.0


@pytest.mark.parametrize("n", [64, 65, 1024])
def test_cx128_exact_spectrum(n):
    rng = np.random.default_rng(1000 + n)
    ex = dse.build(*_spectrum(n, rng, "cluster"), rng, cplx=True)
    A = _to_dd(ex)
    tag, U, S = _evd(A, True)
    assert tag == 0
    assert np.all(S["im_hi"] == 0) and np.all(S["im_lo"] == 0)
    _check(ex, A, U, S, f"cx128 n={n}")
    tag, _, S2 = _evd(A, True, vectors=False)
    assert tag == 0
    assert dse.value_ratio(ex, *_limbs(S2, True)) <= 1.0


@pytest.mark.parametrize("cplx", [False, True])
def test_nan_upper_triangle_is_not_read_and_calls_are_deterministic(cplx):
    rng = np.random.default_rng(7)
    n = 97
    ex = dse.build(*_spectrum(n, rng, "cluster"), rng, cplx=cplx)
    A = _to_dd(ex)
    An = A.copy(order="F")
    iu = np.triu_indices(n, 1)
    for f in An.dtype.names:
        An[f][iu] = np.nan
    tag, U, S = _evd(An, cplx)
    assert tag == 0
    _check(ex, A, U, S, f"{'cx' if cplx else 'fx'}128 NaN upper")  # the residual's GEMM reads the whole (clean) A
    tag2, U2, S2 = _evd(An, cplx)
    assert tag2 == 0 and U.tobytes() == U2.tobytes() and S.tobytes() == S2.tobytes()


def test_nonfinite_input_and_tiny_sizes():
    capi = _capi()
    for cplx in (False, True):
        dt = capi.CX128 if cplx else capi.FX128
        A = np.zeros((5, 5), dtype=dt, order="F")
        (A["re_hi"] if cplx else A["hi"])[np.diag_indices(5)] = [1, 2, 3, 4, 5]
        (A["re_hi"] if cplx else A["hi"])[3, 1] = np.inf
        assert _evd(A, cplx)[0] == NOCONV
        assert _evd(A, cplx, vectors=False)[0] == NOCONV
        (A["re_hi"] if cplx else A["hi"])[3, 1] = np.nan
        assert _evd(A, cplx)[0] == NOCONV
        E = np.zeros((0, 0), dtype=dt, order="F")
        assert _evd(E, cplx)[0] == 0 and _evd(E, cplx, vectors=False)[0] == 0
        A1 = np.zeros((1, 1), dtype=dt, order="F")
        (A1["re_hi"] if cplx else A1["hi"])[0, 0] = 2.0 ** 60
        (A1["re_lo"] if cplx else A1["lo"])[0, 0] = 3.0
        tag, U, S = _evd(A1, cplx)
        assert tag == 0 and S.tobytes() == A1.ravel().tobytes()
        assert (U["re_hi"] if cplx else U["hi"])[0, 0] == 1.0
        tag, _, S = _evd(A1, cplx, vectors=False)  # bisection: to 8 u |a| of the value
        hi, lo = _limbs(S, cplx)
        assert tag == 0 and abs((hi[0] - 2.0 ** 60) + (lo[0] - 3.0)) <= 8 * 2.0 ** -104 * 2.0 ** 60


@pytest.mark.parametrize("cplx", [False, True])
def test_row_major_strided_and_device_operands(cplx):
    import torch
    capi, lib = _capi(), _lib()
    suf, dt, limbs = ("cx128", capi.CX128, (2, 2)) if cplx else ("fx128", capi.FX128, (2,))
    rng = np.random.default_rng(11)
    n = 150
    ex = dse.build(*_spectrum(n, rng, "cluster"), rng, cplx=cplx)
    A = _to_dd(ex)
    tag, U, S = _evd(A, cplx)
    assert tag == 0
    # row-major A, U a strided window of a larger array, S with stride 3 (element units)
    Ar = _to_dd(ex, order="C")
    big = np.zeros((n + 7, 2 * n), dtype=dt, order="F")
    Uw = big[3:3 + n, ::2]
    Sb = np.zeros(3 * n, dtype=dt)
    tag2, _, _ = _evd(Ar, cplx, U=Uw, S=Sb[::3])
    assert tag2 == 0 and Uw.tobytes() == U.tobytes() and Sb[::3].tobytes() == S.tobytes()
    # device operands: row-major A and U, contiguous S
    dev = torch.device("cuda")
    At = capi.DDTensor(torch.from_numpy(Ar.view(np.float64).reshape((n, n) + limbs).copy()).to(dev), cplx)
    Ut = capi.DDTensor(torch.zeros((n, n) + limbs, dtype=torch.float64, device=dev), cplx)
    St = torch.zeros((n,) + limbs, dtype=torch.float64, device=dev)
    p = getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_{suf}")(capi.mat_ref(At), capi.mat_mut(Ut), capi.VecMut(St.data_ptr(), n, 1),
                                                               capi.par_default(), capi.MemAlloc(None, 0), p)
    assert st.tag == 0
    assert St.cpu().numpy().tobytes() == S.tobytes()
    assert np.ascontiguousarray(Ut.t.cpu().numpy()).reshape(n, n, -1).view(dt).reshape(n, n).tobytes() == U.tobytes()


def test_gaps_of_2e_80_straddling_a_double():
    """a tridiagonal input whose eigenvalues are 2^-80 apart around the midpoint of two doubles near 1/3 (the hi limbs differ by
    one ulp, the lo limbs have opposite signs): the divide and conquer's poles and roots need dd_sub_accurate here. Reference:
    mpmath.eigsy at 300 bits; bounds 8 N 2^-104 ||A|| as above."""
    import mpmath
    capi, lib = _capi(), _lib()
    mpmath.mp.prec = 300
    n = 100
    rng = np.random.default_rng(80)
    mid = mpmath.mpf(float(mpmath.mpf(1) / 3)) + mpmath.mpf(2) ** -55
    d = [mid + (i - n // 2) * mpmath.mpf(2) ** -80 for i in range(n)]
    e = [mpmath.mpf(float(x)) * mpmath.mpf(2) ** -81 for x in rng.uniform(0.5, 1.0, n - 1)]
    A = np.zeros((n, n), dtype=capi.FX128, order="F")
    M = mpmath.zeros(n, n)
    for i in range(n):
        vals = [(i, i, d[i])] + ([(i + 1, i, e[i]), (i, i + 1, e[i])] if i + 1 < n else [])
        for r, c, v in vals:
            hi = float(v)
            A["hi"][r, c], A["lo"][r, c] = hi, float(v - mpmath.mpf(hi))
            M[r, c] = mpmath.mpf(A["hi"][r, c]) + mpmath.mpf(A["lo"][r, c])
    ref = sorted(mpmath.eigsy(M, eigvals_only=True))
    nrm = float(max(abs(x) for x in ref))
    bound = dse.P_FACTOR * n * dse.U * nrm
    for vectors in (True, False):
        tag, U, S = _evd(A, False, vectors=vectors)
        assert tag == 0
        err = max(abs(mpmath.mpf(h) + mpmath.mpf(l) - r) for h, l, r in zip(S["hi"], S["lo"], ref))
        ratios = {"values": float(err) / bound}
        if vectors:
            D = np.zeros((n, n), dtype=capi.FX128, order="F")
            D["hi"][np.diag_indices(n)], D["lo"][np.diag_indices(n)] = S["hi"], S["lo"]
            AU = _matmul(lib, False, np.zeros((n, n), dtype=capi.FX128, order="F"), A, U)
            UL = _matmul(lib, False, np.zeros((n, n), dtype=capi.FX128, order="F"), U, D)
            ratios["residual"] = float(np.linalg.norm(_diff(AU, UL, False), axis=0).max() / bound)
            G = _matmul(lib, False, np.zeros((n, n), dtype=capi.FX128, order="F"), U.T.copy(order="F"), U)
            I = np.zeros((n, n), dtype=capi.FX128, order="F")
            I["hi"][np.diag_indices(n)] = 1.0
            ratios["orth"] = float(np.abs(_diff(G, I, False)).max() / (dse.P_FACTOR * n * dse.U))
        print(f"[zz25] 2^-80 gaps, vectors={vectors}: {({k: float(f'{v:.3g}') for k, v in ratios.items()})}")
        for k, v in ratios.items():
            assert v <= 1.0, (k, v)


def test_hi_limbs_agree_with_the_f64_entry_point():
    capi, lib = _capi(), _lib()
    rng = np.random.default_rng(5)
    n = 1000
    X = rng.standard_normal((n, n))
    A64 = np.asfortranarray(X + X.T)
    A = np.zeros((n, n), dtype=capi.FX128, order="F")
    A["hi"] = A64
    _, _, S = _evd(A, False, vectors=False)
    S64 = np.zeros(n)
    p = lib.libfaer_v0_23_SelfAdjointEvdParams_f64()
    st = lib.libfaer_v0_23_self_adjoint_evd_f64(capi.mat_ref(A64), capi.MatMut(None, 0, 0, 0, 0), capi.VecMut(S64.ctypes.data, n, 1),
                                                 capi.par_default(), capi.MemAlloc(None, 0), p)
    assert st.tag == 0
    nrm = np.linalg.norm(A64, 2)
    assert np.abs(S["hi"] - S64).max() <= 8 * n * 2.0 ** -53 * nrm
