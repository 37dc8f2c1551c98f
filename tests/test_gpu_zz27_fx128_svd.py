"""Double-double SVD (fx128 / cx128) through the C ABI (csrc/svd_dd.cu, csrc/ffi_dd.cu) against rectangular matrices whose singular
values need more than 53 bits (tests/dd_rect_exact.py `rectangular`: sigma = 2^s a + b, exact in dd, exact singular vectors).

Every case checks, with vectors: the values against the exact integers (exact limb differences), the residuals
max_j ||A v_j - sigma_j u_j|| and max_j ||A^H u_j - sigma_j v_j||, ||A^H u_j|| for the columns of a full U past min(m, n) and
||A v_j|| for those of a full V, all through the dd GEMM (matmul_fx128 / cx128); the orthogonality max |U^H U - I| and
max |V^H V - I|, also in dd; and the angle between the computed columns of each exact singular value and its exact singular
subspace (left and right; a zero singular value's subspace includes the null space). Also the values-only path against
the same spectrum. Every bound is 8 N 2^-104 ||A|| with N = m + n (orthogonality: 8 N 2^-104; angles: over the gap), fixed here
and not tuned.

Shapes: fx128 1 x 1, 2 x 1, 32^2, 33 x 17, 17 x 33 (wide: the transpose), 200 x 100 (QR first), 128^2 / 129^2 (the divide and
conquer of order 2n crosses its leaf and merge boundaries), 1000 x 999, 2048 x 1024, 4096^2 and 65536 x 64; cx128 64^2, 65 x 40,
40 x 65 and 1024^2. Spectra: clusters 2^60 + j, heavy ties, exact zeros (rank deficiency), and a cluster 2^-80 apart whose hi limbs
straddle a double boundary (exact, and against mpmath.svd_r / svd_c at 300 bits). Also: thin and full U / V, U only and V only,
the QR-first threshold, non-finite input, size 0 with full factors, row-major / strided / device operands for both kinds,
determinism, and the hi limbs of the values against the f64 entry point."""
import ctypes
import time

import numpy as np
import pytest

import dd_rect_exact as dre

pytestmark = pytest.mark.gpu
NOCONV = 1


def _capi():
    import faer_b200
    return faer_b200.capi


def _lib():
    return _capi().load()


def _dt(cplx):
    return _capi().CX128 if cplx else _capi().FX128


def _to_dd(ex, order="F"):
    m, n = ex.shape
    A = np.zeros((m, n), dtype=_dt(ex.cplx), order=order)
    if ex.cplx:
        A["re_hi"], A["re_lo"], A["im_hi"], A["im_lo"] = ex.hr, ex.lr, ex.hi_, ex.li_
    else:
        A["hi"], A["lo"] = ex.hr, ex.lr
    return A


def _svd(A, cplx, ku=None, kv=None, U=None, V=None, S=None, params=None):
    """ku / kv: columns of U / V (None: not computed)"""
    capi, lib = _capi(), _lib()
    suf = "cx128" if cplx else "fx128"
    m, n = A.shape
    dt = _dt(cplx)
    if S is None:
        S = np.zeros(min(m, n), dtype=dt)
    if U is None and ku is not None:
        U = np.zeros((m, ku), dtype=dt, order="F")
    if V is None and kv is not None:
        V = np.zeros((n, kv), dtype=dt, order="F")
    p = params if params is not None else getattr(lib, f"libfaer_v0_23_SvdParams_{suf}")()
    none = capi.MatMut(None, 0, 0, 0, 0)
    st = getattr(lib, f"libfaer_v0_23_svd_{suf}")(capi.mat_ref(A), capi.mat_mut(U) if U is not None else none,
                                                  capi.VecMut(S.ctypes.data, S.shape[0], S.strides[0] // S.itemsize),
                                                  capi.mat_mut(V) if V is not None else none, capi.par_default(),
                                                  capi.MemAlloc(None, 0), p)
    return st.tag, U, S, V


def _limbs(S, cplx):
    return (S["re_hi"], S["re_lo"]) if cplx else (S["hi"], S["lo"])


def _mm(A, B, cplx):
    capi, lib = _capi(), _lib()
    C = np.zeros((A.shape[0], B.shape[1]), dtype=A.dtype, order="F")
    one = np.zeros(1, dtype=A.dtype)
    one[0][0] = 1.0
    getattr(lib, f"libfaer_v0_23_matmul_{'cx128' if cplx else 'fx128'}")(capi.mat_mut(C), 0, capi.mat_ref(A), capi.mat_ref(B),
                                                                         ctypes.c_void_p(one.ctypes.data), capi.par_default())
    return C


def _adj(X, cplx):
    Y = X.T.copy(order="F")
    if cplx:
        Y["im_hi"], Y["im_lo"] = -Y["im_hi"], -Y["im_lo"]
    return Y


def _diff(X, Y, cplx):
    if cplx:
        return ((X["re_hi"] - Y["re_hi"]) + (X["re_lo"] - Y["re_lo"])) + 1j * ((X["im_hi"] - Y["im_hi"]) + (X["im_lo"] - Y["im_lo"]))
    return (X["hi"] - Y["hi"]) + (X["lo"] - Y["lo"])


def _val(X, cplx):
    return ((X["re_hi"] + X["re_lo"]) + 1j * (X["im_hi"] + X["im_lo"])) if cplx else (X["hi"] + X["lo"])


def _hi(X, cplx):
    return (X["re_hi"] + 1j * X["im_hi"]) if cplx else X["hi"]


def _diag(S, cplx):
    p = S.shape[0]
    D = np.zeros((p, p), dtype=S.dtype, order="F")
    D[np.arange(p), np.arange(p)] = S
    return D


def value_ratio(ex, S, cplx):
    m, n = ex.shape
    if min(m, n) == 0:
        return 0.0
    hi, lo = _limbs(S, cplx)
    eh, el = ex.values_dd()
    return float(np.abs((hi - eh) + (lo - el)).max() / (dre.P_FACTOR * (m + n) * dre.U * max(ex.norm(), 1.0)))


def angle_ratio(ex, X, E_all, bound):
    """largest sine between the computed columns of each exact singular value and its exact singular subspace, over bound / gap.
    E_all: the exact singular vectors of the min(m, n) values; the subspace of a zero singular value also holds the null space, so
    its sine is the norm of X's part along the exact vectors of the nonzero values"""
    p = min(ex.shape)
    sig = ex.sigma()
    worst, i = 0.0, 0
    while i < p:
        j = i
        while j + 1 < p and sig[j + 1] == sig[i]:
            j += 1
        gap = min([sig[i - 1] - sig[i]] if i > 0 else [10 ** 40])
        gap = min(gap, sig[j] - sig[j + 1] if j + 1 < p else gap)
        Xc = X[:, i:j + 1]
        if sig[i] == 0:
            s = np.linalg.norm(np.conj(E_all[:, :i].T) @ Xc, 2) if i else 0.0
        else:
            E = E_all[:, i:j + 1]
            s = np.linalg.norm(Xc - E @ (np.conj(E.T) @ Xc), 2)
        worst = max(worst, s / (bound / float(gap)))
        i = j + 1
    return float(worst)


def _check(ex, A, U, S, V, tag):
    cplx = ex.cplx
    m, n = ex.shape
    p = min(m, n)
    N = m + n
    bound = dre.P_FACTOR * N * dre.U * max(ex.norm(), 1.0)
    ratios = {"values": value_ratio(ex, S, cplx)}
    if p:
        D = _diag(S, cplx)
        AV = _mm(A, V, cplx)
        Ah = _adj(A, cplx)
        AhU = _mm(Ah, U, cplx)
        r1 = np.linalg.norm(_diff(AV[:, :p], _mm(U[:, :p].copy(order="F"), D, cplx), cplx), axis=0).max()
        VS = _mm(V[:, :p].copy(order="F"), D, cplx)
        r2 = np.linalg.norm(_diff(AhU[:, :p], VS, cplx), axis=0).max()
        if U.shape[1] > p:
            r2 = max(r2, np.linalg.norm(_val(AhU[:, p:], cplx), axis=0).max())
        if V.shape[1] > p:
            r1 = max(r1, np.linalg.norm(_val(AV[:, p:], cplx), axis=0).max())
        ratios["residual_av"] = float(r1 / bound)
        ratios["residual_ahu"] = float(r2 / bound)
    for name, Q in (("orth_u", U), ("orth_v", V)):
        k = Q.shape[1]
        I = np.zeros((k, k), dtype=Q.dtype, order="F")
        (I["re_hi"] if cplx else I["hi"])[np.arange(k), np.arange(k)] = 1.0
        ratios[name] = float(np.abs(_diff(_mm(_adj(Q, cplx), Q, cplx), I, cplx)).max(initial=0.0) / (dre.P_FACTOR * N * dre.U))
    ratios["angle_u"] = angle_ratio(ex, _hi(U, cplx), ex.U, bound)
    ratios["angle_v"] = angle_ratio(ex, _hi(V, cplx), ex.V, bound)
    print(f"[zz27] {tag}: {({k: float(f'{v:.3g}') for k, v in ratios.items()})}")
    for k, v in ratios.items():
        assert v <= 1.0, (tag, k, v)


def _spectrum(p, rng, kind):
    if kind == "cluster":  # 2^60 + j (some repeated), a group of small values, and exact zeros
        a = np.ones(p, dtype=np.int64)
        b = rng.integers(0, max(p, 2), size=p)
        a[: p // 8] = 0
        b[: p // 16] = 0
        return a, b
    a = rng.integers(0, 3, size=p)  # heavy ties, zeros included
    b = rng.integers(0, 4, size=p)
    return a, b


def _case(m, n, cplx, kind, seed, full):
    rng = np.random.default_rng(seed)
    ex = dre.rectangular(m, n, *_spectrum(min(m, n), rng, kind), rng, cplx=cplx)
    A = _to_dd(ex)
    p = min(m, n)
    t0 = time.time()
    tag, U, S, V = _svd(A, cplx, m if full else p, n if full else p)
    t1 = time.time()
    assert tag == 0
    if cplx:
        assert np.all(S["im_hi"] == 0) and np.all(S["im_lo"] == 0)
    _check(ex, A, U, S, V, f"{'cx' if cplx else 'fx'}128 {m}x{n} {kind} {'full' if full else 'thin'} ({t1 - t0:.2f} s)")
    t1 = time.time()
    tag, _, S2, _ = _svd(A, cplx)
    assert tag == 0
    r = value_ratio(ex, S2, cplx)
    print(f"[zz27] {'cx' if cplx else 'fx'}128 {m}x{n} values only: {r:.3g} ({time.time() - t1:.2f} s)")
    assert r <= 1.0


FX_SHAPES = [(1, 1, True), (2, 1, True), (32, 32, True), (33, 17, True), (17, 33, True), (200, 100, True), (128, 128, False),
             (129, 129, True), (1000, 999, False), (2048, 1024, True), (4096, 4096, False), (65536, 64, False)]


@pytest.mark.parametrize("m,n,full", FX_SHAPES)
def test_fx128_exact_spectrum(m, n, full):
    _case(m, n, False, "cluster" if (m + n) % 2 == 0 else "ties", m * 7 + n, full)


@pytest.mark.parametrize("m,n,full", [(64, 64, True), (65, 40, True), (40, 65, True), (1024, 1024, False)])
def test_cx128_exact_spectrum(m, n, full):
    _case(m, n, True, "cluster" if m % 2 == 0 else "ties", 1000 + m + n, full)


@pytest.mark.parametrize("cplx", [False, True])
def test_u_only_v_only_and_the_qr_threshold(cplx):
    """U only and V only give the same bits as the call with both; a qr_ratio_threshold above m / n bidiagonalizes A itself"""
    lib = _lib()
    for m, n in ((200, 100), (60, 90)):
        rng = np.random.default_rng(m + n)
        ex = dre.rectangular(m, n, *_spectrum(min(m, n), rng, "cluster"), rng, cplx=cplx)
        A = _to_dd(ex)
        tag, U, S, V = _svd(A, cplx, m, n)
        assert tag == 0
        tag, Uo, So, _ = _svd(A, cplx, ku=m)
        assert tag == 0 and Uo.tobytes() == U.tobytes() and So.tobytes() == S.tobytes()
        tag, _, So, Vo = _svd(A, cplx, kv=min(m, n))
        assert tag == 0 and Vo.tobytes() == V[:, :min(m, n)].tobytes() and So.tobytes() == S.tobytes()
        p = getattr(lib, f"libfaer_v0_23_SvdParams_{'cx128' if cplx else 'fx128'}")()
        p.qr_ratio_threshold = 100.0
        tag, U2, S2, V2 = _svd(A, cplx, m, n, params=p)
        assert tag == 0
        _check(ex, A, U2, S2, V2, f"{'cx' if cplx else 'fx'}128 {m}x{n} without QR first")
        if m > n:
            assert U2.tobytes() != U.tobytes()  # the other path was taken


def test_gaps_of_2e_80_straddling_a_double():
    """sigma = 2^80 + 2^27 + j: neighbouring values 2^-80 apart relative to their size, around the midpoint of two doubles (the hi
    limbs of the values below and above it differ by one ulp, their lo limbs have opposite signs). Exact spectrum, and the values
    of a smaller case against mpmath.svd_r / svd_c at 300 bits."""
    import mpmath
    for m, n, cplx in ((96, 64, False), (64, 64, True), (40, 70, False)):
        rng = np.random.default_rng(m + n)
        p = min(m, n)
        a = np.ones(p, dtype=np.int64)
        b = (1 << 27) + rng.permutation(np.arange(-(p // 2), p - p // 2))
        ex = dre.rectangular(m, n, a, b, rng, cplx=cplx, s=80)
        eh, el = ex.values_dd()
        assert len(set(eh)) == 2 and (el > 0).any() and (el < 0).any()
        A = _to_dd(ex)
        tag, U, S, V = _svd(A, cplx, m, n)
        assert tag == 0
        _check(ex, A, U, S, V, f"{'cx' if cplx else 'fx'}128 {m}x{n} 2^-80 straddling")
        tag, _, S2, _ = _svd(A, cplx)
        assert tag == 0 and value_ratio(ex, S2, cplx) <= 1.0
    mpmath.mp.prec = 300
    for cplx in (False, True):
        m, n = 24, 16
        rng = np.random.default_rng(24 + cplx)
        b = (1 << 27) + rng.permutation(np.arange(-8, 8))
        ex = dre.rectangular(m, n, np.ones(n, dtype=np.int64), b, rng, cplx=cplx, s=80)
        A = _to_dd(ex)
        M = mpmath.matrix(m, n)
        for i in range(m):
            for j in range(n):
                re = mpmath.mpf(ex.hr[i, j]) + mpmath.mpf(ex.lr[i, j])
                M[i, j] = mpmath.mpc(re, mpmath.mpf(ex.hi_[i, j]) + mpmath.mpf(ex.li_[i, j])) if cplx else re
        ref = mpmath.svd_c(M, compute_uv=False) if cplx else mpmath.svd_r(M, compute_uv=False)
        ref = sorted((ref[i] for i in range(n)), reverse=True)
        bound = dre.P_FACTOR * (m + n) * dre.U * float(ref[0])
        for ku in (None, m):
            tag, _, S, _ = _svd(A, cplx, ku, n if ku else None)
            assert tag == 0
            hi, lo = _limbs(S, cplx)
            err = max(abs(mpmath.mpf(h) + mpmath.mpf(l) - r) for h, l, r in zip(hi, lo, ref))
            print(f"[zz27] mpmath {'svd_c' if cplx else 'svd_r'} {m}x{n} vectors={ku is not None}: {float(err) / bound:.3g}")
            assert float(err) <= bound


def test_nonfinite_input_and_size_zero():
    for cplx in (False, True):
        dt = _dt(cplx)
        for m, n in ((6, 4), (4, 6), (30, 5)):
            A = np.zeros((m, n), dtype=dt, order="F")
            (A["re_hi"] if cplx else A["hi"])[np.arange(min(m, n)), np.arange(min(m, n))] = np.arange(1, min(m, n) + 1)
            for bad in (np.inf, np.nan):
                (A["re_hi"] if cplx else A["hi"])[m - 1, 1] = bad
                assert _svd(A, cplx)[0] == NOCONV
                assert _svd(A, cplx, m, n)[0] == NOCONV
                assert _svd(A, cplx, min(m, n))[0] == NOCONV
            if cplx:
                A["re_hi"][m - 1, 1] = 0.0
                A["im_lo"][0, n - 1] = np.nan
                assert _svd(A, cplx, m, n)[0] == NOCONV
        # size == 0: a requested full factor is the identity
        for m, n in ((0, 5), (4, 0), (0, 0)):
            A = np.zeros((m, n), dtype=dt, order="F")
            U = np.full((m, m), 7.0, dtype=np.float64).astype(dt) if m else np.zeros((0, 0), dtype=dt)
            V = np.full((n, n), 7.0, dtype=np.float64).astype(dt) if n else np.zeros((0, 0), dtype=dt)
            U, V = np.asfortranarray(U), np.asfortranarray(V)
            if m:
                U[:] = np.zeros(1, dtype=dt)[0]
                (U["re_hi"] if cplx else U["hi"])[:] = 7.0
            if n:
                V[:] = np.zeros(1, dtype=dt)[0]
                (V["re_hi"] if cplx else V["hi"])[:] = 7.0
            tag, U, _, V = _svd(A, cplx, m if m else None, n if n else None, U=U if m else None, V=V if n else None)
            assert tag == 0
            for Q, k in ((U, m), (V, n)):
                if k:
                    assert np.array_equal(_val(Q, cplx), np.eye(k))
            assert _svd(A, cplx)[0] == 0


@pytest.mark.parametrize("cplx", [False, True])
def test_row_major_strided_device_operands_and_determinism(cplx):
    import torch
    capi, lib = _capi(), _lib()
    suf, dt, limbs = ("cx128", capi.CX128, (2, 2)) if cplx else ("fx128", capi.FX128, (2,))
    for m, n in ((150, 90), (70, 110)):
        rng = np.random.default_rng(m * n)
        ex = dre.rectangular(m, n, *_spectrum(min(m, n), rng, "cluster"), rng, cplx=cplx)
        p = min(m, n)
        A = _to_dd(ex)
        tag, U, S, V = _svd(A, cplx, m, p)
        assert tag == 0
        tag, U2, S2, V2 = _svd(A, cplx, m, p)
        assert tag == 0 and U.tobytes() == U2.tobytes() and S.tobytes() == S2.tobytes() and V.tobytes() == V2.tobytes()
        # row-major A, U and V strided windows of larger arrays, S with stride 3 (element units)
        Ar = _to_dd(ex, order="C")
        bigu = np.zeros((m + 7, 2 * m), dtype=dt, order="F")
        bigv = np.zeros((n, 3 * p), dtype=dt, order="C")
        Uw, Vw = bigu[3:3 + m, ::2], bigv[:, ::3]
        Sb = np.zeros(3 * p, dtype=dt)
        tag, _, _, _ = _svd(Ar, cplx, U=Uw, V=Vw, S=Sb[::3])
        assert tag == 0
        assert Uw.tobytes() == U.tobytes() and Vw.tobytes() == V.tobytes() and Sb[::3].tobytes() == S.tobytes()
        # device operands: row-major A, U and V, contiguous S
        dev = torch.device("cuda")
        At = capi.DDTensor(torch.from_numpy(Ar.view(np.float64).reshape((m, n) + limbs).copy()).to(dev), cplx)
        Ut = capi.DDTensor(torch.zeros((m, m) + limbs, dtype=torch.float64, device=dev), cplx)
        Vt = capi.DDTensor(torch.zeros((n, p) + limbs, dtype=torch.float64, device=dev), cplx)
        St = torch.zeros((p,) + limbs, dtype=torch.float64, device=dev)
        prm = getattr(lib, f"libfaer_v0_23_SvdParams_{suf}")()
        st = getattr(lib, f"libfaer_v0_23_svd_{suf}")(capi.mat_ref(At), capi.mat_mut(Ut), capi.VecMut(St.data_ptr(), p, 1),
                                                      capi.mat_mut(Vt), capi.par_default(), capi.MemAlloc(None, 0), prm)
        assert st.tag == 0
        assert St.cpu().numpy().tobytes() == S.tobytes()
        assert np.ascontiguousarray(Ut.t.cpu().numpy()).reshape(m, m, -1).view(dt).reshape(m, m).tobytes() == U.tobytes()
        assert np.ascontiguousarray(Vt.t.cpu().numpy()).reshape(n, p, -1).view(dt).reshape(n, p).tobytes() == V.tobytes()


def test_hi_limbs_agree_with_the_f64_entry_point():
    capi, lib = _capi(), _lib()
    rng = np.random.default_rng(5)
    m, n = 1000, 700
    A64 = np.asfortranarray(rng.standard_normal((m, n)))
    A = np.zeros((m, n), dtype=capi.FX128, order="F")
    A["hi"] = A64
    tag, _, S, _ = _svd(A, False)
    assert tag == 0
    S64 = np.zeros(n)
    p = lib.libfaer_v0_23_SvdParams_f64()
    none = capi.MatMut(None, 0, 0, 0, 0)
    st = lib.libfaer_v0_23_svd_f64(capi.mat_ref(A64), none, capi.VecMut(S64.ctypes.data, n, 1), none, capi.par_default(),
                                   capi.MemAlloc(None, 0), p)
    assert st.tag == 0
    assert np.abs(S["hi"] - S64).max() <= 8 * (m + n) * 2.0 ** -53 * np.linalg.norm(A64, 2)
