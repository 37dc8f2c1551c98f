"""Double-double (fx128 / cx128) `matmul`, triangular solves / inverses, `llt_*` and `partial_piv_lu_*` through the C ABI
(csrc/gemm_dd.cu, csrc/dd_factor.cu, csrc/ffi_dd.cu), checked against exact rational arithmetic where the size allows it and
against residual bounds of order n * 2^-104 otherwise. Host arrays use capi.FX128 / capi.CX128; device operands capi.DDTensor."""
import random
from fractions import Fraction as F

import numpy as np
import pytest

import dd_model as DM

pytestmark = pytest.mark.gpu
U = 2.0 ** -104


def _dd(x, rng, dtype):
    """x (float64 or complex128) -> FX128 / CX128 with a nonzero low limb below half an ulp of the high one"""
    out = np.zeros(x.shape, dtype=dtype, order="F")
    def limbs(v):
        lo = v * 2.0 ** -60 * rng.uniform(-0.5, 0.5, v.shape)
        return v + 0.0, lo
    if dtype == _capi().FX128:
        out["hi"], out["lo"] = limbs(np.real(x))
    else:
        out["re_hi"], out["re_lo"] = limbs(np.real(x))
        out["im_hi"], out["im_lo"] = limbs(np.imag(x))
    return out


def _capi():
    import faer_b200
    return faer_b200.capi


def _frac(a):
    """exact value(s) of one element"""
    if "hi" in a.dtype.names:
        return F(float(a["hi"])) + F(float(a["lo"]))
    return (F(float(a["re_hi"])) + F(float(a["re_lo"])), F(float(a["im_hi"])) + F(float(a["im_lo"])))


def _approx(a):
    if "hi" in a.dtype.names:
        return a["hi"] + a["lo"]
    return (a["re_hi"] + a["re_lo"]) + 1j * (a["im_hi"] + a["im_lo"])


def _cmul(x, y):
    return (x[0] * y[0] - x[1] * y[1], x[0] * y[1] + x[1] * y[0]) if isinstance(x, tuple) else x * y


def _cadd(x, y):
    return (x[0] + y[0], x[1] + y[1]) if isinstance(x, tuple) else x + y


def _cabs(x):
    return abs(x[0]) + abs(x[1]) if isinstance(x, tuple) else abs(x)


def _zero(cx):
    return (F(0), F(0)) if cx else F(0)


def _struct_val(M, i, j, s, cx):
    """element of a structured operand (Block codes of common.cuh)"""
    lower, upper = s in (1, 3, 5), s in (2, 4, 6)
    if s != 0:
        if i == j:
            if s in (5, 6):
                return (F(1), F(0)) if cx else F(1)
            if s in (3, 4):
                return _zero(cx)
        elif (lower and i < j) or (upper and i > j):
            return _zero(cx)
    return _frac(M[i, j])


def _mm(lib, suf, C_, cb, accum, A, ab, B, bb, alpha):
    capi = _capi()
    getattr(lib, f"libfaer_v0_23_matmul_triangular_{suf}")(capi.mat_mut(C_), cb, accum, capi.mat_ref(A), ab, capi.mat_ref(B), bb,
                                                           alpha.ctypes.data, capi.par_default())


def _check_product(C0, C1, A, B, alpha, cb, ab, bb, accum, cx):
    m, n = C1.shape
    k = A.shape[1]
    al = _frac(alpha[0])
    for i in range(m):
        for j in range(n):
            lower, upper = cb in (1, 3, 5), cb in (2, 4, 6)
            written = not ((lower and i < j) or (upper and i > j) or (cb in (3, 4, 5, 6) and i == j))
            if not written:
                assert C1[i, j].tobytes() == C0[i, j].tobytes()
                continue
            acc, mag = _zero(cx), F(0)
            for t in range(k):
                a, b = _struct_val(A, i, t, ab, cx), _struct_val(B, t, j, bb, cx)
                acc = _cadd(acc, _cmul(a, b))
                mag += _cabs(a) * _cabs(b)
            want = _cmul(al, acc)
            if accum:
                want = _cadd(want, _frac(C0[i, j]))
                mag += _cabs(_frac(C0[i, j]))
            got = _frac(C1[i, j])
            err = _cabs(_cadd(got, _cmul((F(-1), F(0)) if cx else F(-1), want)))
            assert err <= 8 * (k + 2) * F(U) * (mag * (1 + _cabs(al))), (i, j, float(err), float(mag))


@pytest.mark.parametrize("suf", ["fx128", "cx128"])
@pytest.mark.parametrize("shape", [(1, 1, 1), (17, 13, 29), (64, 64, 0), (130, 50, 70)])
@pytest.mark.parametrize("accum", [0, 1])
def test_matmul_exact(fb, suf, shape, accum):
    capi, lib = fb.capi, fb.load()
    cx = suf == "cx128"
    dt = capi.CX128 if cx else capi.FX128
    rng = np.random.default_rng(hash((suf, shape, accum)) % 2**32)
    m, k, n = shape
    g = lambda *s: rng.standard_normal(s) + (1j * rng.standard_normal(s) if cx else 0)
    A, B, C0 = _dd(g(m, k), rng, dt), _dd(g(k, n), rng, dt), _dd(g(m, n), rng, dt)
    B = np.ascontiguousarray(B)  # row-major rhs
    if m > 64:
        A = A[::-1]  # negative row stride, several tiles and k slices
    alpha = _dd(np.array([1.5 - (0.25j if cx else 0)]), rng, dt)
    C1 = C0.copy(order="F")
    getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(C1), accum, capi.mat_ref(A), capi.mat_ref(B), alpha.ctypes.data,
                                                capi.par_default())
    _check_product(C0, C1, A, B, alpha, 0, 0, 0, accum, cx)


def test_matmul_triangular_structures(fb):
    capi, lib = fb.capi, fb.load()
    rng = np.random.default_rng(5)
    n = 33
    r = random.Random(7)
    combos = [(0, 0, 0)] + [(r.randrange(7), r.randrange(7), r.randrange(7)) for _ in range(10)]
    for suf in ("fx128", "cx128"):
        cx = suf == "cx128"
        dt = capi.CX128 if cx else capi.FX128
        g = lambda *s: rng.standard_normal(s) + (1j * rng.standard_normal(s) if cx else 0)
        for cb, ab, bb in combos:
            A, B, C0 = _dd(g(n, n), rng, dt), _dd(g(n, n), rng, dt), _dd(g(n, n), rng, dt)
            alpha = _dd(np.array([0.75 + (0.5j if cx else 0)]), rng, dt)
            for accum in (0, 1):
                C1 = C0.copy(order="F")
                _mm(lib, suf, C1, cb, accum, A, ab, B, bb, alpha)
                _check_product(C0, C1, A, B, alpha, cb, ab, bb, accum, cx)


def _llt(lib, capi, suf, A, delta=None, eps=None):
    reg = capi.LltRegularization(None, None)
    keep = []
    if delta is not None:
        d = np.array([(delta, 0.0)], dtype=capi.FX128)
        e = np.array([(eps, 0.0)], dtype=capi.FX128)
        keep += [d, e]
        reg = capi.LltRegularization(d.ctypes.data, e.ctypes.data)
    p = getattr(lib, f"libfaer_v0_23_LltParams_{suf}")()
    return getattr(lib, f"libfaer_v0_23_llt_factor_in_place_{suf}")(capi.mat_mut(A), reg, capi.par_default(), capi.MemAlloc(None, 0), p)


def test_llt_hilbert_12_forward_error(fb):
    """cond(H_12) ~ 1.7e16: the f64 factorization loses every digit; the double-double one solves to ~1e-12 or better"""
    capi, lib = fb.capi, fb.load()
    n = 12
    Hf = [[F(1, i + j + 1) for j in range(n)] for i in range(n)]
    H = np.zeros((n, n), dtype=capi.FX128, order="F")
    for i in range(n):
        for j in range(n):
            hi = float(Hf[i][j])
            H[i, j] = (hi, float(Hf[i][j] - F(hi)))
    xs = [F(1 + (i % 3), 1 + i) for i in range(n)]
    b = np.zeros((n, 1), dtype=capi.FX128, order="F")
    for i in range(n):
        v = sum(Hf[i][j] * xs[j] for j in range(n))
        hi = float(v)
        b[i, 0] = (hi, float(v - F(hi)))
    L = H.copy(order="F")
    st = _llt(lib, capi, "fx128", L)
    assert st.tag == 0 and st.value == 0
    getattr(lib, "libfaer_v0_23_llt_solve_in_place_fx128")(capi.mat_ref(L), 0, capi.mat_mut(b), capi.par_default(), capi.MemAlloc(None, 0))
    err = max(abs(_frac(b[i, 0]) - xs[i]) for i in range(n)) / max(abs(x) for x in xs)
    assert err <= F(1, 10**12), float(err)


@pytest.mark.parametrize("suf", ["fx128", "cx128"])
@pytest.mark.parametrize("n", [1, 7, 70, 300])
def test_llt_reconstruct_and_inverse(fb, cuda_dev, suf, n):
    import torch
    capi, lib = fb.capi, fb.load()
    cx = suf == "cx128"
    dt = capi.CX128 if cx else capi.FX128
    rng = np.random.default_rng(n)
    G = rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0)
    S = G @ G.conj().T + n * np.eye(n)
    A = _dd(S, rng, dt)
    if cx:  # a real diagonal
        A["im_hi"][np.arange(n), np.arange(n)] = 0
        A["im_lo"][np.arange(n), np.arange(n)] = 0
    # device operand through DDTensor, row-major storage
    limbs = 4 if cx else 2
    raw = np.ascontiguousarray(A).view(np.float64).reshape((n, n, 2, 2) if cx else (n, n, 2))
    Ad = torch.from_numpy(raw.copy()).to(cuda_dev)
    st = _llt(lib, capi, suf, capi.DDTensor(Ad, cx))
    assert st.tag == 0
    L = np.ascontiguousarray(Ad.cpu().numpy()).reshape(n * n * limbs).view(dt).reshape(n, n)
    R = np.zeros((n, n), dtype=dt, order="F")
    getattr(lib, f"libfaer_v0_23_llt_reconstruct_{suf}")(capi.mat_mut(R), capi.mat_ref(L), capi.par_default(), capi.MemAlloc(None, 0))
    # lower triangle of R = A within a few n u |A|: compare limb-wise in f64 (hi differences are exact)
    key = ("re_hi", "re_lo", "im_hi", "im_lo") if cx else ("hi", "lo")
    scale = np.abs(S).max()
    low = np.tril(np.ones((n, n), bool))
    for h, l in zip(key[::2], key[1::2]):
        d = (R[h] - A[h]) + (R[l] - A[l])
        assert np.all(np.abs(d[low]) <= 64 * n * U * scale * 4)
    # determinism
    Ad2 = torch.from_numpy(raw.copy()).to(cuda_dev)
    _llt(lib, capi, suf, capi.DDTensor(Ad2, cx))
    assert torch.equal(Ad, Ad2)
    Ainv = np.zeros((n, n), dtype=dt, order="F")
    getattr(lib, f"libfaer_v0_23_llt_inverse_{suf}")(capi.mat_mut(Ainv), capi.mat_ref(L), capi.par_default(), capi.MemAlloc(None, 0))
    Ai = np.tril(_approx(Ainv))
    Ai = Ai + np.tril(Ai, -1).conj().T
    assert np.abs(Ai @ S - np.eye(n)).max() <= 1e-10


def test_llt_nonfinite_and_regularization(fb):
    capi, lib = fb.capi, fb.load()
    A = np.zeros((3, 3), dtype=capi.FX128, order="F")
    A["hi"] = np.eye(3)
    A["hi"][1, 1] = np.nan
    st = _llt(lib, capi, "fx128", A)
    assert st.tag == 1 and st.value == 1
    B = np.zeros((3, 3), dtype=capi.FX128, order="F")
    B["hi"] = np.diag([1.0, -1.0, 4.0])
    st = _llt(lib, capi, "fx128", B.copy(order="F"))
    assert st.tag == 1 and st.value == 1
    st = _llt(lib, capi, "fx128", B, delta=2.0, eps=1e-10)
    assert st.tag == 0 and st.value == 1


@pytest.mark.parametrize("suf", ["fx128", "cx128"])
@pytest.mark.parametrize("shape", [(1, 1), (7, 7), (16, 16), (17, 17), (100, 100), (513, 513), (40, 25), (25, 40)])
def test_lu(fb, oracle, suf, shape):
    capi, lib = fb.capi, fb.load()
    cx = suf == "cx128"
    dt = capi.CX128 if cx else capi.FX128
    m, n = shape
    rng = np.random.default_rng(m * 1000 + n)
    X = rng.standard_normal((m, n)) + (1j * rng.standard_normal((m, n)) if cx else 0)
    A = np.zeros((m, n), dtype=dt, order="F")
    if cx:
        A["re_hi"], A["im_hi"] = X.real, X.imag
    else:
        A["hi"] = X
    # pivots: with lo = 0 inputs the f64 oracle's LU makes the same choices unless two candidates agree to ~1e-16
    want = np.asfortranarray(X.copy())
    perm_o, _, nt_o = oracle.lu(want)
    for it, idt in (("u32", np.uint32), ("u64", np.uint64)):
        LU = A.copy(order="F")
        pf, pb = np.zeros(m, idt), np.zeros(m, idt)
        p = getattr(lib, f"libfaer_v0_23_PartialPivLuParams_{suf}")()
        st = getattr(lib, f"libfaer_v0_23_partial_piv_lu_factor_in_place_{it}_{suf}")(
            capi.mat_mut(LU), capi.slice_mut(pf), capi.slice_mut(pb), capi.par_default(), capi.MemAlloc(None, 0), p)
        assert st.tag == 0
        if m <= 100:
            assert np.array_equal(pf.astype(np.int64), perm_o) and st.value == nt_o
        assert np.array_equal(pb[pf.astype(np.int64)], np.arange(m))
        size = min(m, n)
        L = np.tril(_approx(LU), -1)[:, :size] + np.eye(m, size)
        Uf = np.triu(_approx(LU))[:size, :]
        assert np.abs(L @ Uf - X[pf.astype(np.int64)]).max() <= 1e-13 * size * np.abs(L).max() * np.abs(Uf).max()
        if m > n:
            continue
        R = np.zeros((m, n), dtype=dt, order="F")
        getattr(lib, f"libfaer_v0_23_partial_piv_lu_reconstruct_{it}_{suf}")(
            capi.mat_mut(R), capi.mat_ref(np.asfortranarray(LU[:, :size])), capi.mat_ref(np.asfortranarray(LU[:size, :])),
            capi.slice_mut(pf), capi.slice_mut(pb), capi.par_default(), capi.MemAlloc(None, 0))
        key = ("re_hi", "re_lo", "im_hi", "im_lo") if cx else ("hi", "lo")
        for h, l in zip(key[::2], key[1::2]):
            d = (R[h] - A[h]) + (R[l] - A[l])
            assert np.abs(d).max() <= 64 * size * U * np.abs(L).max() * np.abs(Uf).max() * 4
        if m != n:
            continue
        bx = rng.standard_normal((n, 3)) + (1j * rng.standard_normal((n, 3)) if cx else 0)
        for name, M in (("solve", X), ("solve_transpose", X.T)):
            b = np.zeros((n, 3), dtype=dt, order="F")
            if cx:
                b["re_hi"], b["im_hi"] = bx.real, bx.imag
            else:
                b["hi"] = bx
            getattr(lib, f"libfaer_v0_23_partial_piv_lu_{name}_in_place_{it}_{suf}")(
                capi.mat_ref(LU), capi.mat_ref(LU), 0, capi.slice_mut(pf), capi.slice_mut(pb), capi.mat_mut(b),
                capi.par_default(), capi.MemAlloc(None, 0))
            x = _approx(b)
            assert np.abs(M @ x - bx).max() <= 1e-9 * np.abs(M).max() * np.abs(x).max() * n
        Ainv = np.zeros((n, n), dtype=dt, order="F")
        getattr(lib, f"libfaer_v0_23_partial_piv_lu_inverse_{it}_{suf}")(
            capi.mat_mut(Ainv), capi.mat_ref(LU), capi.mat_ref(LU), capi.slice_mut(pf), capi.slice_mut(pb), capi.par_default(),
            capi.MemAlloc(None, 0))
        assert np.abs(_approx(Ainv) @ X - np.eye(n)).max() <= 1e-8 * n


@pytest.mark.parametrize("suf", ["fx128", "cx128"])
def test_triangular_solves_and_inverses(fb, suf):
    capi, lib = fb.capi, fb.load()
    cx = suf == "cx128"
    dt = capi.CX128 if cx else capi.FX128
    rng = np.random.default_rng(3)
    n, k = 90, 5
    # off-diagonal entries of order 1 / n keep the unit-diagonal factors well conditioned for the f64 residual check
    T = (rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0)) / n + 2 * np.eye(n)
    Td = _dd(T, rng, dt)
    Tv = _approx(Td)
    for name, lower, unit in (("solve_triangular_lower", True, False), ("solve_triangular_upper", False, False),
                              ("solve_unit_triangular_lower", True, True), ("solve_unit_triangular_upper", False, True)):
        M = np.tril(Tv) if lower else np.triu(Tv)
        if unit:
            M = M - np.diag(np.diag(M)) + np.eye(n)
        for conj in ((0, 1) if cx else (0,)):
            bx = rng.standard_normal((n, k)) + (1j * rng.standard_normal((n, k)) if cx else 0)
            b = _dd(bx, rng, dt)
            b0 = _approx(b)
            b = np.ascontiguousarray(b)  # row-major rhs
            getattr(lib, f"libfaer_v0_23_{name}_in_place_{suf}")(capi.mat_ref(Td), conj, capi.mat_mut(b), capi.par_default())
            Mc = M.conj() if conj else M
            assert np.abs(Mc @ _approx(b) - b0).max() <= 1e-12
        inv = name.replace("solve", "inverse")
        D0 = _dd(rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0), rng, dt)
        D = D0.copy(order="F")
        getattr(lib, f"libfaer_v0_23_{inv}_in_place_{suf}")(capi.mat_mut(D), capi.mat_ref(Td), capi.par_default())
        tri = np.tril(np.ones((n, n), bool), -1 if unit else 0) if lower else np.triu(np.ones((n, n), bool), 1 if unit else 0)
        assert D[~tri].tobytes() == D0[~tri].tobytes()
        Dv = np.where(tri, _approx(D), 0) + (np.eye(n) if unit else 0)
        assert np.abs(Dv @ M - np.eye(n)).max() <= 1e-12


def test_large_matmul_against_f64(fb):
    """513 x 1031 x 257: the dd product with lo = 0 inputs agrees with the f64 product to f64 accuracy and is deterministic"""
    capi, lib = fb.capi, fb.load()
    rng = np.random.default_rng(11)
    m, k, n = 513, 1031, 257
    X, Y = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    A = np.zeros((m, k), dtype=capi.FX128, order="F"); A["hi"] = X
    B = np.zeros((k, n), dtype=capi.FX128, order="F"); B["hi"] = Y
    alpha = np.array([(1.0, 0.0)], dtype=capi.FX128)
    outs = []
    for _ in range(2):
        Cm = np.zeros((m, n), dtype=capi.FX128, order="F")
        lib.libfaer_v0_23_matmul_fx128(capi.mat_mut(Cm), 0, capi.mat_ref(A), capi.mat_ref(B), alpha.ctypes.data, capi.par_default())
        outs.append(Cm)
    assert outs[0].tobytes() == outs[1].tobytes()
    ref = X @ Y
    assert np.abs(_approx(outs[0]) - ref).max() <= 4 * k * 2.0 ** -53 * (np.abs(X) @ np.abs(Y)).max()


def _bound_arrays(A, B, cx):
    return np.abs(_approx(A)) @ np.abs(_approx(B))


def _structured(X, s, cx):
    """numpy copy of a structured operand with the excluded half zeroed and a unit / strict diagonal applied"""
    Y = X.copy(order="F")
    n = X.shape[0]
    keys = ("re_hi", "re_lo", "im_hi", "im_lo") if cx else ("hi", "lo")
    if s != 0:
        lower = s in (1, 3, 5)
        mask = np.tril(np.ones(X.shape, bool), -1) if lower else np.triu(np.ones(X.shape, bool), 1)
        for k in keys:
            Y[k][~mask] = np.where(np.eye(n, X.shape[1], dtype=bool), Y[k], 0)[~mask] if s in (1, 2) else 0
        if s in (5, 6):
            Y[keys[0]][np.eye(n, X.shape[1], dtype=bool)] = 1
    return Y


@pytest.mark.parametrize("suf", ["fx128", "cx128"])
def test_matmul_triangular_all_structures(fb, suf):
    """all 7^3 structure triples at n = 80 (several tiles), against the dd model within 8 (k + 2) 2^-104 (|A||B| + |C|)"""
    capi, lib = fb.capi, fb.load()
    cx = suf == "cx128"
    dt = capi.CX128 if cx else capi.FX128
    rng = np.random.default_rng(9)
    n = 80
    g = lambda *s_: rng.standard_normal(s_) + (1j * rng.standard_normal(s_) if cx else 0)
    A, B, C0 = _dd(g(n, n), rng, dt), _dd(g(n, n), rng, dt), _dd(g(n, n), rng, dt)
    alpha = _dd(np.array([0.75 + (0.5j if cx else 0)]), rng, dt)
    al = DM.from_fields(alpha)
    idx = np.arange(n)
    for cb in range(7):
        lower, upper = cb in (1, 3, 5), cb in (2, 4, 6)
        written = np.ones((n, n), bool)
        if lower:
            written = np.tril(written, -1 if cb in (3, 5) else 0)
        if upper:
            written = np.triu(written, 1 if cb in (4, 6) else 0)
        for ab in range(7):
            As = _structured(A, ab, cx)
            for bb in range(7):
                accum = (cb + ab + bb) % 2
                C1 = C0.copy(order="F")
                _mm(lib, suf, C1, cb, accum, A, ab, B, bb, alpha)
                assert C1[~written].tobytes() == C0[~written].tobytes()
                Bs = _structured(B, bb, cx)
                P = DM.matmul(DM.from_fields(As), DM.from_fields(Bs), cx)
                if cx:
                    want = DM.cmul(((al[0][0][0], al[0][1][0]), (al[1][0][0], al[1][1][0])), P)
                    if accum:
                        want = DM.cadd(want, DM.from_fields(C0))
                else:
                    want = DM.mul((al[0][0], al[1][0]), P)
                    if accum:
                        want = DM.add(want, DM.from_fields(C0))
                got = DM.from_fields(C1)
                diff = DM.cadd(got, (DM.neg(want[0]), DM.neg(want[1]))) if cx else DM.add(got, DM.neg(want))
                err = np.abs(DM.approx(diff, cx))
                mag = 2 * _bound_arrays(As, Bs, cx) + accum * np.abs(_approx(C0))
                assert np.all(err[written] <= 8 * (n + 2) * U * mag[written]), (cb, ab, bb)


def test_large_matmul_at_the_dd_bound(fb):
    """513 x 1031 x 257 with nonzero low limbs, against the dd model within 8 k 2^-104 |A||B| (an f64 product misses it by 2^51)"""
    capi, lib = fb.capi, fb.load()
    rng = np.random.default_rng(12)
    m, k, n = 513, 1031, 257
    A, B = _dd(rng.standard_normal((m, k)), rng, capi.FX128), _dd(rng.standard_normal((k, n)), rng, capi.FX128)
    alpha = np.array([(1.0, 0.0)], dtype=capi.FX128)
    Cm = np.zeros((m, n), dtype=capi.FX128, order="F")
    lib.libfaer_v0_23_matmul_fx128(capi.mat_mut(Cm), 0, capi.mat_ref(A), capi.mat_ref(B), alpha.ctypes.data, capi.par_default())
    want = DM.matmul(DM.from_fields(A), DM.from_fields(B), False)
    err = np.abs(DM.approx(DM.add(DM.from_fields(Cm), DM.neg(want)), False))
    assert np.all(err <= 8 * k * U * _bound_arrays(A, B, False))


@pytest.mark.parametrize("suf", ["fx128", "cx128"])
def test_solves_and_inverses_at_the_dd_bound(fb, suf):
    """n = 90 (several leaves): |M x - b| and |X M - I| within 64 n 2^-104 of |M||x| + |b|, computed with the dd model"""
    capi, lib = fb.capi, fb.load()
    cx = suf == "cx128"
    dt = capi.CX128 if cx else capi.FX128
    rng = np.random.default_rng(4)
    n, k = 90, 4
    T = (rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0)) / n + 2 * np.eye(n)
    Td = _dd(T, rng, dt)
    for name, code in (("solve_triangular_lower", 1), ("solve_triangular_upper", 2), ("solve_unit_triangular_lower", 5),
                       ("solve_unit_triangular_upper", 6)):
        Ms = _structured(Td, code, cx)
        b0 = _dd(rng.standard_normal((n, k)) + (1j * rng.standard_normal((n, k)) if cx else 0), rng, dt)
        b = b0.copy(order="F")
        getattr(lib, f"libfaer_v0_23_{name}_in_place_{suf}")(capi.mat_ref(Td), 0, capi.mat_mut(b), capi.par_default())
        r = DM.matmul(DM.from_fields(Ms), DM.from_fields(b), cx)
        diff = DM.cadd(r, (DM.neg(DM.from_fields(b0)[0]), DM.neg(DM.from_fields(b0)[1]))) if cx else DM.add(r, DM.neg(DM.from_fields(b0)))
        mag = _bound_arrays(Ms, b, cx) + np.abs(_approx(b0))
        assert np.all(np.abs(DM.approx(diff, cx)) <= 64 * n * U * mag), name
        inv = name.replace("solve", "inverse")
        D = np.zeros((n, n), dtype=dt, order="F")
        getattr(lib, f"libfaer_v0_23_{inv}_in_place_{suf}")(capi.mat_mut(D), capi.mat_ref(Td), capi.par_default())
        Ds = _structured(D, code, cx)  # the unit inverses' diagonal is not written: it is read as 1
        P = DM.matmul(DM.from_fields(Ds), DM.from_fields(Ms), cx)
        E = DM.approx(P, cx) - np.eye(n)
        assert np.abs(E).max() <= 64 * n * U * _bound_arrays(Ds, Ms, cx).max(), inv


@pytest.mark.parametrize("n", [100, 513])
def test_lu_pivots_match_the_dd_model(fb, n):
    capi, lib = fb.capi, fb.load()
    rng = np.random.default_rng(n + 7)
    A = _dd(rng.standard_normal((n, n)), rng, capi.FX128)
    _, perm, nt = DM.lu(DM.from_fields(A))
    LU = A.copy(order="F")
    pf, pb = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    st = lib.libfaer_v0_23_partial_piv_lu_factor_in_place_u64_fx128(
        capi.mat_mut(LU), capi.slice_mut(pf), capi.slice_mut(pb), capi.par_default(), capi.MemAlloc(None, 0),
        lib.libfaer_v0_23_PartialPivLuParams_fx128())
    assert np.array_equal(pf.astype(np.int64), perm) and st.value == nt


@pytest.mark.parametrize("kind", ["llt", "lu"])
def test_factor_2048_backward_error(fb, kind):
    """n = 2048: the factors reconstruct the input within c n 2^-104 (high-limb differences are exact in f64)"""
    capi, lib = fb.capi, fb.load()
    n = 2048
    rng = np.random.default_rng(2048)
    G = rng.standard_normal((n, n))
    X = G @ G.T / n + np.eye(n) if kind == "llt" else G
    A = np.zeros((n, n), dtype=capi.FX128, order="F")
    A["hi"] = X
    F_ = A.copy(order="F")
    R = np.zeros((n, n), dtype=capi.FX128, order="F")
    if kind == "llt":
        st = _llt(lib, capi, "fx128", F_)
        assert st.tag == 0
        lib.libfaer_v0_23_llt_reconstruct_fx128(capi.mat_mut(R), capi.mat_ref(F_), capi.par_default(), capi.MemAlloc(None, 0))
        mask = np.tril(np.ones((n, n), bool))
        scale = np.abs(X).max()
    else:
        pf, pb = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        lib.libfaer_v0_23_partial_piv_lu_factor_in_place_u32_fx128(capi.mat_mut(F_), capi.slice_mut(pf), capi.slice_mut(pb),
                                                                   capi.par_default(), capi.MemAlloc(None, 0),
                                                                   lib.libfaer_v0_23_PartialPivLuParams_fx128())
        lib.libfaer_v0_23_partial_piv_lu_reconstruct_u32_fx128(capi.mat_mut(R), capi.mat_ref(F_), capi.mat_ref(F_), capi.slice_mut(pf),
                                                               capi.slice_mut(pb), capi.par_default(), capi.MemAlloc(None, 0))
        mask = np.ones((n, n), bool)
        L = np.tril(F_["hi"], -1) + np.eye(n)
        scale = np.abs(L).max() * np.abs(np.triu(F_["hi"])).max()
    d = (R["hi"] - A["hi"]) + (R["lo"] - A["lo"])
    assert np.abs(d[mask]).max() <= 4 * n * U * scale
