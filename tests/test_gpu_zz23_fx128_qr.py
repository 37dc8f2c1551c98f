"""Double-double (fx128 / cx128) Householder QR through the C ABI (csrc/qr_dd.cu, csrc/qr_blocked.cuh, csrc/ffi_dd.cu): factor,
reconstruct, the four `apply_householder_*` variants, the solves and the inverse, checked with exact f64 limb differences and the
dd GEMM against bounds of order m * 2^-104; the output format against the f64 / c64 entry points; the rank logic on exactly
dependent columns; a least-squares fit against its exact rational solution; device operands, determinism and strided views."""
from fractions import Fraction as F

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
U = 2.0 ** -104
KINDS = ["fx128", "cx128"]


def _capi():
    import faer_b200
    return faer_b200.capi


def _dd(x, dt, rng=None):
    """float64 / complex128 -> FX128 / CX128 (column-major); with rng, a nonzero low limb below half an ulp of the high one"""
    out = np.zeros(x.shape, dtype=dt, order="F")
    lo = (lambda v: v * 2.0 ** -60 * rng.uniform(-0.5, 0.5, v.shape)) if rng is not None else (lambda v: 0.0 * v)
    if "hi" in dt.names:
        out["hi"], out["lo"] = np.real(x), lo(np.real(x))
    else:
        out["re_hi"], out["re_lo"] = np.real(x), lo(np.real(x))
        out["im_hi"], out["im_lo"] = np.imag(x), lo(np.imag(x))
    return out


def _hi(a):
    return a["hi"] if "hi" in a.dtype.names else a["re_hi"] + 1j * a["im_hi"]


def _diff(a, b):
    """|a - b| per element from exact limb differences"""
    if "hi" in a.dtype.names:
        return np.abs((a["hi"] - b["hi"]) + (a["lo"] - b["lo"]))
    return np.abs(((a["re_hi"] - b["re_hi"]) + (a["re_lo"] - b["re_lo"])) + 1j * ((a["im_hi"] - b["im_hi"]) + (a["im_lo"] - b["im_lo"])))


def _eye(n, dt):
    return _dd(np.eye(n), dt)


def _rand(rng, m, n, cx):
    return rng.standard_normal((m, n)) + (1j * rng.standard_normal((m, n)) if cx else 0)


def _kind(suf):
    capi = _capi()
    return (capi.CX128 if suf == "cx128" else capi.FX128), suf == "cx128"


def _factor(lib, suf, A, bs, thr=None):
    capi = _capi()
    m, n = A.shape
    dt = A.dtype
    Q = np.zeros((bs, min(m, n)), dtype=dt, order="F")
    p = getattr(lib, f"libfaer_v0_23_QrParams_{suf}")()
    if thr is not None:
        p.blocking_threshold = thr
    st = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{suf}")(capi.mat_mut(A), capi.mat_mut(Q), capi.par_default(),
                                                                capi.MemAlloc(None, 0), p)
    return st.value, Q


def _call(lib, name, suf, *args):
    capi = _capi()
    return getattr(lib, f"libfaer_v0_23_{name}_{suf}")(*args, capi.par_default(), capi.MemAlloc(None, 0))


def _reconstruct(lib, suf, QR, Q):
    capi = _capi()
    m, n = QR.shape
    s = min(m, n)
    out = np.zeros((m, n), dtype=QR.dtype, order="F")
    _call(lib, "qr_reconstruct", suf, capi.mat_mut(out), capi.mat_ref(QR[:, :s]), capi.mat_ref(Q), capi.mat_ref(QR[:s, :]))
    return out


def _apply(lib, suf, name, QR, Q, M, conj=0):
    capi = _capi()
    s = min(QR.shape)
    _call(lib, name, suf, capi.mat_ref(QR[:, :s]), capi.mat_ref(Q), conj, capi.mat_mut(M))
    return M


def _fro(a):
    return float(np.sqrt(np.sum(np.abs(_hi(a)) ** 2)))


SHAPES = [(1, 1), (7, 7), (16, 16), (17, 17), (100, 60), (60, 100), (513, 257)]


@pytest.mark.parametrize("suf", KINDS)
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("bs", [1, 4, 48, "rec", "odd"])
def test_factor_reconstruct(fb, suf, shape, bs):
    lib = fb.load()
    dt, cx = _kind(suf)
    m, n = shape
    if bs == "rec":
        bs = getattr(lib, f"libfaer_v0_23_qr_recommended_block_size_{suf}")(m, n)
    elif bs == "odd":
        bs = max(1, min(m, n) // 2 - 1) if min(m, n) > 3 else 3
    bs = max(1, min(bs, min(m, n)))
    rng = np.random.default_rng(m * 1000 + n + bs)
    A0 = _dd(_rand(rng, m, n, cx), dt, rng)
    for thr in (None, 0, 1 << 60):  # default, sub-blocking always, never
        A = A0.copy(order="F")
        rank, Q = _factor(lib, suf, A, bs, thr)
        assert rank == min(m, n)
        err = _diff(_reconstruct(lib, suf, A, Q), A0).max()
        assert err <= 16 * m * U * _fro(A0), (thr, err)


@pytest.mark.parametrize("suf", KINDS)
@pytest.mark.parametrize("shape,bs", [((2048, 2048), "rec"), ((65536, 64), 32)])
def test_factor_reconstruct_large(fb, suf, shape, bs):
    lib = fb.load()
    dt, cx = _kind(suf)
    m, n = shape
    if bs == "rec":
        bs = getattr(lib, f"libfaer_v0_23_qr_recommended_block_size_{suf}")(m, n)
    rng = np.random.default_rng(m + n)
    A0 = _dd(_rand(rng, m, n, cx), dt, rng)
    A = A0.copy(order="F")
    rank, Q = _factor(lib, suf, A, bs)
    assert rank == n
    err = _diff(_reconstruct(lib, suf, A, Q), A0).max()
    assert err <= 16 * m * U * _fro(A0), err


@pytest.mark.parametrize("suf", KINDS)
@pytest.mark.parametrize("shape,bs", [((60, 60), 8), ((90, 40), 16), ((40, 90), 48)])
def test_q_orthonormal_and_variants(fb, suf, shape, bs):
    capi, lib = fb.capi, fb.load()
    dt, cx = _kind(suf)
    m, n = shape
    rng = np.random.default_rng(7 + m)
    A = _dd(_rand(rng, m, n, cx), dt, rng)
    _, Q = _factor(lib, suf, A, min(bs, m, n))
    Qm = _apply(lib, suf, "apply_householder_on_the_left", A, Q, _eye(m, dt))
    # Q^H Q - I on the dd GEMM (conjugate transpose by flipping the sign of the imaginary limbs)
    QH = Qm.T.copy(order="F")
    if cx:
        QH["im_hi"], QH["im_lo"] = -QH["im_hi"], -QH["im_lo"]
    P = np.zeros((m, m), dtype=dt, order="F")
    one = _dd(np.array([1.0]), dt)
    getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(P), 0, capi.mat_ref(QH), capi.mat_ref(Qm), one.ctypes.data, capi.par_default())
    assert _diff(P, _eye(m, dt)).max() <= 32 * m * U, _diff(P, _eye(m, dt)).max() / (m * U)
    # the four variants against the explicit Q: conj?(Q) M, conj?(Q)^T M, M conj?(Q), M conj?(Q)^T (Conj::Yes conjugates Q for cx128)
    M0 = _dd(_rand(rng, m, 5, cx), dt, rng)
    for conj in ((0, 1) if cx else (0,)):
        Qc = Qm.copy(order="F")
        if conj:
            Qc["im_hi"], Qc["im_lo"] = -Qc["im_hi"], -Qc["im_lo"]
        Qch = Qc.T.copy(order="F")  # transpose_*: conj?(Q)^T
        for name, op in (("apply_householder_on_the_left", Qc), ("apply_householder_transpose_on_the_left", Qch)):
            want = np.zeros((m, 5), dtype=dt, order="F")
            getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(want), 0, capi.mat_ref(op), capi.mat_ref(M0), one.ctypes.data,
                                                        capi.par_default())
            got = _apply(lib, suf, name, A, Q, M0.copy(order="F"), conj)
            assert _diff(got, want).max() <= 16 * m * U * _fro(M0), (name, conj, _diff(got, want).max() / (m * U * _fro(M0)))
        L0 = np.asfortranarray(M0.T)
        for name, op in (("apply_householder_on_the_right", Qc), ("apply_householder_transpose_on_the_right", Qch)):
            want = np.zeros((5, m), dtype=dt, order="F")
            getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(want), 0, capi.mat_ref(L0), capi.mat_ref(op), one.ctypes.data,
                                                        capi.par_default())
            got = _apply(lib, suf, name, A, Q, L0.copy(order="F"), conj)
            assert _diff(got, want).max() <= 16 * m * U * _fro(M0), (name, conj, _diff(got, want).max() / (m * U * _fro(M0)))


@pytest.mark.parametrize("suf", KINDS)
@pytest.mark.parametrize("shape,bs", [((100, 60), 8), ((60, 100), 48), ((200, 200), 32)])
def test_format_matches_f64(fb, suf, shape, bs):
    """with zero low limbs, the high limbs agree with the f64 / c64 entry points: sign of beta, tau and the T-block layout"""
    capi, lib = fb.capi, fb.load()
    dt, cx = _kind(suf)
    m, n = shape
    rng = np.random.default_rng(m * n)
    X = _rand(rng, m, n, cx) + 8 * np.eye(m, n)  # well conditioned: the f64 result is close to the exact one
    A = _dd(X, dt)
    rank, Q = _factor(lib, suf, A, bs)
    ref = "c64" if cx else "f64"
    B = np.asfortranarray(X.astype(np.complex128 if cx else np.float64))
    H = np.zeros((bs, min(m, n)), dtype=B.dtype, order="F")
    p = getattr(lib, f"libfaer_v0_23_QrParams_{ref}")()
    st = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{ref}")(capi.mat_mut(B), capi.mat_mut(H), capi.par_default(),
                                                                capi.MemAlloc(None, 0), p)
    assert st.value == rank == min(m, n)
    tol = 64 * max(m, n) * 2.0 ** -53
    assert np.max(np.abs(_hi(A) - B)) <= tol * max(1.0, np.max(np.abs(B)))
    # only the upper triangle of each T block is defined
    for k in range(0, min(m, n), bs):
        w = min(bs, min(m, n) - k)
        got, want = np.triu(_hi(Q)[:w, k:k + w]), np.triu(H[:w, k:k + w])
        fin = np.isfinite(want)  # +inf: the tau of a reflector without a tail (the last column of a square block)
        assert np.array_equal(fin, np.isfinite(got)), k
        assert np.max(np.abs(got[fin] - want[fin])) <= tol * max(1.0, np.max(np.abs(want[fin]))), k


@pytest.mark.parametrize("suf", KINDS)
def test_rank_dependent_columns(fb, suf):
    capi, lib = fb.capi, fb.load()
    dt, cx = _kind(suf)
    rng = np.random.default_rng(5)
    m, n, bs = 24, 10, 4
    X = rng.integers(-9, 10, (m, n)).astype(np.float64)
    X[:, 3] = X[:, 1] + X[:, 2]
    X[:, 6] = 2 * X[:, 0]
    X[:, 7] = X[:, 3] - X[:, 6]
    A = _dd(X + 0j if cx else X, dt)
    rank, Q = _factor(lib, suf, A, bs)
    B = np.asfortranarray(X + 0j if cx else X)
    H = np.zeros((bs, n), dtype=B.dtype, order="F")
    ref = "c64" if cx else "f64"
    st = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{ref}")(capi.mat_mut(B), capi.mat_mut(H), capi.par_default(),
                                                                capi.MemAlloc(None, 0), getattr(lib, f"libfaer_v0_23_QrParams_{ref}")())
    assert rank == st.value == 7
    # the same staircase: the zero pattern of R's rows
    Rd, Rf = np.triu(_hi(A)[:n, :]), np.triu(B[:n, :])
    assert np.array_equal(np.abs(Rd) > 1e-9, np.abs(Rf) > 1e-9)
    tail = _hi(Q)[:, rank:]
    assert np.all((tail == 0) | np.isinf(tail.real))
    # breaking one dependence by 1e-20 in the low limb gives full rank in dd
    A = _dd(X + 0j if cx else X, dt)
    A[5, 7]["lo" if not cx else "re_lo"] = 1e-20
    rank, _ = _factor(lib, suf, A, bs)
    assert rank == 8


def test_lstsq_vandermonde_exact(fb):
    capi, lib = fb.capi, fb.load()
    m, n = 40, 14
    nodes = [F(i, 39) for i in range(m)]
    def to_dd(fr):
        hi = float(fr)
        return hi, float(fr - F(hi))
    A = np.zeros((m, n), dtype=capi.FX128, order="F")
    Af = [[None] * n for _ in range(m)]
    for i in range(m):
        for j in range(n):
            A[i, j] = to_dd(nodes[i] ** j)
            Af[i][j] = F(float(A[i, j]["hi"])) + F(float(A[i, j]["lo"]))
    xt = [F(k + 1, 7) for k in range(n)]
    b = np.zeros((m, 1), dtype=capi.FX128, order="F")
    bf = []
    for i in range(m):
        b[i, 0] = to_dd(sum(Af[i][j] * xt[j] for j in range(n)) + F((-1) ** i, 10 ** 12))
        bf.append(F(float(b[i, 0]["hi"])) + F(float(b[i, 0]["lo"])))
    # the exact least-squares solution of the stored system: normal equations in rationals
    N = [[sum(Af[k][i] * Af[k][j] for k in range(m)) for j in range(n)] + [sum(Af[k][i] * bf[k] for k in range(m))] for i in range(n)]
    for c in range(n):
        p = next(r for r in range(c, n) if N[r][c] != 0)
        N[c], N[p] = N[p], N[c]
        for r in range(n):
            if r != c and N[r][c] != 0:
                f = N[r][c] / N[c][c]
                N[r] = [x - f * y for x, y in zip(N[r], N[c])]
    x = [N[i][n] / N[i][i] for i in range(n)]
    QR = A.copy(order="F")
    rank, Q = _factor(lib, "fx128", QR, getattr(lib, "libfaer_v0_23_qr_recommended_block_size_fx128")(m, n))
    assert rank == n
    _call(lib, "qr_solve_lstsq_in_place", "fx128", capi.mat_ref(QR), capi.mat_ref(Q), capi.mat_ref(QR), 0, capi.mat_mut(b))
    got = [F(float(b[i, 0]["hi"])) + F(float(b[i, 0]["lo"])) for i in range(n)]
    num = sum((g - w) ** 2 for g, w in zip(got, x))
    den = sum(w ** 2 for w in x)
    assert float(num / den) ** 0.5 <= 1e-18


@pytest.mark.parametrize("suf", KINDS)
def test_square_solves_and_inverse(fb, suf):
    capi, lib = fb.capi, fb.load()
    dt, cx = _kind(suf)
    n, k = 70, 3
    rng = np.random.default_rng(11)
    A0 = _dd(_rand(rng, n, n, cx) + 4 * np.eye(n), dt, rng)
    QR = A0.copy(order="F")
    _, Q = _factor(lib, suf, QR, 16)
    one = _dd(np.array([1.0]), dt)
    mm = lambda Cm, X, Y: getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(Cm), 0, capi.mat_ref(X), capi.mat_ref(Y),
                                                                       one.ctypes.data, capi.par_default())
    B = _dd(_rand(rng, n, k, cx), dt, rng)
    for conj in ((0, 1) if cx else (0,)):
        Ac = A0.copy(order="F")
        if conj:
            Ac["im_hi"], Ac["im_lo"] = -Ac["im_hi"], -Ac["im_lo"]
        for name, op in (("qr_solve_in_place", Ac), ("qr_solve_transpose_in_place", np.asfortranarray(Ac.T))):
            X = B.copy(order="F")
            _call(lib, name, suf, capi.mat_ref(QR), capi.mat_ref(Q), capi.mat_ref(QR), conj, capi.mat_mut(X))
            R = np.zeros((n, k), dtype=dt, order="F")
            mm(R, op, X)
            assert _diff(R, B).max() <= 64 * n * U * _fro(A0) * _fro(X), (name, conj)
    Ai = np.zeros((n, n), dtype=dt, order="F")
    _call(lib, "qr_inverse", suf, capi.mat_mut(Ai), capi.mat_ref(QR), capi.mat_ref(Q), capi.mat_ref(QR))
    P = np.zeros((n, n), dtype=dt, order="F")
    mm(P, A0, Ai)
    assert _diff(P, _eye(n, dt)).max() <= 64 * n * U * _fro(A0) * _fro(Ai)


@pytest.mark.parametrize("suf", KINDS)
def test_device_operands_and_determinism(fb, suf):
    import torch
    capi, lib = fb.capi, fb.load()
    dt, cx = _kind(suf)
    m, n, bs = 3000, 70, 32  # several CTAs in the panel
    rng = np.random.default_rng(3)
    A0 = _dd(_rand(rng, m, n, cx), dt, rng)
    runs = []
    for _ in range(2):
        A = A0.copy(order="F")
        runs.append((_factor(lib, suf, A, bs), A))
    (r1, Q1), A1 = runs[0]
    (r2, Q2), A2 = runs[1]
    assert r1 == r2 and A1.tobytes() == A2.tobytes() and Q1.tobytes() == Q2.tobytes()
    limbs = 4 if cx else 2
    tail = (2, 2) if cx else (2,)

    def dev(X):  # column-major device copy as a DDTensor
        r, c = X.shape
        base = np.stack([X[f] for f in dt.names], axis=-1).transpose(1, 0, 2).reshape((c, r) + tail)
        return torch.from_numpy(np.ascontiguousarray(base)).cuda().transpose(0, 1)

    t, Qd = dev(A0), dev(np.zeros((bs, min(m, n)), dtype=dt))
    p = getattr(lib, f"libfaer_v0_23_QrParams_{suf}")()
    st = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{suf}")(capi.mat_mut(capi.DDTensor(t, cx)), capi.mat_mut(capi.DDTensor(Qd, cx)),
                                                                capi.par_default(), capi.MemAlloc(None, 0), p)
    assert st.value == r1
    for got, want in ((t, A1), (Qd, Q1)):
        g = np.ascontiguousarray(got.cpu().numpy()).reshape(want.shape + (limbs,))
        w = np.stack([want[f] for f in dt.names], axis=-1)
        assert np.array_equal(g.view(np.uint64), w.view(np.uint64))


@pytest.mark.parametrize("suf", KINDS)
def test_strided_and_empty_views(fb, suf):
    lib = fb.load()
    dt, cx = _kind(suf)
    rng = np.random.default_rng(9)
    A0 = _dd(_rand(rng, 50, 30, cx), dt, rng)
    ref = A0.copy(order="F")
    rr, Qr = _factor(lib, suf, ref, 8)
    # row-major storage
    B = np.ascontiguousarray(A0)
    rb, Qb = _factor(lib, suf, B, 8)
    assert rb == rr and B.tobytes() == np.ascontiguousarray(ref).tobytes() and Qb.tobytes() == Qr.tobytes()
    # negative row stride: the factorization of the row-reversed matrix
    Cbuf = np.asfortranarray(A0[::-1])
    C = Cbuf[::-1]
    rc, Qc = _factor(lib, suf, C, 8)
    assert rc == rr and np.ascontiguousarray(C).tobytes() == np.ascontiguousarray(ref).tobytes() and Qc.tobytes() == Qr.tobytes()
    for shape in ((0, 5), (5, 0)):
        E = np.zeros(shape, dtype=dt, order="F")
        r, Q = _factor(lib, suf, E, 1)
        assert r == 0 and Q.shape == (1, 0)


@pytest.mark.parametrize("conj", [0, 1])
def test_cx128_triangular_solve_small_diagonal(fb, conj):
    """the cx128 triangular-solve leaf with diagonal entries of modulus below 1 (the taus of the T blocks, small pivots of R):
    faer's complex recip keeps only about 53 bits there, the scaled reciprocal keeps the residual at 2^-104 scale"""
    capi, lib = fb.capi, fb.load()
    dt = capi.CX128
    n, k = 80, 3
    rng = np.random.default_rng(21 + conj)
    X = 0.05 * np.tril(_rand(rng, n, n, True), -1)
    X[np.diag_indices(n)] = rng.uniform(0.2, 0.9, n) * np.exp(2j * np.pi * rng.uniform(size=n))
    L = _dd(X, dt, rng)
    B = _dd(_rand(rng, n, k, True), dt, rng)
    Xs = B.copy(order="F")
    lib.libfaer_v0_23_solve_triangular_lower_in_place_cx128(capi.mat_ref(L), conj, capi.mat_mut(Xs), capi.par_default())
    Lc = L.copy(order="F")
    if conj:
        Lc["im_hi"], Lc["im_lo"] = -Lc["im_hi"], -Lc["im_lo"]
    R = np.zeros((n, k), dtype=dt, order="F")
    one = _dd(np.array([1.0]), dt)
    lib.libfaer_v0_23_matmul_cx128(capi.mat_mut(R), 0, capi.mat_ref(Lc), capi.mat_ref(Xs), one.ctypes.data, capi.par_default())
    assert _diff(R, B).max() <= 64 * n * U * _fro(L) * _fro(Xs), _diff(R, B).max()
