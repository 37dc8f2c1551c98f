"""General eigendecomposition on the GPU (csrc/schur.cu) through the C ABI `libfaer_v0_23_evd_<T>` and the Python layers, for
f64 / f32 / c64 / c32. Checked against the definitions: A x = lambda x and y^H A = lambda y^H column by column, the eigenvalue
sum against the trace, the packed real convention, and numpy's eigenvalues at sizes where matching them is well conditioned.
f32 / c32 compute in f64 / c64, so their results carry only the rounding of the narrow output: tolerances are the narrow eps."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KINDS = {"f64": np.float64, "f32": np.float32, "c64": np.complex128, "c32": np.complex64}
SIZES = [0, 1, 2, 3, 17, 96, 97, 257, 512, 1024]


def _rand(n, dt, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    if np.issubdtype(dt, np.complexfloating):
        A = A + 1j * rng.standard_normal((n, n))
    return np.asfortranarray(A.astype(dt))


def _call(fb, A, left, right, order="F"):
    n = A.shape[0]
    dt = A.dtype
    cx = np.iscomplexobj(A)
    S, S_im = np.zeros(n, dt), np.zeros(n, dt)
    UL = np.zeros((n, n), dt, order=order) if left else None
    UR = np.zeros((n, n), dt, order=order) if right else None
    fb.linalg.evd(A, S, None if cx else S_im, UL, UR)
    return S, S_im, UL, UR


def _unpack(X, S_im):
    if np.iscomplexobj(X):
        return X.astype(np.complex128)
    V = X.astype(np.complex128)
    for k in np.nonzero(S_im > 0)[0]:
        V[:, k] = X[:, k].astype(np.float64) + 1j * X[:, k + 1]
        V[:, k + 1] = X[:, k].astype(np.float64) - 1j * X[:, k + 1]
    return V


def _check(A, S, S_im, UL, UR, c=200.0):
    n = A.shape[0]
    eps = np.finfo(A.dtype).eps
    A64 = A.astype(np.complex128)
    lam = S.astype(np.complex128) if np.iscomplexobj(A) else S.astype(np.float64) + 1j * S_im.astype(np.float64)
    nA = max(np.linalg.norm(A64), 1e-300)
    tol = c * max(n, 4) * eps
    assert np.all(np.isfinite(lam))
    assert abs(lam.sum() - np.trace(A64)) <= tol * nA * np.sqrt(max(n, 1))
    if not np.iscomplexobj(A):
        first = np.nonzero(S_im > 0)[0]
        assert np.all(S_im[first + 1] == -S_im[first]) and np.all(S[first + 1] == S[first])
        assert np.count_nonzero(S_im < 0) == len(first)
    if n <= 97:
        ref = np.linalg.eigvals(A64)
        d = np.abs(lam[:, None] - ref[None, :])
        if n:
            assert max(d.min(axis=0).max(), d.min(axis=1).max()) <= 1e4 * n * eps * nA
    if UR is not None:
        V = _unpack(UR, S_im)
        r = np.linalg.norm(A64 @ V - V * lam[None, :], axis=0)
        assert np.all(np.linalg.norm(V, axis=0) > 0)
        assert np.all(r <= tol * nA * np.linalg.norm(V, axis=0))
    if UL is not None:
        Y = _unpack(UL, S_im)
        r = np.linalg.norm(Y.conj().T @ A64 - lam[:, None] * Y.conj().T, axis=1)
        assert np.all(np.linalg.norm(Y, axis=0) > 0)
        assert np.all(r <= tol * nA * np.linalg.norm(Y, axis=0))


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("n", SIZES)
def test_evd_with_both_vector_sets(fb, kind, n):
    A = _rand(n, KINDS[kind], 100 + n)
    A0 = A.copy()
    S, S_im, UL, UR = _call(fb, A, True, True)
    assert np.array_equal(A, A0)
    _check(A, S, S_im, UL, UR)


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("n", [3, 130, 257])
def test_every_combination_of_requested_vectors_and_bitwise_equal_values(fb, kind, n):
    """The Schur stage performs the same operations on H whether or not Z is accumulated, so the eigenvalues of every call are
    the same bits; so are the vectors of two identical calls."""
    A = _rand(n, KINDS[kind], 7 + n)
    base = _call(fb, A, True, True)
    for left, right in ((False, False), (True, False), (False, True), (True, True)):
        S, S_im, UL, UR = _call(fb, A, left, right)
        assert (UL is None) == (not left) and (UR is None) == (not right)
        assert np.array_equal(S, base[0]) and np.array_equal(S_im, base[1])
        if left:
            assert np.array_equal(UL, base[2])
        if right:
            assert np.array_equal(UR, base[3])
        _check(A, S, S_im, UL, UR)


@pytest.mark.parametrize("kind", ["f64", "c32"])
def test_strided_transposed_and_negative_stride_views(fb, kind):
    n = 70
    dt = KINDS[kind]
    A = _rand(n, dt, 5)
    ref = _call(fb, A, True, True)
    big = np.zeros((2 * n + 3, 3 * n), dt)
    views = [np.ascontiguousarray(A), big[1:2 * n + 1:2, 2:3 * n:3][:, :n], np.asfortranarray(A)[::-1, ::-1][::-1, ::-1]]
    for v in views:
        v[...] = A
    rev = np.ascontiguousarray(A[::-1, ::-1])[::-1, ::-1]  # negative strides in both directions
    assert np.array_equal(rev, A)
    for Av in views + [rev]:
        for order in ("F", "C"):
            S, S_im, UL, UR = _call(fb, Av, True, True, order=order)
            assert np.array_equal(S, ref[0]) and np.array_equal(UR, ref[3]) and np.array_equal(UL, ref[2])
    # strided, reversed outputs
    cx = np.iscomplexobj(A)
    S, S_im = np.zeros(n, dt), np.zeros(n, dt)
    buf = np.full((2 * n, 2 * n), 7, dt)
    UR = buf[::2, ::2][::-1, :]
    fb.linalg.evd(A, S, None if cx else S_im, None, UR)
    assert np.array_equal(UR, ref[3]) and np.all(buf[1::2, :] == 7) and np.all(buf[:, 1::2] == 7)


@pytest.mark.parametrize("kind", list(KINDS))
def test_device_pointers_and_the_solvers_round_trip(fb, kind):
    import torch
    n = 150
    A = _rand(n, KINDS[kind], 11)
    ref = _call(fb, A, False, True)
    Ad = torch.from_numpy(np.ascontiguousarray(A.T)).cuda().T
    S = torch.zeros(n, dtype=Ad.dtype, device="cuda")
    S_im = torch.zeros(n, dtype=Ad.dtype, device="cuda")
    UR = torch.zeros((n, n), dtype=Ad.dtype, device="cuda").T
    fb.linalg.evd(Ad, S, None if Ad.dtype.is_complex else S_im, None, UR)
    assert np.array_equal(S.cpu().numpy(), ref[0]) and np.array_equal(UR.cpu().numpy(), ref[3])
    assert np.array_equal(Ad.cpu().numpy(), A)
    e = fb.solvers.eigen(A)
    U, lam = e.U(), e.S()
    assert np.iscomplexobj(U) and np.iscomplexobj(lam)
    eps = np.finfo(A.dtype).eps
    A64 = A.astype(np.complex128)
    r = np.linalg.norm(A64 @ U - U * lam[None, :], axis=0)
    assert np.all(r <= 200 * n * eps * np.linalg.norm(A64) * np.linalg.norm(U, axis=0))
    assert np.array_equal(fb.solvers.eigenvalues(A), lam)
    lam_d = fb.solvers.eigenvalues(Ad)
    assert np.array_equal(lam_d.cpu().numpy(), lam)


@pytest.mark.parametrize("kind", ["f64", "c64"])
def test_non_finite_input_reports_no_convergence_and_writes_nothing(fb, kind):
    n = 20
    A = _rand(n, KINDS[kind], 3)
    A[4, 7] = np.nan
    S, S_im = np.full(n, 5, A.dtype), np.full(n, 5, A.dtype)
    UL, UR = np.full((n, n), 5, A.dtype, order="F"), np.full((n, n), 5, A.dtype, order="F")
    with pytest.raises(RuntimeError, match="NoConvergence"):
        fb.linalg.evd(A, S, None if np.iscomplexobj(A) else S_im, UL, UR)
    assert np.all(S == 5) and np.all(S_im == 5) and np.all(UL == 5) and np.all(UR == 5)


def test_special_inputs(fb):
    n = 40
    rng = np.random.default_rng(2)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    rot = np.zeros((n, n))
    for k in range(0, n, 2):
        rot[k, k + 1], rot[k + 1, k] = -(k + 1.0), k + 1.0
    cases = {
        "zeros": np.zeros((n, n)), "identity": np.eye(n), "ones": np.ones((n, n)), "triangular": np.triu(rng.standard_normal((n, n))),
        "repeated": Q @ np.diag(np.r_[np.full(n // 2, 2.0), np.arange(n - n // 2)]) @ Q.T, "rotation": rot,
        "large": rng.standard_normal((n, n)) * 1e100,
    }
    for name, A in cases.items():
        A = np.asfortranarray(A)
        S, S_im, UL, UR = _call(fb, A, True, True)
        _check(A, S, S_im, UL, UR, c=2e4)
        if name == "rotation":
            assert np.count_nonzero(S_im) == n and np.allclose(S, 0, atol=1e-10)


def test_the_callers_shift_count_is_an_upper_bound(fb):
    capi = fb.capi
    A = _rand(200, np.float64, 9)
    lib = fb.load()
    p = lib.libfaer_v0_23_EvdParams_f64()
    keep = capi.SHIFT_COUNT_FN(lambda n, nh: 4)
    p.schur.recommended_shift_count = keep
    S, S_im = np.zeros(200), np.zeros(200)
    UR = np.zeros((200, 200), order="F")
    fb.linalg.evd(A, S, S_im, None, UR, params=p)
    _check(A, S, S_im, None, UR)
    counts = (capi.C.c_longlong * 2)()
    lib.faer_b200_evd_last_sweep_counts(counts)
    few = counts[0]
    fb.linalg.evd(A, S, S_im, None, UR)
    lib.faer_b200_evd_last_sweep_counts(counts)
    assert few > counts[0] > 0  # 2 bulges per sweep need more sweeps than 16
