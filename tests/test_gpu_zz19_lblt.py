"""Bunch-Kaufman LBL^H (`lblt_*`, csrc/lblt.cu) through the C ABI against the numpy restatement of
faer/src/linalg/cholesky/bunch_kaufman (tests/lblt_model.py).

Factor: when the model's smallest decision margin is well above rounding, perm_fwd, perm_bwd and the transposition count must
equal the model's exactly and L, diag and subdiag must agree within tolerance; otherwise the factors must satisfy
P A P^T = L B L^H. A NaN sentinel in subdiag survives exactly where the model leaves it; the strict upper triangle is untouched
(NaN sentinels) except under Full, which scales it. Solve (A_conj No / Yes), reconstruct (all of `out`) and inverse (all n^2
entries) run on the GPU's own factors and are compared with the model applied to them."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lblt_model as M  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32, np.complex128, np.complex64]
STRATS = [M.PARTIAL, M.PARTIAL_DIAG, M.ROOK, M.ROOK_DIAG, M.FULL]


def ueps(dtype):
    return float(np.finfo(dtype).eps)


def is_cx(dtype):
    return np.issubdtype(dtype, np.complexfloating)


def sym(rng, n, dtype):
    X = rng.standard_normal((n, n))
    if is_cx(dtype):
        X = X + 1j * rng.standard_normal((n, n))
    A = (X + np.conj(X.T)) / 2
    A[np.diag_indices(n)] = np.real(np.diag(A))
    return np.asfortranarray(A.astype(dtype))


def run(la, A, strat, bs, it=np.uint64, sub=None):
    n = A.shape[0]
    p = np.zeros(n, dtype=it)
    pi = np.zeros(n, dtype=it)
    sub = np.zeros(n, dtype=A.dtype) if sub is None else sub
    params = la.lblt_params_default()
    params.pivoting = strat
    params.block_size = bs
    info = la.lblt_in_place(A, sub, p, pi, params=params)
    return A, sub, p.astype(np.int64), pi.astype(np.int64), info.transposition_count


def lbl_identity(LB, sub, perm_inv, A, dtype, n):
    R = M.reconstruct(LB.astype(np.complex128 if is_cx(dtype) else np.float64), sub.astype(np.complex128 if is_cx(dtype) else np.float64), perm_inv)
    Rf = np.tril(R) + np.conj(np.tril(R, -1)).T
    return np.abs(Rf - A).max(initial=0) / max(1.0, np.abs(A).max(initial=0))


def check(la, A0, strat, bs, it=np.uint64):
    dtype = A0.dtype
    n = A0.shape[0]
    A_in = A0.copy(order="F")
    if strat != M.FULL:
        A_in[np.triu_indices(n, 1)] = np.nan
    sub0 = np.zeros(n, dtype=dtype)
    if n:
        sub0[-1] = np.nan
    LB, sub, p, pi, cnt = run(la, A_in, strat, bs, it, sub0.copy())
    Aw = A0.astype(np.complex128 if is_cx(dtype) else np.float64)
    mLB, msub, mp, mpi, mcnt, margins = M.factor(Aw if strat == M.FULL else np.tril(Aw), sub0.astype(Aw.dtype), strat, bs)
    tol = 200 * max(n, 1) * ueps(dtype)
    if strat != M.FULL:
        iu = np.triu_indices(n, 1)
        assert np.all(np.isnan(LB[iu])), "strict upper triangle written"
    assert sorted(p.tolist()) == list(range(n)) and np.array_equal(pi[p], np.arange(n))
    if not margins or min(margins) > 1e3 * max(n, 1) * ueps(dtype):
        assert np.array_equal(p, mp) and np.array_equal(pi, mpi) and cnt == mcnt
        sc = max(1.0, np.abs(np.tril(mLB)).max(initial=0))
        assert np.abs(np.tril(LB) - np.tril(mLB)).max(initial=0) <= tol * sc * 10
        nanm = np.isnan(msub)
        assert np.array_equal(np.isnan(sub), nanm), "subdiag written where the reference leaves it"
        assert np.abs(sub[~nanm] - msub[~nanm]).max(initial=0) <= tol * sc * 10
        if strat == M.FULL:
            iu = np.triu_indices(n, 1)
            assert np.abs(LB[iu] - mLB[iu]).max(initial=0) <= tol * 10
    clean = np.where(np.isnan(sub), 0, sub)
    assert lbl_identity(np.tril(LB), clean, pi, Aw, dtype, n) <= tol * 10
    return np.asfortranarray(np.tril(LB)), clean, p, pi


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("strat", STRATS)
@pytest.mark.parametrize("it", [np.uint32, np.uint64])
def test_factor_small(fb, dtype, strat, it):
    la = fb.linalg
    rng = np.random.default_rng(19 + strat)
    for n in (0, 1, 2, 3, 6, 19, 100):
        for bs in (0, 1, 2, 4, 7, 64, 128, n, n + 5):
            check(la, sym(rng, n, dtype), strat, bs, it)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("strat", STRATS)
def test_factor_421(fb, dtype, strat):
    la = fb.linalg
    rng = np.random.default_rng(421)
    n = 421
    for bs in (0, 1, 2, 4, 7, 64, 128, n, n + 5):
        check(la, sym(rng, n, dtype), strat, bs)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("strat", STRATS)
def test_factor_1000(fb, dtype, strat):
    la = fb.linalg
    rng = np.random.default_rng(1000)
    n = 1000
    for bs in (2, 7, 64, 128, n + 5):
        check(la, sym(rng, n, dtype), strat, bs)


@pytest.mark.parametrize("dtype,strat,bs", [
    (np.float64, M.PARTIAL, 64), (np.float64, M.PARTIAL_DIAG, 128), (np.float64, M.ROOK, 128), (np.float64, M.ROOK_DIAG, 64),
    (np.float32, M.PARTIAL_DIAG, 64), (np.complex128, M.PARTIAL_DIAG, 64), (np.complex64, M.ROOK, 64)])
def test_factor_3000(fb, dtype, strat, bs):
    la = fb.linalg
    rng = np.random.default_rng(3000)
    check(la, sym(rng, 3000, dtype), strat, bs)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("strat", STRATS)
def test_zero_column_inside_a_blocked_step(fb, dtype, strat):
    """Columns with nothing to do (gamma == 0: no scaling, no update, subdiag left as given) inside the first step of an
    n = 20, bs = 8 factorization. Variables 0 and 3 form the singular pair [[1, 2], [2, 4]], coupled to nothing else: once one
    of them is eliminated (a 1 x 1 pivot on 3), the other's column is exactly zero, which the column strategies meet at step
    column 3. Variable 5 is decoupled with the largest diagonal entry, which the Diag strategies take first."""
    la = fb.linalg
    rng = np.random.default_rng(8)
    n = 20
    A = sym(rng, n, dtype).astype(np.complex128 if is_cx(dtype) else np.float64) * 0.25
    A[np.diag_indices(n)] = 8.0 + np.arange(n)
    for v in (0, 3, 5):
        A[v, :] = 0
        A[:, v] = 0
    A[0, 0], A[3, 3], A[3, 0], A[0, 3] = 1, 4, 2, 2
    A[5, 5] = 100
    A = np.asfortranarray(A.astype(dtype))
    check(la, A, strat, 8)  # the NaN sentinel of subdiag must survive exactly where the model leaves it
    w = np.complex128 if is_cx(dtype) else np.float64
    _, msub, _, _, _, _ = M.factor(A.astype(w) if strat == M.FULL else np.tril(A).astype(w), np.full(n, np.nan, dtype=w), strat, 8)
    if strat != M.FULL:
        assert np.isnan(msub[:7]).any(), "no nothing-to-do column inside the first blocked step"


def test_exact_small_cases(fb):
    la = fb.linalg
    for dtype in DTYPES:
        for strat in STRATS:
            for bs in (0, 2, 64):
                I = np.eye(5, dtype=dtype, order="F")
                LB, sub, p, pi, cnt = run(la, I.copy(order="F"), strat, bs)
                assert cnt == 0 and np.array_equal(np.tril(LB), np.eye(5))
                Z = np.zeros((4, 4), dtype=dtype, order="F")
                sub0 = np.full(4, 7, dtype=dtype)
                LB, sub, p, pi, cnt = run(la, Z, strat, bs, sub=sub0)
                if strat != M.FULL:  # nothing to do in every column: subdiag untouched
                    assert np.array_equal(sub, np.full(4, 7, dtype=dtype)) and cnt == 0
                X = np.array([[0, 1], [1, 0]], dtype=dtype, order="F")
                LB, sub, p, pi, cnt = run(la, X, strat, bs)
                assert sub[0] == 1 and sub[1] == 0 and LB[1, 0] == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_solve_reconstruct_inverse(fb, dtype):
    la = fb.linalg
    rng = np.random.default_rng(7)
    for n, strat, bs in ((50, M.PARTIAL_DIAG, 4), (100, M.ROOK, 0), (80, M.FULL, 64), (300, M.PARTIAL, 64)):
        A = sym(rng, n, dtype)
        LB, sub, p, pi = check(la, A, strat, bs)
        w = np.complex128 if is_cx(dtype) else np.float64
        tol = 1e3 * n * ueps(dtype)
        for conj in (False, True):
            b = np.asfortranarray(sym(rng, n, dtype)[:, :3])
            x = b.copy(order="F")
            la.lblt_solve_in_place(LB, sub, p.astype(np.uint64), pi.astype(np.uint64), x, la.CONJ_YES if conj else la.CONJ_NO)
            xm = M.solve(LB.astype(w), sub.astype(w), p, pi, b.astype(w), conj=conj)
            assert np.abs(x - xm).max(initial=0) <= tol * max(1.0, np.abs(xm).max(initial=0))
        out = np.full((n, n), np.nan, dtype=dtype, order="F")
        la.lblt_reconstruct(out, LB, sub, p.astype(np.uint32), pi.astype(np.uint32))
        Rm = M.reconstruct(LB.astype(w), sub.astype(w), pi)
        assert not np.isnan(out).any()
        assert np.abs(out - Rm).max(initial=0) <= tol * max(1.0, np.abs(Rm).max(initial=0))
        inv = np.full((n, n), np.nan, dtype=dtype, order="F")
        la.lblt_inverse(inv, LB, sub, p.astype(np.uint64), pi.astype(np.uint64))
        Im = M.solve(LB.astype(w), sub.astype(w), p, pi, np.eye(n, dtype=w))
        assert np.abs(inv - Im).max(initial=0) <= tol * max(1.0, np.abs(Im).max(initial=0))


def test_device_pointers_and_layouts(fb, cuda_dev):
    import torch
    la = fb.linalg
    rng = np.random.default_rng(11)
    n = 200
    for dtype, tdt in ((np.float64, torch.float64), (np.complex64, torch.complex64)):
        A = sym(rng, n, dtype)
        ref = run(la, A.copy(order="F"), M.ROOK_DIAG, 16)
        # device, column-major
        T = torch.from_numpy(A.copy(order="F")).to(cuda_dev).t().contiguous().t()
        sub = torch.zeros(n, dtype=tdt, device=cuda_dev)
        p = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
        pi = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
        params = la.lblt_params_default()
        params.pivoting, params.block_size = M.ROOK_DIAG, 16
        la.lblt_in_place(T, sub, p, pi, params=params)
        assert np.array_equal(p.cpu().numpy(), ref[2])
        assert np.allclose(np.tril(T.cpu().numpy()), np.tril(ref[0]), atol=1e-3, rtol=0)
        # row-major host view and a non-unit row stride
        R = np.ascontiguousarray(A)
        LBr, subr, pr, _, _ = run(la, R, M.ROOK_DIAG, 16)
        assert np.array_equal(pr, ref[2])
        big = np.zeros((2 * n, n), dtype=dtype, order="F")
        big[::2] = A
        S = big[::2]
        LBs, subs, ps, _, _ = run(la, S, M.ROOK_DIAG, 16)
        assert np.array_equal(ps, ref[2]) and np.all(big[1::2] == 0)


def test_f64_6144_partial_diag(fb):
    la = fb.linalg
    rng = np.random.default_rng(6144)
    n = 6144
    A = sym(rng, n, np.float64)
    LB, sub, p, pi, cnt = run(la, A.copy(order="F"), M.PARTIAL_DIAG, 64)
    b = rng.standard_normal((n, 2))
    x = b.copy(order="F")
    la.lblt_solve_in_place(np.asfortranarray(np.tril(LB)), sub, p.astype(np.uint64), pi.astype(np.uint64), x)
    assert np.abs(A @ x - b).max(initial=0) / np.abs(b).max(initial=0) < 1e-6


def test_solvers_lblt_on_kkt(fb):
    s = fb.solvers
    rng = np.random.default_rng(5)
    n, m = 60, 20
    H = rng.standard_normal((n, n))
    H = H @ H.T + n * np.eye(n)
    B = rng.standard_normal((m, n))
    # the saddle-point system with the constraints first: its first pivot is exactly zero, so LDLT without pivoting fails
    K = np.asfortranarray(np.block([[np.zeros((m, m)), B], [B.T, H]]))
    with pytest.raises(s.LdltError):
        s.ldlt(K)
    f = s.lblt(K)
    b = rng.standard_normal((n + m, 1))
    x = f.solve(b)
    assert np.abs(K @ x - b).max(initial=0) < 1e-8 * np.abs(b).max(initial=0) * (n + m)
    assert np.abs(f.reconstruct() - K).max(initial=0) < 1e-10 * np.abs(K).max(initial=0) * (n + m)
    assert np.abs(f.inverse() @ K - np.eye(n + m)).max(initial=0) < 1e-8
