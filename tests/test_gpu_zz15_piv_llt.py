"""Pivoted Cholesky (`piv_llt_*`, csrc/piv_llt.cu) through the C ABI against the numpy restatement of
faer/src/linalg/cholesky/llt_pivoting (tests/piv_llt_model.py).

Factor: status, rank, transposition count, perm_fwd and perm_bwd exact; L[:, :rank] (all rows) within the LLT tests' tolerances;
the strict upper triangle bit for bit (NaN sentinels). Inputs avoid near-ties of the residual diagonal (well-conditioned Gram
matrices in f64 / c64, graded ones in every dtype), so the pivots do not depend on the trailing update's rounding. Solve,
reconstruct and inverse per dtype and index width."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import piv_llt_model as M  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32, np.complex128, np.complex64]


def ueps(dtype):
    return float(np.finfo(dtype).eps)


def randn(rng, shape, dtype):
    x = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.standard_normal(shape)
    return x


def gram(rng, n, dtype, r=None):
    """G G^H / m with G n x m (m = 2n: eigenvalues within a factor 34; m = r < n: rank r)."""
    m = r if r is not None else 2 * n
    G = randn(rng, (n, m), dtype)
    return np.asfortranarray((G @ np.conj(G.T) / max(m, 1)).astype(dtype))


def graded(rng, n, dtype):
    """diag(d) + 0.02 * (well-conditioned Gram), d = 1 + 0.05 * (a permutation of 0..n-1): the pivots follow d, whose gaps
    are far above any rounding difference."""
    d = 1.0 + 0.05 * rng.permutation(n)
    return np.asfortranarray((np.diag(d) + 0.02 * gram(rng, n, np.complex128 if np.issubdtype(dtype, np.complexfloating)
                                                           else np.float64)).astype(dtype))


def with_upper_sentinels(A):
    B = A.copy(order="F")
    B[np.triu_indices(A.shape[0], 1)] = np.nan
    return B


def factor(la, A, bs, it=np.uint64):
    n = A.shape[0]
    p = np.zeros(n, dtype=it)
    pi = np.full(n, 7, dtype=it)
    params = la.piv_llt_params_default()
    params.block_size = bs
    try:
        info = la.piv_llt_in_place(A, p, pi, params=params)
        return ("ok", info.rank, info.transposition_count), p.astype(np.int64), pi.astype(np.int64)
    except la.LltError as e:
        return ("err", e.index, None), p.astype(np.int64), None


def model(A, bs):
    ok, idx, tc, p, pi = M.piv_llt(A, bs)
    return ("ok", idx, tc) if ok else ("err", idx, None), p, pi


def ltol(dtype, n):
    return 64 * ueps(dtype) * max(n, 16)


def check_against_model(la, A0, bs, it=np.uint64):
    n = A0.shape[0]
    Ag = with_upper_sentinels(A0)
    st_g, p_g, pi_g = factor(la, Ag, bs, it)
    Am = A0.copy(order="F")
    st_m, p_m, pi_m = model(Am, bs)
    assert st_g == st_m, (n, bs, st_g, st_m)
    assert np.array_equal(p_g, p_m), (n, bs)
    if st_m[0] == "ok":
        assert np.array_equal(pi_g, pi_m)
        r = st_m[1]
        tol = ltol(A0.dtype, n)
        scale = max(1.0, float(np.abs(Am[:, :r]).max())) if r else 1.0
        Lg, Lm = np.tril(Ag)[:, :r], np.tril(Am)[:, :r]
        assert np.all(np.abs(Lg - Lm) <= tol * scale), (n, bs, float(np.abs(Lg - Lm).max()))
        if r < n:
            assert np.isclose(Ag[r, r], Am[r, r], rtol=1e-2, atol=1e3 * ueps(A0.dtype) * scale)
    iu = np.triu_indices(n, 1)
    assert np.all(np.isnan(Ag[iu])), "the strict upper triangle was written"
    return st_m, Ag, p_g, pi_g


CASES = [(2, 128), (3, 1), (3, 2), (50, 1), (50, 7), (127, 128), (128, 128), (129, 128), (129, 7), (300, 2), (300, 7),
         (300, 128), (1000, 7), (1000, 128)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_factor_full_rank(fb, dtype):
    la = fb.linalg
    rng = np.random.default_rng(1501)
    for n, bs in CASES:
        A = graded(rng, n, dtype)
        st, *_ = check_against_model(la, A, bs)
        assert st == ("ok", n, st[2])
        if dtype in (np.float64, np.complex128):
            st, *_ = check_against_model(la, gram(rng, n, dtype), bs, np.uint32)
            assert st[:2] == ("ok", n)


@pytest.mark.parametrize("dtype", DTYPES)
def test_factor_rank_deficient(fb, dtype):
    la = fb.linalg
    rng = np.random.default_rng(1502)
    for n, r, bs in [(50, 3, 7), (128, 5, 2), (300, 7, 128), (300, 40, 7), (1000, 10, 128)]:
        A = gram(rng, n, dtype, r)
        st, *_ = check_against_model(la, A, bs)
        assert st[:2] == ("ok", r), (n, r, bs, st)


@pytest.mark.parametrize("dtype", DTYPES)
def test_factor_edge_cases(fb, dtype):
    la = fb.linalg
    rng = np.random.default_rng(1503)
    # n = 0
    st, p, pi = factor(la, np.zeros((0, 0), dtype=dtype, order="F"), 128)
    assert st == ("ok", 0, 0) and p.size == 0
    # n = 1: Ok { rank: 1 }, also for a zero entry
    for v in (4.0, 0.0):
        A = np.full((1, 1), v, dtype=dtype, order="F")
        st, p, pi = factor(la, A, 128)
        assert st == ("ok", 1, 0) and A[0, 0] == np.sqrt(v)
    for bs in (1, 2, 7, 128):
        # identity: no swap, rank n; diag with repeated values: first-maximum tie rule
        check_against_model(la, np.eye(9, dtype=dtype, order="F"), bs)
        d = np.array([1, 3, 2, 3, 5, 5, 0.5, 5, 2], dtype=np.float64)
        st, _, p, _ = check_against_model(la, np.asfortranarray(np.diag(d).astype(dtype)), bs)
        assert st == ("ok", 9, 6) and list(p) == [4, 5, 7, 3, 1, 2, 8, 0, 6]
        # zero matrix: NaN at column 1 (index 1)
        st, *_ = check_against_model(la, np.zeros((6, 6), dtype=dtype, order="F"), bs)
        assert st[:2] == ("err", 1)
        # NaN off the diagonal: the first column that reaches it
        A = graded(rng, 12, dtype)
        A[7, 3] = np.nan
        check_against_model(la, A, bs)
    # negative / NaN diagonal entry: index 0, A untouched
    for bad in (-1.0, np.nan):
        A = graded(rng, 40, dtype)
        A[17, 17] = bad
        B = A.copy(order="F")
        st, p, _ = factor(la, B, 128)
        assert st[:2] == ("err", 0) and np.array_equal(p, np.arange(40))
        assert np.array_equal(B, A, equal_nan=True)


@pytest.mark.parametrize("dtype", DTYPES)
def test_factor_device_pointers_and_strides(fb, cuda_dev, dtype):
    import torch
    la = fb.linalg
    rng = np.random.default_rng(1504)
    n, bs = 300, 7
    A0 = graded(rng, n, dtype)
    Am = A0.copy(order="F")
    st_m, p_m, pi_m = model(Am, bs)
    params = la.piv_llt_params_default()
    params.block_size = bs
    for tdt in (torch.int32, torch.int64):
        # device matrix (column-major) and device permutations
        dA = torch.from_numpy(np.ascontiguousarray(with_upper_sentinels(A0).T)).to(cuda_dev).T
        p = torch.zeros(n, dtype=tdt, device=cuda_dev)
        pi = torch.zeros(n, dtype=tdt, device=cuda_dev)
        info = la.piv_llt_in_place(dA, p, pi, params=params)
        assert ("ok", info.rank, info.transposition_count) == st_m
        assert np.array_equal(p.cpu().numpy(), p_m) and np.array_equal(pi.cpu().numpy(), pi_m)
        Ag = dA.cpu().numpy()
        assert np.all(np.abs(np.tril(Ag) - np.tril(Am)) <= ltol(dtype, n) * np.abs(Am).max())
        assert np.all(np.isnan(Ag[np.triu_indices(n, 1)]))
    # a non-unit row stride (every other row of a taller host array) and a row-major matrix
    big = np.full((2 * n, n), np.nan, dtype=dtype, order="F")
    big[::2] = with_upper_sentinels(A0)
    view = big[::2]
    st_g, p_g, pi_g = factor(la, view, bs)
    assert st_g == st_m and np.array_equal(p_g, p_m)
    assert np.all(np.abs(np.tril(view) - np.tril(Am)) <= ltol(dtype, n) * np.abs(Am).max())
    assert np.all(np.isnan(big[1::2]))
    rowmaj = np.ascontiguousarray(with_upper_sentinels(A0))
    st_g, p_g, _ = factor(la, rowmaj, bs)
    assert st_g == st_m and np.array_equal(p_g, p_m)
    assert np.all(np.abs(np.tril(rowmaj) - np.tril(Am)) <= ltol(dtype, n) * np.abs(Am).max())


def test_factor_wide_trailing_update(fb):
    """n = 6144, block 128: the first trailing updates are 47 x 47 lower tiles of 128 x 128 (8 waves), so the SYRK takes the
    wide warp-specialised f64 configuration."""
    la = fb.linalg
    rng = np.random.default_rng(1505)
    n = 6144
    st, *_ = check_against_model(la, graded(rng, n, np.float64), 128)
    assert st[:2] == ("ok", n)


@pytest.mark.parametrize("it", [np.uint32, np.uint64])
@pytest.mark.parametrize("dtype", DTYPES)
def test_solve_reconstruct_inverse(fb, dtype, it):
    la = fb.linalg
    rng = np.random.default_rng(1506)
    u = ueps(dtype)
    for n, bs in [(50, 7), (257, 128)]:
        A = graded(rng, n, dtype)
        L = A.copy(order="F")
        p = np.zeros(n, dtype=it)
        pi = np.zeros(n, dtype=it)
        params = la.piv_llt_params_default()
        params.block_size = bs
        info = la.piv_llt_in_place(L, p, pi, params=params)
        assert info.rank == n
        Af = M.mirror(A).astype(np.complex128)
        # solve, A_conj = No / Yes
        B = np.asfortranarray(randn(rng, (n, 3), dtype).astype(dtype))
        for conj in (la.CONJ_NO, la.CONJ_YES):
            X = B.copy(order="F")
            la.piv_llt_solve_in_place(L, p, pi, X, conj=conj)
            Ac = np.conj(Af) if conj == la.CONJ_YES else Af
            res = np.abs(Ac @ X.astype(np.complex128) - B).max()
            assert res <= 64 * n * u * np.abs(Af).max() * max(1.0, np.abs(X).max()), (n, conj, res)
        # reconstruct: the model's gather of L L^H, the strict upper triangle of out untouched
        out = np.full((n, n), np.nan, dtype=dtype, order="F")
        la.piv_llt_reconstruct(out, L, p, pi)
        want = M.reconstruct(L.astype(np.complex128), pi.astype(np.int64))
        il = np.tril_indices(n)
        assert np.all(np.abs(out[il] - want[il]) <= 64 * n * u * np.abs(Af).max())
        assert np.all(np.abs(out[il] - np.tril(Af)[il]) <= 64 * n * u * np.abs(Af).max())
        assert np.all(np.isnan(out[np.triu_indices(n, 1)]))
        # inverse: A_inv A = I with the lower triangle mirrored
        out = np.full((n, n), np.nan, dtype=dtype, order="F")
        la.piv_llt_inverse(out, L, p, pi)
        assert np.all(np.isnan(out[np.triu_indices(n, 1)]))
        Ai = M.mirror(np.where(np.isnan(out), 0, out)).astype(np.complex128)
        err = np.abs(Ai @ Af - np.eye(n)).max()
        assert err <= 64 * n * u * np.linalg.cond(Af), (n, err)
