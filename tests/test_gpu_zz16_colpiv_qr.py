"""Column-pivoted QR (`colpiv_qr_*`, csrc/colpiv_qr.cu) through the C ABI against the numpy restatement of
faer/src/linalg/qr/col_pivoting (tests/colpiv_qr_model.py).

Factor on graded inputs (pivot gaps far above rounding): perm_fwd, perm_bwd and the transposition count exact; R, the Householder
vectors and Q_coeff within the QR tests' tolerances. On Gaussian and rank-deficient inputs, whatever the ties: the factorization
reproduces A, the pivoting inequality holds and R reveals the rank. Runs are bitwise reproducible. Solve, solve_transpose,
lstsq, reconstruct and inverse per dtype and index width."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import colpiv_qr_model as M  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32, np.complex128, np.complex64]
CX = (np.complex128, np.complex64)


def ueps(dtype):
    return float(np.finfo(dtype).eps)


def randn(rng, shape, dtype):
    x = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.standard_normal(shape)
    return x


def graded(rng, m, n, dtype, hi=1e3):
    """Gaussian columns scaled by a random permutation of a geometric sequence from 1 to `hi`."""
    g = np.geomspace(1.0, hi, max(n, 1))[:n]
    rng.shuffle(g)
    return np.asfortranarray((randn(rng, (m, n), dtype) * g).astype(dtype))


def maxdiff(a, b):
    """max |a - b|, equal infinities (the +inf tau of a reflector with an empty or zero tail) counting as 0"""
    a, b = np.asarray(a), np.asarray(b)
    d = np.where(np.isinf(b) & (a == b), 0.0, np.abs(a - b))
    return np.max(d, initial=0)


def factor(la, A, bs, it=np.uint64):
    m, n = A.shape
    H = np.zeros((bs, min(m, n)), dtype=A.dtype, order="F")
    p = np.zeros(n, dtype=it)
    pi = np.zeros(n, dtype=it)
    info = la.colpiv_qr_in_place(A, H, p, pi)
    return H, p.astype(np.int64), pi.astype(np.int64), info.transposition_count


def check_against_model(la, A0, bs, it=np.uint64, row_stride_one=True, A=None):
    dtype = A0.dtype
    QRm, Hm, pm, pim, cm = M.factor(A0, bs, row_stride_one)  # in the working precision: the branch threshold is sqrt(eps)
    A = np.asfortranarray(A0.copy()) if A is None else A
    H, p, pi, c = factor(la, A, bs, it)
    m, n = A0.shape
    assert (p == pm).all() and (pi == pim).all() and c == cm
    tol = 50 * max(m, n, 1) * ueps(dtype) * max(1.0, np.max(np.abs(QRm), initial=0))
    assert np.max(np.abs(np.asarray(A) - QRm), initial=0) <= tol
    s = min(m, n)
    Tm = np.triu(Hm[:, :s]) if s else Hm
    finite = np.abs(Tm[np.isfinite(Tm)])
    # T = striu(V^H V) + diag(tau): an entry sums up to m products of reflector entries (|v| <= 1), so it carries up to
    # 2 m times the difference of the reflectors themselves
    dV = np.max(np.abs(np.tril(np.asarray(A), -1) - np.tril(QRm, -1)), initial=0)
    assert maxdiff(np.triu(H), Tm) <= 2 * m * dV + 200 * max(m, n, 1) * ueps(dtype) * max(1.0, np.max(finite, initial=0))
    return A, H, p, pi


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [0, 1, 2, 3, 17, 127, 255, 1000])
def test_factor_square_against_model(fb, dtype, n):
    la = fb.linalg
    rng = np.random.default_rng(n)
    single = ueps(dtype) > 1e-10
    # single precision over 1000 columns: neighbouring scales 1e3^(1/999) = 0.7 % apart leave some late pivots of the downdated
    # norms within rounding; a grading up to 1e9 (2.1 % apart) keeps them separated, which the model confirms below by giving
    # the same pivots in single and in double precision
    hi = 1e9 if single and n >= 1000 else 1e3
    A0 = graded(rng, n, n, dtype, hi)
    if single and n >= 1000:
        wide = np.complex128 if dtype in CX else np.float64
        assert (M.factor(A0, 15)[2] == M.factor(A0.astype(wide), 15)[2]).all()
    for bs in sorted({1, 15, max(1, la.qr_recommended_block_size(n, n))}):
        check_against_model(la, A0, bs, np.uint64 if bs != 15 else np.uint32)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(4000, 300), (300, 4000)])
def test_factor_rectangular_against_model(fb, dtype, shape):
    la = fb.linalg
    check_against_model(la, graded(np.random.default_rng(7), *shape, dtype), la.qr_recommended_block_size(*shape))


@pytest.mark.parametrize("dtype", DTYPES)
def test_row_major_and_strided_views(fb, dtype):
    la = fb.linalg
    rng = np.random.default_rng(11)
    A0 = graded(rng, 120, 90, dtype)
    # row-major: the caller's row stride is not 1, so every column takes the recompute branch
    check_against_model(la, A0, 8, row_stride_one=False, A=np.ascontiguousarray(A0))
    sub = np.asfortranarray(np.zeros((300, 120), dtype=dtype))[10:130, 5:95]
    sub[...] = A0
    check_against_model(la, A0, 8, A=sub)


@pytest.mark.parametrize("dtype", DTYPES)
def test_device_pointers(fb, cuda_dev, dtype):
    import torch
    la = fb.linalg
    rng = np.random.default_rng(3)
    A0 = graded(rng, 300, 200, dtype)
    QRm, Hm, pm, _, cm = M.factor(A0, 16)
    dA = torch.from_numpy(np.ascontiguousarray(A0.T)).to(cuda_dev).T
    dH = torch.zeros((200, 16), dtype=dA.dtype, device=cuda_dev).T
    p = torch.zeros(200, dtype=torch.int64, device=cuda_dev)
    pi = torch.zeros(200, dtype=torch.int64, device=cuda_dev)
    info = la.colpiv_qr_in_place(dA, dH, p, pi)
    assert (p.cpu().numpy() == pm).all() and info.transposition_count == cm
    assert np.max(np.abs(dA.cpu().numpy() - QRm)) <= 1e3 * ueps(dtype) * np.max(np.abs(QRm))


def replayed_count(perm, size):
    """The transposition count of the reference's loop that ends in `perm`: step k swaps the chosen column into position k, so
    the swap sequence is determined by the first `size` entries of the final permutation."""
    cur = list(range(len(perm)))
    pos = {c: i for i, c in enumerate(cur)}
    count = 0
    for k in range(size):
        j = pos[int(perm[k])]
        if j != k:
            cur[j], cur[k] = cur[k], cur[j]
            pos[cur[j]], pos[cur[k]] = j, k
            count += 1
    return count


@pytest.mark.parametrize("dtype,shape", [(np.float64, (4096, 4096)), (np.float32, (16384, 1024))])
def test_large_row_split_against_geqp3(fb, dtype, shape):
    """The row-split path at sizes where the numpy model takes minutes: pivots against LAPACK ?geqp3 (f64 arithmetic), the
    transposition count and perm_bwd from them, |diag R| against ?geqp3's, and Q R P^T = A through the T blocks of Q_coeff."""
    import scipy.linalg as sl
    la = fb.linalg
    rng = np.random.default_rng(1)
    A0 = graded(rng, *shape, dtype)
    A = np.asfortranarray(A0.copy())
    bs = 64
    H, p, pi, c = factor(la, A, bs)
    Rg, P = sl.qr(A0.astype(np.float64), pivoting=True, mode="r")
    m, n = shape
    s = min(shape)
    assert (p[:s] == P[:s]).all()
    assert (pi[p] == np.arange(n)).all()
    assert c == replayed_count(p, s)
    dg = np.abs(np.diag(Rg))[:s]
    assert np.max(np.abs(np.abs(np.diag(A))[:s] - dg)) <= 50 * max(m, n) * ueps(dtype) * dg[0]
    out = np.zeros(shape, dtype=dtype, order="F")
    la.colpiv_qr_reconstruct(out, A, H, np.triu(A)[:s], p.astype(np.uint64), pi.astype(np.uint64))
    assert np.linalg.norm(out - A0) <= 50 * max(m, n) * ueps(dtype) * np.linalg.norm(A0)


def contract_checks(la, A0, r=None):
    dtype = A0.dtype
    m, n = A0.shape
    A = np.asfortranarray(A0.copy())
    H, p, pi, c = factor(la, A, 8)
    s = min(m, n)
    R = np.triu(A)[:s]
    QR = np.array(A)
    w = np.complex128 if dtype in CX else np.float64
    tau = np.real(H[np.arange(s) % 8, np.arange(s)]).astype(np.float64)
    out = M.reconstruct(QR.astype(w), tau, p)
    nrm = np.linalg.norm(A0)
    assert np.linalg.norm(out - A0) <= 100 * max(m, n) * ueps(dtype) * nrm
    d = np.abs(np.diag(R))
    for k in range(s):
        colsq = np.sum(np.abs(R[k:s, k + 1:]) ** 2, axis=0)
        assert (d[k] ** 2 >= (1 - 1e-3) * colsq - 1e3 * ueps(dtype) * nrm ** 2).all()
    if r is not None:
        assert (d[r:] <= 1e3 * ueps(dtype) * d[0]).all()
    A2 = np.asfortranarray(A0.copy())
    H2, p2, pi2, c2 = factor(la, A2, 8)
    assert np.asarray(A2).tobytes() == np.asarray(A).tobytes() and H2.tobytes() == H.tobytes()
    assert (p2 == p).all() and (pi2 == pi).all() and c2 == c


@pytest.mark.parametrize("dtype", DTYPES)
def test_contracts_gaussian_and_rank_deficient(fb, dtype):
    la = fb.linalg
    rng = np.random.default_rng(2)
    contract_checks(la, np.asfortranarray(randn(rng, (200, 150), dtype).astype(dtype)))
    B, Cm = randn(rng, (200, 20), dtype), randn(rng, (20, 150), dtype)
    contract_checks(la, np.asfortranarray((B @ Cm).astype(dtype)), r=20)


def test_edge_cases(fb):
    la = fb.linalg
    # a NaN column next to a zero column: nothing qualifies at k = 1, so the pivot stays at k (factor.rs:161-193)
    nan_zero = np.array([[1.0, np.nan, 0.0], [2.0, np.nan, 0.0], [3.0, np.nan, 0.0]])
    for A0 in (np.zeros((6, 5)), np.zeros((0, 3)), np.zeros((3, 0)), np.ones((7, 1)), nan_zero):
        A = np.asfortranarray(A0.copy())
        H, p, pi, c = factor(la, A, 4)
        _, _, pm, _, cm = M.factor(A0, 4)
        assert (p == pm).all() and c == cm
    A = np.asfortranarray(np.zeros((6, 5)))
    factor(la, A, 4)
    assert np.isnan(A).all()
    rng = np.random.default_rng(5)
    for cols in (((2, 0.0),), ((1, np.nan),), ((1, np.nan), (2, 0.0)), ((0, 0.0), (3, 0.0))):
        A0 = graded(rng, 10, 6, np.float64)
        for col, val in cols:
            A0[:, col] = val
        A = np.asfortranarray(A0.copy())
        H, p, pi, c = factor(la, A, 4)
        _, _, pm, _, cm = M.factor(A0, 4)
        assert (p == pm).all() and c == cm


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("it", [np.uint32, np.uint64])
def test_solves_reconstruct_inverse(fb, dtype, it):
    la = fb.linalg
    rng = np.random.default_rng(4)
    n, k = 60, 3
    tol = 1e3 * n * ueps(dtype)
    A0 = np.asfortranarray(randn(rng, (n, n), dtype).astype(dtype))
    QR = np.asfortranarray(A0.copy())
    H = np.zeros((4, n), dtype=dtype, order="F")
    p, pi = np.zeros(n, dtype=it), np.zeros(n, dtype=it)
    la.colpiv_qr_in_place(QR, H, p, pi)
    B = np.asfortranarray(randn(rng, (n, k), dtype).astype(dtype))
    conjs = (la.CONJ_NO, la.CONJ_YES) if dtype in CX else (la.CONJ_NO,)
    for conj in conjs:
        Ac = A0.conj() if conj == la.CONJ_YES else A0
        X = B.copy(order="F")
        la.colpiv_qr_solve_in_place(QR, H, QR, p, pi, X, conj)
        assert np.linalg.norm(Ac @ X - B) <= tol * np.linalg.norm(Ac) * np.linalg.norm(X)
        X = B.copy(order="F")
        la.colpiv_qr_solve_transpose_in_place(QR, H, QR, p, pi, X, conj)
        assert np.linalg.norm(Ac.T @ X - B) <= tol * np.linalg.norm(Ac) * np.linalg.norm(X)
    out = np.zeros((n, n), dtype=dtype, order="F")
    la.colpiv_qr_reconstruct(out, QR, H, QR, p, pi)
    assert np.linalg.norm(out - A0) <= tol * np.linalg.norm(A0)
    la.colpiv_qr_inverse(out, QR, H, QR, p, pi)
    assert np.linalg.norm(A0 @ out - np.eye(n)) <= tol * np.linalg.norm(A0) * np.linalg.norm(out)
    # least squares on a tall rank-deficient input (rank 25) with a consistent right-hand side: backward stable, so the residual
    # is at the rounding level of ||A|| ||x||
    m, n2, r = 150, 40, 25
    A1 = np.asfortranarray((randn(rng, (m, r), dtype) @ randn(rng, (r, n2), dtype)).astype(dtype))
    QR = A1.copy(order="F")
    H = np.zeros((4, n2), dtype=dtype, order="F")
    p, pi = np.zeros(n2, dtype=it), np.zeros(n2, dtype=it)
    la.colpiv_qr_in_place(QR, H, p, pi)
    assert (np.abs(np.diag(QR))[r:] <= 1e3 * ueps(dtype) * abs(QR[0, 0])).all()
    B = np.asfortranarray((A1 @ randn(rng, (n2, k), dtype)).astype(dtype))
    X = B.copy(order="F")
    la.colpiv_qr_solve_lstsq_in_place(QR, H, QR, p, pi, X)
    assert np.linalg.norm(A1 @ X[:n2] - B) <= tol * (np.linalg.norm(A1) * np.linalg.norm(X[:n2]) + np.linalg.norm(B))
    # least squares on a tall full-rank input

    for conj in conjs:
        A1 = np.asfortranarray(randn(rng, (m, n2), dtype).astype(dtype))
        QR = A1.copy(order="F")
        H = np.zeros((4, n2), dtype=dtype, order="F")
        p, pi = np.zeros(n2, dtype=it), np.zeros(n2, dtype=it)
        la.colpiv_qr_in_place(QR, H, p, pi)
        B = np.asfortranarray(randn(rng, (m, k), dtype).astype(dtype))
        X = B.copy(order="F")
        la.colpiv_qr_solve_lstsq_in_place(QR, H, QR, p, pi, X, conj)
        Ac = A1.conj() if conj == la.CONJ_YES else A1
        lhs = Ac.conj().T @ (Ac @ X[:n2]) - Ac.conj().T @ B
        assert np.linalg.norm(lhs) <= tol * np.linalg.norm(Ac) ** 2 * np.linalg.norm(X[:n2])


@pytest.mark.parametrize("dtype", DTYPES)
def test_solvers_colpiv_qr_end_to_end(fb, cuda_dev, dtype):
    """solvers.ColPivQr (solvers.rs:1206-1260, 2462-2560) on host and device matrices."""
    import torch
    sv = fb.solvers
    rng = np.random.default_rng(8)
    n, k = 70, 2
    tol = 1e3 * n * ueps(dtype)
    A0 = randn(rng, (n, n), dtype).astype(dtype)
    B0 = randn(rng, (n, k), dtype).astype(dtype)
    for dev in (False, True):
        A = torch.from_numpy(np.ascontiguousarray(A0.T)).to(cuda_dev).T if dev else np.asfortranarray(A0)
        B = torch.from_numpy(np.ascontiguousarray(B0.T)).to(cuda_dev).T if dev else np.asfortranarray(B0)
        host = (lambda x: x.cpu().numpy()) if dev else (lambda x: np.asarray(x))
        f = sv.ColPivQr.new(A)
        fwd, bwd = (host(x).astype(np.int64) for x in f.P())
        assert (np.sort(fwd) == np.arange(n)).all() and (bwd[fwd] == np.arange(n)).all()
        Q, R = host(f.compute_Q()), host(f.R())
        assert np.linalg.norm(Q @ R - A0[:, fwd]) <= tol * np.linalg.norm(A0)
        d = np.abs(np.diag(R))
        assert (d[:-1] >= d[1:] * (1 - 1e-3)).all()  # the pivoting makes |R_kk| non-increasing
        assert np.linalg.norm(host(f.reconstruct()) - A0) <= tol * np.linalg.norm(A0)
        X = host(f.solve(B))
        assert np.linalg.norm(A0 @ X - B0) <= tol * np.linalg.norm(A0) * np.linalg.norm(X)
        X = host(f.solve_transpose(B))
        assert np.linalg.norm(A0.T @ X - B0) <= tol * np.linalg.norm(A0) * np.linalg.norm(X)
        X = host(f.solve_adjoint(B))
        assert np.linalg.norm(A0.conj().T @ X - B0) <= tol * np.linalg.norm(A0) * np.linalg.norm(X)
        Ai = host(f.inverse())
        assert np.linalg.norm(A0 @ Ai - np.eye(n)) <= tol * np.linalg.norm(A0) * np.linalg.norm(Ai)
        # tall: least squares and the thin factors
        T0 = randn(rng, (3 * n, n), dtype).astype(dtype)
        T = torch.from_numpy(np.ascontiguousarray(T0.T)).to(cuda_dev).T if dev else np.asfortranarray(T0)
        g = sv.ColPivQr.new(T)
        fwd = host(g.P()[0]).astype(np.int64)
        Qt, Rt = host(g.compute_thin_Q()), host(g.thin_R())
        assert Qt.shape == (3 * n, n) and Rt.shape == (n, n)
        assert np.linalg.norm(Qt @ Rt - T0[:, fwd]) <= tol * np.linalg.norm(T0)
        C0 = randn(rng, (3 * n, k), dtype).astype(dtype)
        C = torch.from_numpy(np.ascontiguousarray(C0.T)).to(cuda_dev).T if dev else np.asfortranarray(C0)
        X = host(g.solve_lstsq(C))
        assert X.shape == (n, k)
        res = T0.conj().T @ (T0 @ X - C0)
        assert np.linalg.norm(res) <= tol * np.linalg.norm(T0) ** 2 * np.linalg.norm(X)
