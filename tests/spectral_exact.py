"""Matrices whose eigen- and singular decompositions are known exactly, and error-to-bound checks of computed ones.

Construction. Every matrix is an exact floating-point number set, built in int64 and scaled by a power of two:

  * w is a small-integer vector (entries +-1, a few 0 or +-2; for complex matrices each entry also carries a phase from
    {1, i, -1, -i}) with w^H w = 2^k, so H = I - 2^(1-k) w w^H is unitary, Hermitian and dyadic;
  * self-adjoint: for integer eigenvalues D = diag(d),
        2^(2k) H D H = 2^(2k) D - 2^(k+1) (w (Dw)^H + (Dw) w^H) + 4 (w^H D w) w w^H,
    a rank-2 update computed in O(n^2) int64. The eigenvalues are d_i 2^e and the eigenvectors exactly H e_i;
  * rectangular: A = H_m [diag(s); 0] H_n (one reflector on each side), expanded the same way; A = U S V^H with U = H_m,
    V = H_n;
  * optionally a random signed permutation on each side, which is exact too.
Dividing the integers by 2^(2k) (and multiplying by 2^e) is exact only if they stay below 2^53 (2^24 for f32); the
builders check this by converting back (2^(2k - e) A == M in int64) and raise ValueError for a spectrum that does not
fit instead of rounding it. Two closed-form tridiagonals complete the set: the 1-2-1 Toeplitz matrix (eigenvalues
4 sin^2(j pi / (2 (n + 1))), evaluated with mpmath and rounded once; eigenvectors the sine basis) and the Clement
(Kac-Sylvester) matrix (off-diagonals sqrt(i (n - i)) rounded once; eigenvalues the integers -(n-1), -(n-3), ..., n-1).

Bounds. A backward-stable solver returns the exact decomposition of A + E with ||E||_2 <= p u ||A||_2 and columns
orthonormal to p u, where u = 2^-53 and p = C N with C = 8 fixed here: N is n for the self-adjoint EVD and m + n for the
SVD (the order of the Jordan-Wielandt matrix [0 A; A^H 0], whose eigenproblem the SVD is). This is the form of the error
bounds LAPACK states for its symmetric eigensolvers and SVDs (LAPACK Users' Guide, 3rd ed., sections 4.7 and 4.9), with
the "modestly growing function p(n)" taken as 8 n. With e_in = ||A_stored - A_exact||_2 (0 for the dyadic matrices) and
gamma_m = m u / (1 - m u), the checks are, per column i:

  values     |lam^_i - lam_i| <= p u ||A|| + e_in                                        (Weyl)
  residual   ||A u^_i - lam^_i u^_i|| <= (p u ||A|| + e_in) ||u^_i|| + gamma_{N+2} || |A||u^_i| + |lam^_i||u^_i| ||
             (the second term is the f64 rounding of evaluating the residual); for the SVD both ||A v^_i - s^_i u^_i||
             and ||A^H u^_i - s^_i v^_i||, and ||A^H u^_i|| (||A v^_i||) for the columns of a full U (V) past min(m, n)
  orthogonal |U^H U - I|_ij <= p u + gamma_N ||u^_i|| ||u^_j||
  vectors    sin(u^_i, X_c) <= r / delta_i + e_Q                                          (Davis-Kahan sin theta)
             X_c is the exact invariant subspace of column i's cluster: a maximal run of exact eigenvalues whose
             neighbours are at most 2^10 (p u ||A|| + e_in) apart, so a repeated eigenvalue is one cluster and a pair
             that close is judged as a subspace. r = p u ||A|| + e_in bounds the residual of the exact A, delta_i is
             the distance from lam^_i to the nearest exact eigenvalue outside the cluster (for any unit x and any mu,
             ||(I - X_c X_c^H) x|| <= ||(A - mu) x|| / delta), and e_Q bounds the rounding of applying the exact basis.
             For the SVD (Wedin, through the Jordan-Wielandt matrix) the clusters are taken over +-s_j, plus 0 when
             m != n, the bound is sqrt(2) r / delta_i + e_Q, and it is applied to U and to V; the null space
             columns (s = 0, and a full U's or V's columns past min(m, n)) are judged against the exact null spaces.

For f32 outputs (the f32 entry points compute in f64 and round once) each bound also gets the rounding of the outputs
with u_out = 2^-24: u_out |lam^| on values, u_out (||A|| + 2 |lam^|) on residuals, 2 u_out on orthogonality, u_out on
angles. Every check evaluates in f64 (c128) on the device that holds the matrix, after scaling by an exact power of two
that puts ||A|| in [1/2, 1) (so 2^+-500 inputs neither overflow nor underflow in the check). Each returns the largest
error-to-bound ratio; a pass is <= 1 and a NaN counts as infinite. `loosen` multiplies every bound (used by the tests
that show which wrong results stay rejected with bounds 10^3 looser).
"""
import math
from dataclasses import dataclass
from typing import Callable, Optional

import numpy as np
import torch

U64 = 2.0 ** -53
U32 = 2.0 ** -24
C = 8
CLUSTER = 2.0 ** 10


def gamma(m: int) -> float:
    return m * U64 / (1.0 - m * U64)


# ---------------------------------------------------------------------------------------------------------------- build


def weights(n: int, rng, cplx: bool = False):
    """(w_re, w_im, k): int64 numpy vectors with sum |w|^2 = 2^k, entries mostly of modulus 1, the fewest 0s and 2s."""
    best = None
    for k in range(0, n.bit_length() + 2):
        d = (1 << k) - n  # |w|^2 = n - zeros + 3 twos
        t, z = (-(-d // 3), 3 * (-(-d // 3)) - d) if d >= 0 else (0, -d)
        if t + z <= n and (best is None or t + z < best[0]):
            best = (t + z, k, t, z)
    _, k, t, z = best
    mag = np.ones(n, dtype=np.int64)
    idx = rng.permutation(n)
    mag[idx[:t]] = 2
    mag[idx[t:t + z]] = 0
    mag *= rng.choice(np.array([-1, 1], dtype=np.int64), n)
    if not cplx:
        wr, wi = mag, np.zeros(n, dtype=np.int64)
    else:
        rot = rng.integers(0, 2, n)  # multiply by i where set
        wr, wi = np.where(rot == 0, mag, 0), np.where(rot == 1, mag, 0)
    assert int((wr * wr + wi * wi).sum()) == 1 << k
    return wr, wi, k


def _outer_h(xr, xi, yr, yi):
    """x y^H for Gaussian-integer vectors given as (re, im) int64 tensors."""
    return (xr[:, None] * yr[None, :] + xi[:, None] * yi[None, :], xi[:, None] * yr[None, :] - xr[:, None] * yi[None, :])


def _to_float(Mr, Mi, scale_exp: int, dtype, bits: int, cplx: bool):
    """M 2^scale_exp as `dtype` (real or complex counterpart), checked to be exact."""
    lim = 1 << bits
    if not -1022 <= scale_exp <= 1023:
        raise ValueError(f"spectrum does not fit: scale 2^{scale_exp} is not a normal f64")
    for M in (Mr, Mi):
        if int(M.abs().max()) >= lim:
            raise ValueError(f"spectrum does not fit: integers reach {int(M.abs().max())} >= 2^{bits}")
    parts = []
    for M in (Mr, Mi) if cplx else (Mr,):
        F = M.to(dtype) * math.ldexp(1.0, scale_exp)
        back = F.to(torch.float64) * math.ldexp(1.0, -scale_exp)
        if not bool((back.to(torch.int64) == M).all()) or not bool(torch.isfinite(F).all()):
            raise ValueError("spectrum does not fit: the scaled matrix is not exact")
        parts.append(F)
    return torch.complex(*parts) if cplx else parts[0]


@dataclass
class Basis:
    """A unitary Q known exactly. apply_h(X) = Q^H X; row j of the result belongs to exact value `raw[j]`; `err` bounds
    the f64 rounding of ||Q^H x|| restricted to any set of rows, for a unit x."""
    apply_h: Callable
    raw: torch.Tensor
    err: float


@dataclass
class Exact:
    A: torch.Tensor  # the stored matrix (its exact spectrum is below)
    values: torch.Tensor  # float64: eigenvalues ascending / singular values descending
    norm: float  # ||A_exact||_2
    input_err: float = 0.0  # ||A_stored - A_exact||_2
    value_err: float = 0.0  # relative rounding of `values` (closed forms evaluated in mpmath)
    left: Optional[Basis] = None  # eigenvectors / U
    right: Optional[Basis] = None  # V


def _reflector_basis(wr, wi, k, perm, sign, raw, cplx, device):
    """Q = P H with (P x)[i] = sign[i] x[perm[i]]... as a Basis: Q^H X = H P^T X."""
    w = torch.complex(torch.as_tensor(wr, dtype=torch.float64), torch.as_tensor(wi, dtype=torch.float64)) if cplx else \
        torch.as_tensor(wr, dtype=torch.float64)
    w = w.to(device)
    p = torch.as_tensor(perm, device=device)
    s = torch.as_tensor(sign, dtype=torch.float64, device=device)
    f = 2.0 ** (1 - k)
    n = w.shape[0]

    def apply_h(X):
        Y = torch.empty_like(X)
        Y[p] = s[:, None] * X  # P^T X
        return Y - f * w[:, None] * (w.conj()[None, :] @ Y)

    return Basis(apply_h, raw, 2.0 * gamma(n + 3))


def _signed_perm(n, rng, permute):
    if not permute:
        return np.arange(n), np.ones(n, dtype=np.int64)
    return rng.permutation(n), rng.choice(np.array([-1, 1], dtype=np.int64), n)


def hermitian(d, rng, device="cpu", exp: int = 0, dtype=torch.float64, cplx: bool = False, permute: bool = True) -> Exact:
    """Self-adjoint P H diag(d 2^exp) H P^T with integer d (any order; values may repeat), exact in `dtype`
    (float64 / float32; complex when `cplx`)."""
    d = np.asarray(d, dtype=np.int64)
    n = d.size
    bits = 53 if dtype == torch.float64 else 24
    wr, wi, k = weights(n, rng, cplx)
    if int(np.abs(d).max(initial=0)) >= 1 << max(0, 61 - 2 * k - 5):
        raise ValueError("spectrum does not fit in int64 intermediates")
    t = lambda x: torch.as_tensor(x, dtype=torch.int64, device=device)
    xr, xi, D = t(wr), t(wi), t(d)
    yr, yi = D * xr, D * xi
    c = int((D * (xr * xr + xi * xi)).sum())  # w^H D w (real)
    a1, b1 = _outer_h(xr, xi, yr, yi)
    a2, b2 = _outer_h(yr, yi, xr, xi)
    a3, b3 = _outer_h(xr, xi, xr, xi)
    Mr = (a1 + a2) * -(1 << (k + 1)) + a3 * (4 * c)
    Mi = (b1 + b2) * -(1 << (k + 1)) + b3 * (4 * c)
    del a1, a2, a3, b1, b2, b3
    Mr.diagonal().add_(D << (2 * k))
    perm, sign = _signed_perm(n, rng, permute)
    P, S = t(perm), t(sign)
    ss = S[:, None] * S[None, :]
    Mr = Mr[P][:, P] * ss
    Mi = Mi[P][:, P] * ss
    A = _to_float(Mr, Mi, exp - 2 * k, dtype, bits, cplx)
    del Mr, Mi
    raw = D.to(torch.float64) * math.ldexp(1.0, exp)
    vals = torch.sort(raw).values
    norm = float(vals.abs().max()) if n else 0.0
    return Exact(A, vals, norm, left=_reflector_basis(wr, wi, k, perm, sign, raw, cplx, device))


def rectangular(m: int, n: int, s, rng, device="cpu", exp: int = 0, dtype=torch.float64, cplx: bool = False,
                permute: bool = True) -> Exact:
    """P_m H_m [diag(s 2^exp); 0] H_n P_n^T (m x n) with non-negative integer s of length min(m, n)."""
    s = np.asarray(s, dtype=np.int64)
    size = min(m, n)
    assert s.shape == (size,) and (s >= 0).all()
    bits = 53 if dtype == torch.float64 else 24
    ur, ui, km = weights(m, rng, cplx)
    vr, vi, kn = weights(n, rng, cplx)
    if int(s.max(initial=0)) >= 1 << max(0, 61 - km - kn - 5):
        raise ValueError("spectrum does not fit in int64 intermediates")
    t = lambda x: torch.as_tensor(x, dtype=torch.int64, device=device)
    Ur, Ui, Vr, Vi, Sg = t(ur), t(ui), t(vr), t(vi), t(s)
    z_m = torch.zeros(m - size, dtype=torch.int64, device=device)
    z_n = torch.zeros(n - size, dtype=torch.int64, device=device)
    # 2^(km+kn) A = ab S - 2a (S v) v^H - 2b u (u^H S) + 4 (u^H S v) u v^H with a = 2^km, b = 2^kn
    svr, svi = torch.cat([Sg * Vr[:size], z_m]), torch.cat([Sg * Vi[:size], z_m])  # S v
    tur, tui = torch.cat([Sg * Ur[:size], z_n]), torch.cat([Sg * Ui[:size], z_n])  # (u^H S)^H
    cr = int((Sg * (Ur[:size] * Vr[:size] + Ui[:size] * Vi[:size])).sum())  # u^H S v
    ci = int((Sg * (Ur[:size] * Vi[:size] - Ui[:size] * Vr[:size])).sum())
    a1, b1 = _outer_h(svr, svi, Vr, Vi)
    a2, b2 = _outer_h(Ur, Ui, tur, tui)
    a3, b3 = _outer_h(Ur, Ui, Vr, Vi)
    Mr = a1 * -(1 << (km + 1)) + a2 * -(1 << (kn + 1)) + (a3 * cr - b3 * ci) * 4
    Mi = b1 * -(1 << (km + 1)) + b2 * -(1 << (kn + 1)) + (a3 * ci + b3 * cr) * 4
    del a1, a2, a3, b1, b2, b3
    Mr.diagonal()[:size] += Sg << (km + kn)
    pm, sm = _signed_perm(m, rng, permute)
    pn, sn = _signed_perm(n, rng, permute)
    Pm, Sm, Pn, Sn = t(pm), t(sm), t(pn), t(sn)
    ss = Sm[:, None] * Sn[None, :]
    Mr = Mr[Pm][:, Pn] * ss
    Mi = Mi[Pm][:, Pn] * ss
    A = _to_float(Mr, Mi, exp - km - kn, dtype, bits, cplx)
    del Mr, Mi
    sv = Sg.to(torch.float64) * math.ldexp(1.0, exp)
    raw_u = torch.cat([sv, torch.zeros(m - size, dtype=torch.float64, device=device)])
    raw_v = torch.cat([sv, torch.zeros(n - size, dtype=torch.float64, device=device)])
    vals = torch.sort(sv, descending=True).values
    norm = float(vals.max()) if size else 0.0
    return Exact(A, vals, norm, left=_reflector_basis(ur, ui, km, pm, sm, raw_u, cplx, device),
                 right=_reflector_basis(vr, vi, kn, pn, sn, raw_v, cplx, device))


def toeplitz_121(n: int, device="cpu") -> Exact:
    """tridiag(-1, 2, -1): eigenvalues 4 sin^2(j pi / (2 (n + 1))) (mpmath, rounded once), eigenvectors
    sqrt(2 / (n + 1)) sin(i j pi / (n + 1)); the matrix itself is exact."""
    import mpmath
    with mpmath.workdps(40):
        lam = [float(4 * mpmath.sin(j * mpmath.pi / (2 * (n + 1))) ** 2) for j in range(1, n + 1)]
    A = torch.zeros((n, n), dtype=torch.float64, device=device)
    A.diagonal().fill_(2.0)
    A.diagonal(1).fill_(-1.0)
    A.diagonal(-1).fill_(-1.0)
    raw = torch.tensor(lam, dtype=torch.float64, device=device)
    idx = torch.arange(1, n + 1, device=device, dtype=torch.int64)
    nrm = math.sqrt(2.0 / (n + 1))

    def apply_h(X):
        Q = torch.empty((n, n), dtype=torch.float64, device=device)
        for r0 in range(0, n, 2048):  # (i j mod 2(n+1)) is exact; sin's argument is rounded once: |error| <= 8 u
            r = (idx[r0:r0 + 2048, None] * idx[None, :]) % (2 * (n + 1))
            Q[r0:r0 + 2048] = torch.sin(r.to(torch.float64) * (math.pi / (n + 1))) * nrm
        return Q.to(X.dtype) @ X

    # entries within 16 u of the exact ones: ||dQ||_2 <= ||dQ||_F <= 16 u sqrt(2 n); plus the product's gamma_n
    basis = Basis(apply_h, raw, 16 * U64 * math.sqrt(2 * n) + gamma(n))
    return Exact(A, torch.sort(raw).values, float(raw.max()), value_err=U64, left=basis)


def clement(n: int, device="cpu") -> Exact:
    """Symmetric Clement matrix, off-diagonals sqrt(i (n - i)) rounded once: eigenvalues -(n-1), -(n-3), ..., n-1.
    Each stored entry is within u of the exact one, so ||A_stored - A_exact||_2 <= 2 u max|a_ij| (two per row)."""
    i = torch.arange(1, n, dtype=torch.float64, device=device)
    off = torch.sqrt(i * (n - i))
    A = torch.diag(off, 1) + torch.diag(off, -1)
    vals = torch.arange(-(n - 1), n, 2, dtype=torch.float64, device=device)
    return Exact(A, vals, float(n - 1), input_err=2 * U64 * (float(off.max()) if n > 1 else 0.0))


# ---------------------------------------------------------------------------------------------------------------- check


def _max_ratio(err, bound) -> float:
    r = err / bound
    r = torch.where((err == 0) & (bound == 0), torch.zeros_like(r), r)
    r = torch.nan_to_num(r, nan=float("inf"), posinf=float("inf"))
    return float(r.max()) if r.numel() else 0.0


def _as(x, like, dtype=None):
    t = torch.as_tensor(x) if not torch.is_tensor(x) else x
    t = t.to(like.device)
    if dtype is None:
        dtype = torch.complex128 if t.is_complex() or like.is_complex() else torch.float64
    return t.to(dtype)


def _uo(u_out):
    return u_out / (1.0 - u_out) if u_out > U64 else 0.0


def _scale(ex: Exact):
    """Exact power of two that puts ||A|| in [1/2, 1)."""
    return math.ldexp(1.0, -math.frexp(ex.norm)[1]) if ex.norm > 0 else 1.0


def _clusters(v, tau):
    """Cluster ids (0, 1, ...) of ascending values v: a new cluster starts where the gap exceeds tau; also the per-cluster
    (lo, hi) ranges."""
    brk = torch.zeros_like(v, dtype=torch.int64)
    if v.numel() > 1:
        brk[1:] = (v[1:] - v[:-1] > tau).to(torch.int64)
    cid = torch.cumsum(brk, 0)
    nc = int(cid[-1]) + 1 if v.numel() else 0
    lo = torch.full((nc,), float("inf"), dtype=v.dtype, device=v.device).scatter_reduce(0, cid, v, "amin")
    hi = torch.full((nc,), -float("inf"), dtype=v.dtype, device=v.device).scatter_reduce(0, cid, v, "amax")
    return cid, lo, hi


def _cluster_of(x, lo, hi):
    """Index of the cluster [lo_c, hi_c] that holds each x (x must lie in one)."""
    c = torch.searchsorted(lo, x, right=True) - 1
    assert bool(((c >= 0) & (x <= hi[c.clamp(min=0)])).all()), "value outside every cluster"
    return c


def _delta(mu, cid_col, lo, hi):
    """Distance from mu_i to the nearest cluster other than cid_col[i]."""
    nc = lo.numel()
    up = torch.full_like(mu, float("inf"))
    dn = torch.full_like(mu, float("inf"))
    nxt = (cid_col + 1).clamp(max=nc - 1)
    prv = (cid_col - 1).clamp(min=0)
    up = torch.where(cid_col + 1 < nc, (lo[nxt] - mu).abs(), up)
    dn = torch.where(cid_col > 0, (mu - hi[prv]).abs(), dn)
    return torch.minimum(up, dn)


def _angles(basis: Basis, X, cid_row, cid_col):
    """sin of the angle between each column of X and the exact subspace of its cluster: the part of Q^H x outside the
    rows of that cluster, over ||x||."""
    Cm = basis.apply_h(X)
    Cm = torch.where(cid_row[:, None] == cid_col[None, :], torch.zeros_like(Cm), Cm)
    return torch.linalg.vector_norm(Cm, dim=0) / torch.linalg.vector_norm(X, dim=0)


def _orth(X, pu, uo, loosen):
    n = X.shape[1]
    G = X.mH @ X
    G.diagonal().sub_(1.0)
    nrm = torch.linalg.vector_norm(X, dim=0)
    bound = (pu + 2 * uo) + gamma(X.shape[0]) * nrm[:, None] * nrm[None, :]
    return _max_ratio(G.abs(), bound * loosen) if n else 0.0


def check_values(ex: Exact, vals, u_out: float = U64, N: Optional[int] = None, loosen: float = 1.0) -> float:
    """|lam^_i - lam_i| / (p u ||A|| + e_in + rounding); `vals` in the order of ex.values."""
    s = _scale(ex)
    lam = ex.values * s
    got = _as(vals, lam, torch.float64) * s
    N = N or ex.A.shape[0]
    pu = C * N * U64
    bound = pu * ex.norm * s + ex.input_err * s + _uo(u_out) * got.abs() + ex.value_err * lam.abs()
    return _max_ratio((got - lam).abs(), bound * loosen)


def check_evd(ex: Exact, lam_hat, U_hat=None, u_out: float = U64, loosen: float = 1.0) -> dict:
    """Ratios of a self-adjoint EVD (ascending values, eigenvector columns) against the exact one."""
    A = ex.A
    n = A.shape[0]
    s = _scale(ex)
    As = _as(A, A) * s
    out = {"values": check_values(ex, lam_hat, u_out, n, loosen)}
    if U_hat is None:
        return out
    lh = _as(lam_hat, As, torch.float64) * s
    X = _as(U_hat, As)
    pu, uo, nA = C * n * U64, _uo(u_out), ex.norm * s
    r = pu * nA + ex.input_err * s
    nx = torch.linalg.vector_norm(X, dim=0)
    res = torch.linalg.vector_norm(As @ X - X * lh[None, :], dim=0)
    ev = torch.linalg.vector_norm(As.abs() @ X.abs() + X.abs() * lh.abs()[None, :], dim=0)
    bound = r * nx + gamma(n + 2) * ev + uo * (nA + 2 * lh.abs()) * nx
    out["residual"] = _max_ratio(res, bound * loosen)
    out["orthogonality"] = _orth(X, pu, uo, loosen)
    if ex.left is not None:
        lam = ex.values * s
        tau = CLUSTER * (r + ex.value_err * nA)
        cid, lo, hi = _clusters(lam, tau)
        cid_row = _cluster_of(ex.left.raw * s, lo, hi)
        delta = _delta(lh, cid, lo, hi) - ex.value_err * nA
        sin = _angles(ex.left, X, cid_row, cid)
        bound = (r + uo * (nA + 2 * lh.abs())) / delta + ex.left.err + uo
        out["vectors"] = _max_ratio(sin, bound * loosen)
    return out


def check_svd(ex: Exact, S_hat, U_hat=None, V_hat=None, u_out: float = U64, loosen: float = 1.0) -> dict:
    """Ratios of an SVD (non-increasing values; thin or full U and V, either may be None) against the exact one."""
    A = ex.A
    m, n = A.shape
    size = min(m, n)
    N = m + n
    s = _scale(ex)
    As = _as(A, A) * s
    out = {"values": check_values(ex, S_hat, u_out, N, loosen)}
    if U_hat is None and V_hat is None:
        return out
    sh = _as(S_hat, As, torch.float64) * s
    pu, uo, nA = C * N * U64, _uo(u_out), ex.norm * s
    r = pu * nA + ex.input_err * s
    Xu = None if U_hat is None else _as(U_hat, As)
    Xv = None if V_hat is None else _as(V_hat, As)
    # residuals: A v_i - s_i u_i and A^H u_i - s_i v_i; past min(m, n) just A^H u_i (A v_i)
    res_parts, bnd_parts = [], []
    for X, Y, Op in ((Xv, Xu, As), (Xu, Xv, As.mH)):
        if X is None:
            continue
        k = X.shape[1]
        sv = torch.cat([sh, torch.zeros(k - size, dtype=sh.dtype, device=sh.device)])
        nx = torch.linalg.vector_norm(X, dim=0)
        R = Op @ X
        E = Op.abs() @ X.abs()
        if Y is not None:
            R[:, :size] -= Y[:, :size] * sh[None, :]
            E[:, :size] += Y[:, :size].abs() * sh[None, :]
        keep = slice(0, k) if Y is not None else slice(size, k)  # without the partner only the null-space columns
        res_parts.append(torch.linalg.vector_norm(R, dim=0)[keep])
        bnd_parts.append((r * nx + gamma(N + 2) * torch.linalg.vector_norm(E, dim=0) + uo * (nA + 2 * sv) * nx)[keep])
    out["residual"] = _max_ratio(torch.cat(res_parts), torch.cat(bnd_parts) * loosen)
    out["orthogonality"] = max(_orth(X, pu, uo, loosen) for X in (Xu, Xv) if X is not None)
    # singular subspaces: clusters over the Jordan-Wielandt spectrum +-s (and 0 when m != n)
    sig = ex.values * s
    jw = torch.cat([sig, -sig] + ([torch.zeros(1, dtype=sig.dtype, device=sig.device)] if m != n else []))
    jw = torch.sort(jw).values
    cid, lo, hi = _clusters(jw, CLUSTER * r)
    ang = []
    for X, basis in ((Xu, ex.left), (Xv, ex.right)):
        if X is None:
            continue
        k = X.shape[1]
        zero = torch.zeros(k - size, dtype=sig.dtype, device=sig.device)
        exact_col = torch.cat([sig, zero])
        mu = torch.cat([sh, zero])
        cid_col = _cluster_of(exact_col, lo, hi)
        cid_row = _cluster_of(basis.raw * s, lo, hi)
        sin = _angles(basis, X, cid_row, cid_col)
        bound = math.sqrt(2.0) * (r + uo * 2 * nA) / _delta(mu, cid_col, lo, hi) + basis.err + uo
        ang.append(_max_ratio(sin, bound * loosen))
    out["vectors"] = max(ang)
    return out


def worst(ratios: dict) -> float:
    return max(ratios.values())
