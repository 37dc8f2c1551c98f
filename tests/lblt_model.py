"""numpy restatement of faer's Bunch-Kaufman LBL^H (faer/src/linalg/cholesky/bunch_kaufman/{factor,solve,reconstruct}.rs), the
model the GPU factorization is compared with. It keeps the reference's operation sequence and its quirks:

* `factor(A, strategy, block_size)`: Full -> the full-pivoting path; the other strategies -> the blocked path (left-looking steps
  of at most bs - 1 columns while more than bs columns remain, one product A22(strict lower) -= W Al^H per step, the unblocked
  right-looking path on the rest). bs is 0 when bs < 2 or n <= bs.
* A column whose candidate off-diagonal maximum is 0 (and the last column of the non-Full paths) is "nothing to do": no scaling,
  no update, and subdiag[k] is not written.
* Full scales the whole matrix (strict upper triangle included) by 1 / norm_max and restores only diag and subdiag.

Every pivot decision records the relative margin of each comparison it made (|lhs - rhs| / max(|lhs|, |rhs|)); a GPU result is
compared exactly with the model's pivots when the smallest margin is well above rounding."""
import numpy as np

PARTIAL, PARTIAL_DIAG, ROOK, ROOK_DIAG, FULL = range(5)
TOP_BIT = 1 << 63


def _abs1(x):
    return np.abs(np.real(x)) + np.abs(np.imag(x))


def _abs2(x):
    return np.real(x) ** 2 + np.imag(x) ** 2


def _first_max(v):
    """l1_argmax: first maximum with strict `>` from 0 (None for an empty vector)."""
    if len(v) == 0:
        return None, 0.0
    v = np.where(np.isnan(v), 0.0, v)  # NaN is never > best
    i = int(np.argmax(v))  # the first occurrence of the maximum
    return (i, v[i]) if v[i] > 0 else (0, 0.0)


def _margin(a, b):
    a, b = float(a), float(b)
    d = max(abs(a), abs(b))
    return abs(a - b) / d if d > 0 else np.inf


class _Rec:
    def __init__(self):
        self.margins = []

    def cmp(self, a, b):
        self.margins.append(_margin(a, b))
        return a >= b


def _swap_self_adjoint(A, i, j):
    """factor.rs:37-53 on the square view A."""
    i, j = min(i, j), max(i, j)
    A[j + 1:, [i, j]] = A[j + 1:, [j, i]]
    A[[i, j], :i] = A[[j, i], :i]
    aii = np.real(A[i, i])
    A[i, i] = np.real(A[j, j])
    A[j, j] = aii
    A[j, i] = np.conj(A[j, i])
    x = A[i + 1:j, i].copy()
    y = A[j, i + 1:j].copy()
    A[i + 1:j, i] = np.conj(y)
    A[j, i + 1:j] = np.conj(x)


def _two_by_two(a00, a11, a10):
    d10 = np.abs(a10)
    d10_inv = 1.0 / d10
    d00 = a00 * d10_inv
    d11 = a11 * d10_inv
    t = 1.0 / (d00 * d11 - 1.0)
    d10 = a10 * d10_inv
    d = t * d10_inv
    return d, d00, d11, d10


def _w(x0, x1, d, d00, d11, d10):
    return (x0 * d11 - x1 * d10) * d, (x1 * d00 - x0 * np.conj(d10)) * d


def _offdiag_argmax(A, idx):
    ca, cm = _first_max(_abs1(A[idx + 1:, idx]))
    if ca is not None:
        ca += idx + 1
    ra, rm = _first_max(_abs1(A[idx, :idx]))
    return (ca, cm) if cm > rm else (ra, rm)


def _decide(alpha, diag_re, diag_abs1, col, i0, gamma_i, r, rook, last, blocked, rec, move=lambda: None):
    """The shared decision logic; col(x) -> (argmax, gamma) of candidate column x; move() is called whenever i0 takes the
    candidate's place (the blocked step copies W's second column into the first). Returns (npiv, i0, i1, nothing)."""
    if last or gamma_i == 0:
        return 1, i0, None, True
    if rec.cmp(abs(diag_re(i0)), alpha * gamma_i):
        return 1, i0, None, False
    i1 = r
    if rook:
        while True:
            s, gamma_r = col(i1)
            if rec.cmp(diag_abs1(i1), alpha * gamma_r):
                move()
                return 1, i1, None, False
            if (blocked and s == i0) or gamma_i == gamma_r:
                return 2, i0, i1, False
            move()
            i0, i1, gamma_i = i1, s, gamma_r
    _, gamma_r = col(i1)
    if rec.cmp(abs(diag_re(i0)), (alpha * gamma_r) * (gamma_r / gamma_i)):
        return 1, i0, None, False
    if rec.cmp(abs(diag_re(i1)), alpha * gamma_r):
        move()
        return 1, i1, None, False
    return 2, i0, i1, False


def _unblocked(alpha, A, sub, piv, off, rook, diagonal, rec):
    """lblt_unblocked (factor.rs:784-902) on the trailing view A (its columns are the region's), pivots offset by `off`."""
    n = A.shape[0]
    k = 0
    while k < n:
        T = A[k:, k:]
        i0 = _first_max(_abs1(np.diagonal(T)))[0] if diagonal else 0
        r, gamma_i = _offdiag_argmax(T, i0)
        npiv, i0, i1, nothing = _decide(alpha, lambda x: np.real(T[x, x]), lambda x: _abs1(T[x, x]),
                                        lambda x: _offdiag_argmax(T, x), i0, gamma_i, r, rook, k + 1 == n, False, rec)
        if npiv == 2 and i0 > i1:
            i0, i1 = i1, i0
        if i0 != 0:
            _swap_self_adjoint(T, 0, i0)
            A[[k, k + i0], :k] = A[[k + i0, k], :k]
        if npiv == 2 and i1 != 1:
            _swap_self_adjoint(T, 1, i1)
            A[[k + 1, k + i1], :k] = A[[k + i1, k + 1], :k]
        if not nothing:
            if npiv == 1:
                dg = np.real(T[0, 0])
                sub[off + k] = 0
                L = T[1:, 0].copy()
                w = L * (1.0 / dg)
                S = T[1:, 1:]
                S -= np.tril(np.outer(L, np.conj(w)))
                np.fill_diagonal(S, np.real(np.diagonal(S)))
                T[1:, 0] = w
            else:
                a00, a11, a10 = np.real(T[0, 0]), np.real(T[1, 1]), T[1, 0]
                sub[off + k] = a10
                sub[off + k + 1] = 0
                T[1, 0] = 0
                d, d00, d11, d10 = _two_by_two(a00, a11, a10)
                L0, L1 = T[2:, 0].copy(), T[2:, 1].copy()
                w0, w1 = _w(L0, L1, d, d00, d11, d10)
                S = T[2:, 2:]
                S -= np.tril(np.outer(L0, np.conj(w0)) + np.outer(L1, np.conj(w1)))
                np.fill_diagonal(S, np.real(np.diagonal(S)))
                T[2:, 0], T[2:, 1] = w0, w1
        piv[off + k] = off + k + i0
        if npiv == 2:
            piv[off + k] |= TOP_BIT
            piv[off + k + 1] = (off + k + i1) | TOP_BIT
        k += npiv


def _blocked_step(alpha, A, sub, piv, off, bs, rook, diagonal, rec):
    """lblt_blocked_step (factor.rs:491-699) on the trailing view A (m x m); returns the number of columns done."""
    m = A.shape[0]
    W = np.zeros((m, bs), dtype=A.dtype)
    kmax = min(bs - 1, m)
    k = 0

    def build(k, x, wc):
        Ar, Al, Wl = A[k:, k:], A[k:, :k], W[k:, :k]
        dst = np.concatenate([np.conj(Ar[x, :x]), [0], Ar[x + 1:, x]]).astype(A.dtype)
        dst = dst - Al @ np.conj(Wl[x, :])
        dst[x] = 0
        r, g = _first_max(_abs1(dst))
        dst[x] = np.real(Ar[x, x])
        W[k:, wc] = dst
        return (None, 0.0) if len(dst) == 1 else (r, g)

    while k < kmax:
        Ar = A[k:, k:]
        i0 = _first_max(_abs1(np.diagonal(Ar)))[0] if diagonal else 0
        r, gamma_i = build(k, i0, k)

        def move():
            W[k:, k] = W[k:, k + 1]

        npiv, i0, i1, nothing = _decide(alpha, lambda x: np.real(Ar[x, x]), lambda x: _abs1(Ar[x, x]),
                                        lambda x: build(k, x, k + 1), i0, gamma_i, r, rook, k + 1 == m, True, rec, move)
        if npiv == 2 and i0 > i1:
            W[:, [k, k + 1]] = W[:, [k + 1, k]]
            i0, i1 = i1, i0
        if i0 != 0:
            _swap_self_adjoint(Ar, 0, i0)
            A[[k, k + i0], :k] = A[[k + i0, k], :k]
            W[[k, k + i0], :k + npiv] = W[[k + i0, k], :k + npiv]
        if npiv == 2 and i1 != 1:
            _swap_self_adjoint(Ar, 1, i1)
            A[[k + 1, k + i1], :k] = A[[k + i1, k + 1], :k]
            W[[k + 1, k + i1], :k + 2] = W[[k + i1, k + 1], :k + 2]
        if not nothing:
            if npiv == 1:
                dg = np.real(W[k, k])
                sub[off + k] = 0
                L = W[k + 1:, k] * (1.0 / dg)
                Ar[1:, 0] = L
                idx = np.arange(1, m - k)
                Ar[idx, idx] = np.real(Ar[idx, idx]) - dg * _abs2(L)
            else:
                a00, a11, a10 = np.real(W[k, k]), np.real(W[k + 1, k + 1]), W[k + 1, k]
                sub[off + k] = a10
                sub[off + k + 1] = 0
                W[k + 1, k] = 0
                Ar[1, 0] = 0
                d, d00, d11, d10 = _two_by_two(a00, a11, a10)
                W0, W1 = W[k + 2:, k], W[k + 2:, k + 1]
                w0, w1 = _w(W0, W1, d, d00, d11, d10)
                idx = np.arange(2, m - k)
                Ar[idx, idx] = np.real(Ar[idx, idx] - W0 * np.conj(w0) - W1 * np.conj(w1))
                Ar[2:, 0], Ar[2:, 1] = w0, w1
        piv[off + k] = off + k + i0
        if npiv == 2:
            piv[off + k] |= TOP_BIT
            piv[off + k + 1] = (off + k + i1) | TOP_BIT
        k += npiv
    Ar = A[k:, k:]
    Ar -= np.tril(W[k:, :k] @ np.conj(A[k:, :k]).T, -1)
    np.fill_diagonal(Ar, np.real(np.diagonal(Ar)))
    return k


def _full(A, sub, piv, rec):
    """lblt_full_piv (factor.rs:264-429), the Seq rule for the off-diagonal maximum (column-major first maximum)."""
    alpha = ((1.0 + np.sqrt(17.0)) * 0.125) ** 2
    n = A.shape[0]
    scale_fwd = np.max(np.maximum(np.abs(np.real(A)), np.abs(np.imag(A)))) if n else np.float64(0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        A *= np.float64(1.0) / scale_fwd  # a zero matrix becomes NaN, as in the reference

    def offmax(T):
        """the first maximum of abs2 over the strict lower triangle in column-major order, strict `>` from 0"""
        m = T.shape[0]
        v = np.tril(_abs2(T), -1)
        e, best = _first_max(v.ravel(order="F"))
        return (e % m, e // m, best) if best > 0 else (0, 0, 0.0)

    mi, mj, mo = offmax(A)
    k = 0
    while k < n:
        if mo == 0:
            break
        T = A[k:, k:]
        ms, md = _first_max(_abs2(np.diagonal(T)))
        if rec.cmp(md, alpha * mo):
            npiv, i0, i1 = 1, ms, None
        else:
            npiv, i0, i1 = 2, mj, mi
        if i0 != 0:
            _swap_self_adjoint(T, 0, i0)
            A[[k, k + i0], :k] = A[[k + i0, k], :k]
        if npiv == 2 and i1 != 1:
            _swap_self_adjoint(T, 1, i1)
            A[[k + 1, k + i1], :k] = A[[k + i1, k + 1], :k]
        if npiv == 1:
            dg = np.real(T[0, 0])
            sub[k] = 0
            L = T[1:, 0] * (1.0 / dg)
            T[1:, 0] = L
            S = T[1:, 1:]
            idx = np.arange(S.shape[0])
            S[idx, idx] = np.real(S[idx, idx]) - dg * _abs2(L)
            if S.shape[0]:
                S -= np.tril(np.outer(L, np.conj(L)) * dg, -1)
                mi, mj, mo = offmax(S)
        else:
            a00, a11, a10 = np.real(T[0, 0]), np.real(T[1, 1]), T[1, 0]
            sub[k] = a10
            sub[k + 1] = 0
            T[1, 0] = 0
            d, d00, d11, d10 = _two_by_two(a00, a11, a10)
            L0, L1 = T[2:, 0].copy(), T[2:, 1].copy()
            w0, w1 = _w(L0, L1, d, d00, d11, d10)
            S = T[2:, 2:]
            if S.shape[0]:
                S -= np.tril(np.outer(L0, np.conj(w0)) + np.outer(L1, np.conj(w1)), -1)
                mi, mj, mo = offmax(S)
            idx = np.arange(S.shape[0])
            S[idx, idx] = np.real(S[idx, idx] - L0 * np.conj(w0) - L1 * np.conj(w1))
            T[2:, 0], T[2:, 1] = w0, w1
        piv[k] = k + i0
        if npiv == 2:
            piv[k] |= TOP_BIT
            piv[k + 1] = (k + i1) | TOP_BIT
        k += npiv
    while k < n:
        T = A[k:, k:]
        ms, _ = _first_max(_abs2(np.diagonal(T)))
        if ms != 0:
            T[0, 0], T[ms, ms] = T[ms, ms], T[0, 0]
            A[[k, k + ms], :k] = A[[k + ms, k], :k]
        sub[k] = 0
        piv[k] = k + ms
        k += 1
    idx = np.arange(n)
    A[idx, idx] *= scale_fwd
    sub *= scale_fwd


def factor(A, sub, strategy=PARTIAL_DIAG, block_size=64):
    """cholesky_in_place on copies: returns (A, subdiag, perm_fwd, perm_bwd, transposition_count, margins)."""
    A = np.array(A, copy=True)
    sub = np.array(sub, copy=True)
    n = A.shape[0]
    piv = [0] * n
    rec = _Rec()
    alpha = (1.0 + np.sqrt(17.0)) * 0.125
    if A.dtype in (np.float32, np.complex64):
        alpha = np.float32(alpha)
    if strategy == FULL:
        _full(A, sub, piv, rec)
    else:
        rook, diagonal = strategy in (ROOK, ROOK_DIAG), strategy in (PARTIAL_DIAG, ROOK_DIAG)
        bs = block_size if (block_size >= 2 and n > block_size) else 0
        k = 0
        while k < n:
            if bs < 2 or n - k <= bs:
                _unblocked(alpha, A[k:, k:], sub, piv, k, rook, diagonal, rec)
                # the region's own left columns were swapped inside; columns 0..k here
                nxt = n
            else:
                nxt = k + _blocked_step(alpha, A[k:, k:], sub, piv, k, bs, rook, diagonal, rec)
            for i in range(k, nxt):
                j = piv[i] & ~TOP_BIT
                A[[i, j], :k] = A[[j, i], :k]
            k = nxt
    perm = np.arange(n)
    count = 0
    for i in range(n):
        p = piv[i] & ~TOP_BIT
        if p != i:
            count += 1
        perm[i], perm[p] = perm[p], perm[i]
    inv = np.empty(n, dtype=np.int64)
    inv[perm] = np.arange(n)
    return A, sub, perm, inv, count, rec.margins


def _kinds(sub):
    n = len(sub)
    kind = np.zeros(n, dtype=int)
    i = 0
    while i < n:
        if sub[i] == 0:
            i += 1
        else:
            kind[i], kind[i + 1] = 1, 2
            i += 2
    return kind


def solve(LB, sub, perm, perm_inv, rhs, conj=False, diag=None):
    """solve.rs:35-104."""
    n = LB.shape[0]
    d = np.real(np.diagonal(LB) if diag is None else diag)
    L = np.tril(LB, -1) + np.eye(n)
    if conj:
        L = np.conj(L)
    x = rhs[perm].astype(LB.dtype)
    x = np.linalg.solve(L, x) if n else x
    kind = _kinds(sub)
    i = 0
    while i < n:
        if kind[i] == 0:
            x[i] *= 1.0 / d[i]
            i += 1
        else:
            s = sub[i]
            if conj:
                s = np.conj(s)
            rk = 1.0 / s
            ak, akp1 = np.conj(rk) * d[i], rk * d[i + 1]
            denom = 1.0 / (np.real(ak * akp1) - 1.0)
            xk, xkp1 = x[i] * np.conj(rk), x[i + 1] * rk
            x[i], x[i + 1] = (akp1 * xk - xkp1) * denom, (ak * xkp1 - xk) * denom
            i += 2
    x = np.linalg.solve(np.conj(L).T, x) if n else x
    return x[perm_inv]


def reconstruct(LB, sub, perm_inv):
    """reconstruct.rs:12-87: all of `out` (lower triangle: A; strict upper triangle: the intermediate L B)."""
    n = LB.shape[0]
    out = np.tril(LB, -1) + np.eye(n, dtype=LB.dtype)
    kind = _kinds(sub)
    j = 0
    while j < n:
        if kind[j] == 0:
            out[:, j] *= np.real(LB[j, j])
            j += 1
        else:
            s, ak, akp1 = sub[j], np.real(LB[j, j]), np.real(LB[j + 1, j + 1])
            xk, xkp1 = out[:, j].copy(), out[:, j + 1].copy()
            out[:, j], out[:, j + 1] = xk * ak + xkp1 * s, xkp1 * akp1 + xk * np.conj(s)
            j += 2
    L = np.tril(LB, -1) + np.eye(n)
    tmp = L @ np.conj(out).T
    for jj in range(n):
        pj = perm_inv[jj]
        for ii in range(jj, n):
            pi = perm_inv[ii]
            out[ii, jj] = tmp[pi, pj] if pi >= pj else np.conj(tmp[pj, pi])
    idx = np.arange(n)
    out[idx, idx] = np.real(out[idx, idx])
    return out
