"""Rectangular test matrices with singular values that need more than 53 bits, built exactly in double-double (fx128 / cx128): the
SVD counterpart of tests/dd_spectral_exact.py's self-adjoint `build`, with the same dd unit roundoff U and bound factor P_FACTOR
(every bound p U ||A|| with p = P_FACTOR N, fixed and not tuned).

A = P_m H_m [diag(sigma); 0] H_n^H P_n^T with sigma_i = 2^s a_i + b_i >= 0 for small integers a_i, b_i, H = I - 2^(1-k) w w^H as
in `build`, and P_m, P_n signed permutations. Since 2^(k-1) H is an integer matrix, every entry of A is the exact two_sum of two
doubles and converts to dd with no rounding (asserted); the singular vectors are exact in f64.
"""
import numpy as np

from dd_spectral_exact import P_FACTOR, U, _two_sum  # noqa: F401  (P_FACTOR and U are this module's bounds too)


class DDRect:
    """hi / lo limbs of a rectangular A (m x n, complex for cx128), its exact singular values 2^s a + b (non-increasing) and
    singular vectors (exact f64, U m x min(m, n) and V n x min(m, n), column j for value j)."""

    def __init__(self, hr, lr, hi_, li_, a, b, s, U, V, cplx):
        self.hr, self.lr, self.hi_, self.li_ = hr, lr, hi_, li_
        self.a, self.b, self.s, self.U, self.V, self.cplx = a, b, s, U, V, cplx

    @property
    def shape(self):
        return self.hr.shape

    def sigma(self):
        """the exact singular values as Python ints"""
        return [(int(x) << self.s) + int(y) for x, y in zip(self.a, self.b)]

    def norm(self):
        return float(max(self.sigma(), default=0))

    def values_dd(self):
        return _two_sum(self.a.astype(np.float64) * 2.0 ** self.s, self.b.astype(np.float64))


def _int_reflector(n, rng, cplx):
    """k and w (integer real / imaginary parts, 2^k unit entries in {1, -1} or {1, i, -1, -i}) of H = I - 2^(1-k) w w^H; n = 1:
    k = 1 and w = 0 (H = I)"""
    k = int(np.floor(np.log2(n))) if n > 1 else 1
    wr = np.zeros(n, dtype=np.int64)
    wi = np.zeros(n, dtype=np.int64)
    if n > 1:
        idx = rng.permutation(n)[: 1 << k]
        ph = rng.integers(0, 4 if cplx else 2, size=idx.size)
        wr[idx] = np.where(ph == 0, 1, np.where(ph == 1, -1, 0))
        wi[idx] = np.where(ph == 2, 1, np.where(ph == 3, -1, 0))
    return k, wr, wi


def rectangular(m, n, a, b, rng, cplx=False, s=60):
    """the exact m x n matrix A = P_m H_m [diag(sigma); 0] H_n^H P_n^T with sigma_i = 2^s a_i + b_i >= 0 (int arrays of length
    min(m, n)). With M = 2^(k_m - 1) H_m and N = 2^(k_n - 1) H_n (integer matrices), A = 2^(2 - k_m - k_n) (2^s X_a + X_b) for the
    integer matrices X_x = M [diag(x); 0] N^H, formed here from the rank-one structure of M and N in O(m n); both stay below 2^53
    (asserted), so every entry of A is the exact two_sum of two doubles and converts to dd with no rounding."""
    p = min(m, n)
    a = np.asarray(a, dtype=np.int64)
    b = np.asarray(b, dtype=np.int64)
    assert a.size == p and b.size == p
    assert all((int(x) << s) + int(y) >= 0 for x, y in zip(a, b))
    km, wr, wi = _int_reflector(m, rng, cplx)
    kn, ur, ui = _int_reflector(n, rng, cplx)
    cm, cn = 1 << (km - 1), 1 << (kn - 1)

    def xint(x):
        # M S N^H = cm cn S - cm (S u) u^H - cn w (w^H S) + (w^H S u) w u^H for M = cm I - w w^H, N = cn I - u u^H
        sur, sui = np.zeros(m, dtype=np.int64), np.zeros(m, dtype=np.int64)
        sur[:p], sui[:p] = x * ur[:p], x * ui[:p]
        wsr, wsi = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
        wsr[:p], wsi[:p] = x * wr[:p], -x * wi[:p]
        tr = int(np.sum(x * (wr[:p] * ur[:p] + wi[:p] * ui[:p])))
        ti = int(np.sum(x * (wr[:p] * ui[:p] - wi[:p] * ur[:p])))
        re = np.zeros((m, n), dtype=np.int64)
        im = np.zeros((m, n), dtype=np.int64)
        re[np.arange(p), np.arange(p)] = cm * cn * x
        re -= cm * (np.outer(sur, ur) + np.outer(sui, ui))
        im -= cm * (np.outer(sui, ur) - np.outer(sur, ui))
        re -= cn * (np.outer(wr, wsr) - np.outer(wi, wsi))
        im -= cn * (np.outer(wr, wsi) + np.outer(wi, wsr))
        gr = np.outer(wr, ur) + np.outer(wi, ui)
        gi = np.outer(wi, ur) - np.outer(wr, ui)
        re += tr * gr - ti * gi
        im += tr * gi + ti * gr
        assert np.abs(re).max(initial=0) < 2 ** 53 and np.abs(im).max(initial=0) < 2 ** 53
        return re, im

    ar, ai = xint(a)
    br, bi = xint(b)
    hr, lr = _two_sum(ar.astype(np.float64) * 2.0 ** s, br.astype(np.float64))
    hi_, li_ = _two_sum(ai.astype(np.float64) * 2.0 ** s, bi.astype(np.float64))
    scale = 2.0 ** (2 - km - kn)
    hr, lr, hi_, li_ = hr * scale, lr * scale, hi_ * scale, li_ * scale
    w = wr + 1j * wi if cplx else wr.astype(np.float64)
    u = ur + 1j * ui if cplx else ur.astype(np.float64)
    # the first p columns of H_m and H_n (the full H_m of a tall input would not fit in memory)
    Hm = np.eye(m, p) - (2.0 ** (1 - km) if m > 1 else 0.0) * np.outer(w, np.conj(w[:p]))
    Hn = np.eye(n, p) - (2.0 ** (1 - kn) if n > 1 else 0.0) * np.outer(u, np.conj(u[:p]))
    # signed permutations of the rows and the columns
    pm, pn = rng.permutation(m), rng.permutation(n)
    sm, sn = rng.choice([-1.0, 1.0], size=m), rng.choice([-1.0, 1.0], size=n)
    S = sm[:, None] * sn[None, :]
    hr, lr = S * hr[np.ix_(pm, pn)], S * lr[np.ix_(pm, pn)]
    hi_, li_ = S * hi_[np.ix_(pm, pn)], S * li_[np.ix_(pm, pn)]
    U = sm[:, None] * Hm[pm, :]
    V = sn[:, None] * Hn[pn, :]
    order = sorted(range(p), key=lambda i: -((int(a[i]) << s) + int(b[i])))
    order = np.array(order, dtype=np.int64)
    return DDRect(hr, lr, hi_, li_, a[order], b[order], s, U[:, order], V[:, order], cplx)
