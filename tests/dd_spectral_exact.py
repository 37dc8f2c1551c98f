"""Self-adjoint test matrices with spectra that need more than 53 bits, built exactly in double-double (fx128 / cx128).

A = P H diag(d) H^H P^T with H = I - 2^(1-k) w w^H (w has 2^k unit entries in {1, -1} or {1, i, -1, -i}, so H is unitary and
exact in f64) and P a signed permutation. The eigenvalues are d_i = 2^60 a_i + b_i with small integers a_i, b_i: clusters such as
2^60 + j, whose relative gaps of 2^-60 f64 cannot resolve. With M = 2^(k-1) H (an integer matrix), M diag(x) M^H is an integer
matrix for x = a and for x = b, both within int64 and below 2^53, so A = 2^(2-2k) (2^60 M diag(a) M^H + M diag(b) M^H) and each
entry is the exact two_sum of two exactly representable doubles: every entry converts to dd with no rounding (asserted).

The checks follow tests/spectral_exact.py with the dd unit roundoff u = 2^-104: every bound is p u ||A|| with p = 8 N, fixed here
and not tuned to observed errors; errors are returned as error-to-bound ratios (pass: <= 1).
"""
import numpy as np

U = 2.0 ** -104
P_FACTOR = 8


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


class DDExact:
    """hi / lo limbs of A (n x n, complex for cx128), the exact eigenvalues (a, b: value 2^60 a + b, ascending) and eigenvectors
    (exact f64, column j for value j)."""

    def __init__(self, hr, lr, hi_, li_, a, b, V, cplx):
        self.hr, self.lr, self.hi_, self.li_ = hr, lr, hi_, li_
        self.a, self.b, self.V, self.cplx = a, b, V, cplx

    @property
    def n(self):
        return self.hr.shape[0]

    def norm(self):
        return float(np.max(np.abs(self.a * 2.0 ** 60 + self.b)))

    def values_dd(self):
        return _two_sum(self.a.astype(np.float64) * 2.0 ** 60, self.b.astype(np.float64))


def build(a, b, rng, cplx=False):
    """the exact matrix for eigenvalues 2^60 a + b (int arrays of length n)"""
    a = np.asarray(a, dtype=np.int64)
    b = np.asarray(b, dtype=np.int64)
    n = a.size
    k = int(np.floor(np.log2(n))) if n > 1 else 0
    c = 1 << max(k - 1, 0)
    idx = rng.permutation(n)[: 1 << k] if n > 1 else np.arange(0)
    wr = np.zeros(n, dtype=np.int64)
    wi = np.zeros(n, dtype=np.int64)
    if n > 1:
        ph = rng.integers(0, 4 if cplx else 2, size=idx.size)
        wr[idx] = np.where(ph == 0, 1, np.where(ph == 1, -1, 0))
        wi[idx] = np.where(ph == 2, 1, np.where(ph == 3, -1, 0))
    # p_ij = w_i conj(w_j)
    pr = np.outer(wr, wr) + np.outer(wi, wi)
    pi = np.outer(wi, wr) - np.outer(wr, wi)

    def mdm(x):
        s = int(np.sum(x * (wr * wr + wi * wi)))
        xs = x[:, None] + x[None, :]
        re = -c * pr * xs + s * pr
        im = -c * pi * xs + s * pi
        if n > 1:
            re[np.diag_indices(n)] += c * c * x
        else:
            re[0, 0] = x[0]
        assert np.abs(re).max() < 2 ** 53 and np.abs(im).max() < 2 ** 53
        return re, im

    ar, ai = mdm(a)
    br, bi = mdm(b)
    scale = 2.0 ** (-(2 * k - 2)) if n > 1 else 1.0
    hr, lr = _two_sum(ar.astype(np.float64) * 2.0 ** 60, br.astype(np.float64))
    hi_, li_ = _two_sum(ai.astype(np.float64) * 2.0 ** 60, bi.astype(np.float64))
    # exact: hi + lo == 2^60 A_a + A_b as integers
    for h, l, x, y in ((hr, lr, ar, br), (hi_, li_, ai, bi)):
        assert np.array_equal(np.floor(h), h) and np.array_equal(np.floor(l), l)
        hh = h.astype(object) if n <= 70 else None
        if hh is not None:
            assert all(int(p) + int(q) == (int(u) << 60) + int(v) for p, q, u, v in zip(h.ravel(), l.ravel(), x.ravel(), y.ravel()))
    hr, lr, hi_, li_ = hr * scale, lr * scale, hi_ * scale, li_ * scale
    # exact eigenvectors: H = I - 2^(1-k) w w^H
    w = wr + 1j * wi if cplx else wr.astype(np.float64)
    H = np.eye(n) - (2.0 ** (1 - k) if n > 1 else 0.0) * np.outer(w, np.conj(w))
    # signed permutation
    perm = rng.permutation(n)
    sg = rng.choice([-1.0, 1.0], size=n)
    S = sg[:, None] * sg[None, :]
    hr, lr = S * hr[np.ix_(perm, perm)], S * lr[np.ix_(perm, perm)]
    hi_, li_ = S * hi_[np.ix_(perm, perm)], S * li_[np.ix_(perm, perm)]
    V = sg[:, None] * H[perm, :]
    order = np.lexsort((b, a))
    return DDExact(hr, lr, hi_, li_, a[order], b[order], V[:, order], cplx)


def value_ratio(ex, hi, lo, N=None):
    """max |lambda_hat - lambda| / (8 N u ||A||), from exact limb differences (the limbs of both sides are exact)"""
    N = ex.n if N is None else N
    eh, el = ex.values_dd()
    err = np.abs((hi - eh) + (lo - el))
    return float(err.max() / (P_FACTOR * N * U * ex.norm())) if ex.n else 0.0


def angle_ratio(ex, Uh):
    """largest sine of the angle between the computed columns of each exact eigenvalue and its exact eigenspace, over the
    Davis-Kahan bound 8 N u ||A|| / gap (gap >= 1: integer spectrum)"""
    n = ex.n
    vals = ex.a.astype(object) * (1 << 60) + ex.b.astype(object)
    worst, i = 0.0, 0
    while i < n:
        j = i
        while j + 1 < n and vals[j + 1] == vals[i]:
            j += 1
        gap = min([abs(int(vals[i]) - int(vals[i - 1]))] if i > 0 else [10 ** 30])
        gap = min(gap, abs(int(vals[j + 1]) - int(vals[j])) if j + 1 < n else gap)
        E = ex.V[:, i:j + 1]
        X = Uh[:, i:j + 1]
        R = X - E @ (np.conj(E.T) @ X)
        s = np.linalg.norm(R, 2)
        worst = max(worst, s / (P_FACTOR * n * U * ex.norm() / float(gap)))
        i = j + 1
    return float(worst)
