"""An independent double-double model in numpy (test infrastructure), a second implementation beside csrc/dd.cuh: the product's
error term comes from Dekker's split instead of an FMA, and every operation works on whole arrays. A value is a pair (hi, lo) of
float64 arrays; a complex value a pair of such pairs. Used by the GPU tests as the reference for products, solves and
factorizations too large for exact rational arithmetic, and checked itself against mpmath and exact fractions
(tests/test_dd_model_cpu.py)."""
import numpy as np

_SPLIT = 134217729.0  # 2^27 + 1


def _two_sum(a, b):
    s = a + b
    v = s - a
    return s, (a - (s - v)) + (b - v)


def _split(a):
    t = _SPLIT * a
    hi = t - (t - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _fast(s, e):
    h = s + e
    return h, e - (h - s)


def add(x, y):
    s, e = _two_sum(x[0], y[0])
    return _fast(s, e + (x[1] + y[1]))


def neg(x):
    return (-x[0], -x[1])


def mul(x, y):
    p, e = _two_prod(x[0], y[0])
    return _fast(p, e + (x[0] * y[1] + x[1] * y[0]))


def div(x, y):
    q1 = x[0] / y[0]
    r = mul(y, (q1, np.zeros_like(q1)))
    s, e = _two_sum(x[0], -r[0])
    e = e - r[1] + x[1]
    return _fast(q1, (s + e) / y[0])


def absv(x):
    m = x[0] < 0
    return (np.where(m, -x[0], x[0]), np.where(m, -x[1], x[1]))


def gt(x, y):
    return (x[0] > y[0]) | ((x[0] == y[0]) & (x[1] > y[1]))


def sqrt(x):
    with np.errstate(all="ignore"):
        r = 1.0 / np.sqrt(x[0])
        a = x[0] * r
        sq = mul((a, 0 * a), (a, 0 * a))
        # one Newton step: a + (x - a^2) * r / 2, with the difference kept to both limbs
        d1, d2 = _two_sum(x[0], -sq[0])
        t1, t2 = _two_sum(x[1], -sq[1])
        d2 = d2 + t1
        d1, d2 = _fast(d1, d2)
        d1, d2 = _fast(d1, d2 + t2)
        c = mul((d1, d2), (r * 0.5, 0 * r))
        return add((a, 0 * a), c)


def zeros(shape):
    return (np.zeros(shape), np.zeros(shape))


def from_fields(a):
    """structured FX128 / CX128 array -> dd pair, or pair of dd pairs"""
    if "hi" in a.dtype.names:
        return (np.array(a["hi"], dtype=np.float64), np.array(a["lo"], dtype=np.float64))
    return ((np.array(a["re_hi"], dtype=np.float64), np.array(a["re_lo"], dtype=np.float64)),
            (np.array(a["im_hi"], dtype=np.float64), np.array(a["im_lo"], dtype=np.float64)))


def cmul(x, y):
    return (add(mul(x[0], y[0]), neg(mul(x[1], y[1]))), add(mul(x[0], y[1]), mul(x[1], y[0])))


def cadd(x, y):
    return (add(x[0], y[0]), add(x[1], y[1]))


def _idx(x, key, cx):
    return ((x[0][0][key], x[0][1][key]), (x[1][0][key], x[1][1][key])) if cx else (x[0][key], x[1][key])


def matmul(A, B, cx):
    """A (m x k) B (k x n) with one dd mul_add per term, in k order"""
    a0 = A[0][0] if cx else A[0]
    m, k = a0.shape
    n = (B[0][0] if cx else B[0]).shape[1]
    acc = (zeros((m, n)), zeros((m, n))) if cx else zeros((m, n))
    for t in range(k):
        a = _idx(A, (slice(None), slice(t, t + 1)), cx)
        b = _idx(B, (slice(t, t + 1), slice(None)), cx)
        acc = cadd(cmul(a, b), acc) if cx else add(mul(a, b), acc)
    return acc


def approx(x, cx):
    return (x[0][0] + x[0][1]) + 1j * (x[1][0] + x[1][1]) if cx else x[0] + x[1]


def lu(A):
    """unblocked real partial-pivoting LU in dd (first row with the largest |a|); returns (L U packed, perm_fwd, transpositions)"""
    h, l = A[0].copy(), A[1].copy()
    m, n = h.shape
    perm = np.arange(m)
    nt = 0
    for j in range(min(m, n)):
        ah = np.abs(h[j:, j])
        al = np.where(h[j:, j] < 0, -l[j:, j], l[j:, j])
        # first maximum: the smallest index among the largest (hi, lo), none unless it is > 0
        mhi = ah.max()
        mlo = al[ah == mhi].max()
        best = j
        if mhi > 0 or (mhi == 0 and mlo > 0):
            best = j + int(np.nonzero((ah == mhi) & (al == mlo))[0][0])
        if best != j:
            h[[j, best]], l[[j, best]] = h[[best, j]], l[[best, j]]
            perm[[j, best]] = perm[[best, j]]
            nt += 1
        inv = div((np.ones(1), np.zeros(1)), (h[j:j + 1, j], l[j:j + 1, j]))
        col = mul((h[j + 1:, j], l[j + 1:, j]), inv)
        h[j + 1:, j], l[j + 1:, j] = col
        prod = mul((h[j + 1:, j:j + 1], l[j + 1:, j:j + 1]), (h[j:j + 1, j + 1:], l[j:j + 1, j + 1:]))
        h[j + 1:, j + 1:], l[j + 1:, j + 1:] = add((h[j + 1:, j + 1:], l[j + 1:, j + 1:]), neg(prod))
    return (h, l), perm, nt
