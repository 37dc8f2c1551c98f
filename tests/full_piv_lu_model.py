"""numpy restatement of faer's full-pivoting LU (faer/src/linalg/lu/full_pivoting): the factorization (factor.rs:321-538, both
branches of `lu_in_place`, the scalar search `best_in_matrix_fallback` and its tie rule, the `min_positive` exit), the solves
(solve.rs:21-93), `reconstruct` (reconstruct.rs:13-82) and `inverse` (inverse.rs:12-63).

The working precision is the array's dtype; np.longdouble / np.clongdouble inputs give the "wider" run the GPU tests use to show
that a pivot sequence is not decided by rounding."""
import numpy as np


def min_positive(dtype) -> float:
    dt = np.dtype(dtype)
    real = np.empty(0, dt).real.dtype
    return np.finfo(real).tiny


def abs1(x):
    return np.abs(x.real) + np.abs(x.imag) if np.iscomplexobj(x) else np.abs(x)


def best_in_matrix(X):
    """(row, col, score): the first maximum of abs1 in X's column-major order, strict `>` from 0 (factor.rs:255-273)."""
    m, n = X.shape
    if m == 0 or n == 0:
        return 0, 0, abs1(np.zeros(1, X.dtype))[0]
    s = abs1(X)
    flat = s.T.reshape(-1)  # column-major order
    with np.errstate(invalid="ignore"):
        keep = np.where(np.isnan(flat), 0, flat)
    idx = int(np.argmax(keep))  # the first occurrence of the maximum
    best = keep[idx]
    if not best > 0:
        return 0, 0, best * 0
    return idx % m, idx // m, best


def _cx(dtype, re, im):
    out = np.empty(1, dtype)
    out.real = re
    out.imag = im
    return out[0]


def recip(x):
    """ComplexField::recip: 1 / x for real scalars, faer-traits' recip_impl for complex ones (faer-traits/src/lib.rs:353-383)."""
    if not np.iscomplexobj(x):
        return x.dtype.type(1) / x
    re, im = x.real, x.imag
    R = type(re)
    if np.isnan(re) or np.isnan(im):
        return _cx(x.dtype, np.nan, np.nan)
    if re == 0 and im == 0:
        return _cx(x.dtype, np.inf, np.inf)
    if not (np.isfinite(re) and np.isfinite(im)):
        return x.dtype.type(0)
    tiny = np.finfo(R).tiny
    sml, big = R(np.sqrt(tiny)), R(np.sqrt(R(1) / tiny))
    if abs(re) > big or abs(im) > big:
        a, b = re * sml, im * sml
        inv = R(1) / (a * a + b * b)
        return _cx(x.dtype, (a * inv) * sml, (-b * inv) * sml)
    if abs(re) > 1 or abs(im) > 1:
        inv = R(1) / (re * re + im * im)
        return _cx(x.dtype, re * inv, -im * inv)
    a, b = re * big, im * big
    inv = R(1) / (a * a + b * b)
    return _cx(x.dtype, (a * inv) * big, (-b * inv) * big)


def lu_in_place_unblocked(X, transpose: bool):
    """factor.rs:321-432 on the working matrix X (modified in place). Returns (row_trans, col_trans, n_trans) of X."""
    m, n = X.shape
    size = min(m, n)
    row_t = list(range(size))
    col_t = list(range(size))
    n_trans = 0
    if m == 0 or n == 0:
        return row_t, col_t, 0
    tiny = min_positive(X.dtype)
    r, c, s = best_in_matrix(X)
    for k in range(size):
        if not s >= tiny:
            for t in range(k, size):
                row_t[t] = t
                col_t[t] = t
            break
        row_t[k], col_t[k] = r, c
        if r != k:
            X[[k, r], :] = X[[r, k], :]
            n_trans += 1
        if c != k:
            X[:, [k, c]] = X[:, [c, k]]
            n_trans += 1
        inv = recip(X[k, k])
        if transpose:
            X[k, k + 1:] *= inv
        else:
            X[k + 1:, k] *= inv
        if k + 1 == size:
            break
        with np.errstate(invalid="ignore", over="ignore"):
            X[k + 1:, k + 1:] -= np.outer(X[k + 1:, k], X[k, k + 1:])
        r, c, s = best_in_matrix(X[k + 1:, k + 1:])
        r += k + 1
        c += k + 1
    return row_t, col_t, n_trans


def _perm(length, trans):
    fwd = np.arange(length, dtype=np.int64)
    for i, t in enumerate(trans):
        fwd[i], fwd[t] = fwd[t], fwd[i]
    bwd = np.empty(length, dtype=np.int64)
    bwd[fwd] = np.arange(length, dtype=np.int64)
    return fwd, bwd


def lu_in_place(A, row_major: bool = False):
    """factor.rs:466-538. A (modified in place) is seen with the strides of a column-major array, or of a row-major one with
    `row_major` (the transposed branch: |row_stride| >= |col_stride|; a 1 x n or m x 1 column-major numpy array takes that branch
    too when its strides are equal, which callers pass as row_major=True). Returns (row_fwd, row_bwd, col_fwd, col_bwd, count)."""
    m, n = A.shape
    if not row_major:
        rt, ct, cnt = lu_in_place_unblocked(A, False)
    else:
        XT = A.T.copy()
        ct, rt, cnt = lu_in_place_unblocked(XT, True)
        A[...] = XT.T
    rf, rb = _perm(m, rt)
    cf, cb = _perm(n, ct)
    return rf, rb, cf, cb, cnt


def takes_transposed_branch(rs: int, cs: int) -> bool:
    """factor.rs:492: the transposed branch unless |row_stride| < |col_stride|."""
    return not abs(rs) < abs(cs)


def split(LU):
    """(L, U) of the packed factor: L unit-lower m x size, U upper size x n."""
    m, n = LU.shape
    size = min(m, n)
    L = np.tril(LU[:, :size], -1)
    L[np.arange(size), np.arange(size)] = 1
    U = np.triu(LU[:size, :])
    return L, U


def solve(L, U, rf, rb, cf, cb, rhs, conj=False):
    """solve.rs:21-56: rhs <- (conj A)^-1 rhs."""
    Lc, Uc = (np.conj(L), np.conj(U)) if conj else (L, U)
    x = rhs[rf]
    x = np.linalg.solve(Lc, x)
    x = np.linalg.solve(Uc, x)
    return x[cb]


def solve_transpose(L, U, rf, rb, cf, cb, rhs, conj=False):
    """solve.rs:58-93: rhs <- (conj A)^-T rhs."""
    Lc, Uc = (np.conj(L), np.conj(U)) if conj else (L, U)
    x = rhs[cf]
    x = np.linalg.solve(Uc.T, x)
    x = np.linalg.solve(Lc.T, x)
    return x[rb]


def reconstruct(L, U, rb, cb):
    """reconstruct.rs:13-82: out[i, j] = (L U)[row_bwd[i], col_bwd[j]]."""
    return (L @ U)[np.ix_(rb, cb)]


def inverse(L, U, rb, cb):
    """inverse.rs:12-63: tmp = U^-1 L^-1, out[i, j] = tmp[col_bwd[i], row_bwd[j]]."""
    n = L.shape[0]
    tmp = np.linalg.solve(U, np.linalg.solve(L, np.eye(n, dtype=L.dtype)))
    return tmp[np.ix_(cb, rb)]
