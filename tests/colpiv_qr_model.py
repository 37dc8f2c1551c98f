"""numpy restatement of faer's column-pivoted QR (faer/src/linalg/qr/col_pivoting/factor.rs:112-388) and of the compositions on
its factors (solve.rs:52-184, reconstruct.rs:16-45, inverse.rs:16-50). The GPU factorization (csrc/colpiv_qr.cu) is checked
against it; tests/test_oracle_colpiv_qr_cpu.py pins it to the reference's own tests and to LAPACK ?geqp3.

factor(A, bs, row_stride_one) -> (QR, Q_coeff, perm_fwd, perm_bwd, transposition_count), in the working precision of A."""
import numpy as np


def _norm(x):
    return np.sqrt(np.sum(np.abs(x) ** 2)) if x.size else x.real.dtype.type(0)


def make_householder(head, tail):
    """householder.rs:59-107 (make_householder_imp): returns (tau, new head, scaled tail)."""
    rt = tail.real.dtype.type
    tiny = np.finfo(tail.real.dtype).tiny
    tail_norm = _norm(tail)
    head_norm = abs(head)
    if head_norm < tiny:
        head = head * 0
        head_norm = rt(0)
    if tail_norm < tiny:
        return rt(np.inf), head, tail
    nrm = np.hypot(head_norm, tail_norm)
    sign = head / head_norm if head_norm != 0 else head.dtype.type(1)
    signed_norm = sign * nrm
    inv = 1 / (head + signed_norm)
    tau = rt(0.5) * (1 + (tail_norm * abs(inv)) ** 2)
    return tau, -signed_norm, tail * inv


def factor_unblocked(A, row_stride_one=True):
    """qr_in_place_unblocked (factor.rs:112-320): A is overwritten; returns (taus, perm_fwd, count)."""
    m, n = A.shape
    size = min(m, n)
    rt = A.real.dtype.type
    perm = np.arange(n)
    n_trans = 0
    tau = np.zeros(size, dtype=A.real.dtype)
    if size == 0:
        return tau, perm, 0
    dot = np.zeros(n, dtype=A.dtype)
    norm = np.array([_norm(A[:, j]) for j in range(n)], dtype=A.real.dtype)
    best = rt(0)
    for j in range(n):
        if norm[j] > best:
            best = norm[j]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        scale_fwd = best
        scale_bwd = rt(1) / best
        A *= scale_bwd
        norm = norm * scale_bwd
        best = best * scale_bwd
        threshold = np.sqrt(np.finfo(A.real.dtype).eps)
        best_threshold = best * threshold
        for k in range(size):
            new_best, best_col = rt(0), k
            for j in range(k, n):
                if norm[j] > new_best:
                    new_best, best_col = norm[j], j
            delayed = row_stride_one and k > 0 and new_best >= best_threshold
            if k > 0 and not delayed:
                A[k:, k:] += np.outer(A[k:, k - 1], dot[k:])
                best = rt(0)
                for j in range(k, n):
                    val = _norm(A[k:, j])
                    norm[j] = val
                    if val > best:
                        best, best_col = val, j
                best_threshold = best * threshold
            if best_col != k:
                n_trans += 1
                for arr in (perm, dot, norm):
                    arr[[k, best_col]] = arr[[best_col, k]]
                A[:, [k, best_col]] = A[:, [best_col, k]]
            l = A[k, k - 1] if delayed else A.dtype.type(0)
            r = dot[k]
            if delayed:
                A[k, k] += l * r
                A[k + 1:, k] += r * A[k + 1:, k - 1]
            t, head, tail = make_householder(A[k, k], A[k + 1:, k])
            A[k, k] = head
            A[k + 1:, k] = tail
            tau[k] = t
            tau_inv = rt(1) / t
            if k + 1 == size:
                if delayed:
                    A[k, k + 1:] += l * dot[k + 1:]
                break
            v = A[k + 1:, k]
            if delayed:
                A[k + 1:, k + 1:] += np.outer(A[k + 1:, k - 1], dot[k + 1:])
                tmp = A[k, k + 1:] + l * dot[k + 1:]
                d0 = -(tmp + v.conj() @ A[k + 1:, k + 1:]) * tau_inv
                A[k, k + 1:] = tmp + d0
            else:
                d0 = -(A[k, k + 1:] + v.conj() @ A[k + 1:, k + 1:]) * tau_inv
                A[k, k + 1:] += d0
            dot[k + 1:] = d0
            norm[k + 1:] = np.sqrt(norm[k + 1:] ** 2 - np.abs(A[k, k + 1:]) ** 2)
        iu = np.triu_indices(m, 0, n)
        A[iu] *= scale_fwd
    return tau, perm, n_trans


def t_blocks(QR, tau, bs):
    """factor.rs:367-386 with upgrade_householder_factor: Q_coeff (bs x size), T = striu(V^H V) + diag(tau) per block."""
    m, n = QR.shape
    size = min(m, n)
    H = np.zeros((bs, size), dtype=QR.dtype)
    H[0, :] = tau
    for j in range(0, size, bs):
        b = min(bs, size - j)
        V = np.tril(QR[j:, j:j + b], -1)
        V[np.arange(b), np.arange(b)] = 1
        T = np.triu(V.conj().T @ V, 1)
        T[np.arange(b), np.arange(b)] = tau[j:j + b]
        H[:b, j:j + b] = T
        H[0, j:j + b] = T[0, :]
    return H


def factor(A, bs, row_stride_one=True):
    QR = np.array(A, copy=True)
    tau, perm, count = factor_unblocked(QR, row_stride_one)
    H = t_blocks(QR, tau, bs) if min(QR.shape) > 0 else np.zeros((bs, 0), dtype=QR.dtype)
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    return QR, H, perm, inv, count


def q_matrix(QR, tau):
    """Q = H_0 H_1 ... H_{size-1}, m x m."""
    m, n = QR.shape
    Q = np.eye(m, dtype=QR.dtype)
    for k in reversed(range(min(m, n))):
        v = np.zeros(m, dtype=QR.dtype)
        v[k] = 1
        v[k + 1:] = QR[k + 1:, k]
        if np.isfinite(tau[k]):
            Q -= np.outer(v, v.conj() @ Q) / tau[k]
    return Q


def r_matrix(QR):
    m, n = QR.shape
    return np.triu(QR)[: min(m, n), :]


def reconstruct(QR, tau, perm):
    """out = Q R P^T (reconstruct.rs:16-45)."""
    m, n = QR.shape
    QRm = q_matrix(QR, tau)[:, : min(m, n)] @ r_matrix(QR)
    out = np.empty_like(QRm)
    out[:, perm] = QRm
    return out


def solve_lstsq(QR, tau, perm, B, conj=False):
    """solve.rs:52-80: the unpivoted lstsq, then rows ..n <- rows perm^-1."""
    Q = q_matrix(QR, tau)
    R = r_matrix(QR)
    if conj:
        Q, R = Q.conj(), R.conj()
    n = QR.shape[1]
    y = np.linalg.solve(R[:, :n], (Q.conj().T @ B)[:n])
    x = np.empty_like(y)
    x[perm] = y
    return x
