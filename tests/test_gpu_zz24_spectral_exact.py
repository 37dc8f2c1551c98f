"""GPU tests of the self-adjoint EVD and the SVD, with vectors and values only, against spectra known exactly
(tests/spectral_exact.py: dyadic Householder similarities, the 1-2-1 Toeplitz and the Clement matrix).

The sizes reach the device code's branches:
  * n = 32 / 33 and 64 / 65 cross divide-and-conquer tree levels (tridiag_dc.cu: leaves of 16..32 rows);
  * n = 8193 and 12289 exceed the 8192 rows tridiag.cu keeps in shared memory (TD_CH): each CTA starts on its private
    global-memory slice and switches to shared memory at the column where n - k <= 8192 (k = 1 for 8193, 4097 for 12289);
  * an SVD with 8192 < m and m / n <= 11/6 runs bidiag.cu's 8192-row chunks (BD_CH) over more than one chunk; taller
    matrices take a QR first and bidiagonalise the n x n R; 1100 x 600 and 1101 x 600 sit on the two sides of 11/6;
  * spectra: distinct integers, three values of multiplicity n/3 (exact ties across the tree cuts), a tight dyadic
    cluster, zero eigenvalues of both signs around them, the same matrix scaled by 2^+-500, rank n/2, repeated singular
    values, full U on a tall case; f32 and c64 entry points once each.
Every case checks values, residuals, orthogonality and the angles to the exact eigen- / singular subspaces, and the
values-only path (bisection) on the same input. Each prints its largest error-to-bound ratio and wall time (-s).
"""
import os
import re
import time

import numpy as np
import pytest
import torch

import spectral_exact as se

pytestmark = pytest.mark.gpu
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "faer-rs_b200", "csrc")


def _const(fname, name):
    src = open(os.path.join(CSRC, fname)).read()
    return int(re.search(rf"constexpr int {name} = (\d+);", src).group(1))


TD_CH = _const("tridiag.cu", "TD_CH")
BD_CH = _const("bidiag.cu", "BD_CH")


def _report(tag, ratios, dt):
    print(f"[zz24] {tag}: worst {se.worst(ratios):.3g} {({k: float(f'{v:.3g}') for k, v in ratios.items()})} {dt:.2f} s")


def _sync():
    torch.cuda.synchronize()


def _run_evd(la, ex, tag, host=False, u_out=se.U64, poison_upper=False):
    A = ex.A
    n = A.shape[0]
    if poison_upper:  # only the lower triangle may be read
        A = A.clone()
        A[torch.triu(torch.ones(n, n, dtype=torch.bool, device=A.device), 1)] = float("nan")
    if host:
        A = np.asfortranarray(A.cpu().numpy())
        S = np.zeros(n, dtype=A.dtype)
        U = np.zeros((n, n), dtype=A.dtype, order="F")
    else:
        S = torch.zeros(n, dtype=A.dtype, device=A.device)
        U = torch.zeros((n, n), dtype=A.dtype, device=A.device).T
    _sync()
    t0 = time.perf_counter()
    la.self_adjoint_evd(A, S, U)
    _sync()
    dt = time.perf_counter() - t0
    S = la._real_values(S)
    r = se.check_evd(ex, S, U, u_out=u_out)
    t1 = time.perf_counter()
    vals = la.self_adjoint_eigenvalues(A)
    _sync()
    dv = time.perf_counter() - t1
    r["values (bisection)"] = se.check_values(ex, vals, u_out=u_out)
    _report(f"evd {tag} n={n}", r, dt)
    print(f"[zz24]   self_adjoint_eigenvalues {dv:.2f} s")
    assert se.worst(r) <= 1.0, (tag, n, r)


def _run_svd(la, ex, tag, full_u=False, host=False, u_out=se.U64):
    A = ex.A
    m, n = A.shape
    size = min(m, n)
    ku = m if full_u else size
    if host:
        A = np.asfortranarray(A.cpu().numpy())
        S = np.zeros(size, dtype=A.dtype)
        U = np.zeros((m, ku), dtype=A.dtype, order="F")
        V = np.zeros((n, size), dtype=A.dtype, order="F")
    else:
        S = torch.zeros(size, dtype=A.dtype, device=A.device)
        U = torch.zeros((ku, m), dtype=A.dtype, device=A.device).T
        V = torch.zeros((size, n), dtype=A.dtype, device=A.device).T
    _sync()
    t0 = time.perf_counter()
    la.svd(A, S, U, V)
    _sync()
    dt = time.perf_counter() - t0
    r = se.check_svd(ex, la._real_values(S), U, V, u_out=u_out)
    t1 = time.perf_counter()
    vals = la.singular_values(A)
    _sync()
    dv = time.perf_counter() - t1
    r["values (values only)"] = se.check_values(ex, vals, u_out=u_out, N=m + n)
    _report(f"svd {tag} {m}x{n}{' full U' if full_u else ''}", r, dt)
    print(f"[zz24]   singular_values {dv:.2f} s")
    assert se.worst(r) <= 1.0, (tag, m, n, r)


def _distinct(n, rng, step=1):
    return rng.permutation(np.arange(-(n // 2), n - n // 2, dtype=np.int64)) * step


def _three(n, rng):
    return rng.permutation(np.repeat(np.array([-3, 1, 5], dtype=np.int64), -(-n // 3))[:n])


@pytest.mark.parametrize("n", [32, 33, 64, 65])
def test_evd_tree_levels(fb, cuda_dev, n):
    rng = np.random.default_rng(2400 + n)
    _run_evd(fb.linalg, se.hermitian(_distinct(n, rng, 3), rng, cuda_dev), "distinct", host=True)
    _run_evd(fb.linalg, se.hermitian(_three(n, rng), rng, cuda_dev), "three values", host=True)


def test_evd_hard_spectra_1024(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(2401)
    n = 1024
    # a tight dyadic cluster 1 + j 2^-30 (1000 values) with outliers on both sides
    cl = np.concatenate([(1 << 30) + np.arange(1000), [-(1 << 32), -(1 << 31), 3 << 30, 1 << 32] * 6]).astype(np.int64)
    _run_evd(la, se.hermitian(rng.permutation(cl), rng, cuda_dev, exp=-30), "dyadic cluster", host=True)
    # zero with multiplicity n/2 and both signs around it
    z = np.concatenate([np.zeros(n // 2, np.int64), -np.arange(1, n // 4 + 1), np.arange(1, n // 4 + 1)])
    _run_evd(la, se.hermitian(rng.permutation(z), rng, cuda_dev), "zeros +-")
    d = _distinct(n, rng, 7)
    for e in (500, -500):
        _run_evd(la, se.hermitian(d, rng, cuda_dev, exp=e), f"distinct * 2^{e}")


def test_evd_4097(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(2402)
    n = 4097
    _run_evd(la, se.hermitian(_distinct(n, rng) << 8, rng, cuda_dev), "distinct", poison_upper=True)
    _run_evd(la, se.toeplitz_121(n, cuda_dev), "toeplitz 1-2-1")
    _run_evd(la, se.clement(n, cuda_dev), "clement")


def test_evd_8192_three_values(fb, cuda_dev):
    rng = np.random.default_rng(2403)
    assert 8192 == TD_CH  # the largest size that runs on shared memory only
    _run_evd(fb.linalg, se.hermitian(_three(8192, rng), rng, cuda_dev), "three values")


def test_evd_8193_global_memory_slice(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(2404)
    n = 8193
    assert n > TD_CH and n - 1 <= TD_CH  # global memory for the first column only, then shared memory
    _run_evd(la, se.hermitian(_distinct(n, rng) << 4, rng, cuda_dev), "distinct")
    _run_evd(la, se.toeplitz_121(n, cuda_dev), "toeplitz 1-2-1")
    _run_evd(la, se.clement(n, cuda_dev), "clement")


def test_evd_12289_switch_halfway(fb, cuda_dev):
    rng = np.random.default_rng(2405)
    n = 12289
    assert n - TD_CH == 4097  # global-memory slices for the first 4097 columns, then shared memory
    d = np.concatenate([_distinct(n - n // 4, rng), np.zeros(n // 4, np.int64)])  # distinct plus a zero of multiplicity n/4
    _run_evd(fb.linalg, se.hermitian(rng.permutation(d), rng, cuda_dev), "distinct + zeros")


def test_svd_bidiag_chunks(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(2406)
    assert 9000 > BD_CH and 9000 / 6000 <= 11 / 6  # no QR first: bidiag.cu runs two row chunks
    _run_svd(la, se.rectangular(9000, 6000, rng.permutation(np.arange(1, 6001)), rng, cuda_dev), "distinct")
    half = np.concatenate([np.zeros(3000, np.int64), np.arange(1, 3001)])
    _run_svd(la, se.rectangular(6000, 9000, rng.permutation(half), rng, cuda_dev), "rank n/2 (wide)")


def test_svd_qr_first_full_u(fb, cuda_dev):
    rng = np.random.default_rng(2407)
    assert 12000 / 4000 > 11 / 6
    s = np.repeat(np.array([1, 2, 4, 1000], dtype=np.int64), 1000)
    _run_svd(fb.linalg, se.rectangular(12000, 4000, rng.permutation(s), rng, cuda_dev), "repeated", full_u=True)


@pytest.mark.parametrize("m", [1100, 1101])
def test_svd_qr_threshold(fb, cuda_dev, m):
    la = fb.linalg
    rng = np.random.default_rng(2408 + m)
    n = 600
    assert (m / n > 11 / 6) == (m == 1101)
    _run_svd(la, se.rectangular(m, n, rng.permutation(np.arange(1, n + 1)) * 5, rng, cuda_dev), "distinct", host=True)
    half = np.concatenate([np.zeros(n // 2, np.int64), np.arange(1, n // 2 + 1)])
    _run_svd(la, se.rectangular(m, n, rng.permutation(half), rng, cuda_dev), "rank n/2", full_u=True)
    _run_svd(la, se.rectangular(m, n, np.repeat(np.array([3, 7, 7 << 20], np.int64), n // 3), rng, cuda_dev), "repeated")


def test_f32_entry_points(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(2409)
    n = 256
    ex = se.hermitian(rng.integers(-100, 101, n), rng, cuda_dev, dtype=torch.float32)
    _run_evd(la, ex, "f32", host=True, u_out=se.U32)
    ex = se.rectangular(300, 200, rng.integers(0, 60, 200), rng, cuda_dev, dtype=torch.float32)
    _run_svd(la, ex, "f32", host=True, u_out=se.U32)


def test_c64_through_condensed_drivers(fb, cuda_dev):
    la = fb.linalg
    rng = np.random.default_rng(2410)
    _run_evd(la, se.hermitian(_distinct(1024, rng, 5), rng, cuda_dev, cplx=True), "c64")
    s = np.concatenate([np.zeros(100, np.int64), rng.permutation(np.arange(1, 301))])
    _run_svd(la, se.rectangular(700, 400, s, rng, cuda_dev, cplx=True), "c64 rank 300")
