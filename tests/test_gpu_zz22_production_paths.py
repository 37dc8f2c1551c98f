"""GPU tests of the f64 LLT and LU drivers that serve large matrices, and of the split-K branch of the f64 / f32 GEMM, with
odd, padded and misaligned layouts, against the componentwise backward-error bounds of tests/backward_error.py.

  * LLT, n >= 4096, column-major device matrix: the block-column look-ahead driver (dist.cu) with 512-, 256- and 128-wide
    blocks; ld = n, ld = n + 3 (odd: TMA refused), ld = n + 4, a base one element into its allocation, and row-major (the
    recursive driver). The padding and the strict upper triangle hold NaN sentinels and must come back bit for bit. An odd
    n refuses every TMA-fed trailing update (the panel buffer's leading dimension n - k0 is odd), so its factor is bit for
    bit the one of the cp.async kernel (`gemm_ws` = 0); an even one is not.
  * LLT statuses at n = 12289 in each block tier: isolated negative pivots regularised exactly once each, the first
    negative pivot reported without regularization, and where the tiers begin and end.
  * LU, n >= 4096: permutations bit-exact against the oracle, factors within the bound, sentinels untouched, a zero
    column inside a look-ahead block, and the 1024-wide tier above n = 20000.
  * Split-K GEMM (few output tiles, k >= 4096): every accumulation mode and destination structure, the reduce kernel's
    extra launch counted.
Each case prints its largest error-to-bound ratio and its wall time (run with -s to see them)."""
import time

import numpy as np
import pytest
import torch

from backward_error import (SENTINEL, changed_outside, llt_ratio, lu_ratio, matrix_in, sentinel_buffer)
from test_gpu_parity import S_LOW, S_RECT, S_SLOW, S_SUP, S_ULOW, S_UP, S_UUP, gemm_bound

pytestmark = pytest.mark.gpu

# documented defaults of the drivers' schedules
LOOKAHEAD_MIN_N = 4096           # dist.cu lookahead_min_n(): column-major n >= this takes the look-ahead drivers
LLT_HEAD, LLT_TAIL = 8192, 6144  # dist.cu llt_block_bounds(): 512 wide while more than HEAD columns remain, 128 from TAIL
LU_WIDE_N = 20000                # lu_f64.cu: 512-wide LU blocks up to n = 20000, 1024 beyond
U32 = 2.0 ** -24


def llt_bounds(n):
    """Block boundaries of the single-GPU device-resident LLT at its default widths."""
    b = [0]
    while b[-1] < n:
        rem = n - b[-1]
        w = 128 if rem <= LLT_TAIL else 512 if rem > LLT_HEAD else 256
        b.append(b[-1] + min(w, rem))
    return b


def report(what, ratio, t0):
    torch.cuda.synchronize()
    print(f"\n[zz22] {what}: max error / bound {ratio:.3g}, {time.perf_counter() - t0:.2f} s")


def spd(n, seed, dev):
    """the bench generator: G G^T + n I"""
    g = torch.Generator(device=dev).manual_seed(seed)
    G = torch.randn((n, n), dtype=torch.float64, device=dev, generator=g)
    return torch.addmm(n * torch.eye(n, dtype=torch.float64, device=dev), G, G.T)


def gaussian(n, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn((n, n), dtype=torch.float64, device=dev, generator=g)


LAYOUTS = {"ld": (0, 0, False), "ld+3": (3, 0, False), "ld+4": (4, 0, False), "offset": (0, 1, False), "row": (0, 0, True)}


def placed(A0, layout, lower_only, dev):
    """A0 copied into a sentinel-filled buffer with the given layout. Returns (buffer, view, mask of the elements the
    factorization may write): the lower triangle for LLT (the strict upper part stays sentinel), else the whole matrix."""
    n = A0.shape[0]
    extra, off, row = LAYOUTS[layout]
    ld = n + extra
    buf = sentinel_buffer(off + ld * n + 7, dev)
    A = matrix_in(buf, n, ld, off, row)
    writable = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
    W = matrix_in(writable, n, ld, off, row)
    if lower_only:
        W.copy_(torch.tril(torch.ones((n, n), dtype=torch.bool, device=dev)))
        A.copy_(torch.where(W, A0, A))
    else:
        W.fill_(True)
        A.copy_(A0)
    return buf, A, writable


@pytest.fixture
def ws_option(fb):
    lib = fb.load()
    saved = lib.faer_b200_get_option(b"gemm_ws")
    yield lib
    lib.faer_b200_set_option(b"gemm_ws", saved)


def tril_bits(A):
    return torch.tril(A).contiguous().view(torch.int64)


# ---- 1. LLT on the look-ahead driver, layout matrix -----------------------------------------------------------------
LLT_CASES = [(n, lay) for n in (4095, 4096, 4097, 6146, 8200, 8201) for lay in LAYOUTS] + [(12289, "ld"), (16384, "ld")]


def test_llt_schedule_defaults():
    """The sizes below land where they are meant to: 6146 starts with one 256-wide block and ends ragged in the tail, 8200
    has exactly one 512-wide block, 12289 has every tier and a one-column last block."""
    w = np.diff(llt_bounds(6146))
    assert w[0] == 256 and set(w[1:-1]) == {128} and w[-1] == 6146 - 256 - 128 * 46 == 2
    w = np.diff(llt_bounds(8200))
    assert list(w).count(512) == 1 and w[0] == 512
    w = list(np.diff(llt_bounds(12289)))
    assert w == [512] * 9 + [256] * 7 + [128] * 46 + [1]


@pytest.mark.parametrize("n,layout", LLT_CASES)
def test_llt_layouts(fb, cuda_dev, ws_option, n, layout):
    la = fb.linalg
    t0 = time.perf_counter()
    A0 = spd(n, 2200 + n, cuda_dev)
    buf, A, writable = placed(A0, layout, True, cuda_dev)
    before = buf.clone()
    info = la.cholesky_in_place(A)
    assert info.dynamic_regularization_count == 0
    assert changed_outside(buf, before, writable) == 0, "padding or strict upper triangle written"
    ratio = llt_ratio(A0, A)
    assert ratio <= 1, (n, layout, ratio)
    if layout == "ld":
        # odd n: no operand of a trailing update is TMA-addressable, the cp.async kernel served every one of them
        ref_buf = before.clone()
        R = matrix_in(ref_buf, n, n)
        assert ws_option.faer_b200_set_option(b"gemm_ws", 0) == 0
        la.cholesky_in_place(R)
        same = torch.equal(tril_bits(A), tril_bits(R))
        assert same == (n % 2 == 1), (n, "bit-equal to the cp.async run" if same else "differs from the cp.async run")
    report(f"LLT n={n} {layout}", ratio, t0)


def test_llt_host_pipeline_padded(fb, cuda_dev):
    """host matrix, n = 4097 >= lookahead_min_n, column stride n + 3: the pipelined upload / factor / download driver"""
    la = fb.linalg
    t0 = time.perf_counter()
    n, ld = 4097, 4100
    A0 = spd(n, 2290, cuda_dev)
    dbuf, _, writable = placed(A0, "ld+3", True, cuda_dev)
    buf = dbuf.cpu().numpy()
    A = buf[:ld * n].reshape(n, ld)[:, :n].T
    assert A.strides == (8, 8 * ld)
    before = torch.from_numpy(buf.copy()).to(cuda_dev)
    info = la.cholesky_in_place(A)
    assert info.dynamic_regularization_count == 0
    after = torch.from_numpy(buf).to(cuda_dev)
    assert changed_outside(after, before, writable) == 0
    ratio = llt_ratio(A0, matrix_in(after, n, ld))
    assert ratio <= 1
    report("LLT host n=4097 ld=4100", ratio, t0)


# ---- 2. LLT statuses on every tier (n = 12289) ------------------------------------------------------------------------
N_ST = 12289
B_ST = llt_bounds(N_ST)
TIERS = {512: (0, 4608), 256: (4608, 6400), 128: (6400, N_ST)}
POSITIONS = {512: [1536, 1800, 2047], 256: [4608, 5200, 6399], 128: [6400, 9001, N_ST - 1]}


def test_llt_tiers_at_12289(fb, cuda_dev):
    """The driver's tiers at n = 12289 are where the defaults put them, and the positions used below sit in the tiers
    they are named for: the first, an interior and the last column of a 512-wide block; the first and last column of the
    256 tier; the first column of the tail, an interior one and the one-column last block.
    The library's 512 tier ends at 4608, checked against a run of uniform 512-wide blocks. A 512-wide block is factored
    by halves, so for its own columns it performs the same operations as two 256-wide blocks; the columns after it see one
    k = 512 update instead of two k = 256 updates, which round differently. So the factors agree bit for bit on every
    column before 5120 (512-wide blocks up to 4608, then 256 or 512) and differ on the next 512 columns (the block at
    4608 is not 512 wide)."""
    assert B_ST == list(range(0, 4608, 512)) + list(range(4608, 6400, 256)) + list(range(6400, N_ST, 128)) + [N_ST]
    for w, (lo, hi) in TIERS.items():
        assert all(lo <= j < hi for j in POSITIONS[w])
    assert POSITIONS[512][0] % 512 == 0 and POSITIONS[512][2] % 512 == 511 and B_ST[-2] == N_ST - 1
    la = fb.linalg
    t0 = time.perf_counter()
    A0 = spd(N_ST, 2201, cuda_dev).T  # column-major view
    A = A0.clone(memory_format=torch.preserve_format)
    la.cholesky_in_place(A)
    R = A0.clone(memory_format=torch.preserve_format)
    fail, _ = fb.dist.cholesky_in_place(R, N_ST, nb=512, lookahead=2)  # local run, no look-ahead: uniform blocks
    assert fail == -1
    a, r = tril_bits(A), tril_bits(R)
    assert torch.equal(a[:, :5120], r[:, :5120])
    assert not torch.equal(a[:, 5120:5632], r[:, 5120:5632])
    ratio = llt_ratio(A0, A)
    assert ratio <= 1
    report("LLT n=12289 tier boundary", ratio, t0)


@pytest.mark.parametrize("tier", [512, 256, 128])
def test_llt_regularised_pivots(fb, cuda_dev, tier):
    """Row and column j zeroed except A[j, j] = -1, with regularization (delta, eps) = (4, 1e-8): each pivot is regularised
    exactly once; L[j, j] is the unregularised pivot times recip(sqrt(delta)), -1 * 0.5, exactly; the rest of row and
    column j of L is zero; and the rest of L factors A0 with those rows and columns removed, within the bound.
    (An exactly zero pivot would store a zero diagonal, and the panel solve below it would divide by it: the reference
    turns such a matrix into NaN and fails at a later block, so a negative pivot is the clean construction.)"""
    la = fb.linalg
    t0 = time.perf_counter()
    js = POSITIONS[tier]
    A0 = spd(N_ST, 2202, cuda_dev).T
    idx = torch.tensor(js, device=cuda_dev)
    A0[idx, :] = 0.0
    A0[:, idx] = 0.0
    A0[idx, idx] = -1.0
    A = A0.clone(memory_format=torch.preserve_format)
    info = la.cholesky_in_place(A, regularization=(4.0, 1e-8))
    assert info.dynamic_regularization_count == len(js), (tier, info.dynamic_regularization_count)
    L = torch.tril(A)
    assert torch.equal(L[idx, idx], torch.full((len(js),), -0.5, dtype=torch.float64, device=cuda_dev))
    L[idx, idx] = 0.0
    assert torch.count_nonzero(L[:, idx]) == 0 and torch.count_nonzero(L[idx, :]) == 0
    keep = torch.ones(N_ST, dtype=torch.bool, device=cuda_dev)
    keep[idx] = False
    ratio = llt_ratio(A0[keep][:, keep], L[keep][:, keep])
    assert ratio <= 1, (tier, ratio)
    report(f"LLT n=12289 regularised {js}", ratio, t0)


@pytest.mark.parametrize("js", [[j] for w in POSITIONS for j in POSITIONS[w]] + [[5200, 1800], [9001, 5200], [N_ST - 1, 2047]])
def test_llt_failure_index(fb, cuda_dev, js):
    la = fb.linalg
    A = spd(N_ST, 2203, cuda_dev).T
    for j in js:
        A[j, j] = -1.0
    with pytest.raises(la.LltError) as ei:
        la.cholesky_in_place(A)
    assert ei.value.index == min(js), (js, ei.value.index)


# ---- 3. LU on the look-ahead driver ---------------------------------------------------------------------------------
@pytest.mark.parametrize("n,layout", [(4095, "ld"), (4097, "ld"), (4096, "ld+3"), (4096, "offset"), (4100, "row")])
def test_lu_layouts_vs_oracle(fb, oracle, cuda_dev, n, layout):
    la = fb.linalg
    t0 = time.perf_counter()
    A0 = gaussian(n, 2210 + n, cuda_dev).T
    buf, A, writable = placed(A0, layout, False, cuda_dev)
    before = buf.clone()
    p = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    pi = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    info = la.lu_in_place(A, p, pi)
    t_gpu = time.perf_counter()
    want = np.asfortranarray(A0.cpu().numpy())
    perm_o, pinv_o, nt_o = oracle.lu(want)
    t_oracle = time.perf_counter() - t_gpu
    assert np.array_equal(p.cpu().numpy(), perm_o) and np.array_equal(pi.cpu().numpy(), pinv_o)
    assert info.transposition_count == nt_o
    assert changed_outside(buf, before, writable) == 0, "padding written"
    ratio = lu_ratio(A0, A, perm_o)
    assert ratio <= 1, (n, layout, ratio)
    report(f"LU n={n} {layout} (oracle {t_oracle:.2f} s)", ratio, t0)


def test_lu_zero_column_in_lookahead_block(fb, oracle, cuda_dev):
    """An all-zero column j inside the fourth 512-wide block: no error status; the pivots (first maximum over the NaN
    columns that follow) and the NaN / inf pattern are the oracle's."""
    la = fb.linalg
    t0 = time.perf_counter()
    n, j = 4097, 3 * 512 + 100
    A0 = gaussian(n, 2220, cuda_dev).T
    A0[:, j] = 0.0
    A = A0.clone(memory_format=torch.preserve_format)
    p = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    pi = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    info = la.lu_in_place(A, p, pi)
    want = np.asfortranarray(A0.cpu().numpy())
    perm_o, pinv_o, nt_o = oracle.lu(want)
    assert np.array_equal(p.cpu().numpy(), perm_o) and np.array_equal(pi.cpu().numpy(), pinv_o)
    assert info.transposition_count == nt_o
    got = A.cpu().numpy()
    assert np.isnan(want).any()
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want))
    report("LU n=4097 zero column 1636", 0.0, t0)


def test_lu_wide_tier(fb, cuda_dev):
    """odd n > 20000: 1024-wide look-ahead blocks (too large for the oracle)"""
    la = fb.linalg
    t0 = time.perf_counter()
    n = 20001
    assert n > LU_WIDE_N and n >= LOOKAHEAD_MIN_N
    A0 = gaussian(n, 2230, cuda_dev).T
    A = A0.clone(memory_format=torch.preserve_format)
    p = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    pi = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    la.lu_in_place(A, p, pi)
    ar = torch.arange(n, device=cuda_dev)
    assert torch.equal(torch.sort(p).values, ar) and torch.equal(pi[p], ar)
    assert float(torch.tril(A, -1).abs().max()) <= 1.0
    ratio = lu_ratio(A0, A, p)
    assert ratio <= 1, ratio
    report("LU n=20001", ratio, t0)


# ---- 4. split-K GEMM --------------------------------------------------------------------------------------------------
SPLIT_SHAPES = [(64, 64, 4096), (300, 300, 8192), (513, 129, 65536), (130, 1, 16384)]
MODES = [(False, 1.0), (False, -1.0), (False, 0.5), (True, 1.0), (True, -1.0), (True, 0.5)]


def selected(ds, m, n):
    if ds == S_RECT:
        return np.ones((m, n), bool)
    sel = np.tril(np.ones((m, n), bool)) if ds in (S_LOW, S_SLOW, S_ULOW) else np.triu(np.ones((m, n), bool))
    if ds in (S_SLOW, S_SUP, S_ULOW, S_UUP):
        np.fill_diagonal(sel, False)
    return sel


def splits(dtype, m, n, k, ds, sms):
    """Whether gemm_f64 / gemm_f32 split the contraction: fewer 64 x 64 output tiles than SMs and k >= 4096, except f32
    rectangular products large enough for the wgmma kernel, which never split (gemm_f32.cu)."""
    if dtype == np.float32 and ds == S_RECT and m >= 64 and n >= 64 and 2.0 * m * n * k >= 2.5e8:
        return False
    return -(-m // 64) * -(-n // 64) < sms and k >= 4096


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", SPLIT_SHAPES)
def test_split_k_gemm(fb, oracle, cuda_dev, dtype, shape):
    la = fb.linalg
    lib = fb.load()
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    t0 = time.perf_counter()
    m, n, k = shape
    rng = np.random.default_rng(2240 + k)
    A = np.asfortranarray(rng.standard_normal((m, k)).astype(dtype))
    B = np.asfortranarray(rng.standard_normal((k, n)).astype(dtype))
    if dtype == np.float64:
        # the parity tests' bound: |alpha| gemm_bound + 4 u |want|
        P = np.zeros((m, n), order="F")
        oracle.matmul(P, False, A, B, 1.0)
        err_ab, err_c, err_c0 = gemm_bound(A, B, k), 4 * 2.0 ** -53, 0.0
    else:
        # the f32 tests' bound against the f64 product: 4 k u32 |alpha| |A||B| + 4 u32 (|want| + |C0|)
        A64, B64 = A.astype(np.float64), B.astype(np.float64)
        P = A64 @ B64
        err_ab, err_c, err_c0 = 4 * k * U32 * (np.abs(A64) @ np.abs(B64)) + 1e-30, 4 * U32, 4 * U32
        del A64, B64
    ibits = np.int64 if dtype == np.float64 else np.int32
    dA = torch.from_numpy(np.ascontiguousarray(A.T)).to(cuda_dev).T
    dB = torch.from_numpy(np.ascontiguousarray(B.T)).to(cuda_dev).T
    nan = np.array([SENTINEL], dtype=np.int64).view(np.float64)[0].astype(dtype)
    structs = [S_RECT] + ([S_LOW, S_UP, S_SLOW, S_SUP, S_ULOW, S_UUP] if m == n else [])
    worst = 0.0
    for ds in structs:
        sel = selected(ds, m, n)
        for row_major in ([False, True] if ds == S_RECT else [False]):
            for add, alpha in MODES:
                C0 = rng.standard_normal((m, n)).astype(dtype)
                C0[~sel] = nan
                if not add:
                    C0[...] = nan  # Replace must not read dst
                dC = torch.from_numpy(C0).to(cuda_dev)
                dC = dC if row_major else dC.T.contiguous().T
                mode = la.Accum.Add if add else la.Accum.Replace
                n0 = lib.faer_b200_launch_count()
                la.matmul_triangular(dC, ds, mode, dA, S_RECT, dB, S_RECT, alpha)
                launches = lib.faer_b200_launch_count() - n0
                got = dC.cpu().numpy()
                # an unsplit call of the same kind: same dst layout and structure, k = 1024
                dU = torch.zeros((m, n), dtype=tdt, device=cuda_dev)
                dU = dU if row_major else dU.T.contiguous().T
                n0 = lib.faer_b200_launch_count()
                la.matmul_triangular(dU, ds, mode, dA[:, :1024], S_RECT, dB[:1024], S_RECT, alpha)
                base = lib.faer_b200_launch_count() - n0
                extra = 1 if splits(dtype, m, n, k, ds, sms) else 0  # the reduce kernel
                assert launches == base + extra, (shape, ds, add, alpha, launches, base)
                assert np.array_equal(got[~sel].view(ibits), C0[~sel].view(ibits)), (shape, ds, "unselected part written")
                c = C0.astype(np.float64) if add else 0.0
                want = alpha * P + c
                bound = abs(alpha) * err_ab + err_c * np.abs(want) + err_c0 * np.abs(c)
                err = np.abs(got.astype(np.float64) - want)[sel]
                assert np.all(err <= bound[sel]), (shape, ds, row_major, add, alpha)
                worst = max(worst, float((err / bound[sel]).max()))
    report(f"split-K {np.dtype(dtype).name} {shape}", worst, t0)
