"""The LLT diagonal-block kernel (potf2, one launch for n <= 128 at block size 128) against the reference's unblocked
leaf recurrence, bit for bit: `oracle.llt(A, recursion_threshold=128)` is one leaf at these sizes (oracle/oracle.cpp,
llt_leaf).

  * n from 1 to 128, on both sides of every multiple of 32, f64 and f32, on device matrices: column-major, row-major
    and column-major with ld = n + 3 (the padding and the strict upper triangle hold NaN sentinels and must come back
    bit for bit);
  * regularised pivots (a negative diagonal entry) at the first column, on both sides of each multiple of 32 and at the
    last column, one at a time and all at once: the factor bitwise, the count exactly;
  * a failing pivot (negative or NaN) at the same columns: the index exactly, and A afterwards as the kernel leaves it:
    the columns before the failing one hold their L, the rest of A is untouched;
  * n = 200 (two leaves): the failing index in either leaf, and the count summed over both.
Each call at n <= 128 is checked to be a single kernel launch."""
import numpy as np
import pytest
import torch

from backward_error import SENTINEL

pytestmark = pytest.mark.gpu

NS = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 96, 127, 128]
DTYPES = {np.float32: torch.float32, np.float64: torch.float64}
LAYOUTS = ("col", "row", "ld+3")


def spd(n, dtype, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    return (G @ G.T + n * np.eye(n)).astype(dtype)


def reg(n):
    """(delta, epsilon): a regularised pivot of the size of the others, so that it does not cascade into more"""
    return (4.0 * n, 1e-3)


def boundary_columns(n):
    return sorted({j for j in (0, 31, 32, 63, 64, 95, 96, n - 1) if 0 <= j < n})


def offsets(n, layout):
    """buffer offset of each element (i, j) and the buffer length"""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    if layout == "row":
        return i * n + j, n * n
    ld = n + 3 if layout == "ld+3" else n
    return j * ld + i, n * ld


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view(np.int32 if x.dtype == np.float32 else np.int64)


def check(fb, oracle, dev, A, layout, reg=(0.0, 0.0), one_leaf=True):
    """Factor A's lower triangle on the device and compare with the leaf recurrence (with one_leaf: in one launch, bit
    for bit; otherwise the statuses only). Returns (fail index or -1, count)."""
    la, lib = fb.linalg, fb.load()
    n = A.shape[0]
    want = np.asfortranarray(A.copy())
    want_fail, want_cnt = oracle.llt(want, delta=reg[0], eps=reg[1], recursion_threshold=128)

    off, size = offsets(n, layout)
    low = np.tril(np.ones((n, n), dtype=bool))
    nan = np.array([SENTINEL], dtype=np.int64).view(np.float64)[0].astype(A.dtype)
    host = np.full(size, nan, dtype=A.dtype)
    host[off[low]] = A[low]
    buf = torch.from_numpy(host).to(dev)
    M = torch.as_strided(buf, (n, n), (n, 1) if layout == "row" else (1, n + 3 if layout == "ld+3" else n))

    n0 = lib.faer_b200_launch_count()
    try:
        fail, cnt = -1, la.cholesky_in_place(M, regularization=reg).dynamic_regularization_count
    except la.LltError as e:
        fail, cnt = e.index, None
    torch.cuda.synchronize()
    if one_leaf:
        assert lib.faer_b200_launch_count() - n0 == 1
    assert fail == want_fail, (fail, want_fail)
    if fail < 0:
        assert cnt == want_cnt, (cnt, want_cnt)

    out = buf.cpu().numpy()
    outside = np.ones(size, dtype=bool)
    outside[off[low]] = False
    assert np.array_equal(bits(out[outside]), bits(host[outside])), "padding or strict upper triangle written"
    if not one_leaf:
        return fail, cnt
    got = out[off]
    if fail < 0:
        assert np.array_equal(bits(got[low]), bits(want[low]))
    else:
        done = low & (np.arange(n)[None, :] < fail)  # the columns before the failing one hold their L
        assert np.array_equal(bits(got[done]), bits(want[done]))
        assert np.array_equal(bits(got[low & ~done]), bits(A[low & ~done]))  # the rest is the input
    return fail, cnt


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("n", NS)
def test_potf2_bitwise_layouts(fb, oracle, cuda_dev, n, dtype):
    A = spd(n, dtype, 2600 + n)
    for layout in LAYOUTS:
        assert check(fb, oracle, cuda_dev, A, layout) == (-1, 0)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("n", NS)
def test_potf2_regularised_pivots(fb, oracle, cuda_dev, n, dtype):
    A0 = spd(n, dtype, 2700 + n)
    cols = boundary_columns(n)
    for j in cols:
        A = A0.copy()
        A[j, j] = -1.0
        fail, cnt = check(fb, oracle, cuda_dev, A, "col", reg(n))
        assert fail == -1 and cnt >= 1
    A = A0.copy()
    A[cols, cols] = -1.0
    fail, cnt = check(fb, oracle, cuda_dev, A, "ld+3", reg(n))
    assert fail == -1 and cnt >= len(cols)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("n", NS)
def test_potf2_failing_pivots(fb, oracle, cuda_dev, n, dtype):
    A0 = spd(n, dtype, 2800 + n)
    for j in boundary_columns(n):
        for bad, r in ((-1.0, (0.0, 0.0)), (np.nan, (0.0, 0.0)), (np.nan, reg(n))):
            A = A0.copy()
            A[j, j] = bad
            assert check(fb, oracle, cuda_dev, A, "col", r)[0] == j
    A = A0.copy()
    A[n - 1, n - 1] = -1.0
    assert check(fb, oracle, cuda_dev, A, "row")[0] == n - 1


def test_potf2_two_leaves_statuses(fb, oracle, cuda_dev):
    """n = 200 factors as leaves of 128 and 72 with a panel solve and an update between them: a failure in the first
    leaf stops the second one, and the regularisation counts of both leaves add up."""
    n = 200
    A0 = spd(n, np.float64, 2900)
    for j in (5, 127, 128, 150):
        A = A0.copy()
        A[j, j] = -1.0
        assert check(fb, oracle, cuda_dev, A, "col", one_leaf=False)[0] == j
    A = A0.copy()
    for j in (3, 127, 150, 199):
        A[j, j] = -1.0
    fail, cnt = check(fb, oracle, cuda_dev, A, "col", reg(n), one_leaf=False)
    assert fail == -1 and cnt >= 4
