"""The backward-error checker of tests/backward_error.py discriminates (CPU, n = 600): it accepts the oracle's own LLT and
LU factors and rejects factors rounded to f32, a residual above the bound in one 128 x 128 tile, and one changed bit in the
sentinels around a matrix. Every rejection is by a factor of more than 10^3, so a bound 10^3 times looser would still
reject them: the GPU checks built on it are not too loose to mean anything."""
import numpy as np
import pytest
import torch

from backward_error import (changed_outside, llt_ratio, llt_residual, lu_ratio, lu_residual, matrix_in,
                            sentinel_buffer)

N = 600
TILE = (slice(256, 384), slice(128, 256))  # one 128 x 128 tile strictly below the diagonal


@pytest.fixture(scope="module")
def llt_case(oracle):
    rng = np.random.default_rng(2201)
    G = rng.standard_normal((N, N))
    A0 = np.asfortranarray(G @ G.T + N * np.eye(N))
    L = A0.copy(order="F")
    fail, cnt = oracle.llt(L)
    assert fail == -1 and cnt == 0
    return torch.from_numpy(A0), torch.from_numpy(np.tril(L))


@pytest.fixture(scope="module")
def lu_case(oracle):
    rng = np.random.default_rng(2202)
    A0 = np.asfortranarray(rng.standard_normal((N, N)))
    LU = A0.copy(order="F")
    perm, _, _ = oracle.lu(LU)
    return torch.from_numpy(A0), torch.from_numpy(LU), perm


def test_accepts_oracle_factors(llt_case, lu_case):
    A0, L = llt_case
    r_llt = llt_ratio(A0, L)
    A, LU, perm = lu_case
    r_lu = lu_ratio(A, LU, perm)
    print(f"oracle n={N}: LLT ratio {r_llt:.3g}, LU ratio {r_lu:.3g}")
    assert r_llt <= 1 and r_lu <= 1
    # the strict upper triangles are not read: NaN there changes nothing
    nan_up = torch.triu(torch.full_like(A0, float("nan")), 1)
    assert llt_ratio(A0 + nan_up, L + nan_up) == r_llt


def test_rejects_f32_factors(llt_case, lu_case):
    A0, L = llt_case
    assert llt_ratio(A0, L.float().double()) > 1e3
    A, LU, perm = lu_case
    assert lu_ratio(A, LU.float().double(), perm) > 1e3


def test_rejects_one_bad_tile(llt_case, lu_case):
    """A residual of 1.01e3 times the bound in one tile (added to the input, so the factors are those of a matrix that
    differs from A0 there) is rejected; the rest of the matrix still passes."""
    rng = np.random.default_rng(2203)
    sign = torch.from_numpy(np.where(rng.random((128, 128)) < 0.5, -1.0, 1.0))
    A0, L = llt_case
    _, bound = llt_residual(A0, L)
    Ab = A0.clone()
    Ab[TILE] += 1.01e3 * sign * bound[TILE]
    assert llt_ratio(Ab, L) > 1e3
    err, bound = llt_residual(Ab, L)
    ok = err <= bound
    assert not ok[TILE].any() and int((~ok).sum()) == 128 * 128
    A, LU, perm = lu_case
    _, bound = lu_residual(A, LU, perm)
    Ab = A.clone()
    rows = torch.as_tensor(perm)[TILE[0]]  # rows of A that land in the tile of P A
    Ab[rows, TILE[1]] += 1.01e3 * sign * bound[TILE]
    assert lu_ratio(Ab, LU, perm) > 1e3


def test_rejects_nan_residual(llt_case):
    A0, L = llt_case
    Lb = L.clone()
    Lb[N - 1, N - 1] = float("nan")
    assert llt_ratio(A0, Lb) == float("inf")


@pytest.mark.parametrize("where", ["padding", "offset", "upper"])
def test_sentinel_detects_one_changed_bit(where):
    n, ld, off = 37, 40, 1
    buf = sentinel_buffer(off + ld * n + 5, "cpu")
    M = matrix_in(buf, n, ld, off)
    low = torch.tril(torch.ones(n, n, dtype=torch.bool))
    M.copy_(torch.where(low, torch.randn(n, n, dtype=torch.float64), M))  # lower triangle: data
    writable = torch.zeros(buf.shape, dtype=torch.bool)
    matrix_in(writable, n, ld, off).copy_(low)
    before = buf.clone()
    M.copy_(torch.where(low, 2.0 * M, M))  # a "factorization" that changes the lower triangle only
    assert changed_outside(buf, before, writable) == 0
    raw = buf.view(torch.int64)
    idx = {"padding": off + 3 * ld + n + 1, "offset": 0, "upper": off + 5 * ld + 2}[where]
    assert not writable[idx]
    raw[idx] ^= 1  # the payload's lowest bit: still a NaN, so a NaN-aware comparison would miss it
    assert torch.isnan(buf[idx])
    assert changed_outside(buf, before, writable) == 1
