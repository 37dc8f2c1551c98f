"""GPU tests of the wide (128 x 128 tile) configuration of the TMA-fed f64 GEMM (csrc/gemm_f64_ws.cuh) after its tile store
moved to a storer warp, and of the LLT block schedule that feeds it deeper contractions (512-wide leading blocks):
  * forced wide (`gemm_ws` = 3), triangular destinations, Add and Replace, alpha in {-1, 1, 0.5}, contractions up to 1024,
    sizes that are not tile multiples, against the oracle; the untouched triangle (NaN sentinels) bit for bit. Operand
    and dst strides are even (TMA-addressable); that the ws kernel ran is shown by a result that differs from the
    cp.async kernel's (`gemm_ws` = 0), which a rejected ws launch would fall back to and reproduce bit for bit;
  * Add with alpha = -1: the shared-memory epilogue (staged tiles, TMA store) bit for bit equal to the register epilogue,
    which a destination offset by one element (not 16-byte aligned, so TMA cannot address it) takes for every tile;
  * the single-GPU LLT at n = 12288 and 16384 (512-, 256- and 128-wide blocks) within the LLT tolerance of the parity
    tests, bit for bit equal to the same driver called with the 512-wide tier requested explicitly, and different from
    it without that tier."""
import numpy as np
import pytest

from test_gpu_parity import S_LOW, S_RECT, S_UP, U, gemm_bound, to_dev

pytestmark = pytest.mark.gpu


@pytest.fixture
def wide(fb):
    lib = fb.load()
    saved = lib.faer_b200_get_option(b"gemm_ws")
    assert lib.faer_b200_set_option(b"gemm_ws", 3) == 0
    yield lib
    lib.faer_b200_set_option(b"gemm_ws", saved)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def run_as_cp_async(lib, f):
    """f() on the cp.async kernel (`gemm_ws` = 0), then back to the forced wide configuration"""
    assert lib.faer_b200_set_option(b"gemm_ws", 0) == 0
    try:
        f()
    finally:
        assert lib.faer_b200_set_option(b"gemm_ws", 3) == 0


# even n and k: Fortran operands (ld = n, resp. k) are TMA-readable. (4094, 256): 528 staged-or-diagonal tiles, so a CTA
# takes several tiles (up to 1024 / k) and reuses the dst buffer across staged tiles.
@pytest.mark.parametrize("n,k", [(1000, 1024), (2050, 768), (1100, 512), (386, 258), (4094, 256)])
def test_wide_epilogue_vs_oracle(fb, oracle, cuda_dev, wide, n, k):
    import torch
    la = fb.linalg
    rng = np.random.default_rng(180 + n + k)
    for ds in (S_LOW, S_UP):
        sel = np.tril(np.ones((n, n), bool)) if ds == S_LOW else np.triu(np.ones((n, n), bool))
        for add, alpha in [(True, -1.0), (True, 1.0), (True, 0.5), (False, 1.0), (False, -1.0), (False, 0.5)]:
            A = np.asfortranarray(rng.standard_normal((n, k)))
            B = np.asfortranarray(rng.standard_normal((k, n)))
            C0 = np.asfortranarray(rng.standard_normal((n, n)))
            C0[~sel] = np.nan
            want = C0.copy(order="F")
            oracle.matmul_triangular(want, ds, add, A, S_RECT, B, S_RECT, alpha)
            dA, dB, dC = to_dev(A, cuda_dev), to_dev(B, cuda_dev), to_dev(C0, cuda_dev)
            if not add:
                dC.masked_fill_(torch.from_numpy(sel).to(cuda_dev), float("nan"))
            dC0 = dC.clone()
            mode = la.Accum.Add if add else la.Accum.Replace
            la.matmul_triangular(dC, ds, mode, dA, S_RECT, dB, S_RECT, alpha)
            got = dC.cpu().numpy()
            if add and alpha == -1.0:
                run_as_cp_async(wide, lambda: la.matmul_triangular(dC0, ds, mode, dA, S_RECT, dB, S_RECT, alpha))
                assert not np.array_equal(bits(got[sel]), bits(dC0.cpu().numpy()[sel])), (n, k, ds)
            assert np.array_equal(bits(got[~sel]), bits(C0[~sel])), (n, k, ds, add, alpha)
            bound = abs(alpha) * gemm_bound(A, B, k) + 4 * U * np.abs(want)
            assert np.all(np.abs(got - want)[sel] <= bound[sel]), (n, k, ds, add, alpha)


@pytest.mark.parametrize("ds", [S_LOW, S_UP])
def test_staged_epilogue_bitwise_equals_register_epilogue(fb, cuda_dev, wide, ds):
    import torch
    la = fb.linalg
    torch.manual_seed(181 + ds)
    n, k, ld = 2049, 1024, 2050
    A = torch.randn((k, ld), dtype=torch.float64, device=cuda_dev)[:, :n].T   # n x k, column stride ld (even)
    assert A.stride() == (1, ld) and A.data_ptr() % 16 == 0
    C0 = torch.randn((n, n), dtype=torch.float64, device=cuda_dev).T
    outs = []
    for off in (0, 1):
        buf = torch.empty(1 + ld * n, dtype=torch.float64, device=cuda_dev)
        dC = buf[off:off + ld * n].view(n, ld)[:, :n].T   # column-major n x n, column stride ld
        # off = 0: TMA can address dst, the off-diagonal tiles take the staged epilogue; off = 1: every tile takes the
        # register epilogue
        assert (dC.data_ptr() % 16 == 0) == (off == 0)
        dC.copy_(C0)
        la.matmul_triangular(dC, ds, la.Accum.Add, A, S_RECT, A.T, S_RECT, -1.0)
        outs.append(dC.clone())
    assert torch.equal(outs[0].view(torch.int64), outs[1].view(torch.int64))
    ref = C0.clone(memory_format=torch.preserve_format)
    run_as_cp_async(wide, lambda: la.matmul_triangular(ref, ds, la.Accum.Add, A, S_RECT, A.T, S_RECT, -1.0))
    assert not torch.equal(ref.view(torch.int64), outs[0].view(torch.int64))   # the ws kernel ran
    untouched = torch.triu(C0, 1) if ds == S_LOW else torch.tril(C0, -1)
    kept = torch.triu(outs[0], 1) if ds == S_LOW else torch.tril(outs[0], -1)
    assert torch.equal(kept.view(torch.int64), untouched.view(torch.int64))


@pytest.mark.parametrize("n", [12288, 16384])
def test_llt_wide_leading_blocks(fb, cuda_dev, n):
    """|A - L L^T| <= 8 n 128 u |A|_max (the parity tests' LLT tolerance) and the upper triangle untouched. The entry
    point's factor is bit for bit the one of the same driver asked for the 512-wide tier explicitly (lookahead bits
    1 | 2 | 4), and differs from the 256 / 128 schedule (bits 1 | 2): the tier is in use."""
    import torch
    la = fb.linalg
    torch.manual_seed(182)
    G = torch.randn((n, n), dtype=torch.float64, device=cuda_dev)
    A0 = torch.addmm(n * torch.eye(n, dtype=torch.float64, device=cuda_dev), G, G.T).T
    del G
    A = A0.clone(memory_format=torch.preserve_format)
    info = la.cholesky_in_place(A)
    assert info.dynamic_regularization_count == 0
    assert torch.equal(torch.triu(A, 1), torch.triu(A0, 1))
    L = torch.tril(A)
    amax = float(A0.abs().max())
    assert float((torch.tril(A0) - torch.tril(L @ L.T)).abs().max()) <= 8 * n * 128 * U * amax
    del L
    R = A0.clone(memory_format=torch.preserve_format)
    fail, _ = fb.dist.cholesky_in_place(R, n, nb=256, lookahead=7)
    assert fail == -1
    assert torch.equal(torch.tril(A).view(torch.int64), torch.tril(R).view(torch.int64))
    R.copy_(A0)
    fail, _ = fb.dist.cholesky_in_place(R, n, nb=256, lookahead=3)
    assert fail == -1
    assert not torch.equal(torch.tril(A).view(torch.int64), torch.tril(R).view(torch.int64))
    assert float((torch.tril(A) - torch.tril(R)).abs().max()) <= 64 * n * U * float(torch.tril(A).abs().max())
