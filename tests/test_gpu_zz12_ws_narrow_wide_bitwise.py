"""GPU tests of the TMA-fed f64 GEMM (csrc/gemm_f64_ws.cuh) in its two configurations, narrow (`gemm_ws` = 2, 128 x 64
tiles, two CTAs per SM) and wide (`gemm_ws` = 3, 128 x 128 tiles, one CTA per SM):
  * the LLT's trailing update (lower destination, Add and Replace, alpha = -1, panel P = randn(k, n).T and rhs P^T):
    both configurations share the 32 x 64 warp tile, the fragment mapping and the k order, so they must agree bit for
    bit, for ragged orders, contractions that are not a multiple of the 16-deep k-step and fewer k-steps than ring
    stages. The strict upper triangle stays untouched, the result lies within the forward bound of a reference product,
    and for the deeper contractions it differs from the cp.async kernel's (`gemm_ws` = 0): the ws kernel ran;
  * rectangular m != n updates, every operand and destination layout, against the oracle at the forward bound of the
    ws GEMM tests."""
import itertools

import numpy as np
import pytest

from test_gpu_parity import S_LOW, S_RECT, U, gemm_bound, to_dev

pytestmark = pytest.mark.gpu


@pytest.fixture
def ws_opt(fb):
    lib = fb.load()
    saved = lib.faer_b200_get_option(b"gemm_ws")
    yield lib
    lib.faer_b200_set_option(b"gemm_ws", saved)


@pytest.mark.parametrize("n", [16128, 6016, 1000])
def test_narrow_and_wide_agree_bitwise_on_the_llt_update(fb, cuda_dev, ws_opt, n):
    import torch
    la = fb.linalg
    torch.manual_seed(1200 + n)
    C0 = torch.randn((n, n), dtype=torch.float64, device=cuda_dev).T
    for k in (512, 256, 128, 40, 8):
        P = torch.randn((k, n), dtype=torch.float64, device=cuda_dev).T  # column-major n x k, as the LLT's panel
        for accum in (la.Accum.Add, la.Accum.Replace):
            outs = {}
            for mode in (2, 3, 0):
                if mode == 0 and k < 128:
                    continue
                assert ws_opt.faer_b200_set_option(b"gemm_ws", mode) == 0
                Cm = C0.clone(memory_format=torch.preserve_format)
                la.matmul_triangular(Cm, S_LOW, accum, P, S_RECT, P.T, S_RECT, -1.0)
                outs[mode] = Cm
            assert torch.equal(outs[2].view(torch.int64), outs[3].view(torch.int64)), (n, k, accum)
            assert torch.equal(torch.triu(outs[3], 1).view(torch.int64), torch.triu(C0, 1).view(torch.int64)), (n, k, accum)
            if 0 in outs:
                assert not torch.equal(outs[0].view(torch.int64), outs[3].view(torch.int64)), (n, k, accum)
            want = (C0 if accum == la.Accum.Add else torch.zeros_like(C0)) - P @ P.T
            bound = 2 * k * 2 * U * (P.abs() @ P.abs().T) + 4 * U * want.abs()
            assert bool((torch.tril(outs[3] - want).abs() <= bound).all()), (n, k, accum)
            del outs, want, bound
        del P


@pytest.mark.parametrize("mode", [2, 3])
def test_rectangular_updates_vs_oracle(fb, oracle, cuda_dev, ws_opt, mode):
    la = fb.linalg
    assert ws_opt.faer_b200_set_option(b"gemm_ws", mode) == 0
    rng = np.random.default_rng(1210 + mode)
    for (m, n, k) in [(1000, 300, 512), (300, 1000, 256), (2050, 130, 40), (130, 2050, 8), (517, 1031, 129)]:
        for layout in itertools.product("CF", repeat=3):
            for add, alpha in [(True, -1.0), (False, 1.0)]:
                A = np.array(rng.standard_normal((m, k)), order=layout[0])
                B = np.array(rng.standard_normal((k, n)), order=layout[1])
                C0 = np.array(rng.standard_normal((m, n)), order=layout[2])
                want = C0.copy(order="K")
                if not add:
                    want[...] = np.nan
                oracle.matmul(want, add, A, B, alpha)
                bound = abs(alpha) * gemm_bound(A, B, k) + (2 * U) * np.abs(want) * 2
                dA, dB, dC = to_dev(A, cuda_dev), to_dev(B, cuda_dev), to_dev(C0.copy(order="K"), cuda_dev)
                if not add:
                    dC.fill_(float("nan"))
                la.matmul(dC, la.Accum.Add if add else la.Accum.Replace, dA, dB, alpha)
                got = dC.cpu().numpy()
                assert np.all(np.abs(got - want) <= bound), (m, n, k, layout, add, float(np.nanmax(np.abs(got - want))))
