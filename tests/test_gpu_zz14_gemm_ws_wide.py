"""GPU parity tests of the wide (128 x 128 tile, one CTA per SM) configuration of the TMA-fed warp-specialised f64 GEMM
(csrc/gemm_f64_ws.cuh), forced on with `gemm_ws` = 3, against the oracle: sizes that are not multiples of the tile,
contractions shorter and longer than one stage, rectangular / lower / upper destinations with their strict and unit
variants, Add and Replace, both operand layouts, destinations that TMA cannot address (the register epilogue for every
tile), and the untouched triangle of a triangular destination compared bit for bit, NaN sentinels included."""
import itertools

import numpy as np
import pytest

from test_gpu_parity import S_LOW, S_RECT, S_SLOW, S_SUP, S_ULOW, S_UP, S_UUP, U, gemm_bound, to_dev

pytestmark = pytest.mark.gpu

LOWERS = (S_LOW, S_SLOW, S_ULOW)


@pytest.fixture
def wide(fb):
    lib = fb.load()
    saved = lib.faer_b200_get_option(b"gemm_ws")
    assert lib.faer_b200_set_option(b"gemm_ws", 3) == 0
    yield lib
    lib.faer_b200_set_option(b"gemm_ws", saved)


def kept_mask(n, ds):
    sel = np.tril(np.ones((n, n), bool)) if ds in LOWERS else np.triu(np.ones((n, n), bool))
    if ds in (S_SLOW, S_SUP, S_ULOW, S_UUP):
        np.fill_diagonal(sel, False)
    return sel


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def test_wide_rect_vs_oracle(fb, oracle, cuda_dev, wide):
    la = fb.linalg
    rng = np.random.default_rng(140)
    n0 = wide.faer_b200_launch_count()
    for (m, n, k) in [(1, 129, 15), (127, 1000, 257), (129, 127, 1), (1000, 2049, 128), (2049, 1000, 600), (1000, 1000, 256)]:
        for lay_a, lay_b in itertools.product("CF", repeat=2):
            for add, alpha in [(False, 0.5), (True, -1.0), (True, 0.5)]:
                A = np.array(rng.standard_normal((m, k)), order=lay_a)
                B = np.array(rng.standard_normal((k, n)), order=lay_b)
                C0 = np.asfortranarray(rng.standard_normal((m, n)))
                want = C0.copy(order="F")
                if not add:
                    want[...] = np.nan
                oracle.matmul(want, add, A, B, alpha)
                dA, dB, dC = to_dev(A, cuda_dev), to_dev(B, cuda_dev), to_dev(C0, cuda_dev)
                if not add:
                    dC.fill_(float("nan"))
                la.matmul(dC, la.Accum.Add if add else la.Accum.Replace, dA, dB, alpha)
                got = dC.cpu().numpy()
                bound = abs(alpha) * gemm_bound(A, B, k) + 4 * U * np.abs(want)
                assert np.all(np.abs(got - want) <= bound), (m, n, k, lay_a, lay_b, add, alpha)
    assert wide.faer_b200_launch_count() > n0


@pytest.mark.parametrize("n,k", [(127, 15), (129, 257), (1000, 128), (1000, 1), (2049, 256), (2049, 600)])
def test_wide_triangular_vs_oracle(fb, oracle, cuda_dev, wide, n, k):
    """Every structure, Add and Replace; the untouched part (strict upper triangle of a lower dst, and the diagonal of the
    strict / unit variants) holds NaN sentinels and is compared bit for bit, inside diagonal tiles too."""
    import torch
    la = fb.linalg
    rng = np.random.default_rng(141 + n + k)
    for ds in (S_LOW, S_UP, S_SLOW, S_SUP, S_ULOW, S_UUP):
        sel = kept_mask(n, ds)
        for (lay_a, lay_b), (add, alpha) in zip(itertools.product("CF", repeat=2),
                                                [(True, -1.0), (False, 0.5), (True, 0.5), (False, -1.0)]):
            A = np.array(rng.standard_normal((n, k)), order=lay_a)
            B = np.array(rng.standard_normal((k, n)), order=lay_b)
            C0 = np.asfortranarray(rng.standard_normal((n, n)))
            C0[~sel] = np.nan
            want = C0.copy(order="F")
            oracle.matmul_triangular(want, ds, add, np.asfortranarray(A), S_RECT, np.asfortranarray(B), S_RECT, alpha)
            dA, dB, dC = to_dev(A, cuda_dev), to_dev(B, cuda_dev), to_dev(C0, cuda_dev)
            if not add:
                dC.masked_fill_(torch.from_numpy(sel).to(cuda_dev), float("nan"))
            la.matmul_triangular(dC, ds, la.Accum.Add if add else la.Accum.Replace, dA, S_RECT, dB, S_RECT, alpha)
            got = dC.cpu().numpy()
            assert np.array_equal(bits(got[~sel]), bits(C0[~sel])), (n, k, ds, lay_a, lay_b, add)
            bound = abs(alpha) * gemm_bound(A, B, k) + 4 * U * np.abs(want)
            assert np.all(np.abs(got - want)[sel] <= bound[sel]), (n, k, ds, lay_a, lay_b, add)


def test_wide_unaligned_destination_takes_register_epilogue(fb, oracle, cuda_dev, wide):
    """A dst whose base is not 16-byte aligned, or whose column stride is odd, cannot be addressed by TMA: every tile
    takes the register epilogue, with the same results and the same untouched entries."""
    import torch
    la = fb.linalg
    rng = np.random.default_rng(142)
    n, k = 1000, 256
    A = np.asfortranarray(rng.standard_normal((n, k)))
    dA = to_dev(A, cuda_dev)
    for ld, off in [(n + 1, 0), (n + 2, 1), (n + 3, 1)]:
        for ds in (S_RECT, S_LOW, S_SUP):
            sel = np.ones((n, n), bool) if ds == S_RECT else kept_mask(n, ds)
            buf = torch.from_numpy(rng.standard_normal(off + ld * n)).to(cuda_dev)
            dC = buf[off:off + ld * n].view(n, ld)[:, :n].T   # column-major n x n with column stride ld
            assert dC.stride() == (1, ld) and (dC.data_ptr() % 16 != 0 or ld % 2 == 1)
            C0 = dC.cpu().numpy().copy(order="F")
            want = C0.copy(order="F")
            if ds == S_RECT:
                oracle.matmul(want, True, A, A.T.copy(order="F"), -1.0)
                la.matmul(dC, la.Accum.Add, dA, dA.T, -1.0)
            else:
                oracle.matmul_triangular(want, ds, True, A, S_RECT, np.asfortranarray(A.T), S_RECT, -1.0)
                la.matmul_triangular(dC, ds, la.Accum.Add, dA, S_RECT, dA.T, S_RECT, -1.0)
            got = dC.cpu().numpy()
            assert np.array_equal(bits(got[~sel]), bits(C0[~sel])), (ld, off, ds)
            bound = gemm_bound(A, A.T, k) + 4 * U * np.abs(want)
            assert np.all(np.abs(got - want)[sel] <= bound[sel]), (ld, off, ds)


def test_wide_syrk_matches_narrow_and_cp_async(fb, cuda_dev, wide):
    """The LLT trailing update at the benchmark's shape (lower dst, rhs = lhs^T, k = 256): the wide configuration against the
    cp.async kernel on the same device data (the same products, summed in different orders), and the strict upper
    triangle untouched bit for bit."""
    import torch
    la = fb.linalg
    torch.manual_seed(14)
    n, k = 6016, 256
    A = torch.randn((k, n), dtype=torch.float64, device=cuda_dev).T
    C0 = torch.randn((n, n), dtype=torch.float64, device=cuda_dev).T
    outs = []
    for mode in (0, 3):
        assert wide.faer_b200_set_option(b"gemm_ws", mode) == 0
        Cm = C0.clone(memory_format=torch.preserve_format)
        la.matmul_triangular(Cm, S_LOW, la.Accum.Add, A, S_RECT, A.T, S_RECT, -1.0)
        outs.append(Cm)
    assert torch.equal(torch.triu(outs[1], 1).view(torch.int64), torch.triu(C0, 1).view(torch.int64))
    absprod = A.abs() @ A.abs().T
    assert bool((torch.tril(outs[0] - outs[1]).abs() <= 2 * k * 2 * U * absprod).all())
