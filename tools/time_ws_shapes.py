"""Dev aid: the ws f64 GEMM, narrow (gemm_ws = 2, 128 x 64 tiles) and wide (3, 128 x 128 tiles), against the cp.async kernel
(0) on the trailing-update shapes of LLT / LU.
usage: python tools/time_ws_shapes.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402

dev = torch.device("cuda:0")
lib = faer_b200.load()
lib.faer_b200_set_stream(torch.cuda.current_stream().cuda_stream)


def best(f, reps=5):
    f(); torch.cuda.synchronize(); b = 1e30
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); f(); e1.record(); torch.cuda.synchronize(); b = min(b, e0.elapsed_time(e1))
    return b


# lower-triangular updates of the headline LLT (k = 512 / 256 / 128 by remaining order), and deeper ones; Add (accum 1)
# is the LLT's, Replace (accum 0) skips the old-tile load
for (n, k, accum) in [(16128, 128, 1), (16128, 256, 1), (16128, 512, 1), (16128, 768, 1), (16128, 1024, 1),
                      (16128, 128, 0), (16128, 256, 0), (16128, 512, 0), (16128, 1024, 0),
                      (12288, 256, 1), (10240, 512, 1), (8192, 256, 1), (4096, 256, 1), (1024, 256, 1), (6016, 128, 1),
                      (3072, 128, 1)]:
    P = torch.randn((k, n), dtype=torch.float64, device=dev).T
    Cm = torch.randn((n, n), dtype=torch.float64, device=dev).T
    line = f"SYRK(lower, {'Add' if accum else 'Replace'}) n={n} k={k}:"
    for mode in (0, 2, 3):
        lib.faer_b200_set_option(b"gemm_ws", mode)
        ms = best(lambda: la.matmul_triangular(Cm, 1, accum, P, 0, P.T, 0, -1.0))
        line += f"  mode {mode}: {ms:.3f} ms {n * n * k / ms / 1e9:.2f} TF"
    print(line, flush=True)
    del P, Cm
# rectangular: LU / GEMM updates, and the LLT panel chain's rows x 256 x 256 updates
for (m, n, k) in [(16384, 16384, 256), (16384, 16384, 512), (8192, 8192, 512), (16384, 512, 512), (16128, 256, 256),
                  (8192, 256, 256), (2048, 256, 256)]:
    L = torch.randn((k, m), dtype=torch.float64, device=dev).T
    U = torch.randn((n, k), dtype=torch.float64, device=dev).T
    Cm = torch.randn((n, m), dtype=torch.float64, device=dev).T
    line = f"update m={m} n={n} k={k}:"
    for mode in (0, 2, 3):
        lib.faer_b200_set_option(b"gemm_ws", mode)
        ms = best(lambda: la.matmul(Cm, 1, L, U, -1.0))
        line += f"  mode {mode}: {ms:.3f} ms {2.0 * m * n * k / ms / 1e9:.2f} TF"
    print(line, flush=True)
    del L, U, Cm
lib.faer_b200_set_option(b"gemm_ws", 1)
