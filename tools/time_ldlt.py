"""Dev aid: device-resident f64 LDLT (ldlt_in_place) at n = 4096 and 8192. Its trailing updates are `spicy_matmul`
launches of the ws f64 GEMM (k = 128, lower destination), so this times that path end to end.
usage: python tools/time_ldlt.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402

dev = torch.device("cuda:0")
lib = faer_b200.load()
lib.faer_b200_set_stream(torch.cuda.current_stream().cuda_stream)

for n in (4096, 8192):
    torch.manual_seed(7)
    G = torch.randn((n, n), dtype=torch.float64, device=dev)
    A0 = torch.addmm(n * torch.eye(n, dtype=torch.float64, device=dev), G, G.T).T  # symmetric, column-major view
    del G
    A = A0.clone(memory_format=torch.preserve_format)
    best = 1e30
    for it in range(6):
        A.copy_(A0)
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); la.ldlt_in_place(A); e1.record(); torch.cuda.synchronize()
        if it:  # the first call warms up
            best = min(best, e0.elapsed_time(e1))
    print(f"LDLT f64 n={n}: {best:.3f} ms {n ** 3 / 3 / best / 1e9:.2f} TF (n^3/3 flop), |D| sum {float(A.diagonal().abs().sum()):.6e}",
          flush=True)
    del A, A0
