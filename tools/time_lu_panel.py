"""Dev aid: the LU panel chain in isolation — tall m x w panels through the recursive driver (non-square input => lu_rec on the
current stream, on the grid-barrier panel kernel: the cluster kernels and the fused sub-panel run only inside the
partitioned look-ahead drivers). usage: python tools/time_lu_panel.py [w ...]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402

dev = torch.device("cuda:0")
lib = faer_b200.load()
lib.faer_b200_set_stream(torch.cuda.current_stream().cuda_stream)
ws = [int(x) for x in sys.argv[1:]] or [128, 512]
ms = [int(x) for x in os.environ.get("PANEL_ROWS", "32768,16384,8192,2048,512").split(",")]
for w in ws:
    for m in ms:
        A0 = torch.randn((w, m), dtype=torch.float64, device=dev).T
        A = A0.clone(memory_format=torch.preserve_format)
        p = torch.zeros(m, dtype=torch.int64, device=dev); pi = torch.zeros(m, dtype=torch.int64, device=dev)

        def run():
            A.copy_(A0); la.lu_in_place(A, p, pi)
        run(); torch.cuda.synchronize()
        l0 = lib.faer_b200_launch_count(); run(); nl = lib.faer_b200_launch_count() - l0
        best = 1e30
        for _ in range(3):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); run(); e1.record(); torch.cuda.synchronize(); best = min(best, e0.elapsed_time(e1))
        print(f"panel {m} x {w}: {best:.3f} ms  {1e3 * best / w:.2f} us/column  ({nl} launches)", flush=True)
