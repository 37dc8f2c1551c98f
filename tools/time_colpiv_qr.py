"""Dev aid: device-resident column-pivoted QR (colpiv_qr_in_place) against the unpivoted QR (qr_in_place) on the same Gaussian
inputs, alternated in one process: f64 4096^2 and 8192^2, c64 4096^2, f32 65536 x 4096. Reports the algorithmic traffic of the
BLAS-2 column loop, 2 * s * sum_k (m - k)(n - k) bytes (s = the scalar's size), and the TB/s it implies, then a torch.profiler
split of one f64 8192^2 factorization: the persistent kernel, the T-block GEMMs, the rest. Prints the card, its power limit and SM
clock, then one JSON line per configuration and one for the split; --out also writes the whole document to a file.
usage: python tools/time_colpiv_qr.py [--reps 2] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True).strip()
    except Exception as e:  # pragma: no cover
        out = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": out}


def time_once(fn):
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def colmajor(m, n, dtype, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn((n, m), dtype=dtype, device=dev, generator=g).T


def traffic_bytes(m, n, s):
    size = min(m, n)
    return 2 * s * sum((m - k) * (n - k) for k in range(size))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = faer_b200.load()
    lib.faer_b200_set_stream(torch.cuda.current_stream().cuda_stream)
    doc = {"card": card(), "runs": []}
    print(doc["card"], flush=True)
    for dtype, m, n in ((torch.float64, 4096, 4096), (torch.float64, 8192, 8192), (torch.complex128, 4096, 4096),
                        (torch.float32, 65536, 4096)):
        A0 = colmajor(m, n, dtype, dev, 7)
        A = torch.empty_like(A0.T).T
        bs = la.qr_recommended_block_size(m, n)
        H = torch.zeros((min(m, n), bs), dtype=dtype, device=dev).T
        p = torch.empty(n, dtype=torch.int64, device=dev)
        pi = torch.empty(n, dtype=torch.int64, device=dev)
        cp_ms, qr_ms, info = [], [], None
        for rep in range(args.reps + 1):  # rep 0 warms up both paths
            A.copy_(A0)
            t, info = time_once(lambda: la.colpiv_qr_in_place(A, H, p, pi))
            if rep:
                cp_ms.append(t)
            A.copy_(A0)
            t, _ = time_once(lambda: la.qr_in_place(A, H))
            if rep:
                qr_ms.append(t)
        s = A0.element_size()
        tb = traffic_bytes(m, n, s)
        run = {"dtype": str(dtype).replace("torch.", ""), "m": m, "n": n, "block_size": bs,
               "transpositions": info.transposition_count, "colpiv_qr_ms": cp_ms, "qr_ms": qr_ms,
               "algorithmic_bytes": tb, "colpiv_tb_per_s": tb / (min(cp_ms) / 1e3) / 1e12,
               "bound_ms_at_3.35_tb_per_s": tb / 3.35e12 * 1e3}
        doc["runs"].append(run)
        print(json.dumps(run), flush=True)
        del A, A0, H

    m = n = 8192
    A0 = colmajor(m, n, torch.float64, dev, 11)
    A = A0.clone(memory_format=torch.preserve_format)
    bs = la.qr_recommended_block_size(m, n)
    H = torch.zeros((n, bs), dtype=torch.float64, device=dev).T
    p = torch.empty(n, dtype=torch.int64, device=dev)
    pi = torch.empty(n, dtype=torch.int64, device=dev)
    la.colpiv_qr_in_place(A, H, p, pi)
    A.copy_(A0)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        la.colpiv_qr_in_place(A, H, p, pi)
        torch.cuda.synchronize()
    groups = {"column_loop_kernel": 0.0, "t_blocks": 0.0, "other": 0.0}
    counts = dict.fromkeys(groups, 0)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        key = "column_loop_kernel" if "colpiv_qr_kernel" in ev.name else "t_blocks" if "gemm" in ev.name.lower() else "other"
        groups[key] += ev.device_time / 1e3
        counts[key] += 1
    split = {"dtype": "float64", "m": m, "n": n, "ms": groups, "launches": counts}
    doc["profile_f64_8192"] = split
    print(json.dumps(split), flush=True)
    doc["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
