"""Dev aid: device-resident pivoted Cholesky (piv_llt_in_place) against the unpivoted LLT (cholesky_in_place) on the same
well-conditioned Gram matrices, alternated in one process: f64 at n = 4096, 8192, 16384 and f32 at n = 8192. Then a
torch.profiler split of one f64 n = 16384 pivoted factorization: panel kernel, trailing-update GEMMs, row swaps, the rest.
Prints the card, its power limit and SM clock, then one JSON line per configuration and one for the split; --out also writes the
whole document to a file.
usage: python tools/time_piv_llt.py [--reps 3] [--out FILE]"""
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


def gram(n, dtype, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    G = torch.randn((n, 2 * n), dtype=dtype, device=dev, generator=g)
    A = (G @ G.T) / (2 * n)  # eigenvalues within a factor 34
    del G
    return A.T.contiguous().T  # column-major view


def time_once(fn):
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = faer_b200.load()
    lib.faer_b200_set_stream(torch.cuda.current_stream().cuda_stream)
    doc = {"card": card(), "runs": []}
    print(doc["card"], flush=True)
    for dtype, n in ((torch.float64, 4096), (torch.float64, 8192), (torch.float64, 16384), (torch.float32, 8192)):
        A0 = gram(n, dtype, dev, 7)
        A = torch.empty_like(A0.T).T
        p = torch.empty(n, dtype=torch.int64, device=dev)
        pi = torch.empty(n, dtype=torch.int64, device=dev)
        piv_ms, llt_ms, info = [], [], None
        for rep in range(args.reps + 1):  # rep 0 warms up both paths
            A.copy_(A0)
            t, info = time_once(lambda: la.piv_llt_in_place(A, p, pi))
            if rep:
                piv_ms.append(t)
            A.copy_(A0)
            t, _ = time_once(lambda: la.cholesky_in_place(A))
            if rep:
                llt_ms.append(t)
        run = {"dtype": str(dtype).replace("torch.", ""), "n": n, "rank": info.rank, "transpositions": info.transposition_count,
               "piv_llt_ms": piv_ms, "llt_ms": llt_ms, "ratio_best": min(piv_ms) / min(llt_ms),
               "piv_llt_tflops_n3_over_3": n ** 3 / 3 / min(piv_ms) / 1e9}
        doc["runs"].append(run)
        print(json.dumps(run), flush=True)
        del A, A0

    # kernel split of one f64 n = 16384 pivoted factorization
    n = 16384
    A0 = gram(n, torch.float64, dev, 11)
    A = A0.clone(memory_format=torch.preserve_format)
    p = torch.empty(n, dtype=torch.int64, device=dev)
    pi = torch.empty(n, dtype=torch.int64, device=dev)
    la.piv_llt_in_place(A, p, pi)
    A.copy_(A0)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        la.piv_llt_in_place(A, p, pi)
        torch.cuda.synchronize()
    groups = {"panel": 0.0, "trailing_gemm": 0.0, "row_swaps": 0.0, "other": 0.0}
    counts = dict.fromkeys(groups, 0)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name
        key = ("panel" if "piv_llt_panel" in name else "row_swaps" if "laswp" in name
               else "trailing_gemm" if "gemm" in name.lower() else "other")
        groups[key] += ev.device_time / 1e3
        counts[key] += 1
    split = {"n": n, "ms": groups, "launches": counts}
    doc["profile_f64_16384"] = split
    print(json.dumps(split), flush=True)
    doc["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)

if __name__ == "__main__":
    main()
