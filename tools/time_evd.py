"""Timing of the general eigendecomposition (`evd_*`) on device-resident Gaussian inputs, values only and with both eigenvector
sets, next to `self_adjoint_evd` with vectors at the same size. Writes profiles/r10_evd_timing.json (or the path given) with the
card name and power limit. Each figure is the median of `--reps` calls after one warm-up call, CUDA events around the call; the
sweep and window counts are the library's own. For one size a separate profiled call splits the kernel time by stage
(torch.profiler, CUDA activity): Hessenberg + Z, window kernels, off-window GEMMs and their copies, eigenvectors."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402


def gaussian(n, dtype):
    g = torch.Generator(device="cuda").manual_seed(n)
    return torch.randn(n, n, dtype=dtype, device="cuda", generator=g).t().contiguous().t()


def outputs(n, dtype, vectors):
    S, S_im = (torch.zeros(n, dtype=dtype, device="cuda") for _ in range(2))
    UL, UR = ((torch.zeros(n, n, dtype=dtype, device="cuda").t() for _ in range(2)) if vectors else (None, None))
    return S, (None if dtype.is_complex else S_im), UL, UR


def timed(fn, reps):
    ts = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts[1:]))


def profile_split(n, dtype):
    from torch.profiler import ProfilerActivity, profile

    A = gaussian(n, dtype)
    out = outputs(n, dtype, True)
    la.evd(A, *out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        la.evd(A, *out)
        torch.cuda.synchronize()
    fam = {"window_kernels": 0.0, "scan": 0.0, "gemm": 0.0, "copies": 0.0, "eigenvectors": 0.0, "hessenberg_and_other": 0.0}
    count = {k: 0 for k in fam}
    for ev in prof.key_averages():
        us = getattr(ev, "self_device_time_total", None)
        if us is None:
            us = getattr(ev, "self_cuda_time_total", 0)
        if not us:
            continue
        name = ev.key
        k = ("window_kernels" if "schur_window" in name else "scan" if "schur_scan" in name else
             "eigenvectors" if "evd_from_schur" in name or "schur_norm" in name else "gemm" if "gemm" in name else
             "copies" if "Memcpy" in name or "memcpy" in name else "hessenberg_and_other")
        fam[k] += us / 1e3
        count[k] += ev.count
    return {"n": n, "dtype": str(dtype).replace("torch.", ""), "kernel_ms": {k: round(v, 2) for k, v in fam.items()}, "launches": count}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r10_evd_timing.json"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="*", default=[1024, 2048, 4096])
    ap.add_argument("--complex-size", type=int, default=2048)
    ap.add_argument("--profile-size", type=int, default=1024)
    a = ap.parse_args()
    lib = faer_b200.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    rows = []
    counts = (ctypes.c_longlong * 2)()
    for n, dt in [(n, torch.float64) for n in a.sizes] + ([(a.complex_size, torch.complex128)] if a.complex_size else []):
        A = gaussian(n, dt)
        for vectors in (False, True):
            out = outputs(n, dt, vectors)
            ms = timed(lambda: la.evd(A, *out), a.reps)
            lib.faer_b200_evd_last_sweep_counts(counts)
            rows.append({"op": "evd", "n": n, "dtype": str(dt).replace("torch.", ""), "vectors": "both" if vectors else "none",
                         "ms": round(ms, 1), "sweeps": counts[0], "windows": counts[1]})
            print(json.dumps(rows[-1]), flush=True)
        H = ((A + A.mH) / 2).t().contiguous().t()
        S = torch.zeros(n, dtype=dt, device="cuda")
        U = torch.zeros(n, n, dtype=dt, device="cuda").t()
        rows.append({"op": "self_adjoint_evd", "n": n, "dtype": str(dt).replace("torch.", ""), "vectors": "yes",
                     "ms": round(timed(lambda: la.self_adjoint_evd(H, S, U), a.reps), 1)})
        print(json.dumps(rows[-1]), flush=True)
    split = None
    if a.profile_size:
        try:
            split = profile_split(a.profile_size, torch.float64)
            print(json.dumps(split), flush=True)
        except Exception as e:  # the timings above stand without the split
            print("profile split failed:", repr(e), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump({"card_and_power_limit": card, "rows": rows, "split_both_vectors": split}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
