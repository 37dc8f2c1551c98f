"""Timing of the Bunch-Kaufman LBL^H (`lblt_*`) on device-resident Gaussian symmetric inputs, next to the LDLT (on a diagonally
shifted input it can factor) and the pivoted / unpivoted LLT (on a positive definite input) of the same size. Writes
profiles/r09_lblt_timing.json (or the path given) with the card name and power limit. Each figure is the median of `--reps`
calls, CUDA events around the call. For f64 n = 16384 with the default parameters, a separate profiled call splits the kernel
time into panel launches, trailing products (GEMM), left-column swaps and the rest (torch.profiler, CUDA activity)."""
import argparse
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

PIV = {"partial": 0, "partial_diag": 1, "rook": 2, "rook_diag": 3, "full": 4}


def sym(n, dtype, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(n)
    X = torch.randn(n, n, dtype=dtype, device="cuda", generator=g)
    A = (X + X.mH) / 2 + shift * torch.eye(n, dtype=dtype, device="cuda")
    return A.t().contiguous().t()


def timed(fn, make, reps):
    ts = []
    for _ in range(reps + 1):
        args = make()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*args)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts[1:]))


def lblt_case(n, dtype, piv, bs, reps):
    def make():
        A = sym(n, dtype)
        return (A, torch.zeros(n, dtype=dtype, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda"),
                torch.zeros(n, dtype=torch.int64, device="cuda"))

    params = la.lblt_params_default()
    params.pivoting = PIV[piv]
    params.block_size = bs

    def fn(A, s, p, pi):
        la.lblt_in_place(A, s, p, pi, params=params)

    return timed(fn, make, reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r09_lblt_timing.json"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="f64 n = 8192 default parameters only")
    a = ap.parse_args()
    faer_b200.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    rows = []
    cases = [(8192, torch.float64, "partial_diag", 64)]
    if not a.quick:
        cases += [(16384, torch.float64, "partial_diag", 64), (8192, torch.float64, "partial_diag", 128),
                  (16384, torch.float64, "partial_diag", 128), (8192, torch.float64, "rook", 64), (16384, torch.float64, "rook", 64),
                  (4096, torch.float64, "full", 64), (8192, torch.float64, "full", 64), (8192, torch.float32, "partial_diag", 64),
                  (4096, torch.complex128, "partial_diag", 64)]
    for n, dt, piv, bs in cases:
        ms = lblt_case(n, dt, piv, bs, a.reps)
        row = {"op": "lblt", "n": n, "dtype": str(dt).replace("torch.", ""), "pivoting": piv, "block_size": bs, "ms": round(ms, 2)}
        if piv == "full":
            row["algorithmic_TBps"] = round(2 * 8 * sum((n - k) ** 2 / 2 for k in range(n)) / (ms * 1e-3) / 1e12, 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    for n in sorted({c[0] for c in cases if c[1] == torch.float64}):
        def make_ldlt():
            return (sym(n, torch.float64, shift=2.0 * np.sqrt(n)),)

        def make_spd():
            return (sym(n, torch.float64, shift=3.0 * np.sqrt(n)),)  # Gershgorin-free margin: eigenvalues of the Gaussian part < 2 sqrt(n)

        def make_piv():
            A = make_spd()[0]
            return A, torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda")

        for op, fn, make in (("ldlt", lambda A: la.ldlt_in_place(A), make_ldlt), ("llt", lambda A: la.cholesky_in_place(A), make_spd),
                             ("piv_llt", lambda A, p, pi: la.piv_llt_in_place(A, p, pi), make_piv)):
            rows.append({"op": op, "n": n, "dtype": "float64", "ms": round(timed(fn, make, a.reps), 2)})
            print(json.dumps(rows[-1]), flush=True)
    split = None
    if not a.quick:
        try:
            split = profile_split(16384)
        except Exception as e:  # the timings above stand without the split
            print("profile split failed:", repr(e), flush=True)
    if split:
        print(json.dumps(split), flush=True)
    json.dump({"card_and_power_limit": card, "rows": rows, "split_f64_16384_default": split}, open(a.out, "w"), indent=1)


def profile_split(n):
    """Kernel time of one f64 lblt_in_place call (default parameters) by kernel family, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    A = sym(n, torch.float64)
    s = torch.zeros(n, dtype=torch.float64, device="cuda")
    p, pi = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(2))
    la.lblt_in_place(A.clone(), s.clone(), p, pi)  # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0.record()
        la.lblt_in_place(A, s, p, pi)
        e1.record()
        torch.cuda.synchronize()
    fam = {"panel": 0.0, "trailing_gemm": 0.0, "left_swaps": 0.0, "right_looking_tail": 0.0, "other": 0.0}
    count = {k: 0 for k in fam}
    for ev in prof.key_averages():
        us = getattr(ev, "self_device_time_total", None)
        if us is None:
            us = getattr(ev, "self_cuda_time_total", 0)
        if not us:
            continue
        name = ev.key
        k = ("panel" if "lblt_panel_kernel" in name else "right_looking_tail" if "lblt_rl_kernel" in name else
             "left_swaps" if "laswp" in name else "trailing_gemm" if "gemm" in name else "other")
        fam[k] += us / 1e3
        count[k] += ev.count
    return {"n": n, "wall_ms_profiled": round(e0.elapsed_time(e1), 2), "kernel_ms": {k: round(v, 2) for k, v in fam.items()},
            "launches": count}


if __name__ == "__main__":
    main()
