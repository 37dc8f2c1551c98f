"""Dev aid: device-resident full-pivoting LU (full_piv_lu_in_place) against the partial-pivoting LU (lu_in_place) of the same
Gaussian inputs, alternated in one process: f64 4096^2 and 8192^2, f32 8192^2, c64 4096^2, plus the L2-resident f64 1024^2 that
gives the fixed cost per step. Per case: the call time from CUDA events, the persistent kernel's time from torch.profiler and the
rest of the call, the algorithmic traffic of the rank-one updates, 2 * s * sum_k (m - k - 1)(n - k - 1) bytes (s = the scalar's
size), and the TB/s it implies. Prints the card, its power limit and SM clock, then one JSON line per case; --out also writes the
whole document to a file.
usage: python tools/time_full_piv_lu.py [--reps 2] [--out FILE]"""
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
    return 2 * s * sum((m - k - 1) * (n - k - 1) for k in range(size))


def kernel_ms(calls):
    """Device time of the persistent kernel of each call, in order, from ONE profiler session (each call launches it once)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls:
            fn()
            torch.cuda.synchronize()
    evs = sorted((ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
                  and "full_piv_lu_kernel" in ev.name), key=lambda ev: ev.time_range.start)
    return [ev.device_time / 1e3 for ev in evs]


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
    cases = ((torch.float64, 1024), (torch.float64, 4096), (torch.float64, 8192), (torch.float32, 8192), (torch.complex64, 4096))
    for dtype, n in cases:
        A0 = colmajor(n, n, dtype, dev, 7)
        A = torch.empty_like(A0.T).T
        ps = [torch.empty(n, dtype=torch.int64, device=dev) for _ in range(4)]
        fp_ms, lu_ms, info = [], [], None
        for rep in range(args.reps + 1):  # rep 0 warms up both paths
            A.copy_(A0)
            t, info = time_once(lambda: la.full_piv_lu_in_place(A, *ps))
            if rep:
                fp_ms.append(t)
            A.copy_(A0)
            t, _ = time_once(lambda: la.lu_in_place(A, ps[0], ps[1]))
            if rep:
                lu_ms.append(t)
        tb = traffic_bytes(n, n, A0.element_size())
        best = min(fp_ms)
        run = {"dtype": str(dtype).replace("torch.", ""), "m": n, "n": n, "transpositions": info.transposition_count,
               "full_piv_lu_ms": fp_ms, "partial_piv_lu_ms": lu_ms, "algorithmic_bytes": tb,
               "call_tb_per_s": tb / (best / 1e3) / 1e12, "bound_ms_at_3.35_tb_per_s": tb / 3.35e12 * 1e3}
        doc["runs"].append(run)
        print(json.dumps(run), flush=True)
        del A, A0

    def one_call(dtype, n):
        def fn():
            A = colmajor(n, n, dtype, dev, 7).clone(memory_format=torch.preserve_format)
            ps = [torch.empty(n, dtype=torch.int64, device=dev) for _ in range(4)]
            torch.cuda.synchronize()
            la.full_piv_lu_in_place(A, *ps)
        return fn

    kms = kernel_ms([one_call(dtype, n) for dtype, n in cases])
    if len(kms) != len(cases):
        doc["profile_error"] = f"{len(kms)} kernel records for {len(cases)} calls"
        kms = []
    for run, k in zip(doc["runs"], kms):
        best = min(run["full_piv_lu_ms"])
        run.update({"kernel_ms": k, "rest_of_call_ms": best - k, "kernel_tb_per_s": run["algorithmic_bytes"] / (k / 1e3) / 1e12,
                    "kernel_us_per_step": k * 1e3 / run["n"]})
        print(json.dumps({k_: run[k_] for k_ in ("dtype", "n", "kernel_ms", "rest_of_call_ms", "kernel_tb_per_s",
                                                  "kernel_us_per_step")}), flush=True)
    doc["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
