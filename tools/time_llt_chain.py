"""Where the f64 LLT panel chain's time goes at the headline size (n = 16384, bench.py's input and call), in one run on
one card:
  * the card's name and power limit;
  * the chain pieces at the shapes the step uses, each run on an otherwise idle GPU: the diagonal-block LLT at 128 (one
    potf2), 256 and 512; the panel solve and the look-ahead column update (diagonal block: lower-triangular SYRK; below
    it: GEMM) at (rows, width) = (16000, 512), (8000, 256) and (6000, 128). For each: the call time with CUDA events over
    many calls (the LLT calls include the C ABI's status read-back), and the device time per call of every kernel it
    launched, from torch.profiler;
  * the step time of the schedule the FAER_B200_* variables in the environment select.
usage: python tools/time_llt_chain.py [out_dir] [tag]   (writes out_dir/llt_chain[_tag].json)"""
import json
import os
import re
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
tag = sys.argv[2] if len(sys.argv) > 2 else ""
n = 16384
dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
lib = faer_b200.load()
stream = torch.cuda.current_stream()
lib.faer_b200_set_stream(stream.cuda_stream)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def call_us(f, reps):
    f(); torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def kernels_us(f, reps):
    """device time per call of each kernel f launches (copies and memsets left out)"""
    f(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            f()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or "memcpy" in e.name.lower() or "memset" in e.name.lower():
            continue
        m = re.search(r"(\w+_kernel)\b", e.name)
        d = per.setdefault(m.group(1) if m else e.name[:80], {"us_per_call": 0.0, "launches_per_call": 0.0})
        d["us_per_call"] += (e.time_range.end - e.time_range.start) / reps
        d["launches_per_call"] += 1.0 / reps
    return per


def spd(m, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    G = torch.randn((m, m), dtype=torch.float64, device=dev, generator=g)
    return torch.addmm(m * torch.eye(m, dtype=torch.float64, device=dev), G, G.T).T  # column-major view


res = {"card": card(), "n": n, "env": {k: v for k, v in os.environ.items() if k.startswith("FAER_B200_")}, "isolated": {}}
iso = res["isolated"]
for w in (128, 256, 512):
    D0 = spd(w, w)
    D = D0.clone(memory_format=torch.preserve_format)
    f = lambda: (D.copy_(D0), la.cholesky_in_place(D))  # noqa: E731
    iso[f"diag_llt_{w}"] = {"call_us": call_us(f, 200), "kernels": kernels_us(f, 50)}
for rows, w in ((16000, 512), (8000, 256), (6000, 128)):
    L = torch.linalg.cholesky(spd(w, 7).T).T.contiguous().T  # lower factor, column-major
    B = torch.randn((w, rows), dtype=torch.float64, device=dev).T  # the panel below the diagonal block, column-major
    f = lambda: la.solve_lower_triangular_in_place(L, B.T)  # noqa: E731  (values drift; the time does not depend on them)
    iso[f"panel_trsm_{rows}x{w}"] = {"call_us": call_us(f, 50), "kernels": kernels_us(f, 20)}
    Wp = torch.randn((w, rows + w), dtype=torch.float64, device=dev).T
    Wj, Wb = Wp[:w], Wp[w:]
    Cd = torch.randn((w, w), dtype=torch.float64, device=dev).T
    Cb = torch.randn((w, rows), dtype=torch.float64, device=dev).T
    f = lambda: (la.matmul_triangular(Cd, 1, 1, Wj, 0, Wj.T, 0, -1.0), la.matmul(Cb, 1, Wb, Wj.T, -1.0))  # noqa: E731
    iso[f"col_update_{rows}x{w}"] = {"call_us": call_us(f, 50), "kernels": kernels_us(f, 20)}

A0 = spd(n, 1234)
A = A0.clone(memory_format=torch.preserve_format)
steps = []
for i in range(6):
    A.copy_(A0)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); la.cholesky_in_place(A); e1.record(); torch.cuda.synchronize()
    if i >= 2:
        steps.append(e0.elapsed_time(e1))
res["step_ms"] = {"min": min(steps), "median": sorted(steps)[len(steps) // 2], "all": steps}
print(json.dumps(res, indent=1))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, f"llt_chain{'_' + tag if tag else ''}.json"), "w") as fh:
    json.dump(res, fh, indent=1)
