"""Per-kernel breakdown of ONE f64 LLT step of the headline workload (n = 16384, bench.py's input and call) with
torch.profiler: device time per kernel name, summed over the step; how much of the step no kernel covers (exposed gaps);
and the largest trailing update (lower-triangular n = 16128, k = 256) timed on its own with CUDA events.
usage: python tools/profile_llt_step.py [out_dir]   (writes out_dir/llt_step_profile.json)"""
import json
import os
import re
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import faer_b200  # noqa: E402
from faer_b200 import linalg as la  # noqa: E402

n = 16384
out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
lib = faer_b200.load()
stream = torch.cuda.current_stream()
lib.faer_b200_set_stream(stream.cuda_stream)

torch.manual_seed(1234)
G = torch.randn((n, n), dtype=torch.float64, device=dev)
A0 = torch.addmm(n * torch.eye(n, dtype=torch.float64, device=dev), G, G.T).T
del G
A = A0.clone(memory_format=torch.preserve_format)
for _ in range(2):
    A.copy_(A0); la.cholesky_in_place(A)
A.copy_(A0)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    la.cholesky_in_place(A)
    torch.cuda.synchronize()

kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
           and "memset" not in e.name.lower()]
spans = sorted((e.time_range.start, e.time_range.end) for e in kernels)
t0, t1 = spans[0][0], max(s[1] for s in spans)
busy, cur_s, cur_e = 0.0, None, None
for s, e in spans:
    if cur_e is None or s > cur_e:
        if cur_e is not None:
            busy += cur_e - cur_s
        cur_s, cur_e = s, e
    else:
        cur_e = max(cur_e, e)
busy += cur_e - cur_s
per = {}
for e in kernels:
    m = re.search(r"(\w+_kernel)\b", e.name)
    name = m.group(1) if m else e.name[:80]
    d = per.setdefault(name, {"ms": 0.0, "launches": 0})
    d["ms"] += (e.time_range.end - e.time_range.start) / 1e3
    d["launches"] += 1
per = dict(sorted(per.items(), key=lambda kv: -kv[1]["ms"]))

# the largest trailing update on its own: dst(lower, 16128^2) -= P P^T, P 16128 x 256 (the shape of the first block step)
m, k = n - 256, 256
P = torch.randn((k, m), dtype=torch.float64, device=dev).T
Cm = torch.randn((m, m), dtype=torch.float64, device=dev).T
f = lambda: la.matmul_triangular(Cm, 1, 1, P, 0, P.T, 0, -1.0)
f(); torch.cuda.synchronize()
best = 1e30
for _ in range(10):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); f(); e1.record(); torch.cuda.synchronize()
    best = min(best, e0.elapsed_time(e1))
res = {"n": n, "step_ms": (t1 - t0) / 1e3, "kernel_busy_ms": busy / 1e3, "exposed_gap_ms": (t1 - t0 - busy) / 1e3,
       "kernels": per,
       "largest_update": {"m": m, "k": k, "ms": best, "tflops": m * (m + 1.0) * k / (best * 1e-3) / 1e12}}
print(json.dumps(res, indent=1))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "llt_step_profile.json"), "w") as fh:
    json.dump(res, fh, indent=1)
