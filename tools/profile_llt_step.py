"""Per-kernel breakdown of ONE f64 LLT step of the headline workload (n = 16384, bench.py's input and call) with
torch.profiler: device time per kernel name, summed over the step; how much of the step no kernel covers (exposed gaps);
per CUDA stream (the look-ahead driver's bulk-update stream and its high-priority panel stream), the busy time and the
kernel time per name, and the wall time during which only the panel stream is busy; the same split per block tier (the
512-wide head, the 256 tier and the 128 tail, told apart by their potf2 launches: 4, 2 and 1 per block column), with the
chain kernels' mean time per launch; and the largest trailing update (lower-triangular n = 16128, k = 256) timed on its
own with CUDA events. The FAER_B200_* variables in the environment select the schedule as in the library.
usage: python tools/profile_llt_step.py [out_dir]   (writes out_dir/llt_step_profile.json)"""
import json
import os
import re
import sys
import tempfile

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


def union(iv):
    out = []
    for s, e in sorted(iv):
        if out and s <= out[-1][1]:
            out[-1][1] = max(out[-1][1], e)
        else:
            out.append([s, e])
    return out


# per-stream split from the trace (the stream id is only exported there)
with tempfile.TemporaryDirectory() as td:
    path = os.path.join(td, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        trace = json.load(fh)
streams = {}
for ev in trace.get("traceEvents", []):
    if ev.get("cat") != "kernel":
        continue
    st = ev.get("args", {}).get("stream")
    m = re.search(r"(\w+_kernel)\b", ev["name"])
    name = m.group(1) if m else ev["name"][:80]
    d = streams.setdefault(st, {"iv": [], "kernels": {}})
    d["iv"].append((ev["ts"], ev["ts"] + ev["dur"]))
    k = d["kernels"].setdefault(name, {"ms": 0.0, "launches": 0})
    k["ms"] += ev["dur"] / 1e3
    k["launches"] += 1
# the bulk stream is the one with the most gemm time; any other stream counts as the panel chain
by_gemm = sorted(streams, key=lambda s: -streams[s]["kernels"].get("gemm_f64_ws_kernel", {"ms": 0})["ms"]
                 - streams[s]["kernels"].get("gemm_f64_kernel", {"ms": 0})["ms"])
per_stream = {}
if by_gemm:
    bulk = union(streams[by_gemm[0]]["iv"])
    panel = union([iv for s in by_gemm[1:] for iv in streams[s]["iv"]])
    # wall time in which the panel streams are busy and the bulk stream is not
    only_panel = 0.0
    for s, e in panel:
        cur = s
        for bs, be in bulk:
            if be <= cur or bs >= e:
                continue
            if bs > cur:
                only_panel += bs - cur
            cur = max(cur, be)
        if cur < e:
            only_panel += e - cur
    for i, s in enumerate(by_gemm):
        per_stream[f"{'bulk' if i == 0 else 'panel'}_stream_{s}"] = {
            "busy_ms": sum(e - b for b, e in union(streams[s]["iv"])) / 1e3,
            "kernels": dict(sorted(streams[s]["kernels"].items(), key=lambda kv: -kv[1]["ms"]))}
    per_stream["only_panel_busy_ms"] = only_panel / 1e3

    # per tier: potf2 launches in time order; the head has 16 block columns of 4, the 256 tier 8 of 2, the tail 1 each
    kev = [ev for ev in trace.get("traceEvents", []) if ev.get("cat") == "kernel"]
    tr0, tr1 = min(ev["ts"] for ev in kev), max(ev["ts"] + ev["dur"] for ev in kev)  # the trace's own clock
    potf2 = sorted(ev["ts"] for ev in kev if "potf2" in ev["name"])
    edges = [tr0, potf2[64], potf2[80], tr1] if len(potf2) == 128 else None

    def clip(iv, lo, hi):
        return [(max(s, lo), min(e, hi)) for s, e in iv if e > lo and s < hi]

    def length(iv):
        return sum(e - s for s, e in union(iv))

    def minus(a, b):  # length of union(a) not covered by union(b)
        return length(a) - length([(max(s, bs), min(e, be)) for s, e in union(a) for bs, be in union(b)
                                   if min(e, be) > max(s, bs)])

    if edges:
        tiers = {}
        all_iv = [iv for s in streams for iv in streams[s]["iv"]]
        for name, lo, hi in (("512", edges[0], edges[1]), ("256", edges[1], edges[2]), ("128_tail", edges[2], edges[3])):
            chain = {}
            for s in by_gemm[1:]:
                for ev in trace["traceEvents"]:
                    if ev.get("cat") != "kernel" or ev.get("args", {}).get("stream") != s or not lo <= ev["ts"] < hi:
                        continue
                    m = re.search(r"(\w+_kernel)\b", ev["name"])
                    d = chain.setdefault(m.group(1) if m else ev["name"][:80], {"ms": 0.0, "launches": 0})
                    d["ms"] += ev["dur"] / 1e3
                    d["launches"] += 1
            for d in chain.values():
                d["us_per_launch"] = d["ms"] * 1e3 / d["launches"]
            tiers[name] = {"wall_ms": (hi - lo) / 1e3,
                           "only_panel_busy_ms": minus(clip(panel, lo, hi), clip(bulk, lo, hi)) / 1e3,
                           "no_kernel_ms": (hi - lo - length(clip(all_iv, lo, hi))) / 1e3,
                           "panel_kernels": dict(sorted(chain.items(), key=lambda kv: -kv[1]["ms"]))}
        per_stream["tiers"] = tiers

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
res = {"n": n, "env": {k: v for k, v in os.environ.items() if k.startswith("FAER_B200_")},
       "step_ms": (t1 - t0) / 1e3, "kernel_busy_ms": busy / 1e3, "exposed_gap_ms": (t1 - t0 - busy) / 1e3,
       "kernels": per, "streams": per_stream,
       "largest_update": {"m": m, "k": k, "ms": best, "tflops": m * (m + 1.0) * k / (best * 1e-3) / 1e12}}
print(json.dumps(res, indent=1))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "llt_step_profile.json"), "w") as fh:
    json.dump(res, fh, indent=1)
