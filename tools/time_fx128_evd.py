"""Times the double-double self-adjoint EVD (self_adjoint_evd_fx128 / _cx128) on device-resident operands, with the fx128 GEMM at
n = 4096 in the same run as the rate to compare against: the median of 3 calls after a warm-up, with CUDA events, and the card name
and power limit read in the same run. Writes profiles/r14_fx128_evd_timing.json (or the path given as the first argument).

Cases: fx128 at n = 1024 / 2048 / 4096 and cx128 at 2048, each values only and with vectors. Work model in dd multiply-adds:
(2/3) n^3 for the reduction, (2/3) n^3 for the divide-and-conquer merges and n^3 for the back-transform (vectors only; a cx128
multiply-add counts as 4 real ones), against the bound 0.77e12 dd multiply-adds per second (profiles/r03_f64_peaks.log / 20) and
this run's GEMM rate (a cx128 multiply-add counts as 4 real ones on both sides). A torch.profiler pass over one call splits its
kernel time into "reduction" (the tridiagonal reduction), "solve" (bisection, or divide and conquer with its merge GEMMs),
"back_transform" (D Z, the T-factor builds and the block-reflector products) and "other" (the copies and the extraction of the
tridiagonal), by the kernels that open and close each phase (see split)."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import faer_b200  # noqa: E402
from time_fx128 import BOUND, dd_tensor, timed  # noqa: E402


def split(lib, fn):
    """kernel time of one call by phase, from one torch.profiler trace. The phases run one after the other, so the library's
    kernels are assigned in start order by the kernels that open and close them: everything before the extraction of the
    tridiagonal is the reduction (except the copy of A), everything between it and the lift of Z (or the values' store) the
    solve, everything from the lift to the store of U the back-transform. This does not depend on every launch having a record:
    large traces can lose a few, and the row reports how many records the trace holds against the launches the library logged
    (faer_b200_launch_log_begin / _end)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    tags = np.zeros(1 << 20, dtype=np.int8)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lib.faer_b200_launch_log_begin(tags.ctypes.data, tags.size)
        fn()
        torch.cuda.synchronize()
        count = lib.faer_b200_launch_log_end()
    kernels = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "fb::" in e.name),
                     key=lambda e: e.time_range.start)
    cats = {"reduction": 0.0, "solve": 0.0, "back_transform": 0.0, "other": 0.0}
    phase = "reduction"
    for e in kernels:
        name, ms = e.name, e.time_range.elapsed_us() / 1e3
        if "ed_copy_kernel" in name or "ed_extract_kernel" in name or "ed_values_out_kernel" in name or "ed_store_kernel" in name:
            cats["other"] += ms
            if "ed_extract_kernel" in name:
                phase = "solve"
            continue
        if "ed_lift_kernel" in name:
            phase = "back_transform"
        cats[phase] += ms
    missing = {k: v for k, v in cats.items() if v == 0.0 and k != "back_transform"}
    assert not missing, f"phase markers not found in the trace: {missing}"
    return {**cats, "kernel_records": len(kernels), "logged_launches": int(count)}


def main() -> int:
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r14_fx128_evd_timing.json")
    dev = torch.device("cuda:0")
    capi, lib = faer_b200.capi, faer_b200.load()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    par, mem = capi.par_default(), capi.MemAlloc(None, 0)
    rng = np.random.default_rng(0)
    rows = []
    n = 4096
    A, B = dd_tensor(rng.standard_normal((n, n)), False, dev), dd_tensor(rng.standard_normal((n, n)), False, dev)
    Cm = torch.zeros_like(A)
    alpha = np.array([1.0, 0.0])
    ms = timed(lambda: lib.libfaer_v0_23_matmul_fx128(capi.mat_mut(capi.DDTensor(Cm, False)), 0, capi.mat_ref(capi.DDTensor(A, False)),
                                                      capi.mat_ref(capi.DDTensor(B, False)), alpha.ctypes.data, par))
    gemm_rate = n ** 3 / (ms * 1e-3)
    rows.append({"kind": "fx128", "op": "gemm", "n": n, "ms": ms, "dd_madd_per_s": gemm_rate})
    print(rows[-1], flush=True)
    del A, B, Cm
    for suf, cx, n in (("fx128", False, 1024), ("fx128", False, 2048), ("fx128", False, 4096), ("cx128", True, 2048)):
        w = 4 if cx else 1
        X = rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0)
        X = X + np.conj(X.T)
        Ad = dd_tensor(X, cx, dev)
        S = torch.zeros((n, 2, 2) if cx else (n, 2), dtype=torch.float64, device=dev)
        p = getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}")()
        for vectors in (False, True):
            Ud = torch.zeros_like(Ad) if vectors else None

            def evd():
                uv = capi.mat_mut(capi.DDTensor(Ud, cx)) if vectors else capi.MatMut(None, 0, 0, 0, 0)
                st = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_{suf}")(capi.mat_ref(capi.DDTensor(Ad, cx)), uv,
                                                                           capi.VecMut(S.data_ptr(), n, 1), par, mem, p)
                assert st.tag == 0
            ms = timed(evd)
            madd = w * (2 * n ** 3 / 3 + ((2 * n ** 3 / 3 + n ** 3) if vectors else 0))
            row = {"kind": suf, "n": n, "vectors": vectors, "ms": ms, "model_dd_madd": madd,
                   "dd_madd_per_s": madd / (ms * 1e-3), "split_ms": split(lib, evd)}
            row["frac_of_bound"] = row["dd_madd_per_s"] / BOUND
            row["frac_of_gemm_rate"] = row["dd_madd_per_s"] / gemm_rate
            rows.append(row)
            print(row, flush=True)
            del Ud
        del Ad, S
    big = next(r for r in rows if r.get("vectors") and r["n"] == 4096)
    doc = {"card": q, "bound_dd_madd_per_s": BOUND, "gemm_dd_madd_per_s": gemm_rate,
           "how": "CUDA events, median of 3 calls after one warm-up, device operands; split_ms from one torch.profiler pass",
           "rows": rows, "aims_met": {"fx128_4096_with_vectors_under_3_s": big["ms"] < 3000.0}}
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(doc, open(out, "w"), indent=1)
    print(json.dumps(doc["aims_met"]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
