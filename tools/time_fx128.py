"""Times the double-double (fx128 / cx128) GEMM, LLT and partial-pivoting LU at n = 1024 / 2048 / 4096 on device-resident
operands: the median of several calls after a warm-up, with CUDA events, and the card name and power limit read in the same run.
Writes profiles/r11_fx128_timing.json (or the path given as the first argument).
Rate: dd multiply-adds per second (GEMM n^3, LLT n^3 / 3, LU 2 n^3 / 3; a cx128 multiply-add counts as 4 real ones), compared with the
bound 15.4e12 FP64 instructions per second (profiles/r03_f64_peaks.log) / 20 instructions per real dd multiply-add."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import faer_b200  # noqa: E402

BOUND = 15.4e12 / 20


def dd_tensor(x, cx, dev):
    t = torch.zeros(x.shape + ((2, 2) if cx else (2,)), dtype=torch.float64, device=dev)
    if cx:
        t[..., 0, 0], t[..., 1, 0] = torch.from_numpy(x.real).to(dev), torch.from_numpy(x.imag).to(dev)
    else:
        t[..., 0] = torch.from_numpy(x).to(dev)
    return t


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main() -> int:
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r11_fx128_timing.json")
    dev = torch.device("cuda:0")
    capi, lib = faer_b200.capi, faer_b200.load()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    par, mem = capi.par_default(), capi.MemAlloc(None, 0)
    rng = np.random.default_rng(0)
    rows = []
    for suf, cx in (("fx128", False), ("cx128", True)):
        w = 4 if cx else 1
        alpha = np.array([1.0, 0.0, 0.0, 0.0] if cx else [1.0, 0.0])
        for n in (1024, 2048, 4096):
            g = lambda: rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cx else 0)
            A, B = dd_tensor(g(), cx, dev), dd_tensor(g(), cx, dev)
            Cm = torch.zeros_like(A)
            ms = timed(lambda: getattr(lib, f"libfaer_v0_23_matmul_{suf}")(capi.mat_mut(capi.DDTensor(Cm, cx)), 0,
                                                                          capi.mat_ref(capi.DDTensor(A, cx)),
                                                                          capi.mat_ref(capi.DDTensor(B, cx)), alpha.ctypes.data, par))
            rows.append({"kind": suf, "op": "gemm", "n": n, "ms": ms, "dd_madd_per_s": w * n ** 3 / (ms * 1e-3)})
            G = g()
            S = dd_tensor(G @ G.conj().T / n + np.eye(n), cx, dev)
            W = torch.empty_like(S)
            p = getattr(lib, f"libfaer_v0_23_LltParams_{suf}")()

            def llt():
                W.copy_(S)
                st = getattr(lib, f"libfaer_v0_23_llt_factor_in_place_{suf}")(capi.mat_mut(capi.DDTensor(W, cx)),
                                                                              capi.LltRegularization(None, None), par, mem, p)
                assert st.tag == 0
            ms = timed(llt)
            rows.append({"kind": suf, "op": "llt", "n": n, "ms": ms, "dd_madd_per_s": w * n ** 3 / 3 / (ms * 1e-3)})
            pf, pb = torch.zeros(n, dtype=torch.int64, device=dev), torch.zeros(n, dtype=torch.int64, device=dev)
            lp = getattr(lib, f"libfaer_v0_23_PartialPivLuParams_{suf}")()

            def lu():
                W.copy_(A)
                getattr(lib, f"libfaer_v0_23_partial_piv_lu_factor_in_place_u64_{suf}")(
                    capi.mat_mut(capi.DDTensor(W, cx)), capi.slice_mut(pf), capi.slice_mut(pb), par, mem, lp)
            ms = timed(lu)
            rows.append({"kind": suf, "op": "lu", "n": n, "ms": ms, "dd_madd_per_s": w * 2 * n ** 3 / 3 / (ms * 1e-3)})
            print(rows[-3:], flush=True)
    for r in rows:
        r["frac_of_bound"] = r["dd_madd_per_s"] / BOUND
    doc = {"card": q, "bound_dd_madd_per_s": BOUND, "how": "CUDA events, median of 3 calls after one warm-up, device operands "
           "(LLT / LU time includes the copy that restores the input)", "rows": rows}
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(doc, open(out, "w"), indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
