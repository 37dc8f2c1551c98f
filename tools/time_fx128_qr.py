"""Times the double-double Householder QR (qr_factor_in_place_fx128 / _cx128) on device-resident operands, with the fx128 GEMM at
n = 4096 in the same run as the rate to compare against: the median of 3 calls after a warm-up, with CUDA events, and the card name
and power limit read in the same run. Writes profiles/r12_fx128_qr_timing.json (or the path given as the first argument).

Cases: fx128 QR at n = 1024 / 2048 / 4096, cx128 QR at 2048, fx128 at 65536 x 256 followed by qr_solve_lstsq with one right-hand
side. Rate: dd multiply-adds per second (GEMM n^3; QR m n^2 - n^3 / 3, i.e. 2 n^3 / 3 when square, two thirds of a GEMM's; a
cx128 multiply-add counts as 4 real ones). A separate torch.profiler pass over one QR call splits its kernel time into the panel
kernels, the products of the block-reflector applies (their GEMMs and triangular-solve leaves), the T-factor builds and the rest,
from the phase the library logs for each launch."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import faer_b200  # noqa: E402
from time_fx128 import BOUND, dd_tensor, timed  # noqa: E402


def split(lib, fn):
    """kernel time of one call by phase: the library logs the phase of each of its launches in launch order
    (faer_b200_launch_log_begin / _end), which is zipped with the library's kernels of a torch.profiler trace in start order"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    tags = np.zeros(1 << 20, dtype=np.int8)
    # the first trace of a process can miss a kernel record; a trace counts only when it holds every logged launch
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lib.faer_b200_launch_log_begin(tags.ctypes.data, tags.size)
            fn()
            torch.cuda.synchronize()
            count = lib.faer_b200_launch_log_end()
        kernels = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "fb::" in e.name),
                         key=lambda e: e.time_range.start)
        if count <= tags.size and len(kernels) == count:
            break
    assert count <= tags.size and len(kernels) == count, (len(kernels), count)
    names = {0: "other", 1: "panel", 2: "products", 3: "t_builds"}
    cats = {v: 0.0 for v in names.values()}
    for e, t in zip(kernels, tags[:count]):
        cats[names[int(t)]] += e.time_range.elapsed_us() / 1e3
    return cats


def main() -> int:
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r12_fx128_qr_timing.json")
    dev = torch.device("cuda:0")
    capi, lib = faer_b200.capi, faer_b200.load()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    par, mem = capi.par_default(), capi.MemAlloc(None, 0)
    rng = np.random.default_rng(0)
    rows = []
    # the GEMM rate of this run
    n = 4096
    A, B = dd_tensor(rng.standard_normal((n, n)), False, dev), dd_tensor(rng.standard_normal((n, n)), False, dev)
    Cm = torch.zeros_like(A)
    alpha = np.array([1.0, 0.0])
    ms = timed(lambda: lib.libfaer_v0_23_matmul_fx128(capi.mat_mut(capi.DDTensor(Cm, False)), 0, capi.mat_ref(capi.DDTensor(A, False)),
                                                      capi.mat_ref(capi.DDTensor(B, False)), alpha.ctypes.data, par))
    gemm_rate = n ** 3 / (ms * 1e-3)
    rows.append({"kind": "fx128", "op": "gemm", "m": n, "n": n, "ms": ms, "dd_madd_per_s": gemm_rate})
    print(rows[-1], flush=True)
    del A, B, Cm
    for suf, cx, m, n in (("fx128", False, 1024, 1024), ("fx128", False, 2048, 2048), ("fx128", False, 4096, 4096),
                          ("cx128", True, 2048, 2048), ("fx128", False, 65536, 256)):
        w = 4 if cx else 1
        X = rng.standard_normal((m, n)) + (1j * rng.standard_normal((m, n)) if cx else 0)
        S = dd_tensor(X, cx, dev)
        Wt = torch.empty_like(S)
        bs = getattr(lib, f"libfaer_v0_23_qr_recommended_block_size_{suf}")(m, n)
        Qc = torch.zeros((bs, n) + ((2, 2) if cx else (2,)), dtype=torch.float64, device=dev)
        p = getattr(lib, f"libfaer_v0_23_QrParams_{suf}")()

        def qr():
            Wt.copy_(S)
            st = getattr(lib, f"libfaer_v0_23_qr_factor_in_place_{suf}")(capi.mat_mut(capi.DDTensor(Wt, cx)),
                                                                        capi.mat_mut(capi.DDTensor(Qc, cx)), par, mem, p)
            assert st.value == n
        ms = timed(qr)
        madd = w * (m * n * n - n ** 3 / 3)  # Householder QR: 2 m n^2 - 2 n^3 / 3 flop = half as many multiply-adds
        row = {"kind": suf, "op": "qr", "m": m, "n": n, "block_size": bs, "ms": ms, "dd_madd_per_s": madd / (ms * 1e-3),
               "frac_of_gemm_rate": madd / (ms * 1e-3) / gemm_rate / w if not cx else None, "split_ms": split(lib, qr)}
        rows.append(row)
        print(row, flush=True)
        if m == 65536:
            b0 = dd_tensor(rng.standard_normal((m, 1)), False, dev)
            bt = torch.empty_like(b0)

            def lstsq():
                bt.copy_(b0)
                lib.libfaer_v0_23_qr_solve_lstsq_in_place_fx128(capi.mat_ref(capi.DDTensor(Wt, False)), capi.mat_ref(capi.DDTensor(Qc, False)),
                                                                capi.mat_ref(capi.DDTensor(Wt, False)), 0, capi.mat_mut(capi.DDTensor(bt, False)),
                                                                par, mem)
            rows.append({"kind": suf, "op": "qr_solve_lstsq", "m": m, "n": n, "rhs": 1, "ms": timed(lstsq)})
            print(rows[-1], flush=True)
        del S, Wt, Qc
    for r in rows:
        if "dd_madd_per_s" in r:
            r["frac_of_bound"] = r["dd_madd_per_s"] / BOUND
    sq = next(r for r in rows if r["op"] == "qr" and r["m"] == 4096)
    tall = next(r for r in rows if r["op"] == "qr" and r["m"] == 65536)
    aims = {"fx128_4096_qr_at_least_half_the_gemm_rate": sq["frac_of_gemm_rate"] >= 0.5,
            "tall_skinny_panel_below_products": tall["split_ms"]["panel"] < tall["split_ms"]["products"] + tall["split_ms"]["t_builds"]}
    doc = {"card": q, "bound_dd_madd_per_s": BOUND, "how": "CUDA events, median of 3 calls after one warm-up, device operands (the "
           "QR time includes the copy that restores the input); split_ms from one torch.profiler pass", "rows": rows, "aims_met": aims}
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(doc, open(out, "w"), indent=1)
    print(json.dumps(aims))
    return 0


if __name__ == "__main__":
    sys.exit(main())
