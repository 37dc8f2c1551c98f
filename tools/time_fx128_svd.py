"""Times the double-double SVD (svd_fx128 / _cx128) on device-resident operands, with the fx128 GEMM at n = 4096 in the same run as
the rate to compare against: the median of 3 calls after a warm-up, with CUDA events, and the card name and power limit read in
the same run. Writes profiles/r16_fx128_svd_timing.json (or the path given as the first argument).

Cases: fx128 1024^2 / 2048^2 / 4096^2, each values only and with thin U, V; fx128 65536 x 256 (QR first) and cx128 2048^2, both
ways too. A torch.profiler pass over one call splits its kernel time by phase (see split): "qr_first" (the QR of a tall input),
"reduction" (the bidiagonalization), "solve" (bisection, or the Golub-Kahan divide and conquer), "stabilisation_qrs" (the two dd
QRs, their Q formations and the sort), "back_transform" (the T-factor builds and block-reflector products of U and V) and
"other" (copies, the finiteness check, the extraction of the bidiagonal and the stores)."""
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
from time_fx128 import dd_tensor, timed  # noqa: E402

OTHER = ("sd_copy_kernel", "sd_finite_kernel", "sd_copy_upper_kernel", "sd_extract_kernel", "sd_store_kernel", "sd_values_out_kernel")


def split(lib, fn):
    """kernel time of one call by phase, from one torch.profiler trace. The phases run one after the other, so the library's
    kernels are assigned in start order by the kernels that open them: the first left reflector opens the reduction (before it:
    the QR of a tall input), the extraction of the bidiagonal the solve, the v parts of the Golub-Kahan eigenvectors the
    stabilisation QRs, and the first embedding of U_B or V_B the back-transform. The row also reports how many records the trace
    holds against the launches the library logged (faer_b200_launch_log_begin / _end)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    tags = np.zeros(1 << 22, dtype=np.int8)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lib.faer_b200_launch_log_begin(tags.ctypes.data, tags.size)
        fn()
        torch.cuda.synchronize()
        count = lib.faer_b200_launch_log_end()
    kernels = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "fb::" in e.name),
                     key=lambda e: e.time_range.start)
    cats = {"qr_first": 0.0, "reduction": 0.0, "solve": 0.0, "stabilisation_qrs": 0.0, "back_transform": 0.0, "other": 0.0}
    phase = "qr_first"
    for e in kernels:
        name, ms = e.name, e.time_range.elapsed_us() / 1e3
        if "sd_left_house_kernel" in name and phase == "qr_first":
            phase = "reduction"
        elif "sd_extract_kernel" in name:
            phase = "solve"
        elif "sd_vparts_kernel" in name:
            phase = "stabilisation_qrs"
        elif "sd_embed_kernel" in name:
            phase = "back_transform"
        if any(k in name for k in OTHER):
            cats["other"] += ms
            continue
        cats[phase] += ms
    assert cats["reduction"] > 0.0 and cats["solve"] > 0.0, cats
    return {**cats, "kernel_records": len(kernels), "logged_launches": int(count)}


def main() -> int:
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r16_fx128_svd_timing.json")
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
    for suf, cx, m, n in (("fx128", False, 1024, 1024), ("fx128", False, 2048, 2048), ("fx128", False, 4096, 4096),
                          ("fx128", False, 65536, 256), ("cx128", True, 2048, 2048)):
        X = rng.standard_normal((m, n)) + (1j * rng.standard_normal((m, n)) if cx else 0)
        Ad = dd_tensor(X, cx, dev)
        lim = (2, 2) if cx else (2,)
        S = torch.zeros((n,) + lim, dtype=torch.float64, device=dev)
        p = getattr(lib, f"libfaer_v0_23_SvdParams_{suf}")()
        for vectors in (False, True):
            Ud = torch.zeros((m, n) + lim, dtype=torch.float64, device=dev) if vectors else None
            Vd = torch.zeros((n, n) + lim, dtype=torch.float64, device=dev) if vectors else None

            def svd():
                none = capi.MatMut(None, 0, 0, 0, 0)
                uv = capi.mat_mut(capi.DDTensor(Ud, cx)) if vectors else none
                vv = capi.mat_mut(capi.DDTensor(Vd, cx)) if vectors else none
                st = getattr(lib, f"libfaer_v0_23_svd_{suf}")(capi.mat_ref(capi.DDTensor(Ad, cx)), uv, capi.VecMut(S.data_ptr(), n, 1),
                                                              vv, par, mem, p)
                assert st.tag == 0
            ms = timed(svd)
            row = {"kind": suf, "m": m, "n": n, "vectors": vectors, "ms": ms, "split_ms": split(lib, svd)}
            rows.append(row)
            print(row, flush=True)
            del Ud, Vd
            torch.cuda.empty_cache()
        del Ad, S
    big = {r["vectors"]: r["ms"] for r in rows if r.get("m") == 4096 and r.get("n") == 4096}
    doc = {"card": q, "gemm_dd_madd_per_s": gemm_rate,
           "how": "CUDA events, median of 3 calls after one warm-up, device operands; split_ms from one torch.profiler pass",
           "rows": rows, "aims_met": {"fx128_4096_with_vectors_under_10_s": big[True] < 10000.0,
                                      "fx128_4096_values_only_under_2_s": big[False] < 2000.0}}
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(doc, open(out, "w"), indent=1)
    print(json.dumps(doc["aims_met"]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
