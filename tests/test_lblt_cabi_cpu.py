"""CPU-side checks of the Bunch-Kaufman LBLT's C ABI (include/faer_b200_lblt.h, included by include/faer_b200.h):

* its 68 prototypes are exactly the reference header's `lblt_*` / `LbltParams_*` prototypes for f32 / f64 / c32 / c64
  (tests/golden/faer_ffi_lblt_prototypes.json, extracted from faer-ffi/faer.h with the parser of make_ffi_prototypes.py);
* libfaer_b200.so exports every one of them;
* `LbltStatus` / `LbltParams` have faer.h's layouts and `LbltParams_<T>()` is the reference default {PartialDiag, 128 * 128, 64};
* the `*_scratch` queries return the reference's layouts (factor.rs:1128-1140, solve.rs:11-18, reconstruct.rs:4-10,
  inverse.rs:3-9)."""
import ctypes as C
import importlib.util
import json
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_lblt.h")


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_lblt_prototypes_match_the_reference_header():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_lblt_prototypes.json")))["prototypes"]
    ours = _parser().prototypes(open(HDR).read())
    assert len(gold) == 68
    assert ours == gold


def test_main_header_includes_the_lblt_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_lblt.h"' in txt


def test_library_exports_every_lblt_symbol(fb):
    lib = fb.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", hdr)))
    assert len(syms) == 68
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def test_lblt_status_layout_params_and_scratch(fb):
    capi = fb.capi
    assert C.sizeof(capi.LbltStatus) == 16 and capi.LbltStatus.body.offset == 8
    assert C.sizeof(capi.LbltParams) == 24 and capi.LbltParams.block_size.offset == 16
    lib = fb.load()
    par = capi.par_default()
    for suf, sz in (("f64", 8), ("f32", 4), ("c64", 16), ("c32", 8)):
        p = getattr(lib, f"libfaer_v0_23_LbltParams_{suf}")()
        assert (p.pivoting, p.par_threshold, p.block_size) == (capi.PIVOTING_PARTIAL_DIAG, 128 * 128, 64)
        for it in ("u32", "u64"):
            f = getattr(lib, f"libfaer_v0_23_lblt_factor_in_place_scratch_{it}_{suf}")
            # StackReq::new::<usize>(dim).and(temp_mat_scratch::<T>(dim, bs)), bs = 0 when bs < 2 or dim <= bs
            lay = f(100, par, p)
            assert (lay.len_bytes, lay.align_bytes) == (832 + 100 * 64 * sz, 64)
            assert f(64, par, p).len_bytes == 512
            q = capi.LbltParams(capi.PIVOTING_ROOK, 0, 1)
            assert f(100, par, q).len_bytes == 832
            assert getattr(lib, f"libfaer_v0_23_lblt_solve_in_place_scratch_{it}_{suf}")(100, 3, par).len_bytes == 100 * 3 * sz
            assert getattr(lib, f"libfaer_v0_23_lblt_reconstruct_scratch_{it}_{suf}")(50, par).len_bytes == 50 * 50 * sz
            assert getattr(lib, f"libfaer_v0_23_lblt_inverse_scratch_{it}_{suf}")(50, par).len_bytes == 50 * 50 * sz
