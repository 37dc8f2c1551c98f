"""CPU-side checks of the pivoted Cholesky's C ABI (include/faer_b200_piv_llt.h, included by include/faer_b200.h):

* its 68 prototypes are exactly the reference header's `piv_llt_*` / `PivLltParams_*` prototypes for f32 / f64 / c32 / c64
  (tests/golden/faer_ffi_piv_llt_prototypes.json, extracted from faer-ffi/faer.h with the parser of make_ffi_prototypes.py);
* libfaer_b200.so exports every one of them;
* `PivLltStatus` has faer.h's layout (24 bytes, body at offset 8) and `PivLltParams_<T>()` is the reference default {128};
* the `*_scratch` queries return the reference's layouts (factor.rs:36-45, solve.rs:4-11, reconstruct.rs:4-10, inverse.rs:4-11)."""
import ctypes as C
import importlib.util
import json
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_piv_llt.h")


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_piv_llt_prototypes_match_the_reference_header():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_piv_llt_prototypes.json")))["prototypes"]
    ours = _parser().prototypes(open(HDR).read())
    assert len(gold) == 68
    assert ours == gold


def test_main_header_includes_the_piv_llt_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_piv_llt.h"' in txt


def test_library_exports_every_piv_llt_symbol(fb):
    lib = fb.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", hdr)))
    assert len(syms) == 68
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def test_piv_llt_status_layout_params_and_scratch(fb):
    capi = fb.capi
    assert C.sizeof(capi.PivLltStatus) == 24 and capi.PivLltStatus.body.offset == 8
    assert C.sizeof(capi.PivLltParams) == 8
    lib = fb.load()
    par = capi.par_default()
    for suf, real, sz in (("f64", 8, 8), ("f32", 4, 4), ("c64", 8, 16), ("c32", 4, 8)):
        p = getattr(lib, f"libfaer_v0_23_PivLltParams_{suf}")()
        assert p.block_size == 128
        for it in ("u32", "u64"):
            assert getattr(lib, f"libfaer_v0_23_piv_llt_factor_in_place_scratch_{it}_{suf}")(100, par, p).len_bytes == 100 * 2 * real
            assert getattr(lib, f"libfaer_v0_23_piv_llt_solve_in_place_scratch_{it}_{suf}")(100, 3, par).len_bytes == 100 * 3 * sz
            assert getattr(lib, f"libfaer_v0_23_piv_llt_reconstruct_scratch_{it}_{suf}")(50, par).len_bytes == 50 * 50 * sz
            assert getattr(lib, f"libfaer_v0_23_piv_llt_inverse_scratch_{it}_{suf}")(50, par).len_bytes == 50 * 50 * sz
