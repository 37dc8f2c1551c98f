"""CPU-side checks of the full-pivoting LU's C ABI (include/faer_b200_full_piv_lu.h, included by include/faer_b200.h):

* its 84 prototypes are exactly the reference header's `full_piv_lu_*` / `FullPivLuParams_*` prototypes for f32 / f64 / c32 / c64
  (tests/golden/faer_ffi_full_piv_lu_prototypes.json, extracted from faer-ffi/faer.h with the parser of make_ffi_prototypes.py);
* libfaer_b200.so exports every one of them;
* `FullPivLuStatus` has faer.h's layout (16 bytes, body at offset 8) and `FullPivLuParams_<T>()` is the reference default;
* the `*_scratch` queries return the reference's layouts (factor.rs:450-461, solve.rs:4-19, reconstruct.rs:4-11, inverse.rs:4-10)."""
import ctypes as C
import importlib.util
import json
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_full_piv_lu.h")


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_full_piv_lu_prototypes_match_the_reference_header():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_full_piv_lu_prototypes.json")))["prototypes"]
    ours = _parser().prototypes(open(HDR).read())
    assert len(gold) == 84
    assert ours == gold


def test_main_header_includes_the_full_piv_lu_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_full_piv_lu.h"' in txt


def test_library_exports_every_full_piv_lu_symbol(fb):
    lib = fb.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", hdr)))
    assert len(syms) == 84
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s
    assert len([s for s in exported if "full_piv_lu" in s]) == 80


def test_full_piv_lu_status_layout_params_and_scratch(fb):
    capi = fb.capi
    assert C.sizeof(capi.FullPivLuStatus) == 16 and capi.FullPivLuStatus.body.offset == 8
    assert C.sizeof(capi.FullPivLuParams) == 8
    lib = fb.load()
    par = capi.par_default()
    for suf, sz in (("f64", 8), ("f32", 4), ("c64", 16), ("c32", 8)):
        p = getattr(lib, f"libfaer_v0_23_FullPivLuParams_{suf}")()
        assert p.par_threshold == 256 * 512
        for it in ("u32", "u64"):
            pre = "libfaer_v0_23_full_piv_lu_"
            # (dim, block_size) forwarded as (nrows, ncols): two usize arrays of min(dim, block_size), whatever the index type
            lay = getattr(lib, f"{pre}factor_in_place_scratch_{it}_{suf}")(100, 70, par, p)
            assert (lay.len_bytes, lay.align_bytes) == (2 * 70 * 8, 8)
            assert getattr(lib, f"{pre}factor_in_place_scratch_{it}_{suf}")(30, 70, par, p).len_bytes == 2 * 30 * 8
            # permute_rows_in_place_scratch (dim x rhs_ncols)
            assert getattr(lib, f"{pre}solve_in_place_scratch_{it}_{suf}")(50, 3, par).len_bytes == 50 * 3 * sz
            assert getattr(lib, f"{pre}solve_transpose_in_place_scratch_{it}_{suf}")(50, 3, par).len_bytes == 50 * 3 * sz
            # temp_mat_scratch (nrows x ncols) / (dim x dim)
            assert getattr(lib, f"{pre}reconstruct_scratch_{it}_{suf}")(100, 50, par).len_bytes == 100 * 50 * sz
            assert getattr(lib, f"{pre}inverse_scratch_{it}_{suf}")(50, par).len_bytes == 50 * 50 * sz
