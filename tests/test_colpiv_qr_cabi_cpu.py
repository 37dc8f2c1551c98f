"""CPU-side checks of the column-pivoted QR's C ABI (include/faer_b200_colpiv_qr.h, included by include/faer_b200.h):

* its 100 prototypes are exactly the reference header's `colpiv_qr_*` / `ColPivQrParams_*` prototypes for f32 / f64 / c32 / c64
  (tests/golden/faer_ffi_colpiv_qr_prototypes.json, extracted from faer-ffi/faer.h with the parser of make_ffi_prototypes.py);
* libfaer_b200.so exports every one of them;
* `ColPivQrStatus` has faer.h's layout (16 bytes, body at offset 8) and `ColPivQrParams_<T>()` is the reference default;
* the `*_scratch` queries return the reference's layouts (factor.rs:323-336, solve.rs:3-50, reconstruct.rs:3-14, inverse.rs:4-14)."""
import ctypes as C
import importlib.util
import json
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_colpiv_qr.h")


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_colpiv_qr_prototypes_match_the_reference_header():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_colpiv_qr_prototypes.json")))["prototypes"]
    ours = _parser().prototypes(open(HDR).read())
    assert len(gold) == 100
    assert ours == gold


def test_main_header_includes_the_colpiv_qr_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_colpiv_qr.h"' in txt


def test_library_exports_every_colpiv_qr_symbol(fb):
    lib = fb.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", hdr)))
    assert len(syms) == 100
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def _and(a_len, b_len):
    """StackReq::and of two 64-byte aligned requests: the second placed after the first."""
    return (a_len + 63) // 64 * 64 + b_len


def test_colpiv_qr_status_layout_params_and_scratch(fb):
    capi = fb.capi
    assert C.sizeof(capi.ColPivQrStatus) == 16 and capi.ColPivQrStatus.body.offset == 8
    assert C.sizeof(capi.ColPivQrParams) == 16
    lib = fb.load()
    par = capi.par_default()
    for suf, sz in (("f64", 8), ("f32", 4), ("c64", 16), ("c32", 8)):
        p = getattr(lib, f"libfaer_v0_23_ColPivQrParams_{suf}")()
        assert (p.blocking_threshold, p.par_threshold) == (48 * 48, 192 * 256)
        for it in ("u32", "u64"):
            pre = "libfaer_v0_23_colpiv_qr_"
            assert getattr(lib, f"{pre}factor_in_place_scratch_{it}_{suf}")(100, 70, 8, par, p).len_bytes == 70 * 2 * sz
            # the unpivoted solve scratch (block_size x rhs_ncols) and permute_rows_in_place_scratch (ncols x rhs_ncols)
            assert getattr(lib, f"{pre}solve_lstsq_in_place_scratch_{it}_{suf}")(100, 50, 4, 3, par).len_bytes == _and(4 * 3 * sz, 50 * 3 * sz)
            assert getattr(lib, f"{pre}solve_in_place_scratch_{it}_{suf}")(50, 4, 3, par).len_bytes == _and(4 * 3 * sz, 50 * 3 * sz)
            assert getattr(lib, f"{pre}solve_transpose_in_place_scratch_{it}_{suf}")(50, 4, 3, par).len_bytes == _and(4 * 3 * sz, 50 * 3 * sz)
            # StackReq::or of the block-Householder apply and permute_cols_in_place_scratch (nrows x ncols)
            assert getattr(lib, f"{pre}reconstruct_scratch_{it}_{suf}")(100, 50, 4, par).len_bytes == 100 * 50 * sz
            assert getattr(lib, f"{pre}inverse_scratch_{it}_{suf}")(50, 4, par).len_bytes == 50 * 50 * sz
