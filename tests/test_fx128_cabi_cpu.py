"""CPU-side checks of the double-double C ABI (include/faer_b200_fx128.h, included by include/faer_b200.h):

* its 80 prototypes are exactly the reference header's fx128 / cx128 `matmul*`, triangular solve / inverse, `llt_*` and
  `partial_piv_lu_*` prototypes (tests/golden/faer_ffi_fx128_prototypes.json, extracted by tests/golden/make_fx128_prototypes.py);
* libfaer_b200.so exports every one of them;
* `LltParams_*` / `PartialPivLuParams_*` return the f64 defaults, and the scratch queries give the f64 formulas with 16 / 32-byte
  elements, for u32 and u64."""
import json
import os
import re
import subprocess
import importlib.util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_fx128.h")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_fx128_prototypes.json")))


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)


def test_fx128_prototypes_match_the_reference_header():
    ours = _parser().prototypes(open(HDR).read())
    assert len(GOLD["prototypes"]) == 80
    assert ours == GOLD["prototypes"]


def test_main_header_includes_the_fx128_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_fx128.h"' in txt


def test_library_exports_every_fx128_symbol(fb):
    lib = fb.load()
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", _header())))
    assert len(syms) == 80
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def test_params_defaults_and_scratch(fb):
    lib, capi = fb.load(), fb.capi
    par = capi.par_default()
    f64_llt = lib.libfaer_v0_23_LltParams_f64()
    f64_lu = lib.libfaer_v0_23_PartialPivLuParams_f64()
    for suf, es in (("fx128", 16), ("cx128", 32)):
        p = getattr(lib, f"libfaer_v0_23_LltParams_{suf}")()
        assert (p.recursion_threshold, p.block_size) == (f64_llt.recursion_threshold, f64_llt.block_size) == (64, 128)
        q = getattr(lib, f"libfaer_v0_23_PartialPivLuParams_{suf}")()
        assert (q.recursion_threshold, q.block_size, q.par_threshold) == \
            (f64_lu.recursion_threshold, f64_lu.block_size, f64_lu.par_threshold) == (16, 64, 128 * 128)
        lay = lambda name, *a: (lambda r: (r.len_bytes, r.align_bytes))(getattr(lib, f"libfaer_v0_23_{name}_{suf}")(*a))
        assert lay("llt_factor_in_place_scratch", 100, par, p) == (100 * es, 64)
        assert lay("llt_solve_in_place_scratch", 100, 3, par) == (0, 1)
        assert lay("llt_reconstruct_scratch", 100, par) == (0, 1)
        assert lay("llt_inverse_scratch", 100, par) == (100 * 100 * es, 64)
        for it, ib in (("u32", 4), ("u64", 8)):
            assert lay(f"partial_piv_lu_factor_in_place_scratch_{it}", 70, 50, par, q) == (50 * ib, ib)
            assert lay(f"partial_piv_lu_solve_in_place_scratch_{it}", 70, 3, par) == (70 * 3 * es, 64)
            assert lay(f"partial_piv_lu_solve_transpose_in_place_scratch_{it}", 70, 3, par) == (70 * 3 * es, 64)
            assert lay(f"partial_piv_lu_reconstruct_scratch_{it}", 70, 50, par) == (70 * 50 * es, 64)
            assert lay(f"partial_piv_lu_inverse_scratch_{it}", 70, par) == (70 * 70 * es, 64)
