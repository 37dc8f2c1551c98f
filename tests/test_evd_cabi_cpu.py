"""CPU-side checks of the general eigendecomposition's C ABI (include/faer_b200_evd.h, included by include/faer_b200.h):

* its 20 prototypes are exactly the reference header's `evd_*` / `evd_scratch_*` / `EvdParams_*` / `SchurParams_*` /
  `EvdFromSchurParams_*` prototypes for f32 / f64 / c32 / c64 (tests/golden/faer_ffi_evd_prototypes.json, extracted from
  faer-ffi/faer.h by tests/golden/make_evd_prototypes.py), and the three parameter structs have faer.h's fields in order;
* libfaer_b200.so exports every one of them;
* the ctypes mirrors have the C layouts and `EvdParams_<T>()` returns the reference defaults (evd/mod.rs:74-81,
  evd/schur/mod.rs:26-107, evd/hessenberg.rs:17-23), its callbacks reproducing the reference's tables."""
import ctypes as C
import importlib.util
import json
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_evd.h")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_evd_prototypes.json")))


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)


def test_evd_prototypes_match_the_reference_header():
    ours = _parser().prototypes(open(HDR).read())
    assert len(GOLD["prototypes"]) == 20
    assert ours == GOLD["prototypes"]


def test_parameter_structs_have_the_reference_fields():
    hdr = _header()
    for name, fields in GOLD["structs"].items():
        body = re.search(r"typedef struct FaerV0_24_%s \{(.*?)\} FaerV0_24_%s;" % (name, name), hdr, re.S).group(1)
        assert [re.sub(r"\s+", " ", f).strip() for f in body.split(";") if f.strip()] == fields


def test_main_header_includes_the_evd_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_evd.h"' in txt


def test_library_exports_every_evd_symbol(fb):
    lib = fb.load()
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", _header())))
    assert len(syms) == 20
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def test_layouts_defaults_and_scratch(fb):
    capi = fb.capi
    assert C.sizeof(capi.EvdFromSchurParams) == 8
    assert C.sizeof(capi.SchurParams) == 32 and capi.SchurParams.blocking_threshold.offset == 16
    assert C.sizeof(capi.EvdParams) == 56 and capi.EvdParams.schur.offset == 16 and capi.EvdParams.evd_from_schur.offset == 48
    lib = fb.load()
    shift = {29: 2, 30: 4, 59: 4, 60: 12, 149: 12, 150: 32, 589: 32, 590: 64, 2999: 64, 3000: 128, 5999: 128, 6000: 256}
    window = {29: 2, 59: 4, 149: 10, 150: 20, 589: 64, 590: 96, 3000: 192, 6000: 384}
    for suf, sz in (("f64", 8), ("f32", 4), ("c64", 16), ("c32", 8)):
        p = getattr(lib, f"libfaer_v0_23_EvdParams_{suf}")()
        assert (p.hessenberg.par_threshold, p.hessenberg.blocking_threshold) == (192 * 256, 256 * 256)
        assert (p.schur.blocking_threshold, p.schur.nibble_threshold, p.evd_from_schur.recursion_threshold) == (75, 50, 64)
        sp = getattr(lib, f"libfaer_v0_23_SchurParams_{suf}")()
        assert (sp.blocking_threshold, sp.nibble_threshold) == (75, 50)
        for n, v in shift.items():
            assert p.schur.recommended_shift_count(n, n) == v and sp.recommended_shift_count(n, 1) == v
        for n, v in window.items():
            assert p.schur.recommended_deflation_window(n, n) == v
        assert getattr(lib, f"libfaer_v0_23_EvdFromSchurParams_{suf}")().recursion_threshold == 64
        lay = getattr(lib, f"libfaer_v0_23_evd_scratch_{suf}")(100, 1, 1, capi.par_default(), p)
        assert (lay.len_bytes, lay.align_bytes) == (100 * 100 * sz, 64)
