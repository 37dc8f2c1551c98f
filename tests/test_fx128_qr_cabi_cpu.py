"""CPU-side checks of the double-double QR C ABI (include/faer_b200_fx128_qr.h, included by include/faer_b200.h):

* its 44 prototypes are exactly the reference header's fx128 / cx128 `qr_*` and `apply_householder_*` prototypes
  (tests/golden/faer_ffi_fx128_qr_prototypes.json, extracted by tests/golden/make_fx128_qr_prototypes.py);
* libfaer_b200.so exports every one of them;
* `QrParams_*` returns the f64 defaults, `qr_recommended_block_size_*` the f64 shape rule, and the scratch queries the c64
  formulas with 16 / 32-byte elements;
* the dd scalar helpers the Householder scalars use (faer's abs_impl as fx128 hypot and cx128 modulus) match mpmath at 300 bits
  within 2^-104-relative bounds, across scales near sqrt_min_positive / sqrt_max_positive, through the host build of dd.cuh;
* so does the complex reciprocal of the panel and the cx128 triangular-solve leaf (cdd_recip_scaled), with moduli near 1, on
  the normal range up to its guards, and its special values (0, infinities, NaN) taken from faer's recip."""
import ctypes as C
import json
import os
import re
import subprocess
import importlib.util

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_fx128_qr.h")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_fx128_qr_prototypes.json")))


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S)


def test_fx128_qr_prototypes_match_the_reference_header():
    ours = _parser().prototypes(open(HDR).read())
    assert len(GOLD["prototypes"]) == 44
    assert ours == GOLD["prototypes"]


def test_main_header_includes_the_fx128_qr_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_fx128_qr.h"' in txt


def test_library_exports_every_fx128_qr_symbol(fb):
    lib = fb.load()
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", _header())))
    assert len(syms) == 44
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def test_params_block_size_and_scratch(fb):
    lib = fb.load()
    f64 = lib.libfaer_v0_23_QrParams_f64()
    for suf, es in (("fx128", 16), ("cx128", 32)):
        p = getattr(lib, f"libfaer_v0_23_QrParams_{suf}")()
        assert (p.blocking_threshold, p.par_threshold) == (f64.blocking_threshold, f64.par_threshold) == (48 * 48, 192 * 256)
        rec = getattr(lib, f"libfaer_v0_23_qr_recommended_block_size_{suf}")
        for m in (0, 1, 5, 16, 17, 33, 100, 513, 1024, 2048, 4097, 65536):
            for n in (0, 1, 7, 32, 64, 257, 1024, 8192):
                assert rec(m, n) == lib.libfaer_v0_23_qr_recommended_block_size_f64(m, n), (m, n)
        c64 = lambda name, *a: (lambda r: (r.len_bytes, r.align_bytes))(getattr(lib, f"libfaer_v0_23_{name}_c64")(*a))
        lay = lambda name, *a: (lambda r: (r.len_bytes, r.align_bytes))(getattr(lib, f"libfaer_v0_23_{name}_{suf}")(*a))
        par = fb.capi.par_default()
        q = c64("qr_factor_in_place_scratch", 70, 50, 8, par, p)
        assert lay("qr_factor_in_place_scratch", 70, 50, 8, par, p) == (q[0] // 16 * es, q[1]) == (8 * 50 * es, 64)
        for name in ("apply_householder_on_the_left", "apply_householder_transpose_on_the_left", "apply_householder_on_the_right",
                     "apply_householder_transpose_on_the_right"):
            assert lay(f"{name}_scratch", 70, 8, 3) == (8 * 3 * es, 64) == (c64(f"{name}_scratch", 70, 8, 3)[0] // 16 * es, 64)
        assert lay("qr_solve_lstsq_in_place_scratch", 70, 50, 8, 3, par) == (8 * 3 * es, 64)
        assert lay("qr_solve_in_place_scratch", 70, 8, 3, par) == (8 * 3 * es, 64)
        assert lay("qr_solve_transpose_in_place_scratch", 70, 8, 3, par) == (8 * 3 * es, 64)
        assert lay("qr_reconstruct_scratch", 70, 50, 8, par) == (8 * 50 * es, 64) == (c64("qr_reconstruct_scratch", 70, 50, 8, par)[0] // 16 * es, 64)
        assert lay("qr_inverse_scratch", 70, 8, par) == (8 * 70 * es, 64) == (c64("qr_inverse_scratch", 70, 8, par)[0] // 16 * es, 64)


@pytest.fixture(scope="module")
def ddh(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ddh") / "dd_host.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tools", "emul", "dd_host.cpp")])
    lib = C.CDLL(out)
    lib.dd_host_op.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]
    lib.dd_host_op.restype = C.c_int
    return lib


def _op(lib, op, a, b):
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    out = np.zeros_like(a)
    assert lib.dd_host_op(op, a.ctypes.data, b.ctypes.data, out.ctypes.data, len(a) // 2) == 0
    return out


def test_dd_hypot_and_complex_abs_match_mpmath(ddh):
    import mpmath
    mpmath.mp.prec = 300
    mp = lambda hi, lo: mpmath.mpf(float(hi)) + mpmath.mpf(float(lo))
    sml = _op(ddh, 13, [0.0, 0.0], [0.0, 0.0])
    big = _op(ddh, 14, [0.0, 0.0], [0.0, 0.0])
    assert abs(mp(*sml) - mpmath.sqrt(mpmath.mpf(2.2250738585072014e-308))) <= 2.0 ** -104 * mp(*sml)
    assert abs(mp(*big) - mpmath.sqrt(1 / mpmath.mpf(2.2250738585072014e-308))) <= 2.0 ** -104 * mp(*big)
    rng = np.random.default_rng(0)
    scales = [2.0 ** e for e in (-1000, -540, -512, -511, -480, -60, -1, 0, 1, 60, 480, 510, 511, 512, 540, 1000)]
    a, b = [], []
    for s in scales:
        for t in scales:
            for _ in range(4):
                x, y = rng.uniform(0.5, 2.0) * s * rng.choice([-1, 1]), rng.uniform(0.5, 2.0) * t * rng.choice([-1, 1])
                a += [x, x * 2.0 ** -60 * rng.uniform(-0.5, 0.5)]
                b += [y, y * 2.0 ** -60 * rng.uniform(-0.5, 0.5)]
    a, b = np.array(a), np.array(b)
    for op in (11, 12):
        got = _op(ddh, op, a, b)
        for i in range(0, len(a), 2):
            want = mpmath.sqrt(mp(a[i], a[i + 1]) ** 2 + mp(b[i], b[i + 1]) ** 2)
            g = mp(got[i], got[i + 1])
            # relative, plus the spacing of the low limb's subnormals when the result is tiny
            assert abs(g - want) <= 2.0 ** -102 * want + 2.0 ** -1070, (op, a[i], b[i], float(g), float(want))


def test_cdd_recip_scaled_matches_mpmath(ddh):
    import mpmath
    mpmath.mp.prec = 300
    mp = lambda hi, lo: mpmath.mpf(float(hi)) + mpmath.mpf(float(lo))
    rng = np.random.default_rng(1)
    # moduli near 1 (where faer's scaling loses the low limb), the whole normal range up to the lower guard (MIN_POSITIVE) and
    # close to the largest finite values
    scales = [2.0 ** e for e in (-1021, -1000, -970, -500, -60, -1, 0, 1, 60, 500, 970, 1000, 1021)]
    a, b = [], []
    for s in scales:
        for t in scales + [0.0]:
            for _ in range(3):
                x = rng.uniform(0.5, 2.0) * s * rng.choice([-1, 1])
                y = rng.uniform(0.5, 2.0) * t * rng.choice([-1, 1])
                a += [x, x * 2.0 ** -60 * rng.uniform(-0.5, 0.5)]
                b += [y, y * 2.0 ** -60 * rng.uniform(-0.5, 0.5)]
    a, b = np.array(a), np.array(b)
    re, im = _op(ddh, 15, a, b), _op(ddh, 16, a, b)
    for i in range(0, len(a), 2):
        z = mpmath.mpc(mp(a[i], a[i + 1]), mp(b[i], b[i + 1]))
        w = 1 / z
        g = mpmath.mpc(mp(re[i], re[i + 1]), mp(im[i], im[i + 1]))
        # relative to |1/z|, plus the spacing of the low limb's subnormals for tiny results
        assert abs(g - w) <= 2.0 ** -101 * abs(w) + 2.0 ** -1070, (a[i], b[i], complex(g), complex(w))
    # special values come from faer's recip: 1/0 = inf, 1/inf = 0, NaN stays NaN
    sp = np.array([0.0, 0.0, np.inf, 0.0, np.nan, 0.0])
    z0 = np.zeros(6)
    r = _op(ddh, 15, sp, z0)
    assert np.isinf(r[0]) and r[2] == 0.0 and np.isnan(r[4])
