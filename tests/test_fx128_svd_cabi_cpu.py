"""CPU-side checks of the double-double SVD C ABI (include/faer_b200_fx128_svd.h, included by include/faer_b200.h): its 8
prototypes are exactly the reference header's fx128 / cx128 `BidiagParams`, `SvdParams`, `svd_scratch` and `svd`
(tests/golden/faer_ffi_fx128_svd_prototypes.json, extracted by tests/golden/make_fx128_svd_prototypes.py); libfaer_b200.so exports
all of them; the params queries return faer's defaults and the scratch query the f64 / c64 formula with 16 / 32-byte elements.
Also: the exact rectangular dd test matrices of tests/dd_rect_exact.py are what they claim (their limbs reproduce the integer
matrix, and LAPACK on the hi limbs finds the singular values within f64 bounds)."""
import importlib.util
import json
import os
import re
import subprocess
import sys
from fractions import Fraction as F

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_fx128_svd.h")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_fx128_svd_prototypes.json")))


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_fx128_svd_prototypes_match_the_reference_header():
    ours = _parser().prototypes(open(HDR).read())
    assert len(GOLD["prototypes"]) == 8
    assert ours == GOLD["prototypes"]


def test_main_header_includes_the_fx128_svd_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_fx128_svd.h"' in txt


def test_library_exports_every_fx128_svd_symbol(fb):
    lib = fb.load()
    syms = sorted(set(re.findall(r"\b(libfaer_v0_23_\w+)\s*\(", re.sub(r"/\*.*?\*/", "", open(HDR).read(), flags=re.S))))
    assert len(syms) == 8
    out = subprocess.check_output(["nm", "-D", "--defined-only", fb.capi.LIB_PATH], text=True)
    exported = set(re.findall(r"\b(libfaer_v0_23_\w+)", out))
    for s in syms:
        assert hasattr(lib, s) and s in exported, s


def test_params_and_scratch(fb):
    lib = fb.load()
    par = fb.capi.par_default()
    for suf, es in (("fx128", 16), ("cx128", 32)):
        ref = "f64" if suf == "fx128" else "c64"
        b = getattr(lib, f"libfaer_v0_23_BidiagParams_{suf}")()
        assert b.par_threshold == getattr(lib, f"libfaer_v0_23_BidiagParams_{ref}")().par_threshold == 192 * 256
        p = getattr(lib, f"libfaer_v0_23_SvdParams_{suf}")()
        q = getattr(lib, f"libfaer_v0_23_SvdParams_{ref}")()
        assert bytes(p) == bytes(q)
        assert (p.bidiag.par_threshold, p.recursion_threshold, p.qr_ratio_threshold) == (192 * 256, 128, 11.0 / 6.0)
        for m, n in ((0, 0), (1, 1), (33, 17), (17, 33), (1000, 999), (65536, 64)):
            for cu in (0, 1, 2):
                for cv in (0, 1, 2):
                    r = getattr(lib, f"libfaer_v0_23_svd_scratch_{suf}")(m, n, cu, cv, par, p)
                    s = getattr(lib, f"libfaer_v0_23_svd_scratch_{ref}")(m, n, cu, cv, par, q)
                    assert (r.len_bytes, r.align_bytes) == (m * n * es, 64) == (s.len_bytes * 2, s.align_bytes)


def test_exact_rectangular_dd_matrices():
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import dd_rect_exact as dre
    rng = np.random.default_rng(4)
    for m, n, cplx, s in ((1, 1, False, 60), (2, 1, False, 60), (33, 17, False, 60), (17, 33, True, 60), (40, 65, True, 60),
                          (200, 100, False, 60), (64, 64, False, 80), (300, 257, True, 60)):
        p = min(m, n)
        a = rng.integers(0, 3, size=p)
        b = rng.integers(0, 4 * p, size=p) + (2 ** 27 if s == 80 else 0)
        ex = dre.rectangular(m, n, a, b, rng, cplx=cplx, s=s)
        A = (ex.hr + 1j * ex.hi_) if cplx else ex.hr
        # the limbs are a valid dd split (|lo| <= ulp(hi) / 2)
        for h, lo in ((ex.hr, ex.lr), (ex.hi_, ex.li_)):
            assert np.all(np.abs(lo) <= np.spacing(np.abs(h)) / 2)
        # U and V have orthonormal columns, and U^H A V = diag(sigma) in f64 on the hi limbs, to f64 accuracy
        sig = np.array([float(x) for x in ex.sigma()])
        assert np.all(np.diff(sig) <= 0)
        for Q in (ex.U, ex.V):
            assert Q.shape[1] == p and np.abs(np.conj(Q.T) @ Q - np.eye(p)).max(initial=0.0) < 1e-15 * Q.shape[0]
        D = np.diag(sig)
        nrm = max(1.0, sig.max(initial=0.0))
        assert np.abs(np.conj(ex.U.T) @ A @ ex.V - D).max() <= 8 * (m + n) * 2.0 ** -53 * nrm
        assert np.abs(np.linalg.svd(A, compute_uv=False) - sig).max() <= 8 * (m + n) * 2.0 ** -53 * nrm
        if m * n <= 33 * 17 and not cplx:  # exact rational check: (hi + lo) V = U diag(sigma)
            Af = [[F(ex.hr[i, j]) + F(ex.lr[i, j]) for j in range(n)] for i in range(m)]
            sf = [F(x) for x in ex.sigma()]
            for j in range(p):
                for i in range(m):
                    assert sum(Af[i][k] * F(ex.V[k, j]) for k in range(n)) == F(ex.U[i, j]) * sf[j]
