"""CPU-side checks of the double-double self-adjoint EVD C ABI (include/faer_b200_fx128_evd.h, included by include/faer_b200.h):
its 8 prototypes are exactly the reference header's fx128 / cx128 `TridiagParams`, `SelfAdjointEvdParams`,
`self_adjoint_evd_scratch` and `self_adjoint_evd` (tests/golden/faer_ffi_fx128_evd_prototypes.json, extracted by
tests/golden/make_fx128_evd_prototypes.py); libfaer_b200.so exports all of them; the params queries return faer's defaults and the
scratch query the f64 / c64 formula with 16 / 32-byte elements. Also: the exact dd test matrices of tests/dd_spectral_exact.py
are what they claim (their limbs reproduce the integer matrix, and LAPACK on the hi limbs finds the spectrum within f64 bounds)."""
import json
import os
import re
import subprocess
import importlib.util

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "faer_b200_fx128_evd.h")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "faer_ffi_fx128_evd_prototypes.json")))


def _parser():
    spec = importlib.util.spec_from_file_location("make_ffi_prototypes", os.path.join(ROOT, "tests", "golden", "make_ffi_prototypes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_fx128_evd_prototypes_match_the_reference_header():
    ours = _parser().prototypes(open(HDR).read())
    assert len(GOLD["prototypes"]) == 8
    assert ours == GOLD["prototypes"]


def test_main_header_includes_the_fx128_evd_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "faer_b200.h")).read(), flags=re.S)
    assert '#include "faer_b200_fx128_evd.h"' in txt


def test_library_exports_every_fx128_evd_symbol(fb):
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
        t = getattr(lib, f"libfaer_v0_23_TridiagParams_{suf}")()
        assert t.par_threshold == lib.libfaer_v0_23_TridiagParams_f64().par_threshold == 192 * 256
        p = getattr(lib, f"libfaer_v0_23_SelfAdjointEvdParams_{suf}")()
        assert (p.tridiag.par_threshold, p.recursion_threshold) == (192 * 256, 128)
        ref = "f64" if suf == "fx128" else "c64"
        for n in (0, 1, 33, 1000, 4096):
            for cu in (0, 1):
                r = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_scratch_{suf}")(n, cu, par, p)
                q = getattr(lib, f"libfaer_v0_23_self_adjoint_evd_scratch_{ref}")(n, cu, par, p)
                assert (r.len_bytes, r.align_bytes) == (n * n * es, 64) == (q.len_bytes * 2, q.align_bytes)


def test_exact_dd_matrices():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import dd_spectral_exact as dse
    from fractions import Fraction as F
    rng = np.random.default_rng(3)
    for n, cplx in ((1, False), (5, False), (33, False), (40, True), (300, False), (257, True)):
        a = rng.integers(-1, 2, size=n)
        b = rng.integers(-n, n, size=n)
        ex = dse.build(a, b, rng, cplx=cplx)
        # hermitian, and the limbs are a valid dd split (|lo| <= ulp(hi) / 2)
        A = (ex.hr + 1j * ex.hi_) if cplx else ex.hr
        assert np.array_equal(A, np.conj(A.T))
        assert np.all(np.abs(ex.lr) <= np.spacing(np.abs(ex.hr)) / 2)
        # V is unitary and A V = V diag(lambda) in f64 on the hi limbs, to f64 accuracy
        V = ex.V
        assert np.abs(np.conj(V.T) @ V - np.eye(n)).max() < 1e-15 * n
        lam = ex.a * 2.0 ** 60 + ex.b
        assert np.abs(A @ V - V * lam).max() <= 8 * n * 2.0 ** -53 * max(1.0, np.abs(lam).max())
        assert np.allclose(np.linalg.eigvalsh(A), np.sort(lam), rtol=0, atol=8 * n * 2.0 ** -53 * np.abs(lam).max())
        if n <= 40 and not cplx:  # exact rational check: (hi + lo) V = V diag(2^60 a + b)
            Af = [[F(ex.hr[i, j]) + F(ex.lr[i, j]) for j in range(n)] for i in range(n)]
            Vf = [[F(V[i, j]) for j in range(n)] for i in range(n)]
            lamf = [F(int(x)) * 2 ** 60 + F(int(y)) for x, y in zip(ex.a, ex.b)]
            for j in range(n):
                for i in range(n):
                    assert sum(Af[i][k] * Vf[k][j] for k in range(n)) == Vf[i][j] * lamf[j]
