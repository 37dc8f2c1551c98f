"""The double-double (fx128) Golub-Kahan bisection of csrc/svd_dd.cu's values-only path (bidiag_sv.cuh with tridiag_dd.cuh's
bsv::Lim<dd>), run on the CPU by tools/emul/bidiag_sv_dd_host.cpp, against mpmath.svd_r at 300 bits.

Bidiagonals: the graded one of faer's `test_zink` (tests/golden/svd_zink.json), whose smallest singular value is far below the
largest; a cluster with relative gaps near 2^-80 around the midpoint of two doubles near 1/3 (the hi limbs of neighbouring values
differ by one ulp and their lo limbs have opposite signs) with a superdiagonal near 2^-81; and one with an exact zero singular
value (a zero on the diagonal). Each check is an error-to-bound ratio with the bound p 2^-104 ||B||, p = 8 n fixed here and not
tuned. Negative control: the reference values rounded to f64 are rejected on the cluster."""
import ctypes as C
import json
import os
import subprocess

import mpmath
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -104
P = 8
D = C.c_void_p


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("bsvdd") / "libbsvdd.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out,
                           os.path.join(ROOT, "tools", "emul", "bidiag_sv_dd_host.cpp")])
    lib = C.CDLL(out)
    lib.bsvdd_values.argtypes = [D] * 4 + [C.c_int, D, D]
    return lib


def _split(x):
    hi = float(x)
    return hi, float(x - mpmath.mpf(hi))


def _dd(v):
    if not len(v):
        return np.zeros(1), np.zeros(1)
    h, l = zip(*[_split(x) for x in v])
    return np.array(h + (0.0,), dtype=np.float64), np.array(l + (0.0,), dtype=np.float64)


def _reference(dh, dl, fh, fl, n):
    """singular values (non-increasing) of the dd bidiagonal, exactly as stored, through mpmath.svd_r at 300 bits"""
    B = mpmath.zeros(n, n)
    for i in range(n):
        B[i, i] = mpmath.mpf(dh[i]) + mpmath.mpf(dl[i])
        if i + 1 < n:
            B[i, i + 1] = mpmath.mpf(fh[i]) + mpmath.mpf(fl[i])
    s = mpmath.svd_r(B, compute_uv=False)
    return sorted((s[i] for i in range(n)), reverse=True)


def _case(name):
    mpmath.mp.prec = 300
    if name == "zink":
        fx = json.load(open(os.path.join(ROOT, "tests", "golden", "svd_zink.json")))
        n = len(fx["diag"])
        d = [mpmath.mpf(x) for x in fx["diag"]]
        f = [mpmath.mpf(x) for x in fx["subdiag"][: n - 1]]
    elif name == "cluster":
        n = 60
        rng = np.random.default_rng(80)
        mid = mpmath.mpf(float(mpmath.mpf(1) / 3)) + mpmath.mpf(2) ** -55
        d = [mid + (i - n // 2) * mpmath.mpf(2) ** -80 for i in range(n)]
        f = [mpmath.mpf(float(x)) * mpmath.mpf(2) ** -81 for x in rng.uniform(0.5, 1.0, n - 1)]
    else:  # a zero on the diagonal: one singular value is exactly zero
        n = 40
        rng = np.random.default_rng(0)
        d = [mpmath.mpf(float(x)) for x in rng.uniform(-2.0, 2.0, n)]
        d[n // 3] = mpmath.mpf(0)
        f = [mpmath.mpf(float(x)) for x in rng.uniform(-2.0, 2.0, n - 1)]
    dh, dl = _dd(d)
    fh, fl = _dd(f)
    return n, dh, dl, fh, fl


def _ratio(ref, sh, sl, n):
    nrm = float(max(abs(x) for x in ref))
    err = max(abs(mpmath.mpf(h) + mpmath.mpf(l) - r) for h, l, r in zip(sh, sl, ref))
    return float(err) / (P * n * U * nrm)


@pytest.mark.parametrize("name", ["zink", "cluster", "zero"])
def test_dd_bisection_against_mpmath(lib, name):
    n, dh, dl, fh, fl = _case(name)
    ref = _reference(dh, dl, fh, fl, n)
    sh, sl = np.zeros(n), np.zeros(n)
    lib.bsvdd_values(dh.ctypes.data, dl.ctypes.data, fh.ctypes.data, fl.ctypes.data, n, sh.ctypes.data, sl.ctypes.data)
    assert np.all(np.diff(sh + sl) <= 0)
    r = _ratio(ref, sh, sl, n)
    print(f"[bsvdd] {name} n={n}: {r:.3g}")
    assert r <= 1.0
    if name == "zero":
        assert sh[-1] + sl[-1] <= P * n * U * float(ref[0])
    if name == "cluster":  # f64-accurate values do not pass the dd bound
        assert _ratio(ref, [float(x) for x in ref], [0.0] * n, n) > 1.0
