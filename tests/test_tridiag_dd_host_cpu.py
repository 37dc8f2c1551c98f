"""The double-double (fx128) instantiations of the tridiagonal scalar cores (csrc/tridiag_dd.cuh: tridiag_dc_core.cuh's divide
and conquer and tridiag_ev.cuh's bisection), run on the CPU by tools/emul/tridiag_dd_host.cpp with evd_dd.cu's glue as plain
loops, against mpmath at 300 bits.

Matrices (n up to 200): the 1-2-1 Toeplitz matrix and the Clement matrix (closed-form spectra evaluated in mpmath: 2 - 2 cos(k pi /
(n + 1)) and -(n-1), -(n-3), ..., n-1; Clement's off-diagonal sqrt(i (n - i)) is rounded to dd, which moves the spectrum by less
than 2^-105 ||T||); Wilkinson's W21+, whose two largest eigenvalues agree to about 7e-14; and a spectrum with relative gaps near
2^-80 (diagonal m + i 2^-80 around the midpoint m of two doubles near 1/3, off-diagonal about 2^-81: nothing deflates, the merges' poles are 2^-80 apart), both through
mpmath.eigsy at 300 bits.

Checks, each as an error-to-bound ratio with the bound p 2^-104 ||T||, p = 8 n fixed here and not tuned: the eigenvalues of both
paths against mpmath, and for divide and conquer the residual max_j ||T q_j - lambda_j q_j|| and max |Q^T Q - I| (over p 2^-104),
both accumulated in dd. Negative controls: f64-accurate eigenvalues are rejected, and so is divide and conquer built with faer's
own dd subtraction in place of dd_sub_accurate (tools/emul/tridiag_dd_host.cpp -DTDD_SLOPPY) on the 2^-80 spectrum."""
import ctypes as C
import os
import subprocess

import mpmath
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -104
P = 8  # p = P n
D = C.c_void_p


def _build(tmp, sloppy):
    out = str(tmp / ("libtdd_sloppy.so" if sloppy else "libtdd.so"))
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    flags = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out,
             os.path.join(ROOT, "tools", "emul", "tridiag_dd_host.cpp")]
    subprocess.check_call(flags + (["-DTDD_SLOPPY"] if sloppy else []))
    lib = C.CDLL(out)
    lib.tdd_values.argtypes = [D] * 4 + [C.c_int, D, D]
    lib.tdd_eig.argtypes = [D] * 4 + [C.c_int] + [D] * 4
    lib.tdd_eig.restype = C.c_int
    lib.tdd_check.argtypes = [D] * 4 + [C.c_int] + [D] * 5
    return lib


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("tdd")
    return _build(tmp, False), _build(tmp, True)


def _split(x):
    """an mpf -> (hi, lo) doubles: the dd nearest to x"""
    hi = float(x)
    return hi, float(x - mpmath.mpf(hi))


def _dd(v):
    h, l = zip(*[_split(x) for x in v]) if len(v) else ((), ())
    return np.array(h, dtype=np.float64), np.array(l, dtype=np.float64)


def _ptr(a):
    return a.ctypes.data


class Case:
    def __init__(self, name, d, e, ref):
        self.name, self.ref = name, ref  # ref: ascending mpf eigenvalues of the dd matrix
        self.dh, self.dl = _dd(d)
        self.eh, self.el = _dd(e)
        self.n = len(d)
        self.norm = float(max(abs(x) for x in ref)) if ref else 0.0


def _exact_mpf(h, l):
    return [mpmath.mpf(a) + mpmath.mpf(b) for a, b in zip(h, l)]


def _eigsy_ref(dh, dl, eh, el):
    n = len(dh)
    d, e = _exact_mpf(dh, dl), _exact_mpf(eh, el)
    A = mpmath.zeros(n, n)
    for i in range(n):
        A[i, i] = d[i]
        if i + 1 < n:
            A[i, i + 1] = A[i + 1, i] = e[i]
    return sorted(mpmath.eigsy(A, eigvals_only=True))


def _cases():
    mpmath.mp.prec = 300
    out = []
    n = 200
    out.append(Case("toeplitz_121_200", [mpmath.mpf(2)] * n, [mpmath.mpf(1)] * (n - 1),
                    sorted(2 - 2 * mpmath.cos(k * mpmath.pi / (n + 1)) for k in range(1, n + 1))))
    out.append(Case("clement_200", [mpmath.mpf(0)] * n, [mpmath.sqrt(i * (n - i)) for i in range(1, n)],
                    [mpmath.mpf(-(n - 1) + 2 * k) for k in range(n)]))
    d = [mpmath.mpf(abs(10 - i)) for i in range(21)]
    e = [mpmath.mpf(1)] * 20
    c = Case("wilkinson_w21", d, e, [])
    c.ref = _eigsy_ref(c.dh, c.dl, c.eh, c.el)
    c.norm = float(max(abs(x) for x in c.ref))
    out.append(c)
    rng = np.random.default_rng(80)
    n = 100
    # centred on the midpoint between two doubles near 1/3, so that the hi limbs of the cluster differ by one ulp and their lo
    # limbs have opposite signs: faer's subtraction then rounds a.lo - b.lo, an error of order 2^-107 against gaps of 2^-80
    mid = mpmath.mpf(float(mpmath.mpf(1) / 3)) + mpmath.mpf(2) ** -55
    d = [mid + (i - n // 2) * mpmath.mpf(2) ** -80 for i in range(n)]
    e = [mpmath.mpf(float(x)) * mpmath.mpf(2) ** -81 for x in rng.uniform(0.5, 1.0, n - 1)]
    c = Case("gaps_2e-80", d, e, [])
    c.ref = _eigsy_ref(c.dh, c.dl, c.eh, c.el)
    c.norm = float(max(abs(x) for x in c.ref))
    out.append(c)
    return out


@pytest.fixture(scope="module")
def cases():
    return _cases()


def _value_ratio(c, h, l):
    err = max(abs((mpmath.mpf(a) + mpmath.mpf(b)) - r) for a, b, r in zip(h, l, c.ref))
    return float(err) / (P * c.n * U * c.norm)


def _dc(lib, c):
    n = c.n
    lh, ll = np.zeros(n), np.zeros(n)
    qh, ql = np.zeros(n * n), np.zeros(n * n)
    assert lib.tdd_eig(_ptr(c.dh), _ptr(c.dl), _ptr(c.eh), _ptr(c.el), n, _ptr(lh), _ptr(ll), _ptr(qh), _ptr(ql)) == 0
    out = np.zeros(2)
    lib.tdd_check(_ptr(c.dh), _ptr(c.dl), _ptr(c.eh), _ptr(c.el), n, _ptr(lh), _ptr(ll), _ptr(qh), _ptr(ql), _ptr(out))
    return {"values": _value_ratio(c, lh, ll), "residual": out[0] / (P * n * U * c.norm), "orth": out[1] / (P * n * U)}


def test_divide_and_conquer_and_bisection_reach_dd_accuracy(libs, cases):
    lib = libs[0]
    for c in cases:
        r = _dc(lib, c)
        vh, vl = np.zeros(c.n), np.zeros(c.n)
        lib.tdd_values(_ptr(c.dh), _ptr(c.dl), _ptr(c.eh), _ptr(c.el), c.n, _ptr(vh), _ptr(vl))
        r["bisection"] = _value_ratio(c, vh, vl)
        print(c.name, {k: float(f"{v:.3g}") for k, v in r.items()})
        for k, v in r.items():
            assert v <= 1.0, (c.name, k, v)


def test_f64_accurate_values_are_rejected(cases):
    for c in cases:
        h = np.array([float(x) for x in c.ref])
        r = _value_ratio(c, h, np.zeros(c.n))
        print(c.name, "f64 values", f"{r:.3g}")
        if c.name != "clement_200":  # Clement's integer spectrum is exact in f64
            assert r > 1.0, (c.name, r)


def test_faer_subtraction_in_the_secular_solver_is_rejected(libs, cases):
    c = next(c for c in cases if c.name == "gaps_2e-80")
    r = _dc(libs[1], c)
    print("sloppy dc_sub", {k: float(f"{v:.3g}") for k, v in r.items()})
    assert max(r.values()) > 1.0, r
