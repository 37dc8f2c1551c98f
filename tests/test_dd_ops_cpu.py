"""The double-double scalar of csrc/dd.cuh, built for the host (tools/emul/dd_host.cpp, -ffp-contract=off), against the reference's
quad.hpp (tests/golden/dd_ops.npz, written by tests/golden/make_dd_ops_fixture.py): +, *, /, sqrt, faer's recip, abs and the
comparisons reproduce every output bit for random operands over many magnitudes and for the special cases (signed zeros, subnormal
high parts, infinities, NaN in either limb, a non-normalised low limb). NaN outputs match as NaN in the same limbs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = ["add", "mul", "div", "sqrt", "recip", "abs", "lt", "le", "gt", "ge", "eq"]


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


def host_op(lib, op, a, b):
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    out = np.zeros_like(a)
    assert lib.dd_host_op(op, a.ctypes.data, b.ctypes.data, out.ctypes.data, len(a)) == 0
    return out


@pytest.mark.parametrize("op", range(len(OPS)), ids=OPS)
def test_host_build_reproduces_quad_hpp(ddh, op):
    g = np.load(os.path.join(ROOT, "tests", "golden", "dd_ops.npz"))
    a, b = g["a"].view(np.float64), g["b"].view(np.float64)
    want = g[OPS[op]]
    got = host_op(ddh, op, a, b).view(np.uint64)
    wn, gn = np.isnan(want.view(np.float64)), np.isnan(got.view(np.float64))
    assert np.array_equal(wn, gn)
    bad = np.nonzero((want != got) & ~wn)
    assert bad[0].size == 0, (OPS[op], a[bad[0][:3]], b[bad[0][:3]], want[bad[0][:3]].view(np.float64), got[bad[0][:3]].view(np.float64))
