"""Generator of tests/golden/dd_ops.npz: input and output bit patterns of the reference's double-double operations (faer-ffi/quad.hpp,
the only statement of qd::Quad's arithmetic in the reference tree) for +, *, /, sqrt, faer's recip (0 when |hi| is infinite, 1 / x
otherwise; faer-traits/src/lib.rs:5179-5186), abs and the comparisons. A throw-away driver is compiled against quad.hpp in a
temporary directory; only the .npz is kept. Run where the reference is present: python tests/golden/make_dd_ops_fixture.py.
tests/test_dd_ops_cpu.py checks that the host build of csrc/dd.cuh reproduces every output bit for bit."""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
QUAD = "/root/reference/faer-ffi/quad.hpp"
OPS = ["add", "mul", "div", "sqrt", "recip", "abs", "lt", "le", "gt", "ge", "eq"]

DRIVER = r"""
#include <cstdio>
#include <vector>
#include "quad.hpp"
using quad::Quad;
int main(int argc, char** argv) {
  long n; int op;
  FILE* f = fopen(argv[1], "rb"); fread(&op, 4, 1, f); fread(&n, 8, 1, f);
  std::vector<double> a(2 * n), b(2 * n), o(2 * n);
  fread(a.data(), 8, 2 * n, f); fread(b.data(), 8, 2 * n, f); fclose(f);
  for (long i = 0; i < n; ++i) {
    Quad x{a[2 * i], a[2 * i + 1]}, y{b[2 * i], b[2 * i + 1]}, r{0.0, 0.0};
    switch (op) {
      case 0: r = x + y; break;
      case 1: r = x * y; break;
      case 2: r = x / y; break;
      case 3: r = quad::sqrt(x); break;
      case 4: r = std::isinf(x.x0) ? Quad{0.0, 0.0} : Quad{1.0} / x; break;
      case 5: r = quad::abs(x); break;
      case 6: r = Quad{x < y ? 1.0 : 0.0, 0.0}; break;
      case 7: r = Quad{x <= y ? 1.0 : 0.0, 0.0}; break;
      case 8: r = Quad{x > y ? 1.0 : 0.0, 0.0}; break;
      case 9: r = Quad{x >= y ? 1.0 : 0.0, 0.0}; break;
      case 10: r = Quad{x == y ? 1.0 : 0.0, 0.0}; break;
    }
    o[2 * i] = r.x0; o[2 * i + 1] = r.x1;
  }
  f = fopen(argv[2], "wb"); fwrite(o.data(), 8, 2 * n, f); fclose(f);
  return 0;
}
"""


def operands(rng, n):
    """n {hi, lo} pairs: random normalised values over many magnitudes, then the special cases"""
    hi = rng.standard_normal(n) * 10.0 ** rng.integers(-300, 300, n)
    lo = hi * 2.0 ** -53 * rng.uniform(-0.5, 0.5, n)
    x = np.stack([hi, lo], 1)
    inf, nan, sub = np.inf, np.nan, 5e-324
    special = [(0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (sub, 0.0), (-3 * sub, 0.0), (2.2e-308, 1e-324), (inf, 0.0),
               (-inf, 0.0), (inf, inf), (nan, 0.0), (1.0, nan), (nan, nan), (1.0, 0.75), (1.0, -1.0), (3.0, 1e-300),
               (1.0, 2.0 ** -53), (1.0, -2.0 ** -54), (1e308, 1e291), (-1e-308, 0.0), (2.0, 0.0), (0.5, 1e-17)]
    return x, np.array(special, dtype=np.float64)


def main() -> int:
    rng = np.random.default_rng(20261017)
    rnd_a, sp = operands(rng, 1500)
    rnd_b, _ = operands(rng, 1500)
    # every pair of special cases, and each special case against random operands
    sa = np.repeat(sp, len(sp), 0)
    sb = np.tile(sp, (len(sp), 1))
    a = np.concatenate([rnd_a, sa, np.repeat(sp, 20, 0), rnd_a[:len(sp) * 20]])
    b = np.concatenate([rnd_b, sb, rnd_b[:len(sp) * 20], np.repeat(sp, 20, 0)])
    # equal high parts, so that the comparisons reach the low limbs
    a[:200, 0] = b[:200, 0]
    out = {"a": a.view(np.uint64), "b": b.view(np.uint64)}
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "drv.cpp")
        open(src, "w").write(DRIVER)
        exe = os.path.join(tmp, "drv")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", os.path.dirname(QUAD), "-o", exe, src])
        for op, name in enumerate(OPS):
            inp, res = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
            with open(inp, "wb") as f:
                f.write(np.int32(op).tobytes() + np.int64(len(a)).tobytes() + a.tobytes() + b.tobytes())
            subprocess.check_call([exe, inp, res])
            out[name] = np.fromfile(res, dtype=np.uint64).reshape(-1, 2)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "dd_ops.npz"), **out)
    print(len(a), "operand pairs,", len(OPS), "operations")
    return 0


if __name__ == "__main__":
    sys.exit(main())
