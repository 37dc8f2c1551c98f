// Host build of the double-double scalar (faer-rs_b200/csrc/dd.cuh) as a plain C++ library, for tests/test_dd_ops_cpu.py: the same
// source the GPU runs, compiled with -ffp-contract=off so that every FP64 step is the one rounding the device intrinsics perform.
// dd_host_op(op, a, b, out, n): a, b, out hold n {hi, lo} pairs; comparisons write (result, 0).
#include <cstring>

#include "../../faer-rs_b200/csrc/dd.cuh"

using fb::dd;

extern "C" int dd_host_op(int op, const double* a, const double* b, double* out, long n) {
  for (long i = 0; i < n; ++i) {
    const dd x(a[2 * i], a[2 * i + 1]), y(b[2 * i], b[2 * i + 1]);
    dd r(0.0);
    switch (op) {
      case 0: r = x + y; break;
      case 1: r = x * y; break;
      case 2: r = x / y; break;
      case 3: r = fb::sqrt(x); break;
      case 4: r = fb::dd_recip(x); break;
      case 5: r = fb::fabs(x); break;
      case 6: r = dd(x < y ? 1.0 : 0.0); break;
      case 7: r = dd(x <= y ? 1.0 : 0.0); break;
      case 8: r = dd(x > y ? 1.0 : 0.0); break;
      case 9: r = dd(x >= y ? 1.0 : 0.0); break;
      case 10: r = dd(x == y ? 1.0 : 0.0); break;
      case 11: r = fb::dd_hypot(x, y); break;                   // fx128 hypot
      case 12: r = fb::cdd_abs(fb::cdd{x, y}); break;           // |x + i y| of cx128
      case 13: r = fb::dd_sqrt_min_positive(); break;
      case 14: r = fb::dd_sqrt_max_positive(); break;
      case 15: r = fb::cdd_recip_scaled(fb::cdd{x, y}).re; break;   // 1 / (x + i y) of cx128
      case 16: r = fb::cdd_recip_scaled(fb::cdd{x, y}).im; break;
      default: return -1;
    }
    out[2 * i] = r.hi;
    out[2 * i + 1] = r.lo;
  }
  return 0;
}
