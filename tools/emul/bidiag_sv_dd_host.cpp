// Host run of the double-double (fx128) singular values of an upper-bidiagonal matrix as csrc/svd_dd.cu computes them: the SAME
// scalar routine the GPU kernel calls (bidiag_sv.cuh's gk_kth_largest through its dd instantiation, tridiag_dd.cuh) with the
// bound of sd_gk_bound_kernel written as the same loop. Test infrastructure for tests/test_bidiag_sv_dd_host_cpu.py, not product
// code. Build with -ffp-contract=off (dd.cuh's host arithmetic must not be fused).
#include <vector>

#include "../../faer-rs_b200/csrc/tridiag_dd.cuh"

using fb::dd;

extern "C" {

// d (n), f (n - 1 used): limbs; s: the n singular values, non-increasing
void bsvdd_values(const double* dh, const double* dl, const double* fh, const double* fl, int n, double* sh, double* sl) {
  std::vector<dd> d((size_t)n + 1, dd(0.0)), f((size_t)n + 1, dd(0.0));
  for (int i = 0; i < n; ++i) {
    d[(size_t)i] = dd(dh[i], dl[i]);
    if (i + 1 < n) f[(size_t)i] = dd(fh[i], fl[i]);
  }
  dd bound(0.0), b2(0.0);
  for (int i = 0; i < n; ++i) {
    const dd a = fabs(d[(size_t)i]), b = i + 1 < n ? fabs(f[(size_t)i]) : dd(0.0), c = i > 0 ? fabs(f[(size_t)i - 1]) : dd(0.0);
    bound = fmax(bound, fmax(a + b, a + c));
    b2 = fmax(b2, fmax(a * a, b * b));
  }
  bound = bound * (dd(1.0) + dd(4.0) * fb::bsv::Lim<dd>::eps()) + fb::bsv::Lim<dd>::safmin();
  for (int k = 0; k < n; ++k) {
    const dd s = fb::bsv::gk_kth_largest<dd>(d.data(), f.data(), n, 1, 1, k, bound, b2);
    sh[k] = s.hi;
    sl[k] = s.lo;
  }
}

}  // extern "C"
