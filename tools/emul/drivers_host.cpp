// Host build of the flat-map DRIVERS themselves — faer-rs_b200/csrc/{cplx_condensed,ldlt_types,reconstruct_types}.cu are included
// here as they are and compiled by a plain C++ compiler against hostcuda/cuda_runtime.h — so that their control flow, view
// arithmetic, workspace sizes and the flags they pass to the building blocks run end to end on the CPU
// (tests/test_drivers_host_cpu.py). The building blocks they call (structured products, triangular solves, Householder sequences,
// the real tridiagonal / bidiagonal solvers) are forwarded to a callback the test registers, which executes them with the oracle /
// LAPACK. "Device" workspace comes from a checking allocator: fresh blocks are filled with NaN patterns, both ends carry guard
// words that are verified on release.
// TEST INFRASTRUCTURE: nothing in the product links this file.
#include "mock_blocks.hpp"

static long long g_guard_errors = 0, g_live_blocks = 0;

namespace fb {

unsigned long long g_launch_count = 0;
int g_launch_tag = 0;
signed char* g_launch_log = nullptr;
size_t g_launch_log_len = 0, g_launch_log_cap = 0;

// ---- checking allocator ----
namespace {
constexpr size_t GUARD = 64;
struct Hdr {
  size_t bytes;
};
}  // namespace
void* ws_alloc(size_t bytes) {
  if (bytes == 0) bytes = 256;
  unsigned char* raw = (unsigned char*)malloc(sizeof(Hdr) + GUARD + bytes + GUARD);
  ((Hdr*)raw)->bytes = bytes;
  memset(raw + sizeof(Hdr), 0xA5, GUARD);
  memset(raw + sizeof(Hdr) + GUARD, 0xFF, bytes);  // NaN for every floating-point type: a read of unwritten workspace shows
  memset(raw + sizeof(Hdr) + GUARD + bytes, 0x5A, GUARD);
  ++g_live_blocks;
  return raw + sizeof(Hdr) + GUARD;
}
void ws_free(void* p) {
  unsigned char* user = (unsigned char*)p;
  unsigned char* raw = user - GUARD - sizeof(Hdr);
  const size_t bytes = ((Hdr*)raw)->bytes;
  for (size_t k = 0; k < GUARD; ++k) {
    if (raw[sizeof(Hdr) + k] != 0xA5) ++g_guard_errors;
    if (user[bytes + k] != 0x5A) ++g_guard_errors;
  }
  --g_live_blocks;
  free(raw);
}

}  // namespace fb

// ---- the drivers, as they are ----------------------------------------------------------------------------------------------------
#include "../../faer-rs_b200/csrc/cplx_condensed.cu"
#include "../../faer-rs_b200/csrc/ldlt_types.cu"
#include "../../faer-rs_b200/csrc/reconstruct_types.cu"

// ---- C entry points for the test -------------------------------------------------------------------------------------------------
using namespace fb;
template <class R>
static View<R> vw(const MockMat& m) { return View<R>{(R*)m.ptr, m.nrows, m.ncols, m.rs, m.cs}; }
template <class R>
static View<const R> cvw(const MockMat& m) { return View<const R>{(const R*)m.ptr, m.nrows, m.ncols, m.rs, m.cs}; }

// kind: 0 f32, 1 f64, 2 c32, 3 c64. which: 0 llt_reconstruct, 1 llt_inverse, 2 lu_reconstruct, 3 lu_inverse, 4 qr_reconstruct, 5 qr_inverse
template <class R, bool CX>
static void recon(int which, MockMat out, MockMat a, MockMat b, MockMat c, const long long* perm) {
  switch (which) {
    case 0: llt_reconstruct_t<R, CX>(nullptr, vw<R>(out), cvw<R>(a)); break;
    case 1: llt_inverse_t<R, CX>(nullptr, vw<R>(out), cvw<R>(a)); break;
    case 2: lu_reconstruct_t<R, CX>(nullptr, vw<R>(out), cvw<R>(a), cvw<R>(b), perm); break;
    case 3: lu_inverse_t<R, CX>(nullptr, vw<R>(out), cvw<R>(a), cvw<R>(b), perm); break;
    case 4: qr_reconstruct_t<R, CX>(nullptr, vw<R>(out), cvw<R>(a), cvw<R>(b), cvw<R>(c)); break;
    case 5: qr_inverse_t<R, CX>(nullptr, vw<R>(out), cvw<R>(a), cvw<R>(b), cvw<R>(c)); break;
  }
}
// which: 0 factor (info[0] = failure index or -1, info[1] = count), 1 solve (conj in flag), 2 reconstruct, 3 inverse
template <class R, bool CX>
static void ldlt(int which, MockMat a, MockMat b, const void* D, long long dstride, const signed char* signs, double delta, double eps,
                 int flag, long long* info) {
  switch (which) {
    case 0: {
      const LdltResult r = ldlt_in_place_t<R, CX>(nullptr, vw<R>(a), (R)delta, (R)eps, signs);
      info[0] = r.ok ? -1 : (long long)r.zero_pivot_index;
      info[1] = r.ok ? (long long)r.dynamic_regularization_count : 0;
      break;
    }
    case 1: ldlt_solve_in_place_t<R, CX>(nullptr, cvw<R>(a), (const R*)D, dstride, flag != 0, vw<R>(b)); break;
    case 2: ldlt_reconstruct_t<R, CX>(nullptr, vw<R>(b), cvw<R>(a), (const R*)D, dstride); break;
    case 3: ldlt_inverse_t<R, CX>(nullptr, vw<R>(b), cvw<R>(a), (const R*)D, dstride); break;
  }
}
extern "C" {
void drivers_set_callback(mock_cb_t cb) { g_cb = cb; }
void drivers_set_reverse(int r) { fb::flat_map_host_reverse = r != 0; }
long long drivers_guard_errors() { return g_guard_errors; }
long long drivers_live_blocks() { return g_live_blocks; }

// is_double: c64 / c32. U / V with ptr == null: not wanted. S: complex entries, sstride apart.
int drv_svd(int is_double, MockMat A, MockMat U, void* S, long long sstride, MockMat V) {
  if (is_double) return svd_cx<double>(nullptr, cvw<double>(A), vw<double>(U), (double*)S, sstride, vw<double>(V));
  return svd_cx<float>(nullptr, cvw<float>(A), vw<float>(U), (float*)S, sstride, vw<float>(V));
}
int drv_evd(int is_double, MockMat A, MockMat U, void* S, long long sstride) {
  if (is_double) return self_adjoint_evd_cx<double>(nullptr, cvw<double>(A), vw<double>(U), (double*)S, sstride);
  return self_adjoint_evd_cx<float>(nullptr, cvw<float>(A), vw<float>(U), (float*)S, sstride);
}
void drv_recon(int kind, int which, MockMat out, MockMat a, MockMat b, MockMat c, const long long* perm) {
  switch (kind) {
    case 0: recon<float, false>(which, out, a, b, c, perm); break;
    case 1: recon<double, false>(which, out, a, b, c, perm); break;
    case 2: recon<float, true>(which, out, a, b, c, perm); break;
    case 3: recon<double, true>(which, out, a, b, c, perm); break;
  }
}
void drv_ldlt(int kind, int which, MockMat a, MockMat b, const void* D, long long dstride, const signed char* signs, double delta,
              double eps, int flag, long long* info) {
  switch (kind) {
    case 0: ldlt<float, false>(which, a, b, D, dstride, signs, delta, eps, flag, info); break;
    case 2: ldlt<float, true>(which, a, b, D, dstride, signs, delta, eps, flag, info); break;
    case 3: ldlt<double, true>(which, a, b, D, dstride, signs, delta, eps, flag, info); break;
  }
}
// f64 reconstruct / inverse of the LDLT (the factorization itself stays on ldlt_f64.cu)
void drv_ldlt_f64(int which, MockMat a, MockMat b, const void* D, long long dstride) {
  if (which == 2) ldlt_reconstruct_t<double, false>(nullptr, vw<double>(b), cvw<double>(a), (const double*)D, dstride);
  else ldlt_inverse_t<double, false>(nullptr, vw<double>(b), cvw<double>(a), (const double*)D, dstride);
}
}
