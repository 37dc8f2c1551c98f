// extern "C" boundary of the double-double kinds (include/faer_b200_fx128*.h): fx128 = <dd, false>, cx128 = <dd, true>. The
// families they share with the IEEE kinds are ffi_entries.cuh's bodies, instantiated here; their drivers are gemm_dd.cu,
// dd_factor.cu, qr_dd.cu and the <dd, CX> instantiations of the reconstruct_types.cu compositions. The self-adjoint EVD
// (evd_dd.cu) and the SVD (svd_dd.cu) are dd only. Same conventions as ffi.cu (by-value PODs, synchronous on return, abort() on precondition violations,
// host buffers staged, device buffers used in place, `Par` ignored); scratch sizes are the f64 / c64 formulas with 16 / 32-byte
// elements.
#include "../../include/faer_b200.h"
#include "dd.cuh"
#include "ffi_common.cuh"
#include "ffi_entries.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

using namespace fb;

namespace {

// self-adjoint EVD (evd/mod.rs:270-418): the f64 / c64 entries' semantics (ffi.cu, ffi_types.cu); S holds (value, 0) for cx128
template <bool CX>
FaerV0_24_EvdStatus self_adjoint_evd_entry_dd(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = A.nrows, e = elem_bytes<dd, CX>();
  FB_ASSERT(A.ncols == n && S.len == n && (n == 0 || S.stride >= 1), "self_adjoint_evd: square A, S of length n, positive stride");
  const bool want_u = U.ncols != 0;
  if (want_u) FB_ASSERT(U.nrows == n && U.ncols == n, "self_adjoint_evd: U must be n x n (or have no columns)");
  if (n == 0) return evd_status(true);
  StagedMat a = stage<dd, CX>(A, st);
  dd* s_dev = (dd*)ws_alloc(n * e);
  bool ok;
  if (want_u) {
    StagedMat u = stage<dd, CX>(U, false, st);
    ok = self_adjoint_evd_dd<CX>(st, a.view<const dd>(), u.view<dd>(), s_dev);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * e, s_dev, e, e, n, cudaMemcpyDefault, st));
    finish_all(st, {&a, &u});
  } else {
    ok = self_adjoint_evd_dd<CX>(st, a.view<const dd>(), View<dd>{nullptr, 0, 0, 1, 1}, s_dev);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * e, s_dev, e, e, n, cudaMemcpyDefault, st));
    finish_all(st, {&a});
  }
  ws_free(s_dev);
  return evd_status(ok);
}

// SVD (svd/mod.rs:530-672): the f64 / c64 entries' semantics (ffi.cu, ffi_types.cu); U.ncols == 0 / V.ncols == 0 mean "do not
// compute" (faer-ffi/src/lib.rs:2354-2355); S holds (value, 0) for cx128
template <bool CX>
FaerV0_24_SvdStatus svd_entry_dd(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S, FaerV0_24_MatMut V,
                                 double qr_ratio_threshold) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols, e = elem_bytes<dd, CX>();
  FB_ASSERT(S.len == size && (size == 0 || S.stride >= 1), "svd: S must have min(nrows, ncols) entries and a positive stride");
  const bool want_u = U.ncols != 0, want_v = V.ncols != 0;
  if (want_u) FB_ASSERT(U.nrows == A.nrows && (U.ncols == A.nrows || U.ncols == size), "svd: U must be nrows x {size, nrows}");
  if (want_v) FB_ASSERT(V.nrows == A.ncols && (V.ncols == A.ncols || V.ncols == size), "svd: V must be ncols x {size, ncols}");
  const double ratio = qr_ratio_threshold > 0.0 ? qr_ratio_threshold : 11.0 / 6.0;
  if (size == 0 && !want_u && !want_v) return svd_status(true);
  StagedMat a = stage<dd, CX>(A, st);
  dd* s_dev = (dd*)ws_alloc((size + 1) * e);
  StagedMat u = stage<dd, CX>(U, false, st), v = stage<dd, CX>(V, false, st);
  const View<dd> none{nullptr, 0, 0, 1, 1};
  const bool ok = svd_dd<CX>(st, a.view<const dd>(), want_u ? u.view<dd>() : none, s_dev, want_v ? v.view<dd>() : none, ratio);
  if (ok && size) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * e, s_dev, e, e, size, cudaMemcpyDefault, st));
  finish_all(st, {&a, &u, &v});
  ws_free(s_dev);
  return svd_status(ok);
}

}  // namespace

extern "C" {

FB_MATMUL_FFI(fx128, dd, false)
FB_MATMUL_FFI(cx128, dd, true)
FB_TRSM_FFI(fx128, dd, false)
FB_TRSM_FFI(cx128, dd, true)
FB_TRI_INV_FFI(fx128, dd, false)
FB_TRI_INV_FFI(cx128, dd, true)
FB_LLT_FFI(fx128, dd, false)
FB_LLT_FFI(cx128, dd, true)
FB_LLT_RECON_FFI(fx128, dd, false)
FB_LLT_RECON_FFI(cx128, dd, true)
FB_LU_FFI(fx128, dd, false)
FB_LU_FFI(cx128, dd, true)
FB_LU_RECON_FFI(fx128, dd, false)
FB_LU_RECON_FFI(cx128, dd, true)
FB_QR_FFI(fx128, dd, false)
FB_QR_FFI(cx128, dd, true)
FB_QR_RECON_FFI(fx128, dd, false)
FB_QR_RECON_FFI(cx128, dd, true)
FB_QR_INV_FFI(fx128, dd, false)
FB_QR_INV_FFI(cx128, dd, true)

// ---- self-adjoint EVD: faer's defaults (evd/mod.rs:82-90) and the f64 / c64 scratch formula with 16 / 32-byte elements ----
#define FB_DD_EVD_FFI(SUF, CX)                                                                                                   \
  FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_##SUF(void) { return FaerV0_24_TridiagParams{192 * 256}; }               \
  FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_##SUF(void) {                                              \
    return FaerV0_24_SelfAdjointEvdParams{FaerV0_24_TridiagParams{192 * 256}, 128};                                            \
  }                                                                                                                            \
  FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_##SUF(size_t dim, FaerV0_24_ComputeEigenvectors compute_U,           \
                                                                FaerV0_24_Par par, FaerV0_24_SelfAdjointEvdParams params) {    \
    (void)compute_U; (void)par; (void)params;                                                                                  \
    return FaerV0_24_Layout{dim * dim * elem_bytes<dd, CX>(), 64};                                                             \
  }                                                                                                                            \
  FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_##SUF(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S,         \
                                                           FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                          \
                                                           FaerV0_24_SelfAdjointEvdParams params) {                            \
    (void)par; (void)mem; (void)params;                                                                                        \
    return self_adjoint_evd_entry_dd<CX>(A, U, S);                                                                             \
  }
FB_DD_EVD_FFI(fx128, false)
FB_DD_EVD_FFI(cx128, true)
#undef FB_DD_EVD_FFI

// ---- SVD: faer's defaults (svd/mod.rs:49-58, as ffi.cu's f64 / f32 entries) and the f64 / c64 scratch formula with 16 / 32-byte
// elements ----
#define FB_DD_SVD_FFI(SUF, CX)                                                                                                   \
  FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_##SUF(void) { return FaerV0_24_BidiagParams{192 * 256}; }                 \
  FaerV0_24_SvdParams libfaer_v0_23_SvdParams_##SUF(void) {                                                                    \
    return FaerV0_24_SvdParams{FaerV0_24_BidiagParams{192 * 256}, FaerV0_24_QrParams{48 * 48, 192 * 256}, 128, 11.0 / 6.0};    \
  }                                                                                                                            \
  FaerV0_24_Layout libfaer_v0_23_svd_scratch_##SUF(size_t nrows, size_t ncols, FaerV0_24_ComputeSvdVectors compute_U,         \
                                                   FaerV0_24_ComputeSvdVectors compute_V, FaerV0_24_Par par,                  \
                                                   FaerV0_24_SvdParams params) {                                              \
    (void)compute_U; (void)compute_V; (void)par; (void)params;                                                                 \
    return FaerV0_24_Layout{nrows * ncols * elem_bytes<dd, CX>(), 64};                                                         \
  }                                                                                                                            \
  FaerV0_24_SvdStatus libfaer_v0_23_svd_##SUF(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S, FaerV0_24_MatMut V,  \
                                              FaerV0_24_Par par, FaerV0_24_MemAlloc mem, FaerV0_24_SvdParams params) {        \
    (void)par; (void)mem;                                                                                                      \
    return svd_entry_dd<CX>(A, U, S, V, params.qr_ratio_threshold);                                                           \
  }
FB_DD_SVD_FFI(fx128, false)
FB_DD_SVD_FFI(cx128, true)
#undef FB_DD_SVD_FFI

}  // extern "C"
