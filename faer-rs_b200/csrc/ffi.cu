// extern "C" boundary: the symbols declared in include/faer_b200.h. The entry points every scalar kind shares are written once
// in ffi_entries.cuh and instantiated here for f64, f32, c64 and c32 (ffi_types.cu: the entry points whose drivers are the
// flat-map files; ffi_dd.cu: fx128 / cx128; helpers shared by all: ffi_common.cuh). What stays here is f64 / f32 only: LDLT f64,
// the real `svd` / `self_adjoint_evd`, and the extensions.
// Each entry point mirrors the faer-ffi function of the same name (faer-ffi/src/lib.rs, cited per function in the
// header): same argument order and meaning, by-value PODs, synchronous on return, abort() on precondition
// violations. Host buffers are staged; device buffers are used in place.
#include "../../include/faer_b200.h"
#include "ffi_common.cuh"
#include "ffi_entries.cuh"
#include "gemm_f32.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

#include <atomic>
#include <cstring>
#include <vector>

using namespace fb;

namespace {

std::atomic<int> g_par_tag{FaerV0_24_ParTag_Rayon};
std::atomic<size_t> g_par_threads{0};

// ---- self-adjoint eigendecomposition (evd/mod.rs:270-418): eigenvalues by bisection when U is not wanted, divide and
// conquer + Householder back-transform otherwise. Non-finite input -> EvdStatus::NoConvergence, as the reference ----
template <class T>
FaerV0_24_EvdStatus self_adjoint_evd_entry(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = A.nrows;
  FB_ASSERT(A.ncols == n && S.len == n && (n == 0 || S.stride >= 1), "self_adjoint_evd: square A, S of length n, positive stride");
  const bool want_u = U.ncols != 0;
  if (want_u) FB_ASSERT(U.nrows == n && U.ncols == n, "self_adjoint_evd: U must be n x n (or have no columns)");
  if (n == 0) return evd_status(true);
  StagedMat a = stage<T, false>(A, st);
  T* s_dev = (T*)ws_alloc(n * sizeof(T));
  bool ok;
  if (want_u) {
    StagedMat u = stage<T, false>(U, false, st);
    ok = self_adjoint_evd_with_vectors<T>(st, a.view<const T>(), u.view<T>(), s_dev, 1);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * sizeof(T), s_dev, sizeof(T), sizeof(T), n, cudaMemcpyDefault, st));
    finish_all(st, {&a, &u});
  } else {
    ok = self_adjoint_eigenvalues<T>(st, a.view<const T>(), s_dev);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * sizeof(T), s_dev, sizeof(T), sizeof(T), n, cudaMemcpyDefault, st));
    finish_all(st, {&a});
  }
  ws_free(s_dev);
  return evd_status(ok);
}
// ---- SVD (svd/mod.rs:530-672): U.ncols == 0 / V.ncols == 0 mean "do not compute" (faer-ffi/src/lib.rs:2354-2355) ----
template <class T>
FaerV0_24_SvdStatus svd_entry(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S, FaerV0_24_MatMut V,
                              double qr_ratio_threshold) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols;
  FB_ASSERT(S.len == size && (size == 0 || S.stride >= 1), "svd: S must have min(nrows, ncols) entries and a positive stride");
  const bool want_u = U.ncols != 0, want_v = V.ncols != 0;
  if (want_u) FB_ASSERT(U.nrows == A.nrows && (U.ncols == A.nrows || U.ncols == size), "svd: U must be nrows x {size, nrows}");
  if (want_v) FB_ASSERT(V.nrows == A.ncols && (V.ncols == A.ncols || V.ncols == size), "svd: V must be ncols x {size, ncols}");
  const double ratio = qr_ratio_threshold > 0.0 ? qr_ratio_threshold : 11.0 / 6.0;
  if (size == 0 && !want_u && !want_v) return svd_status(true);
  StagedMat a = stage<T, false>(A, st);
  T* s_dev = (T*)ws_alloc((size + 1) * sizeof(T));
  bool ok;
  if (want_u || want_v) {
    StagedMat u = stage<T, false>(U, false, st), v = stage<T, false>(V, false, st);
    View<T> uv = want_u ? u.view<T>() : View<T>{nullptr, 0, 0, 1, 1};
    View<T> vv = want_v ? v.view<T>() : View<T>{nullptr, 0, 0, 1, 1};
    ok = svd_with_vectors<T>(st, a.view<const T>(), uv, s_dev, 1, vv, ratio);
    if (ok && size)
      FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * sizeof(T), s_dev, sizeof(T), sizeof(T), size, cudaMemcpyDefault, st));
    finish_all(st, {&a, &u, &v});
  } else {
    ok = singular_values<T>(st, a.view<const T>(), s_dev, ratio);
    // strided scatter into the caller's vector (host or device)
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * sizeof(T), s_dev, sizeof(T), sizeof(T), size, cudaMemcpyDefault, st));
    finish_all(st, {&a});
  }
  ws_free(s_dev);
  return svd_status(ok);
}

// widening / narrowing copies of the f32 LU (below)
template <class TD, class TS>
__global__ void ffi_cast_kernel(TD* __restrict__ dst, i64 drs, i64 dcs, const TS* __restrict__ src, i64 srs, i64 scs, i64 m,
                                i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < m) dst[i * drs + j * dcs] = (TD)src[i * srs + j * scs];
}
template <class TD, class TS>
void ffi_cast(cudaStream_t st, TD* dst, i64 drs, i64 dcs, const TS* src, i64 srs, i64 scs, i64 m, i64 n) {
  if (m == 0 || n == 0) return;
  for (i64 c0 = 0; c0 < n; c0 += 65535) {
    const i64 nc = std::min<i64>(65535, n - c0);
    ffi_cast_kernel<TD, TS><<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(dst, drs, dcs, src, srs, scs, m, c0);
    note_launch();
  }
  FB_CUDA_CHECK(cudaGetLastError());
}
}  // namespace

// f32 partial-pivoting LU, like the f32 `svd` / `self_adjoint_evd`, computed in f64: the f64 drivers (fused sub-panel kernel,
// TMA-fed GEMM, SM partition) factor the widened matrix. The pivot search sees f64 values, so a pivot can differ from an all-f32
// elimination's where two candidates agree to f32 precision (either choice is a valid partial pivot). The f32 solves run on the
// native f32 triangular solves.
size_t fb::lu_partial_piv_in_place_f32_via_f64(cudaStream_t st, VF A, long long* perm_fwd, long long* perm_bwd) {
  const i64 m = A.nrows, n = A.ncols;
  const i64 ld = std::max<i64>(1, (m + 1) & ~(i64)1);
  double* W = (double*)ws_alloc((size_t)ld * (size_t)std::max<i64>(n, 1) * 8);
  ffi_cast<double, float>(st, W, 1, ld, A.ptr, A.rs, A.cs, m, n);
  const size_t count = lu_partial_piv_in_place_f64(st, VD{W, m, n, 1, ld}, perm_fwd, perm_bwd);
  ffi_cast<float, double>(st, A.ptr, A.rs, A.cs, W, 1, ld, m, n);
  ws_free(W);
  return count;
}

extern "C" {

// ---- the families every kind shares (ffi_entries.cuh); the reconstruct / inverse entries of these kinds are in ffi_types.cu ----
FB_MATMUL_FFI(f64, double, false)
FB_MATMUL_FFI(f32, float, false)
FB_MATMUL_FFI(c64, double, true)
FB_MATMUL_FFI(c32, float, true)
FB_TRSM_FFI(f64, double, false)
FB_TRSM_FFI(f32, float, false)
FB_TRSM_FFI(c64, double, true)
FB_TRSM_FFI(c32, float, true)
FB_LLT_FFI(f64, double, false)
FB_LLT_FFI(f32, float, false)
FB_LLT_FFI(c64, double, true)
FB_LLT_FFI(c32, float, true)
FB_LU_FFI(f64, double, false)
FB_LU_FFI(f32, float, false)
FB_LU_FFI(c64, double, true)
FB_LU_FFI(c32, float, true)
FB_QR_FFI(f64, double, false)
FB_QR_FFI(f32, float, false)
FB_QR_FFI(c64, double, true)
FB_QR_FFI(c32, float, true)

// ---- LDLT (no pivoting), f64: ldlt_f64.cu (the other dtypes, reconstruct and inverse: ffi_types.cu / ldlt_types.cu) ----
FaerV0_24_LdltParams libfaer_v0_23_LdltParams_f64(void) {
  return FaerV0_24_LdltParams{64, 128};  // reference defaults: ldlt/factor.rs:705-714
}
FaerV0_24_Layout libfaer_v0_23_ldlt_factor_in_place_scratch_f64(size_t dim, FaerV0_24_Par par, FaerV0_24_LdltParams params) {
  (void)par; (void)params;
  return FaerV0_24_Layout{dim * sizeof(double), 64};  // temp_mat_scratch::<T>(dim, 1), ldlt/factor.rs:715-724
}
FaerV0_24_LdltStatus libfaer_v0_23_ldlt_factor_in_place_f64(FaerV0_24_MatMut A, FaerV0_24_LdltRegularization regularization,
                                                            FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
                                                            FaerV0_24_LdltParams params) {
  (void)par; (void)mem;
  FB_ENTRY();
  FB_ASSERT(A.nrows == A.ncols, "LDLT needs a square matrix");
  cudaStream_t st = current_stream();
  double delta = 0.0, eps = 0.0;
  if (regularization.dynamic_regularization_delta) read_scalar<double>(regularization.dynamic_regularization_delta, &delta);
  if (regularization.dynamic_regularization_epsilon) read_scalar<double>(regularization.dynamic_regularization_epsilon, &eps);
  // expected signs: i8 slice, null = none (faer-ffi/src/lib.rs:838-848); host slices are mirrored on the device
  const signed char* d_signs = nullptr;
  signed char* signs_mirror = nullptr;
  const FaerV0_24_SliceMut sg = regularization.dynamic_regularization_signs;
  if (sg.ptr != nullptr && A.nrows > 0) {
    FB_ASSERT(sg.len >= A.nrows, "dynamic_regularization_signs is shorter than the matrix dimension");
    if (is_device_pointer(sg.ptr)) {
      d_signs = (const signed char*)sg.ptr;
    } else {
      signs_mirror = (signed char*)ws_alloc(A.nrows);
      FB_CUDA_CHECK(cudaMemcpyAsync(signs_mirror, sg.ptr, A.nrows, cudaMemcpyHostToDevice, st));
      d_signs = signs_mirror;
    }
  }
  StagedMat a = stage<double, false>(A, true, st);
  const LdltResult r = ldlt_in_place_f64(st, a.view<double>(), delta, eps, d_signs,
                                         LltParams{params.recursion_threshold, params.block_size});
  finish_all(st, {&a});
  if (signs_mirror) ws_free(signs_mirror);
  return ldlt_status(r);
}
FaerV0_24_Layout libfaer_v0_23_ldlt_solve_in_place_scratch_f64(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)dim; (void)rhs_ncols; (void)par;
  return FaerV0_24_Layout{0, 1};  // StackReq::EMPTY (ldlt/solve.rs:3-10)
}
void libfaer_v0_23_ldlt_solve_in_place_f64(FaerV0_24_MatRef L, FaerV0_24_VecRef D, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs,
                                           FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)par; (void)mem;
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && D.len == n && rhs.nrows == n, "LDLT solve shape mismatch");
  if (n == 0 || rhs.ncols == 0) return;
  StagedMat l = stage<double, false>(L, st), r = stage<double, false>(rhs, true, st);
  // D: usually the diagonal of the factored matrix (stride = row_stride + col_stride). A host vector is gathered into a
  // compact device copy; a device vector is read in place.
  const double* d_ptr = (const double*)D.ptr;
  i64 d_stride = (i64)D.stride;
  double* d_mirror = nullptr;
  if (!is_device_pointer(D.ptr)) {
    std::vector<double> h(n);
    for (size_t i = 0; i < n; ++i) h[i] = ((const double*)D.ptr)[(ptrdiff_t)i * D.stride];
    d_mirror = (double*)ws_alloc(n * sizeof(double));
    FB_CUDA_CHECK(cudaMemcpyAsync(d_mirror, h.data(), n * sizeof(double), cudaMemcpyHostToDevice, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));  // `h` is pageable and local
    d_ptr = d_mirror;
    d_stride = 1;
  }
  ldlt_solve_in_place_f64(st, l.view<const double>(), d_ptr, d_stride, r.view<double>());
  finish_all(st, {&l, &r});
  if (d_mirror) ws_free(d_mirror);
}

// ---- SVD (svd.cu: values by bisection; svd_vectors.cu: with U / V) ----
#define FB_SVD_FFI(SUF, T)                                                                                             \
  FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_##SUF(void) { return FaerV0_24_BidiagParams{192 * 256}; }          \
  FaerV0_24_SvdParams libfaer_v0_23_SvdParams_##SUF(void) {                                                            \
    /* svd/mod.rs:49-58: recursion_threshold 128, qr_ratio_threshold 11/6 */                                          \
    return FaerV0_24_SvdParams{FaerV0_24_BidiagParams{192 * 256}, FaerV0_24_QrParams{48 * 48, 192 * 256}, 128, 11.0 / 6.0}; \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_svd_scratch_##SUF(size_t nrows, size_t ncols, FaerV0_24_ComputeSvdVectors compute_U,  \
                                                   FaerV0_24_ComputeSvdVectors compute_V, FaerV0_24_Par par,           \
                                                   FaerV0_24_SvdParams params) {                                       \
    (void)compute_U; (void)compute_V; (void)par; (void)params;                                                         \
    /* the GPU path keeps its workspace (a copy of A) in the device pool; reported so that callers size like faer */   \
    return FaerV0_24_Layout{nrows * ncols * sizeof(T), 64};                                                            \
  }                                                                                                                    \
  FaerV0_24_SvdStatus libfaer_v0_23_svd_##SUF(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S, FaerV0_24_MatMut V, \
                                              FaerV0_24_Par par, FaerV0_24_MemAlloc mem, FaerV0_24_SvdParams params) { \
    (void)par; (void)mem;                                                                                              \
    return svd_entry<T>(A, U, S, V, params.qr_ratio_threshold);                                                        \
  }
FB_SVD_FFI(f64, double)
FB_SVD_FFI(f32, float)
#undef FB_SVD_FFI

// ---- self-adjoint EVD (evd.cu: values by bisection; svd_vectors.cu + tridiag_dc.cu: with eigenvectors) ----
#define FB_EVD_FFI(SUF, T)                                                                                             \
  FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_##SUF(void) { return FaerV0_24_TridiagParams{192 * 256}; }       \
  FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_##SUF(void) {                                      \
    return FaerV0_24_SelfAdjointEvdParams{FaerV0_24_TridiagParams{192 * 256}, 128}; /* evd/mod.rs:82-90 */             \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_##SUF(size_t dim, FaerV0_24_ComputeEigenvectors compute_U,   \
                                                                FaerV0_24_Par par, FaerV0_24_SelfAdjointEvdParams params) { \
    (void)compute_U; (void)par; (void)params;                                                                          \
    return FaerV0_24_Layout{dim * dim * sizeof(T), 64}; /* the copy of A (kept in the device pool here) */             \
  }                                                                                                                    \
  FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_##SUF(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S, \
                                                           FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                  \
                                                           FaerV0_24_SelfAdjointEvdParams params) {                    \
    (void)par; (void)mem; (void)params;                                                                                \
    return self_adjoint_evd_entry<T>(A, U, S);                                                                         \
  }
FB_EVD_FFI(f64, double)
FB_EVD_FFI(f32, float)
#undef FB_EVD_FFI

// ---- global par / alloc ----
FaerV0_24_Par libfaer_v0_23_get_global_par(void) {
  FaerV0_24_Par p;
  p.tag = (FaerV0_24_ParTag)g_par_tag.load();
  p.nthreads = g_par_threads.load();
  return p;
}
void libfaer_v0_23_set_global_par(FaerV0_24_Par par) {
  g_par_tag.store((int)par.tag);
  g_par_threads.store(par.nthreads);
}
void* libfaer_v0_23_alloc(size_t size, size_t align) {
  // reference: std::alloc::alloc(Layout::from_size_align(size, align)) (faer-ffi/src/lib.rs:2537-2552)
  if (align < sizeof(void*)) align = sizeof(void*);
  void* p = nullptr;
  if (posix_memalign(&p, align, size ? size : 1) != 0) return nullptr;
  return p;
}
void libfaer_v0_23_dealloc(void* ptr, size_t size, size_t align) {
  (void)size; (void)align;
  free(ptr);
}

// ---- extensions ----
int faer_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return n;
}
void faer_b200_set_stream(void* cuda_stream) { std::lock_guard<std::recursive_mutex> lock(entry_mutex()); set_current_stream((cudaStream_t)cuda_stream); }
unsigned long long faer_b200_launch_count(void) { return g_launch_count; }
void faer_b200_launch_log_begin(signed char* tags, size_t capacity) {
  std::lock_guard<std::recursive_mutex> lock(entry_mutex());
  g_launch_log = tags;
  g_launch_log_cap = capacity;
  g_launch_log_len = 0;
}
size_t faer_b200_launch_log_end(void) {
  std::lock_guard<std::recursive_mutex> lock(entry_mutex());
  g_launch_log = nullptr;
  return g_launch_log_len;
}
void faer_b200_release_workspace(void) { std::lock_guard<std::recursive_mutex> lock(entry_mutex()); ws_release_all(); }
void faer_b200_profile_begin(void) { std::lock_guard<std::recursive_mutex> lock(entry_mutex()); profile_begin(); }
void faer_b200_profile_end(double* flops, double* ms, unsigned long long* count) {
  std::lock_guard<std::recursive_mutex> lock(entry_mutex()); 
  profile_end(flops, ms, count);
}
// ---- multi-GPU extensions (dist.cu) ----
int faer_b200_dist_unique_id(void* out128) { return dist_unique_id(out128); }
int faer_b200_dist_init(int rank, int nranks, const void* id128) {
  std::lock_guard<std::recursive_mutex> lock(entry_mutex()); 
  return dist_init(rank, nranks, id128);
}
void faer_b200_dist_finalize(void) { std::lock_guard<std::recursive_mutex> lock(entry_mutex()); dist_finalize(); }
FaerV0_24_LltStatus faer_b200_dist_llt_factor_in_place_f64(void* A_local, size_t ld, size_t n, size_t nb,
                                                           FaerV0_24_LltRegularization regularization, int lookahead) {
  double delta = 0.0, eps = 0.0;
  if (regularization.dynamic_regularization_delta) read_scalar<double>(regularization.dynamic_regularization_delta, &delta);
  if (regularization.dynamic_regularization_epsilon) read_scalar<double>(regularization.dynamic_regularization_epsilon, &eps);
  FB_ASSERT(n == 0 || is_device_pointer(A_local), "distributed entry points take device-resident local matrices");
  return llt_status(dist_llt_f64((double*)A_local, (i64)ld, (i64)n, (i64)nb, delta, eps, lookahead));
}

size_t faer_b200_dist_partial_piv_lu_factor_in_place_f64(void* A_local, size_t ld, size_t n, size_t nb, long long* perm_fwd,
                                                         long long* perm_inv, int lookahead) {
  FB_ASSERT(n == 0 || is_device_pointer(A_local), "distributed entry points take device-resident local matrices");
  return dist_lu_f64((double*)A_local, (i64)ld, (i64)n, (i64)nb, perm_fwd, perm_inv, lookahead);
}

long long faer_b200_dist_qr_factor_in_place_f64(void* A_local, size_t ld, size_t nrows, size_t ncols, size_t block_size, void* Q_coeff,
                                                int flags) {
  FB_ASSERT(ncols == 0 || (is_device_pointer(A_local) && is_device_pointer(Q_coeff)), "distributed entry points take device-resident matrices");
  return dist_qr_f64((double*)A_local, (i64)ld, (i64)nrows, (i64)ncols, (i64)block_size, (double*)Q_coeff, flags);
}
long long faer_b200_dist_qr_factor_in_place_f32(void* A_local, size_t ld, size_t nrows, size_t ncols, size_t block_size, void* Q_coeff,
                                                int flags) {
  FB_ASSERT(ncols == 0 || (is_device_pointer(A_local) && is_device_pointer(Q_coeff)), "distributed entry points take device-resident matrices");
  return dist_qr_f32((float*)A_local, (i64)ld, (i64)nrows, (i64)ncols, (i64)block_size, (float*)Q_coeff, flags);
}


void faer_b200_spicy_matmul_f64(FaerV0_24_MatMut C, FaerV0_24_Block C_block, const unsigned long long* row_idx, size_t nrow_idx,
                                const unsigned long long* col_idx, size_t ncol_idx, FaerV0_24_Accum accum, FaerV0_24_MatRef A,
                                FaerV0_24_MatRef B, const double* D, const FaerV0_24_Scalar* alpha) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(A.ncols == B.nrows, "spicy_matmul shape mismatch");
  FB_ASSERT(!row_idx || nrow_idx == A.nrows, "spicy_matmul: one row index per row of A");
  FB_ASSERT(!col_idx || ncol_idx == B.ncols, "spicy_matmul: one column index per column of B");
  if (row_idx && !is_device_pointer(row_idx))
    for (size_t i = 0; i < nrow_idx; ++i) FB_ASSERT(row_idx[i] < C.nrows, "spicy_matmul: row index out of range");
  if (col_idx && !is_device_pointer(col_idx))
    for (size_t j = 0; j < ncol_idx; ++j) FB_ASSERT(col_idx[j] < C.ncols, "spicy_matmul: column index out of range");
  double a;
  read_scalar<double>(alpha, &a);
  // scattered destinations keep the untouched entries: always stage the old contents
  StagedMat c = stage<double, false>(C, true, st), lhs = stage<double, false>(A, st), rhs = stage<double, false>(B, st);
  // indices and diagonal: device copies of host arrays
  auto to_dev = [&](const void* p, size_t bytes) -> void* {
    if (!p || bytes == 0) return nullptr;
    if (is_device_pointer(p)) return (void*)p;
    void* d = ws_alloc(bytes);
    FB_CUDA_CHECK(cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, st));
    return d;
  };
  void* dri = to_dev(row_idx, nrow_idx * 8);
  void* dci = to_dev(col_idx, ncol_idx * 8);
  void* dd = to_dev(D, (size_t)A.ncols * 8);
  spicy_matmul_f64(st, c.view<double>(), (int)C_block, (const long long*)dri, (const long long*)dci,
                   accum == FaerV0_24_Accum_Add ? 1 : 0, lhs.view<const double>(), rhs.view<const double>(), (const double*)dd, 1, a);
  finish_all(st, {&c, &lhs, &rhs});
  if (dri && dri != (void*)row_idx) ws_free(dri);
  if (dci && dci != (void*)col_idx) ws_free(dci);
  if (dd && dd != (void*)D) ws_free(dd);
}

// ---- inner seam: the type-erased product call faer makes in three places (private_gemm_x86::gemm at
// faer/src/linalg/matmul/mod.rs:1373-1411, matmul/triangular.rs:641-680, matmul/internal/mod.rs:143-201), same parameter list.
void faer_b200_gemm(int dtype, int itype, int instr_set, size_t m, size_t n, size_t k, void* dst, ptrdiff_t dst_rs, ptrdiff_t dst_cs,
                    const void* row_idx, const void* col_idx, int dst_kind, int accum, const void* lhs, ptrdiff_t lhs_rs,
                    ptrdiff_t lhs_cs, bool conj_lhs, const void* diag, ptrdiff_t diag_stride, const void* rhs, ptrdiff_t rhs_rs,
                    ptrdiff_t rhs_cs, bool conj_rhs, const void* alpha, size_t n_threads) {
  (void)instr_set; (void)n_threads;
  FB_ASSERT(dtype >= 0 && dtype <= 3, "faer_b200_gemm: dtype must be FaerB200_GemmDType_{F32,F64,C32,C64}");
  FB_ASSERT(dst_kind >= 0 && dst_kind <= 2, "faer_b200_gemm: dst_kind must be FaerB200_GemmDstKind_{Lower,Upper,Full}");
  const FaerV0_24_Accum acc = accum ? FaerV0_24_Accum_Add : FaerV0_24_Accum_Replace;
  const int block = dst_kind == FaerB200_GemmDstKind_Full ? (int)FaerV0_24_Block_Rectangular
                                                          : dst_kind == FaerB200_GemmDstKind_Lower ? (int)FaerV0_24_Block_TriangularLower
                                                                                                   : (int)FaerV0_24_Block_TriangularUpper;
  if (block != (int)FaerV0_24_Block_Rectangular) FB_ASSERT(m == n, "faer_b200_gemm: a triangular destination is square");
  const bool plain = !row_idx && !col_idx && !diag;
  FaerV0_24_MatRef A{lhs, m, k, lhs_rs, lhs_cs}, B{rhs, k, n, rhs_rs, rhs_cs};
  if (plain && dtype != FaerB200_GemmDType_F64) {
    FaerV0_24_MatMut C{dst, m, n, dst_rs, dst_cs};
    const FaerV0_24_Scalar* a = (const FaerV0_24_Scalar*)alpha;
    if (dtype == FaerB200_GemmDType_F32) matmul_entry<float, false>(C, block, acc, A, 0, B, 0, a);
    else if (dtype == FaerB200_GemmDType_C64) matmul_entry<double, true>(C, block, acc, A, 0, B, 0, a, conj_lhs, conj_rhs);
    else matmul_entry<float, true>(C, block, acc, A, 0, B, 0, a, conj_lhs, conj_rhs);
    return;
  }
  FB_ASSERT(dtype == FaerB200_GemmDType_F64, "faer_b200_gemm: scatter indices / diagonal scaling are built for f64 only");
  FB_ENTRY();
  cudaStream_t st = current_stream();
  // index arrays as 64-bit device arrays; the destination's extent is what the indices reach
  auto host_idx = [&](const void* p, size_t cnt) {
    std::vector<unsigned long long> v(cnt);
    if (!p) return v;
    const size_t w = itype == FaerB200_GemmIType_U32 ? 4 : 8;
    std::vector<unsigned char> raw(cnt * w);
    if (is_device_pointer(p)) FB_CUDA_CHECK(cudaMemcpy(raw.data(), p, raw.size(), cudaMemcpyDeviceToHost));
    else memcpy(raw.data(), p, raw.size());
    for (size_t i = 0; i < cnt; ++i) v[i] = w == 4 ? (unsigned long long)((const uint32_t*)raw.data())[i] : ((const uint64_t*)raw.data())[i];
    return v;
  };
  const std::vector<unsigned long long> ri = host_idx(row_idx, m), ci = host_idx(col_idx, n);
  size_t c_rows = m, c_cols = n;
  if (row_idx) { c_rows = 0; for (auto x : ri) c_rows = std::max<size_t>(c_rows, (size_t)x + 1); }
  if (col_idx) { c_cols = 0; for (auto x : ci) c_cols = std::max<size_t>(c_cols, (size_t)x + 1); }
  auto to_dev = [&](const void* p, size_t bytes) -> void* {
    if (bytes == 0) return nullptr;
    void* d = ws_alloc(bytes);
    FB_CUDA_CHECK(cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, st));
    return d;
  };
  void* dri = row_idx ? to_dev(ri.data(), m * 8) : nullptr;
  void* dci = col_idx ? to_dev(ci.data(), n * 8) : nullptr;
  // diagonal: device pointers are used in place (with their stride), host ones are gathered into a compact device copy
  const double* dd = (const double*)diag;
  void* dd_own = nullptr;
  i64 dstride = (i64)diag_stride;
  std::vector<double> hd;
  if (diag && !is_device_pointer(diag)) {
    hd.resize(k);
    for (size_t q = 0; q < k; ++q) hd[q] = ((const double*)diag)[(ptrdiff_t)q * diag_stride];
    dd_own = to_dev(hd.data(), k * 8);
    dd = (const double*)dd_own;
    dstride = 1;
  }
  double a;
  read_scalar<double>(alpha, &a);
  FaerV0_24_MatMut C{dst, c_rows, c_cols, dst_rs, dst_cs};
  const bool keep_old = accum != 0 || row_idx || col_idx || block != (int)FaerV0_24_Block_Rectangular;
  StagedMat c = stage<double, false>(C, keep_old, st), l = stage<double, false>(A, st), r = stage<double, false>(B, st);
  if (m > 0 && n > 0)
    spicy_matmul_f64(st, c.view<double>(), block, (const long long*)dri, (const long long*)dci, accum ? 1 : 0,
                     l.view<const double>(), r.view<const double>(), dd, dstride, a);
  finish_all(st, {&c, &l, &r});  // synchronises the stream: the host vectors above may go
  if (dri) ws_free(dri);
  if (dci) ws_free(dci);
  if (dd_own) ws_free(dd_own);
}

int faer_b200_set_option(const char* name, long long value) { return set_option_by_name(name, value) ? 0 : -1; }
long long faer_b200_get_option(const char* name) { return get_option_by_name(name); }

const char* faer_b200_version(void) { return "faer_b200 0.1 (faer-ffi v0_23 ABI subset, sm_90a)"; }

}  // extern "C"
