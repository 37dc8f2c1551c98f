// extern "C" boundary: the symbols declared in include/faer_b200.h (second translation unit: ffi_types.cu, the entry points whose
// drivers are the flat-map files; helpers shared by both: ffi_common.cuh).
// Each entry point mirrors the faer-ffi function of the same name (faer-ffi/src/lib.rs, cited per function in the
// header): same argument order and meaning, by-value PODs, synchronous on return, abort() on precondition
// violations. Host buffers are staged; device buffers are used in place.
#include "../../include/faer_b200.h"
#include "ffi_common.cuh"
#include "gemm_f32.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

#include <atomic>
#include <cstring>
#include <memory>
#include <vector>

using namespace fb;

namespace {

std::atomic<int> g_par_tag{FaerV0_24_ParTag_Rayon};
std::atomic<size_t> g_par_threads{0};

inline size_t scalar_elem_f64() { return sizeof(double); }

struct Mat {
  StagedMat s;
  Mat(FaerV0_24_MatRef m, cudaStream_t st)
      : s(m.ptr, (i64)m.nrows, (i64)m.ncols, (i64)m.row_stride, (i64)m.col_stride, sizeof(double), true, false, st) {}
  Mat(FaerV0_24_MatMut m, bool copy_in, cudaStream_t st)
      : s(m.ptr, (i64)m.nrows, (i64)m.ncols, (i64)m.row_stride, (i64)m.col_stride, sizeof(double), copy_in, true, st) {}
};

template <class S>
void solve_tri(FaerV0_24_MatRef T, FaerV0_24_MatMut rhs, bool lower, bool unit) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(T.nrows == T.ncols && rhs.nrows == T.ncols, "triangular solve shape mismatch");
  StagedMat t(T.ptr, (i64)T.nrows, (i64)T.ncols, (i64)T.row_stride, (i64)T.col_stride, sizeof(S), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, sizeof(S), true, true, st);
  if (lower) solve_lower(st, t.view<const S>(), unit, r.view<S>());  // tensor_ops.cuh: f64 / f32 spellings of trsm.cu
  else solve_upper(st, t.view<const S>(), unit, r.view<S>());
  finish_all(st, {&t, &r});
}

// ---- Householder QR (no pivoting) + block-Householder sequence application, f64 and f32 ----
template <class T>
FaerV0_24_QrStatus qr_entry(FaerV0_24_MatMut A, FaerV0_24_MatMut Q) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols;
  FB_ASSERT(Q.nrows > 0 && Q.ncols == size, "Q_coeff must be block_size x min(nrows, ncols)");
  StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, sizeof(T), true, true, st);
  StagedMat q(Q.ptr, (i64)Q.nrows, (i64)Q.ncols, (i64)Q.row_stride, (i64)Q.col_stride, sizeof(T), true, true, st);
  // the reference leaves the strict lower part of each T block untouched and zero-fills nothing for full rank
  const i64 rank = qr_in_place<T>(st, a.view<T>(), q.view<T>());
  finish_all(st, {&a, &q});
  FaerV0_24_QrStatus out;
  memset(&out, 0, sizeof(out));
  if (rank < 0) {
    out.tag = FaerV0_24_QrStatus_Unknown;
  } else {
    out.tag = FaerV0_24_QrStatus_Ok;
    out.ok.rank = (size_t)rank;
  }
  return out;
}
template <class T>
void householder_seq_entry(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_MatMut rhs, bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat b(basis.ptr, (i64)basis.nrows, (i64)basis.ncols, (i64)basis.row_stride, (i64)basis.col_stride, sizeof(T), true, false, st);
  StagedMat f(factor.ptr, (i64)factor.nrows, (i64)factor.ncols, (i64)factor.row_stride, (i64)factor.col_stride, sizeof(T), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, sizeof(T), true, true, st);
  if (transpose) apply_block_householder_sequence_transpose_on_the_left<T>(st, b.view<const T>(), f.view<const T>(), r.view<T>());
  else apply_block_householder_sequence_on_the_left<T>(st, b.view<const T>(), f.view<const T>(), r.view<T>());
  finish_all(st, {&b, &f, &r});
}
// ---- solves on the QR factors (qr/no_pivoting/solve.rs; SURVEY.md §8f rank 1) ----
// mode 0: solve_lstsq_in_place_with_conj (solve.rs:38-76): rhs <- Q^H rhs, then R[..size, ..] x = rhs[..size, ..]
// mode 1: solve_in_place_with_conj (solve.rs:96-119): the same on a square factorization
// mode 2: solve_transpose_in_place_with_conj (solve.rs:140-176): rhs <- R^-T rhs (lower solve on the transposed view),
//         then rhs <- conj(Q) rhs. Real scalar types only: the conj arguments are no-ops.
template <class T>
void qr_solve_entry(FaerV0_24_MatRef Qb, FaerV0_24_MatRef Qc, FaerV0_24_MatRef R, FaerV0_24_MatMut rhs, int mode) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t m = Qb.nrows, n = Qb.ncols, size = m < n ? m : n;
  FB_ASSERT(Qc.nrows > 0 && rhs.nrows == m && m >= n && Qc.ncols == size && R.nrows >= size && R.ncols == n,
            "QR solve shape mismatch");
  if (mode != 0) FB_ASSERT(m == n && R.nrows == n, "QR solve: the factorization must be square");
  if (size == 0 || rhs.ncols == 0) return;
  StagedMat b(Qb.ptr, (i64)m, (i64)n, (i64)Qb.row_stride, (i64)Qb.col_stride, sizeof(T), true, false, st);
  StagedMat f(Qc.ptr, (i64)Qc.nrows, (i64)Qc.ncols, (i64)Qc.row_stride, (i64)Qc.col_stride, sizeof(T), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, sizeof(T), true, true, st);
  // callers normally pass the packed QR matrix for both Q_basis and R (solve.rs:232-246): stage it once
  const bool alias = R.ptr == Qb.ptr && R.row_stride == Qb.row_stride && R.col_stride == Qb.col_stride;
  std::unique_ptr<StagedMat> rr;
  if (!alias)
    rr.reset(new StagedMat(R.ptr, (i64)size, (i64)n, (i64)R.row_stride, (i64)R.col_stride, sizeof(T), true, false, st));
  View<const T> Rv = (alias ? b.view<const T>() : rr->view<const T>()).sub(0, 0, (i64)size, (i64)n);
  View<T> x = r.view<T>();
  if (mode == 2) {
    solve_lower(st, Rv.t(), false, x);
    apply_block_householder_sequence_on_the_left<T>(st, b.view<const T>(), f.view<const T>(), x);
  } else {
    apply_block_householder_sequence_transpose_on_the_left<T>(st, b.view<const T>(), f.view<const T>(), x);
    solve_upper(st, Rv, false, x.sub(0, 0, (i64)size, x.ncols));
  }
  finish_all(st, {&b, &f, &r});
  if (rr) rr->finish();
}
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
  FaerV0_24_EvdStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_EvdStatus_Ok;
  if (n == 0) return out;
  StagedMat a(A.ptr, (i64)n, (i64)n, (i64)A.row_stride, (i64)A.col_stride, sizeof(T), true, false, st);
  T* s_dev = (T*)ws_alloc(n * sizeof(T));
  bool ok;
  if (want_u) {
    StagedMat u(U.ptr, (i64)n, (i64)n, (i64)U.row_stride, (i64)U.col_stride, sizeof(T), false, true, st);
    ok = self_adjoint_evd_with_vectors<T>(st, a.view<const T>(), u.view<T>(), s_dev, 1);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * sizeof(T), s_dev, sizeof(T), sizeof(T), n, cudaMemcpyDefault, st));
    finish_all(st, {&a, &u});
  } else {
    ok = self_adjoint_eigenvalues<T>(st, a.view<const T>(), s_dev);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * sizeof(T), s_dev, sizeof(T), sizeof(T), n, cudaMemcpyDefault, st));
    finish_all(st, {&a});
  }
  ws_free(s_dev);
  if (!ok) out.tag = FaerV0_24_EvdStatus_NoConvergence;
  return out;
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
  FaerV0_24_SvdStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_SvdStatus_Ok;
  const double ratio = qr_ratio_threshold > 0.0 ? qr_ratio_threshold : 11.0 / 6.0;
  if (size == 0 && !want_u && !want_v) return out;
  StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, sizeof(T), true, false, st);
  T* s_dev = (T*)ws_alloc((size + 1) * sizeof(T));
  bool ok;
  if (want_u || want_v) {
    StagedMat u(U.ptr, (i64)U.nrows, (i64)U.ncols, (i64)U.row_stride, (i64)U.col_stride, sizeof(T), false, true, st);
    StagedMat v(V.ptr, (i64)V.nrows, (i64)V.ncols, (i64)V.row_stride, (i64)V.col_stride, sizeof(T), false, true, st);
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
  if (!ok) out.tag = FaerV0_24_SvdStatus_NoConvergence;
  return out;
}
}  // namespace

// widening / narrowing copies and the f32 row gather of the f32 LU entry points (below)
namespace {
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
__global__ void ffi_gather_rows_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, i64 rs, i64 cs, i64 nrows,
                                           const long long* __restrict__ perm) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 c = blockIdx.y;
  if (i < nrows) dst[c * nrows + i] = src[perm[i] * rs + c * cs];
}
}  // namespace



// ---- complex (c64 / c32) triangular solves, LLT and partial-pivoting LU: cplx.cu, templated over the real type R; the device
// views are in complex-unit strides on an R* base, as the complex GEMMs take them ----
inline void cplx_solve_lower(cudaStream_t st, View<const double> t, bool unit, bool conj, View<double> r) { solve_lower_triangular_in_place_c64(st, t, unit, conj, r); }
inline void cplx_solve_lower(cudaStream_t st, View<const float> t, bool unit, bool conj, View<float> r) { solve_lower_triangular_in_place_c32(st, t, unit, conj, r); }
inline void cplx_solve_upper(cudaStream_t st, View<const double> t, bool unit, bool conj, View<double> r) { solve_upper_triangular_in_place_c64(st, t, unit, conj, r); }
inline void cplx_solve_upper(cudaStream_t st, View<const float> t, bool unit, bool conj, View<float> r) { solve_upper_triangular_in_place_c32(st, t, unit, conj, r); }
inline LltResult cplx_llt(cudaStream_t st, View<double> a, double delta, double eps) { return llt_cholesky_in_place_c64(st, a, delta, eps); }
inline LltResult cplx_llt(cudaStream_t st, View<float> a, float delta, float eps) { return llt_cholesky_in_place_c32(st, a, delta, eps); }
inline void cplx_llt_solve(cudaStream_t st, View<const double> l, bool conj, View<double> r) { llt_solve_in_place_c64(st, l, conj, r); }
inline void cplx_llt_solve(cudaStream_t st, View<const float> l, bool conj, View<float> r) { llt_solve_in_place_c32(st, l, conj, r); }
inline size_t cplx_lu(cudaStream_t st, View<double> a, long long* pf, long long* pb) { return lu_partial_piv_in_place_c64(st, a, pf, pb); }
inline size_t cplx_lu(cudaStream_t st, View<float> a, long long* pf, long long* pb) { return lu_partial_piv_in_place_c32(st, a, pf, pb); }
inline void cplx_lu_solve(cudaStream_t st, View<const double> l, View<const double> u, bool conj, const long long* p, View<double> r) { lu_solve_in_place_c64(st, l, u, conj, p, r); }
inline void cplx_lu_solve(cudaStream_t st, View<const float> l, View<const float> u, bool conj, const long long* p, View<float> r) { lu_solve_in_place_c32(st, l, u, conj, p, r); }
inline void cplx_lu_solve_t(cudaStream_t st, View<const double> l, View<const double> u, bool conj, const long long* p, View<double> r) { lu_solve_transpose_in_place_c64(st, l, u, conj, p, r); }
inline void cplx_lu_solve_t(cudaStream_t st, View<const float> l, View<const float> u, bool conj, const long long* p, View<float> r) { lu_solve_transpose_in_place_c32(st, l, u, conj, p, r); }

template <class R>
void solve_tri_cplx(FaerV0_24_MatRef T, FaerV0_24_Conj conj, FaerV0_24_MatMut rhs, bool lower, bool unit) {
  FB_ENTRY();
  FB_ASSERT(T.nrows == T.ncols && rhs.nrows == T.nrows, "triangular solve shape mismatch");
  cudaStream_t st = current_stream();
  StagedMat t(T.ptr, (i64)T.nrows, (i64)T.ncols, (i64)T.row_stride, (i64)T.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, 2 * sizeof(R), true, true, st);
  if (lower) cplx_solve_lower(st, t.view<const R>(), unit, conj == FaerV0_24_Conj_Yes, r.view<R>());
  else cplx_solve_upper(st, t.view<const R>(), unit, conj == FaerV0_24_Conj_Yes, r.view<R>());
  finish_all(st, {&t, &r});
}
template <class R>
FaerV0_24_LltStatus llt_factor_cplx(FaerV0_24_MatMut A, FaerV0_24_LltRegularization regularization) {
  FB_ENTRY();
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  cudaStream_t st = current_stream();
  R delta = 0, eps = 0;  // the regularisation parameters are T::Real
  if (regularization.dynamic_regularization_delta) delta = read_real(regularization.dynamic_regularization_delta, R());
  if (regularization.dynamic_regularization_epsilon) eps = read_real(regularization.dynamic_regularization_epsilon, R());
  StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, 2 * sizeof(R), true, true, st);
  const LltResult r = cplx_llt(st, a.view<R>(), delta, eps);
  finish_all(st, {&a});
  FaerV0_24_LltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LltStatus_NonPositivePivot;
    out.non_positive_pivot.index = r.non_positive_pivot_index;
  }
  return out;
}
template <class R>
void llt_solve_cplx(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs) {
  FB_ENTRY();
  FB_ASSERT(L.nrows == L.ncols && rhs.nrows == L.nrows, "LLT solve shape mismatch");
  cudaStream_t st = current_stream();
  StagedMat l(L.ptr, (i64)L.nrows, (i64)L.ncols, (i64)L.row_stride, (i64)L.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, 2 * sizeof(R), true, true, st);
  cplx_llt_solve(st, l.view<const R>(), A_conj == FaerV0_24_Conj_Yes, r.view<R>());
  finish_all(st, {&l, &r});
}
template <class R>
FaerV0_24_PartialPivLuStatus lu_entry_cplx(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, int idx_bytes) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(A.nrows == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, 2 * sizeof(R), true, true, st);
  std::vector<long long> pf(A.nrows), pb(A.nrows);
  const size_t cnt = cplx_lu(st, a.view<R>(), pf.data(), pb.data());
  finish_all(st, {&a});
  write_perm(perm_fwd.ptr, pf, idx_bytes);
  write_perm(perm_bwd.ptr, pb, idx_bytes);
  FaerV0_24_PartialPivLuStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_PartialPivLuStatus_Ok;
  out.ok.transposition_count = cnt;
  return out;
}
template <class R>
void lu_solve_entry_cplx(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj conj, FaerV0_24_SliceRef perm_slice, FaerV0_24_MatMut rhs,
                         int idx_bytes, bool transpose = false) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "LU solve shape mismatch");
  std::vector<long long> perm = read_perm(perm_slice.ptr, n, idx_bytes);
  for (size_t i = 0; i < n; ++i) FB_ASSERT(perm[i] >= 0 && (size_t)perm[i] < n, "invalid permutation entry");
  StagedMat l(L.ptr, (i64)L.nrows, (i64)L.ncols, (i64)L.row_stride, (i64)L.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat u(U.ptr, (i64)U.nrows, (i64)U.ncols, (i64)U.row_stride, (i64)U.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, 2 * sizeof(R), true, true, st);
  // transpose = false: perm is perm_fwd (solve.rs:21-54); transpose = true: perm is perm_bwd (solve.rs:55-86)
  if (transpose) cplx_lu_solve_t(st, l.view<const R>(), u.view<const R>(), conj == FaerV0_24_Conj_Yes, perm.data(), r.view<R>());
  else cplx_lu_solve(st, l.view<const R>(), u.view<const R>(), conj == FaerV0_24_Conj_Yes, perm.data(), r.view<R>());
  finish_all(st, {&l, &u, &r});
}


// complex Householder QR / block-Householder sequences / QR solves (cplx.cu)
inline i64 cplx_qr(cudaStream_t st, View<double> a, View<double> q, i64 thr) { return qr_in_place_c64(st, a, q, thr); }
inline i64 cplx_qr(cudaStream_t st, View<float> a, View<float> q, i64 thr) { return qr_in_place_c32(st, a, q, thr); }
inline void cplx_hh_seq(cudaStream_t st, View<const double> b, View<const double> f, bool conj, View<double> r, bool tr) { apply_householder_sequence_left_c64(st, b, f, conj, r, tr); }
inline void cplx_hh_seq(cudaStream_t st, View<const float> b, View<const float> f, bool conj, View<float> r, bool tr) { apply_householder_sequence_left_c32(st, b, f, conj, r, tr); }
template <class V>
inline V cplx_sub(V v, i64 i, i64 j, i64 m, i64 n) { return V{v.ptr + 2 * (i * v.rs + j * v.cs), m, n, v.rs, v.cs}; }

template <class R>
FaerV0_24_QrStatus qr_entry_cplx(FaerV0_24_MatMut A, FaerV0_24_MatMut Q, FaerV0_24_QrParams params) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols;
  FB_ASSERT(Q.nrows > 0 && Q.ncols == size, "Q_coeff must be block_size x min(nrows, ncols)");
  StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, 2 * sizeof(R), true, true, st);
  StagedMat q(Q.ptr, (i64)Q.nrows, (i64)Q.ncols, (i64)Q.row_stride, (i64)Q.col_stride, 2 * sizeof(R), true, true, st);
  const i64 rank = cplx_qr(st, a.view<R>(), q.view<R>(), (i64)params.blocking_threshold);
  finish_all(st, {&a, &q});
  FaerV0_24_QrStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_QrStatus_Ok;
  out.ok.rank = (size_t)rank;
  return out;
}
template <class R>
void householder_seq_entry_cplx(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, FaerV0_24_MatMut rhs, bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat b(basis.ptr, (i64)basis.nrows, (i64)basis.ncols, (i64)basis.row_stride, (i64)basis.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat f(factor.ptr, (i64)factor.nrows, (i64)factor.ncols, (i64)factor.row_stride, (i64)factor.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, 2 * sizeof(R), true, true, st);
  cplx_hh_seq(st, b.view<const R>(), f.view<const R>(), conj == FaerV0_24_Conj_Yes, r.view<R>(), transpose);
  finish_all(st, {&b, &f, &r});
}
// qr/no_pivoting/solve.rs:38-176 for complex T. mode 0: least squares (m >= n), 1: square solve, 2: transpose solve
template <class R>
void qr_solve_entry_cplx(FaerV0_24_MatRef Qb, FaerV0_24_MatRef Qc, FaerV0_24_MatRef Rm, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, int mode) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t m = Qb.nrows, n = Qb.ncols, size = m < n ? m : n;
  FB_ASSERT(Qc.nrows > 0 && rhs.nrows == m && m >= n && Qc.ncols == size && Rm.nrows >= size && Rm.ncols == n, "QR solve shape mismatch");
  if (mode != 0) FB_ASSERT(m == n && Rm.nrows == n, "QR solve: the factorization must be square");
  if (size == 0 || rhs.ncols == 0) return;
  const bool conj = A_conj == FaerV0_24_Conj_Yes;
  StagedMat b(Qb.ptr, (i64)m, (i64)n, (i64)Qb.row_stride, (i64)Qb.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat f(Qc.ptr, (i64)Qc.nrows, (i64)Qc.ncols, (i64)Qc.row_stride, (i64)Qc.col_stride, 2 * sizeof(R), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, 2 * sizeof(R), true, true, st);
  const bool alias = Rm.ptr == Qb.ptr && Rm.row_stride == Qb.row_stride && Rm.col_stride == Qb.col_stride;
  std::unique_ptr<StagedMat> rr;
  if (!alias) rr.reset(new StagedMat(Rm.ptr, (i64)size, (i64)n, (i64)Rm.row_stride, (i64)Rm.col_stride, 2 * sizeof(R), true, false, st));
  View<const R> Rv = cplx_sub(alias ? b.view<const R>() : rr->view<const R>(), 0, 0, (i64)size, (i64)n);
  View<R> x = r.view<R>();
  if (mode == 2) {
    cplx_solve_lower(st, Rv.t(), false, conj, x);               // op(R)^T y = rhs
    cplx_hh_seq(st, b.view<const R>(), f.view<const R>(), !conj, x, false);  // the forward sequence with conj composed with Yes
  } else {
    cplx_hh_seq(st, b.view<const R>(), f.view<const R>(), !conj, x, true);   // op(Q)^H rhs
    cplx_solve_upper(st, Rv, false, conj, cplx_sub(x, 0, 0, (i64)size, x.ncols));
  }
  finish_all(st, {&b, &f, &r});
  if (rr) rr->finish();
}

extern "C" {

void libfaer_v0_23_matmul_f64(FaerV0_24_MatMut C, FaerV0_24_Accum accum, FaerV0_24_MatRef A, FaerV0_24_MatRef B,
                              const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  const double a = read_scalar_f64(alpha);
  Mat c(C, accum == FaerV0_24_Accum_Add, st);
  Mat lhs(A, st), rhs(B, st);
  gemm_f64(st, c.s.view<double>(), RECT, accum == FaerV0_24_Accum_Add ? 1 : 0, lhs.s.view<const double>(), RECT,
           rhs.s.view<const double>(), RECT, a);
  finish_all(st, {&c.s, &lhs.s, &rhs.s});
}

void libfaer_v0_23_matmul_triangular_f64(FaerV0_24_MatMut C, FaerV0_24_Block C_block, FaerV0_24_Accum accum,
                                         FaerV0_24_MatRef A, FaerV0_24_Block A_block, FaerV0_24_MatRef B,
                                         FaerV0_24_Block B_block, const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  const double a = read_scalar_f64(alpha);
  const bool copy_in = accum == FaerV0_24_Accum_Add || C_block != FaerV0_24_Block_Rectangular;
  Mat c(C, copy_in, st);
  Mat lhs(A, st), rhs(B, st);
  gemm_f64(st, c.s.view<double>(), (int)C_block, accum == FaerV0_24_Accum_Add ? 1 : 0, lhs.s.view<const double>(),
           (int)A_block, rhs.s.view<const double>(), (int)B_block, a);
  finish_all(st, {&c.s, &lhs.s, &rhs.s});
}

// ---- f32 matmul (3xTF32 tensor-core kernel) ----
static void matmul_f32_impl(FaerV0_24_MatMut C, int C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, int A_block,
                            FaerV0_24_MatRef B, int B_block, const FaerV0_24_Scalar* alpha) {
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  FB_ASSERT(alpha != nullptr, "null scalar pointer");
  float a;
  if (is_device_pointer(alpha)) FB_CUDA_CHECK(cudaMemcpy(&a, alpha, 4, cudaMemcpyDeviceToHost));
  else memcpy(&a, alpha, 4);
  const bool copy_in = accum == FaerV0_24_Accum_Add || C_block != FaerV0_24_Block_Rectangular;
  StagedMat c(C.ptr, (i64)C.nrows, (i64)C.ncols, (i64)C.row_stride, (i64)C.col_stride, 4, copy_in, true, st);
  StagedMat l(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, 4, true, false, st);
  StagedMat r(B.ptr, (i64)B.nrows, (i64)B.ncols, (i64)B.row_stride, (i64)B.col_stride, 4, true, false, st);
  gemm_f32(st, c.view<float>(), C_block, accum == FaerV0_24_Accum_Add ? 1 : 0, l.view<const float>(), A_block,
           r.view<const float>(), B_block, a);
  finish_all(st, {&c, &l, &r});
}
void libfaer_v0_23_matmul_f32(FaerV0_24_MatMut C, FaerV0_24_Accum accum, FaerV0_24_MatRef A, FaerV0_24_MatRef B,
                              const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  matmul_f32_impl(C, 0, accum, A, 0, B, 0, alpha);
}
void libfaer_v0_23_matmul_triangular_f32(FaerV0_24_MatMut C, FaerV0_24_Block C_block, FaerV0_24_Accum accum,
                                         FaerV0_24_MatRef A, FaerV0_24_Block A_block, FaerV0_24_MatRef B,
                                         FaerV0_24_Block B_block, const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  matmul_f32_impl(C, (int)C_block, accum, A, (int)A_block, B, (int)B_block, alpha);
}

// ---- c64 matmul (interleaved complex<f64>; `alpha` points to a complex scalar) ----
static void matmul_c64_impl(FaerV0_24_MatMut C, int C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, int A_block,
                            FaerV0_24_MatRef B, int B_block, const FaerV0_24_Scalar* alpha, bool conj_a = false,
                            bool conj_b = false) {
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  FB_ASSERT(alpha != nullptr, "null scalar pointer");
  double a[2];
  if (is_device_pointer(alpha)) FB_CUDA_CHECK(cudaMemcpy(a, alpha, 16, cudaMemcpyDeviceToHost));
  else memcpy(a, alpha, 16);
  const bool copy_in = accum == FaerV0_24_Accum_Add || C_block != FaerV0_24_Block_Rectangular;
  StagedMat c(C.ptr, (i64)C.nrows, (i64)C.ncols, (i64)C.row_stride, (i64)C.col_stride, 16, copy_in, true, st);
  StagedMat l(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, 16, true, false, st);
  StagedMat r(B.ptr, (i64)B.nrows, (i64)B.ncols, (i64)B.row_stride, (i64)B.col_stride, 16, true, false, st);
  // StagedMat views are in 16-byte element units; reinterpret the base as double* keeping complex strides
  auto as_c = [](const StagedMat& s) { return s.view<double>(); };
  VD dv = as_c(c);
  VD lv0 = as_c(l), rv0 = as_c(r);
  // view<double>() scaled pointer arithmetic by 8 bytes, but strides are in complex units: rebuild from the raw pointer
  gemm_c64(st, dv, C_block, accum == FaerV0_24_Accum_Add ? 1 : 0, cv(lv0), A_block, conj_a, cv(rv0), B_block, conj_b, a[0],
           a[1]);
  finish_all(st, {&c, &l, &r});
}
void libfaer_v0_23_matmul_c64(FaerV0_24_MatMut C, FaerV0_24_Accum accum, FaerV0_24_MatRef A, FaerV0_24_MatRef B,
                              const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  matmul_c64_impl(C, 0, accum, A, 0, B, 0, alpha);
}
void libfaer_v0_23_matmul_triangular_c64(FaerV0_24_MatMut C, FaerV0_24_Block C_block, FaerV0_24_Accum accum,
                                         FaerV0_24_MatRef A, FaerV0_24_Block A_block, FaerV0_24_MatRef B,
                                         FaerV0_24_Block B_block, const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  matmul_c64_impl(C, (int)C_block, accum, A, (int)A_block, B, (int)B_block, alpha);
}

static void matmul_c32_impl(FaerV0_24_MatMut C, int C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, int A_block,
                            FaerV0_24_MatRef B, int B_block, const FaerV0_24_Scalar* alpha, bool conj_a = false,
                            bool conj_b = false) {
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  FB_ASSERT(alpha != nullptr, "null scalar pointer");
  float a[2];
  if (is_device_pointer(alpha)) FB_CUDA_CHECK(cudaMemcpy(a, alpha, 8, cudaMemcpyDeviceToHost));
  else memcpy(a, alpha, 8);
  const bool copy_in = accum == FaerV0_24_Accum_Add || C_block != FaerV0_24_Block_Rectangular;
  // elements are 8-byte (re, im) pairs; the views keep strides in complex units and a float* base
  StagedMat c(C.ptr, (i64)C.nrows, (i64)C.ncols, (i64)C.row_stride, (i64)C.col_stride, 8, copy_in, true, st);
  StagedMat l(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, 8, true, false, st);
  StagedMat r(B.ptr, (i64)B.nrows, (i64)B.ncols, (i64)B.row_stride, (i64)B.col_stride, 8, true, false, st);
  VF dv = c.view<float>();
  VF lv0 = l.view<float>(), rv0 = r.view<float>();
  gemm_c32(st, dv, C_block, accum == FaerV0_24_Accum_Add ? 1 : 0, cv(lv0), A_block, conj_a, cv(rv0), B_block, conj_b, a[0],
           a[1]);
  finish_all(st, {&c, &l, &r});
}
void libfaer_v0_23_matmul_c32(FaerV0_24_MatMut C, FaerV0_24_Accum accum, FaerV0_24_MatRef A, FaerV0_24_MatRef B,
                              const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  matmul_c32_impl(C, 0, accum, A, 0, B, 0, alpha);
}
void libfaer_v0_23_matmul_triangular_c32(FaerV0_24_MatMut C, FaerV0_24_Block C_block, FaerV0_24_Accum accum,
                                         FaerV0_24_MatRef A, FaerV0_24_Block A_block, FaerV0_24_MatRef B,
                                         FaerV0_24_Block B_block, const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {
  (void)par;
  matmul_c32_impl(C, (int)C_block, accum, A, (int)A_block, B, (int)B_block, alpha);
}

#define FB_TRSM_FFI(SUF, T)                                                                                            \
  void libfaer_v0_23_solve_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs, \
                                                           FaerV0_24_Par par) {                                        \
    (void)L_conj; (void)par;                                                                                           \
    solve_tri<T>(L, rhs, true, false);                                                                                 \
  }                                                                                                                    \
  void libfaer_v0_23_solve_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs, \
                                                           FaerV0_24_Par par) {                                        \
    (void)U_conj; (void)par;                                                                                           \
    solve_tri<T>(U, rhs, false, false);                                                                                \
  }                                                                                                                    \
  void libfaer_v0_23_solve_unit_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj,             \
                                                                FaerV0_24_MatMut rhs, FaerV0_24_Par par) {             \
    (void)L_conj; (void)par;                                                                                           \
    solve_tri<T>(L, rhs, true, true);                                                                                  \
  }                                                                                                                    \
  void libfaer_v0_23_solve_unit_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj,             \
                                                                FaerV0_24_MatMut rhs, FaerV0_24_Par par) {             \
    (void)U_conj; (void)par;                                                                                           \
    solve_tri<T>(U, rhs, false, true);                                                                                 \
  }
FB_TRSM_FFI(f64, double)
FB_TRSM_FFI(f32, float)
#undef FB_TRSM_FFI

// ---- LLT ----
FaerV0_24_LltParams libfaer_v0_23_LltParams_f64(void) {
  // reference defaults: faer/src/linalg/cholesky/ldlt/factor.rs:705-714
  return FaerV0_24_LltParams{64, 128};
}

FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_f64(size_t dim, FaerV0_24_Par par,
                                                               FaerV0_24_LltParams params) {
  (void)par; (void)params;
  // reference: temp_mat_scratch::<T>(dim, 1) (llt/factor.rs:58-66). The GPU path keeps its (tiny) workspace in
  // the internal device pool, but reports the reference's requirement so callers allocate identically.
  return FaerV0_24_Layout{dim * sizeof(double), 64};
}

FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_f64(FaerV0_24_MatMut A, FaerV0_24_LltRegularization regularization,
                                                          FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
                                                          FaerV0_24_LltParams params) {
  (void)par; (void)mem;
  FB_ENTRY();
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  cudaStream_t st = current_stream();
  double delta = 0.0, eps = 0.0;
  if (regularization.dynamic_regularization_delta)
    delta = read_scalar_f64((const FaerV0_24_Scalar*)regularization.dynamic_regularization_delta);
  if (regularization.dynamic_regularization_epsilon)
    eps = read_scalar_f64((const FaerV0_24_Scalar*)regularization.dynamic_regularization_epsilon);
  LltResult r;
  if (A.nrows > 0 && !is_device_pointer(A.ptr) && A.row_stride == 1 && A.col_stride >= (ptrdiff_t)A.nrows &&
      (i64)A.nrows >= lookahead_min_n()) {
    // host matrix: upload / factor / download pipelined block column by block column (dist.cu)
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    const i64 nb = lookahead_block() ? lookahead_block() : 256;
    r = llt_host_pipelined_f64((double*)A.ptr, (i64)A.col_stride, (i64)A.nrows, nb, delta, eps);
  } else {
    Mat a(A, true, st);
    r = llt_cholesky_in_place_f64(st, a.s.view<double>(), delta, eps,
                                  LltParams{params.recursion_threshold, params.block_size});
    finish_all(st, {&a.s});
  }
  FaerV0_24_LltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LltStatus_NonPositivePivot;
    out.non_positive_pivot.index = r.non_positive_pivot_index;
  }
  return out;
}

// ---- f32 LLT (llt.cu: the templated leaf kernel and recursive driver instantiated for float) ----
static float read_real_f32(const void* p) {
  float v;
  if (is_device_pointer(p)) FB_CUDA_CHECK(cudaMemcpy(&v, p, sizeof(float), cudaMemcpyDeviceToHost));
  else memcpy(&v, p, sizeof(float));
  return v;
}
FaerV0_24_LltParams libfaer_v0_23_LltParams_f32(void) { return FaerV0_24_LltParams{64, 128}; }
FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_f32(size_t dim, FaerV0_24_Par par, FaerV0_24_LltParams params) {
  (void)par; (void)params;
  return FaerV0_24_Layout{dim * sizeof(float), 64};  // temp_mat_scratch::<T>(dim, 1), llt/factor.rs:58-66
}
FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_f32(FaerV0_24_MatMut A, FaerV0_24_LltRegularization regularization,
                                                          FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
                                                          FaerV0_24_LltParams params) {
  (void)par; (void)mem;
  FB_ENTRY();
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  cudaStream_t st = current_stream();
  float delta = 0.0f, eps = 0.0f;
  if (regularization.dynamic_regularization_delta) delta = read_real_f32(regularization.dynamic_regularization_delta);
  if (regularization.dynamic_regularization_epsilon) eps = read_real_f32(regularization.dynamic_regularization_epsilon);
  StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, sizeof(float), true, true, st);
  const LltResult r = llt_cholesky_in_place_f32(st, a.view<float>(), delta, eps,
                                                LltParams{params.recursion_threshold, params.block_size});
  finish_all(st, {&a});
  FaerV0_24_LltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LltStatus_NonPositivePivot;
    out.non_positive_pivot.index = r.non_positive_pivot_index;
  }
  return out;
}
FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_f32(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)dim; (void)rhs_ncols; (void)par;
  return FaerV0_24_Layout{0, 1};
}
void libfaer_v0_23_llt_solve_in_place_f32(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,
                                          FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)par; (void)mem;
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(L.nrows == L.ncols && rhs.nrows == L.nrows, "LLT solve shape mismatch");
  StagedMat l(L.ptr, (i64)L.nrows, (i64)L.ncols, (i64)L.row_stride, (i64)L.col_stride, sizeof(float), true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, sizeof(float), true, true, st);
  llt_solve_in_place_f32(st, l.view<const float>(), r.view<float>());
  finish_all(st, {&l, &r});
}

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
  if (regularization.dynamic_regularization_delta)
    delta = read_scalar_f64((const FaerV0_24_Scalar*)regularization.dynamic_regularization_delta);
  if (regularization.dynamic_regularization_epsilon)
    eps = read_scalar_f64((const FaerV0_24_Scalar*)regularization.dynamic_regularization_epsilon);
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
  Mat a(A, true, st);
  const LdltResult r = ldlt_in_place_f64(st, a.s.view<double>(), delta, eps, d_signs,
                                         LltParams{params.recursion_threshold, params.block_size});
  finish_all(st, {&a.s});
  if (signs_mirror) ws_free(signs_mirror);
  FaerV0_24_LdltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LdltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LdltStatus_ZeroPivot;
    out.zero_pivot.index = r.zero_pivot_index;
  }
  return out;
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
  Mat l(L, st);
  Mat r(rhs, true, st);
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
  ldlt_solve_in_place_f64(st, l.s.view<const double>(), d_ptr, d_stride, r.s.view<double>());
  finish_all(st, {&l.s, &r.s});
  if (d_mirror) ws_free(d_mirror);
}

// ---- c64 / c32 triangular solves and LLT (cplx.cu: faer's recursions on the complex GEMMs + scalar complex leaf kernels) ----
#define FB_CPLX_TRSM_LLT(SUF, R)                                                                                                \
  void libfaer_v0_23_solve_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs,     \
                                                           FaerV0_24_Par par) {                                                 \
    (void)par;                                                                                                                  \
    solve_tri_cplx<R>(L, L_conj, rhs, true, false);                                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_solve_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs,     \
                                                           FaerV0_24_Par par) {                                                 \
    (void)par;                                                                                                                  \
    solve_tri_cplx<R>(U, U_conj, rhs, false, false);                                                                            \
  }                                                                                                                             \
  void libfaer_v0_23_solve_unit_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs, \
                                                                FaerV0_24_Par par) {                                            \
    (void)par;                                                                                                                  \
    solve_tri_cplx<R>(L, L_conj, rhs, true, true);                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_solve_unit_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs, \
                                                                FaerV0_24_Par par) {                                            \
    (void)par;                                                                                                                  \
    solve_tri_cplx<R>(U, U_conj, rhs, false, true);                                                                             \
  }                                                                                                                             \
  FaerV0_24_LltParams libfaer_v0_23_LltParams_##SUF(void) { return FaerV0_24_LltParams{64, 128}; }                              \
  FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_##SUF(size_t dim, FaerV0_24_Par par, FaerV0_24_LltParams params) { \
    (void)par; (void)params;                                                                                                    \
    return FaerV0_24_Layout{dim * 2 * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, 1), llt/factor.rs:58-66 */                  \
  }                                                                                                                             \
  FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_LltRegularization regularization,   \
                                                              FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                        \
                                                              FaerV0_24_LltParams params) {                                     \
    (void)par; (void)mem; (void)params;                                                                                         \
    return llt_factor_cplx<R>(A, regularization);                                                                               \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {            \
    (void)dim; (void)rhs_ncols; (void)par;                                                                                      \
    return FaerV0_24_Layout{0, 1};                                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_llt_solve_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs,                  \
                                              FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                      \
    (void)par; (void)mem;                                                                                                       \
    llt_solve_cplx<R>(L, A_conj, rhs);                                                                                          \
  }
FB_CPLX_TRSM_LLT(c64, double)
FB_CPLX_TRSM_LLT(c32, float)
#undef FB_CPLX_TRSM_LLT

// ---- partial-pivoting LU ----
FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_f64(void) {
  // reference defaults: faer/src/linalg/lu/partial_pivoting/factor.rs:212-222
  return FaerV0_24_PartialPivLuParams{16, 64, 128 * 128};
}

FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_f64(size_t nrows, size_t ncols, FaerV0_24_Par par,
                                                                              FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)params;
  return lu_scratch(nrows, ncols, 4);
}
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_f64(size_t nrows, size_t ncols, FaerV0_24_Par par,
                                                                              FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)params;
  return lu_scratch(nrows, ncols, 8);
}

static FaerV0_24_PartialPivLuStatus lu_entry(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd,
                                             FaerV0_24_PartialPivLuParams params, int idx_bytes) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  // NB: faer.hpp fills SliceMut.len with BYTES while the Rust side reads elements (SURVEY.md appendix A), so the
  // permutation length is taken from A.nrows, never from `len`.
  FB_ASSERT(A.nrows == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  Mat a(A, true, st);
  size_t cnt = lu_partial_piv_in_place_f64(st, a.s.view<double>(), perm_fwd.ptr, perm_bwd.ptr, idx_bytes,
                                           PartialPivLuParams{params.recursion_threshold, params.block_size,
                                                              params.par_threshold});
  finish_all(st, {&a.s});
  FaerV0_24_PartialPivLuStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_PartialPivLuStatus_Ok;
  out.ok.transposition_count = cnt;
  return out;
}
FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_f64(
    FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
    FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)mem;
  return lu_entry(A, perm_fwd, perm_bwd, params, 4);
}
FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_f64(
    FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
    FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)mem;
  return lu_entry(A, perm_fwd, perm_bwd, params, 8);
}

// ---- f32 partial-pivoting LU: computed in f64, like the f32 `svd` / `self_adjoint_evd`. The f32 matrix is widened on the
// device, factored by the f64 drivers (fused sub-panel kernel, TMA-fed GEMM, SM partition) and rounded back: the factors carry
// one f32 rounding instead of an f32 elimination's accumulated ones, and the pivot search sees f64 values (so a pivot can
// differ from an all-f32 elimination's where two candidates agree to f32 precision — either choice is a valid partial
// pivot). The solves run on the native f32 triangular solves.
FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_f32(void) { return libfaer_v0_23_PartialPivLuParams_f64(); }
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_f32(size_t nrows, size_t ncols, FaerV0_24_Par par,
                                                                              FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)params;
  return lu_scratch(nrows, ncols, 4);
}
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_f32(size_t nrows, size_t ncols, FaerV0_24_Par par,
                                                                              FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)params;
  return lu_scratch(nrows, ncols, 8);
}
static FaerV0_24_PartialPivLuStatus lu_entry_f32(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd,
                                                 FaerV0_24_PartialPivLuParams params, int idx_bytes) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(A.nrows == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  const i64 m = (i64)A.nrows, n = (i64)A.ncols;
  StagedMat a(A.ptr, m, n, (i64)A.row_stride, (i64)A.col_stride, 4, true, true, st);
  VF av = a.view<float>();
  const i64 ld = std::max<i64>(1, (m + 1) & ~(i64)1);
  double* W = (double*)ws_alloc((size_t)ld * (size_t)std::max<i64>(n, 1) * 8);
  ffi_cast<double, float>(st, W, 1, ld, av.ptr, av.rs, av.cs, m, n);
  const size_t cnt = lu_partial_piv_in_place_f64(st, VD{W, m, n, 1, ld}, perm_fwd.ptr, perm_bwd.ptr, idx_bytes,
                                                 PartialPivLuParams{params.recursion_threshold, params.block_size,
                                                                    params.par_threshold});
  ffi_cast<float, double>(st, av.ptr, av.rs, av.cs, W, 1, ld, m, n);
  finish_all(st, {&a});
  ws_free(W);
  FaerV0_24_PartialPivLuStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_PartialPivLuStatus_Ok;
  out.ok.transposition_count = cnt;
  return out;
}
FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_f32(
    FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
    FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)mem;
  return lu_entry_f32(A, perm_fwd, perm_bwd, params, 4);
}
FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_f32(
    FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,
    FaerV0_24_PartialPivLuParams params) {
  (void)par; (void)mem;
  return lu_entry_f32(A, perm_fwd, perm_bwd, params, 8);
}

// ---- Householder QR (no pivoting) + block-Householder sequence application, f64 and f32 (helpers above) ----
#define FB_QR_FFI(SUF, T)                                                                                              \
  FaerV0_24_QrParams libfaer_v0_23_QrParams_##SUF(void) { return FaerV0_24_QrParams{48 * 48, 192 * 256}; }             \
  size_t libfaer_v0_23_qr_recommended_block_size_##SUF(size_t nrows, size_t ncols) {                                   \
    return (size_t)qr_recommended_block_size((i64)nrows, (i64)ncols);                                                  \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,       \
                                                                  FaerV0_24_Par par, FaerV0_24_QrParams params) {      \
    (void)nrows; (void)par; (void)params;                                                                              \
    return FaerV0_24_Layout{block_size * ncols * sizeof(T), 64}; /* temp_mat_scratch(block_size, ncols) */            \
  }                                                                                                                    \
  FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatMut Q_coeff, FaerV0_24_Par par, \
                                                            FaerV0_24_MemAlloc mem, FaerV0_24_QrParams params) {       \
    (void)par; (void)mem; (void)params;                                                                                \
    return qr_entry<T>(A, Q_coeff);                                                                                    \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols) { \
    (void)dim;                                                                                                         \
    return FaerV0_24_Layout{block_size * rhs_ncols * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_##SUF(size_t dim, size_t block_size,  \
                                                                                        size_t rhs_ncols) {            \
    (void)dim;                                                                                                         \
    return FaerV0_24_Layout{block_size * rhs_ncols * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  void libfaer_v0_23_apply_householder_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, \
                                                         FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)conj; (void)par; (void)mem;                                                                                  \
    householder_seq_entry<T>(basis, factor, rhs, false);                                                               \
  }                                                                                                                    \
  void libfaer_v0_23_apply_householder_transpose_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,    \
                                                                   FaerV0_24_Conj conj, FaerV0_24_MatMut rhs,          \
                                                                   FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {        \
    (void)conj; (void)par; (void)mem;                                                                                  \
    householder_seq_entry<T>(basis, factor, rhs, true);                                                                \
  }                                                                                                                    \
  /* on the right = the transposed sequence on the left of the transposed view, and vice versa (householder.rs:813-854) */ \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_##SUF(size_t dim, size_t block_size, size_t lhs_nrows) { \
    (void)dim;                                                                                                         \
    return FaerV0_24_Layout{block_size * lhs_nrows * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_##SUF(size_t dim, size_t block_size, \
                                                                                         size_t lhs_nrows) {           \
    (void)dim;                                                                                                         \
    return FaerV0_24_Layout{block_size * lhs_nrows * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  void libfaer_v0_23_apply_householder_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, \
                                                          FaerV0_24_MatMut lhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)conj; (void)par; (void)mem;                                                                                  \
    householder_seq_entry<T>(basis, factor, transposed(lhs), true);                                                    \
  }                                                                                                                    \
  void libfaer_v0_23_apply_householder_transpose_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,   \
                                                                    FaerV0_24_Conj conj, FaerV0_24_MatMut lhs,         \
                                                                    FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {       \
    (void)conj; (void)par; (void)mem;                                                                                  \
    householder_seq_entry<T>(basis, factor, transposed(lhs), false);                                                   \
  }                                                                                                                    \
  /* scratch: apply_block_householder_sequence_[transpose_]on_the_left_in_place_scratch (solve.rs:3-37) */           \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,  \
                                                                       size_t rhs_ncols, FaerV0_24_Par par) {          \
    (void)nrows; (void)ncols; (void)par;                                                                               \
    return FaerV0_24_Layout{block_size * rhs_ncols * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols,      \
                                                                 FaerV0_24_Par par) {                                  \
    (void)dim; (void)par;                                                                                              \
    return FaerV0_24_Layout{block_size * rhs_ncols * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_##SUF(size_t dim, size_t block_size,              \
                                                                           size_t rhs_ncols, FaerV0_24_Par par) {      \
    (void)dim; (void)par;                                                                                              \
    return FaerV0_24_Layout{block_size * rhs_ncols * sizeof(T), 64};                                                   \
  }                                                                                                                    \
  void libfaer_v0_23_qr_solve_lstsq_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R, \
                                                   FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,     \
                                                   FaerV0_24_MemAlloc mem) {                                           \
    (void)A_conj; (void)par; (void)mem;                                                                                \
    qr_solve_entry<T>(Q_basis, Q_coeff, R, rhs, 0);                                                                    \
  }                                                                                                                    \
  void libfaer_v0_23_qr_solve_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R,   \
                                             FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,           \
                                             FaerV0_24_MemAlloc mem) {                                                 \
    (void)A_conj; (void)par; (void)mem;                                                                                \
    qr_solve_entry<T>(Q_basis, Q_coeff, R, rhs, 1);                                                                    \
  }                                                                                                                    \
  void libfaer_v0_23_qr_solve_transpose_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,             \
                                                       FaerV0_24_MatRef R, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, \
                                                       FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                    \
    (void)A_conj; (void)par; (void)mem;                                                                                \
    qr_solve_entry<T>(Q_basis, Q_coeff, R, rhs, 2);                                                                    \
  }
FB_QR_FFI(f64, double)
FB_QR_FFI(f32, float)
#undef FB_QR_FFI

// ---- complex Householder QR, block-Householder sequences and the QR solves (cplx.cu) ----
#define FB_QR_CPLX_FFI(SUF, R)                                                                                                  \
  FaerV0_24_QrParams libfaer_v0_23_QrParams_##SUF(void) { return FaerV0_24_QrParams{48 * 48, 192 * 256}; }                      \
  size_t libfaer_v0_23_qr_recommended_block_size_##SUF(size_t nrows, size_t ncols) {                                            \
    return (size_t)qr_recommended_block_size((i64)nrows, (i64)ncols);                                                           \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,                \
                                                                  FaerV0_24_Par par, FaerV0_24_QrParams params) {               \
    (void)nrows; (void)par; (void)params;                                                                                       \
    return FaerV0_24_Layout{block_size * ncols * 2 * sizeof(R), 64};                                                            \
  }                                                                                                                             \
  FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatMut Q_coeff, FaerV0_24_Par par,    \
                                                            FaerV0_24_MemAlloc mem, FaerV0_24_QrParams params) {                \
    (void)par; (void)mem;                                                                                                       \
    return qr_entry_cplx<R>(A, Q_coeff, params);                                                                                \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols) { \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * rhs_ncols * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_##SUF(size_t dim, size_t block_size,           \
                                                                                        size_t rhs_ncols) {                     \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * rhs_ncols * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj,  \
                                                         FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {     \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_entry_cplx<R>(basis, factor, conj, rhs, false);                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_transpose_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,             \
                                                                   FaerV0_24_Conj conj, FaerV0_24_MatMut rhs,                   \
                                                                   FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                 \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_entry_cplx<R>(basis, factor, conj, rhs, true);                                                              \
  }                                                                                                                             \
  /* on the right = the transposed sequence on the left of the transposed view, and vice versa (householder.rs:813-854) */     \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_##SUF(size_t dim, size_t block_size, size_t lhs_nrows) { \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * lhs_nrows * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_##SUF(size_t dim, size_t block_size,          \
                                                                                         size_t lhs_nrows) {                    \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * lhs_nrows * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, \
                                                          FaerV0_24_MatMut lhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {    \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_entry_cplx<R>(basis, factor, conj, transposed(lhs), true);                                                  \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_transpose_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,            \
                                                                    FaerV0_24_Conj conj, FaerV0_24_MatMut lhs,                  \
                                                                    FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_entry_cplx<R>(basis, factor, conj, transposed(lhs), false);                                                 \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,           \
                                                                       size_t rhs_ncols, FaerV0_24_Par par) {                   \
    (void)nrows; (void)ncols; (void)par;                                                                                        \
    return FaerV0_24_Layout{block_size * rhs_ncols * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols,               \
                                                                 FaerV0_24_Par par) {                                           \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{block_size * rhs_ncols * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_##SUF(size_t dim, size_t block_size,                       \
                                                                           size_t rhs_ncols, FaerV0_24_Par par) {               \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{block_size * rhs_ncols * 2 * sizeof(R), 64};                                                        \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_lstsq_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef Rm,     \
                                                   FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,              \
                                                   FaerV0_24_MemAlloc mem) {                                                    \
    (void)par; (void)mem;                                                                                                       \
    qr_solve_entry_cplx<R>(Q_basis, Q_coeff, Rm, A_conj, rhs, 0);                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef Rm,           \
                                             FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,                    \
                                             FaerV0_24_MemAlloc mem) {                                                          \
    (void)par; (void)mem;                                                                                                       \
    qr_solve_entry_cplx<R>(Q_basis, Q_coeff, Rm, A_conj, rhs, 1);                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_transpose_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,                      \
                                                       FaerV0_24_MatRef Rm, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs,        \
                                                       FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                             \
    (void)par; (void)mem;                                                                                                       \
    qr_solve_entry_cplx<R>(Q_basis, Q_coeff, Rm, A_conj, rhs, 2);                                                               \
  }
FB_QR_CPLX_FFI(c64, double)
FB_QR_CPLX_FFI(c32, float)
#undef FB_QR_CPLX_FFI

// ---- solves on top of the factors ----
FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_f64(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)dim; (void)rhs_ncols; (void)par;
  return FaerV0_24_Layout{0, 1};  // reference: StackReq::EMPTY (llt/solve.rs:3-10)
}
void libfaer_v0_23_llt_solve_in_place_f64(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,
                                          FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)par; (void)mem;
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(L.nrows == L.ncols && rhs.nrows == L.nrows, "LLT solve shape mismatch");
  Mat l(L, st);
  Mat r(rhs, true, st);
  llt_solve_in_place_f64(st, l.s.view<const double>(), r.s.view<double>());
  finish_all(st, {&l.s, &r.s});
}

// transpose = false: perm is perm_fwd (solve.rs:21-54); transpose = true: perm is perm_bwd (solve.rs:55-86)
static void lu_solve_entry(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_SliceRef perm_slice, FaerV0_24_MatMut rhs,
                           int idx_bytes, bool transpose = false) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "LU solve shape mismatch");
  std::vector<long long> perm = read_perm(perm_slice.ptr, n, idx_bytes);  // length from L.nrows (see lu_entry note)
  for (size_t i = 0; i < n; ++i) FB_ASSERT(perm[i] >= 0 && (size_t)perm[i] < n, "invalid permutation entry");
  Mat l(L, st), u(U, st);
  Mat r(rhs, true, st);
  if (transpose)
    lu_solve_transpose_in_place_f64(st, l.s.view<const double>(), u.s.view<const double>(), perm.data(), r.s.view<double>());
  else
    lu_solve_in_place_f64(st, l.s.view<const double>(), u.s.view<const double>(), perm.data(), r.s.view<double>());
  finish_all(st, {&l.s, &u.s, &r.s});
}
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)par;
  return FaerV0_24_Layout{dim * rhs_ncols * sizeof(double), 64};  // permute_rows_in_place_scratch (perm/mod.rs)
}
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)par;
  return FaerV0_24_Layout{dim * rhs_ncols * sizeof(double), 64};
}
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_f64(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,
                                                         FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,
                                                         FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)perm_bwd; (void)par; (void)mem;
  lu_solve_entry(L, U, perm_fwd, rhs, 4);
}
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_f64(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,
                                                         FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,
                                                         FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)perm_bwd; (void)par; (void)mem;
  lu_solve_entry(L, U, perm_fwd, rhs, 8);
}
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)par;
  return FaerV0_24_Layout{dim * rhs_ncols * sizeof(double), 64};
}
FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {
  (void)par;
  return FaerV0_24_Layout{dim * rhs_ncols * sizeof(double), 64};
}
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_f64(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,
                                                                   FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,
                                                                   FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)perm_fwd; (void)par; (void)mem;
  lu_solve_entry(L, U, perm_bwd, rhs, 4, true);
}
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_f64(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,
                                                                   FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,
                                                                   FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)A_conj; (void)perm_fwd; (void)par; (void)mem;
  lu_solve_entry(L, U, perm_bwd, rhs, 8, true);
}

// f32 LU solves (lu/partial_pivoting/solve.rs:21-86) on the native f32 triangular solves
static void lu_solve_entry_f32(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_SliceRef perm_slice, FaerV0_24_MatMut rhs,
                               int idx_bytes, bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "LU solve shape mismatch");
  std::vector<long long> perm = read_perm(perm_slice.ptr, n, idx_bytes);
  for (size_t i = 0; i < n; ++i) FB_ASSERT(perm[i] >= 0 && (size_t)perm[i] < n, "invalid permutation entry");
  StagedMat l(L.ptr, (i64)L.nrows, (i64)L.ncols, (i64)L.row_stride, (i64)L.col_stride, 4, true, false, st);
  StagedMat u(U.ptr, (i64)U.nrows, (i64)U.ncols, (i64)U.row_stride, (i64)U.col_stride, 4, true, false, st);
  StagedMat r(rhs.ptr, (i64)rhs.nrows, (i64)rhs.ncols, (i64)rhs.row_stride, (i64)rhs.col_stride, 4, true, true, st);
  VCF lv = l.view<const float>(), uv = u.view<const float>();
  VF rv = r.view<float>();
  const i64 k = rv.ncols;
  auto permute = [&]() {  // rhs[i, :] <- rhs[perm[i], :]
    if (n == 0 || k == 0) return;
    FB_ASSERT(k < 65536, "too many right-hand sides for one permutation launch");
    long long* d_perm = (long long*)ws_alloc(n * 8);
    float* tmp = (float*)ws_alloc(n * (size_t)k * 4);
    FB_CUDA_CHECK(cudaMemcpyAsync(d_perm, perm.data(), n * 8, cudaMemcpyHostToDevice, st));
    ffi_gather_rows_f32_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)k), 256, 0, st>>>(tmp, rv.ptr, rv.rs, rv.cs, (i64)n, d_perm);
    note_launch();
    ffi_cast<float, float>(st, rv.ptr, rv.rs, rv.cs, tmp, 1, (i64)n, (i64)n, k);
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    ws_free(tmp);
    ws_free(d_perm);
  };
  if (!transpose) {
    permute();
    solve_lower_triangular_in_place_f32(st, lv, true, rv);
    solve_upper_triangular_in_place_f32(st, uv, false, rv);
  } else {
    solve_lower_triangular_in_place_f32(st, uv.t(), false, rv);
    solve_upper_triangular_in_place_f32(st, lv.t(), true, rv);
    permute();
  }
  finish_all(st, {&l, &u, &r});
}
#define FB_LU_SOLVE_F32(IT, BYTES)                                                                                              \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_##IT##_f32(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * sizeof(float), 64};                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_in_place_##IT##_f32(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,    \
                                                             FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,          \
                                                             FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)A_conj; (void)perm_bwd; (void)par; (void)mem;                                                                         \
    lu_solve_entry_f32(L, U, perm_fwd, rhs, BYTES, false);                                                                      \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_##IT##_f32(size_t dim, size_t rhs_ncols,       \
                                                                                            FaerV0_24_Par par) {                \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * sizeof(float), 64};                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_##IT##_f32(                                                        \
      FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,   \
      FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                                        \
    (void)A_conj; (void)perm_fwd; (void)par; (void)mem;                                                                         \
    lu_solve_entry_f32(L, U, perm_bwd, rhs, BYTES, true);                                                                       \
  }
FB_LU_SOLVE_F32(u32, 4)
FB_LU_SOLVE_F32(u64, 8)
#undef FB_LU_SOLVE_F32

// ---- c64 / c32 partial-pivoting LU (cplx.cu) ----
FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_c64(void) { return libfaer_v0_23_PartialPivLuParams_f64(); }
FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_c32(void) { return libfaer_v0_23_PartialPivLuParams_f64(); }
#define FB_LU_CPLX(IT, BYTES, SUF, R)                                                                                           \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_##IT##_##SUF(size_t nrows, size_t ncols, FaerV0_24_Par par, \
                                                                                     FaerV0_24_PartialPivLuParams params) {    \
    (void)par; (void)params;                                                                                                    \
    return lu_scratch(nrows, ncols, BYTES);                                                                                     \
  }                                                                                                                             \
  FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_##IT##_##SUF(                                       \
      FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,   \
      FaerV0_24_PartialPivLuParams params) {                                                                                    \
    (void)par; (void)mem; (void)params;                                                                                         \
    return lu_entry_cplx<R>(A, perm_fwd, perm_bwd, BYTES);                                                                      \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * 2 * sizeof(R), 64};                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,  \
                                                               FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,        \
                                                               FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)perm_bwd; (void)par; (void)mem;                                                                                       \
    lu_solve_entry_cplx<R>(L, U, A_conj, perm_fwd, rhs, BYTES);                                                                 \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols,     \
                                                                                              FaerV0_24_Par par) {              \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * 2 * sizeof(R), 64};                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_##IT##_##SUF(                                                      \
      FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,   \
      FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                                        \
    (void)perm_fwd; (void)par; (void)mem;                                                                                       \
    lu_solve_entry_cplx<R>(L, U, A_conj, perm_bwd, rhs, BYTES, true);                                                           \
  }
FB_LU_CPLX(u32, 4, c64, double)
FB_LU_CPLX(u64, 8, c64, double)
FB_LU_CPLX(u32, 4, c32, float)
FB_LU_CPLX(u64, 8, c32, float)
#undef FB_LU_CPLX

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

// ---- reconstruct / inverse on the factors (reconstruct.cu; f64, qr_reconstruct also f32) ----
FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_f64(size_t dim, FaerV0_24_Par par) {
  (void)dim; (void)par;
  return FaerV0_24_Layout{0, 1};  // StackReq::EMPTY (llt/reconstruct.rs:3-6)
}
void libfaer_v0_23_llt_reconstruct_f64(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)par; (void)mem;
  FB_ENTRY();
  cudaStream_t st = current_stream();
  Mat a(A, true, st);  // only the lower triangle is written: the rest of A must survive the round trip
  Mat l(L, st);
  llt_reconstruct_f64(st, a.s.view<double>(), l.s.view<const double>());
  finish_all(st, {&a.s, &l.s});
}
FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_f64(size_t dim, FaerV0_24_Par par) {
  (void)par;
  return FaerV0_24_Layout{dim * dim * sizeof(double), 64};  // temp_mat_scratch(dim, dim) (llt/inverse.rs:3-8)
}
void libfaer_v0_23_llt_inverse_f64(FaerV0_24_MatMut A_inv, FaerV0_24_MatRef L, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)par; (void)mem;
  FB_ENTRY();
  cudaStream_t st = current_stream();
  Mat a(A_inv, true, st);
  Mat l(L, st);
  llt_inverse_f64(st, a.s.view<double>(), l.s.view<const double>());
  finish_all(st, {&a.s, &l.s});
}
static void lu_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_SliceRef perm, int idx_bytes,
                           bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t m = L.nrows;
  std::vector<long long> p = read_perm(perm.ptr, m, idx_bytes);
  for (size_t i = 0; i < m; ++i) FB_ASSERT(p[i] >= 0 && (size_t)p[i] < m, "invalid permutation entry");
  Mat a(A, false, st);
  Mat l(L, st), u(U, st);
  if (inverse) lu_inverse_f64(st, a.s.view<double>(), l.s.view<const double>(), u.s.view<const double>(), p.data());
  else lu_reconstruct_f64(st, a.s.view<double>(), l.s.view<const double>(), u.s.view<const double>(), p.data());
  finish_all(st, {&a.s, &l.s, &u.s});
}
#define FB_LU_RECON_FFI(IT, BYTES)                                                                                     \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_##IT##_f64(size_t nrows, size_t ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                         \
    return FaerV0_24_Layout{nrows * ncols * sizeof(double), 64};                                                       \
  }                                                                                                                    \
  void libfaer_v0_23_partial_piv_lu_reconstruct_##IT##_f64(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U, \
                                                           FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,   \
                                                           FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                \
    (void)perm_fwd; (void)par; (void)mem;                                                                              \
    lu_recon_entry(A, L, U, perm_bwd, BYTES, false);                                                                   \
  }                                                                                                                    \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_##IT##_f64(size_t dim, FaerV0_24_Par par) {            \
    (void)par;                                                                                                         \
    return FaerV0_24_Layout{dim * dim * sizeof(double), 64};                                                           \
  }                                                                                                                    \
  void libfaer_v0_23_partial_piv_lu_inverse_##IT##_f64(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,     \
                                                       FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,       \
                                                       FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                    \
    (void)perm_bwd; (void)par; (void)mem;                                                                              \
    lu_recon_entry(A, L, U, perm_fwd, BYTES, true);                                                                    \
  }
FB_LU_RECON_FFI(u32, 4)
FB_LU_RECON_FFI(u64, 8)
#undef FB_LU_RECON_FFI
#define FB_QR_RECON_FFI(SUF, T)                                                                                        \
  FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size, FaerV0_24_Par par) { \
    (void)nrows; (void)par;                                                                                            \
    return FaerV0_24_Layout{block_size * ncols * sizeof(T), 64};                                                       \
  }                                                                                                                    \
  void libfaer_v0_23_qr_reconstruct_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,      \
                                          FaerV0_24_MatRef R, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {             \
    (void)par; (void)mem;                                                                                              \
    FB_ENTRY();                                                                                                        \
    cudaStream_t st = current_stream();                                                                                \
    StagedMat a(A.ptr, (i64)A.nrows, (i64)A.ncols, (i64)A.row_stride, (i64)A.col_stride, sizeof(T), false, true, st);  \
    StagedMat b(Q_basis.ptr, (i64)Q_basis.nrows, (i64)Q_basis.ncols, (i64)Q_basis.row_stride, (i64)Q_basis.col_stride, sizeof(T), true, false, st); \
    StagedMat f(Q_coeff.ptr, (i64)Q_coeff.nrows, (i64)Q_coeff.ncols, (i64)Q_coeff.row_stride, (i64)Q_coeff.col_stride, sizeof(T), true, false, st); \
    StagedMat r(R.ptr, (i64)R.nrows, (i64)R.ncols, (i64)R.row_stride, (i64)R.col_stride, sizeof(T), true, false, st);  \
    qr_reconstruct<T>(st, a.view<T>(), b.view<const T>(), f.view<const T>(), r.view<const T>());                       \
    finish_all(st, {&a, &b, &f, &r});                                                                                  \
  }
FB_QR_RECON_FFI(f64, double)
FB_QR_RECON_FFI(f32, float)
#undef FB_QR_RECON_FFI
FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_f64(size_t dim, size_t block_size, FaerV0_24_Par par) {
  (void)par;
  return FaerV0_24_Layout{block_size * dim * sizeof(double), 64};
}
void libfaer_v0_23_qr_inverse_f64(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R,
                                  FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {
  (void)par; (void)mem;
  FB_ENTRY();
  cudaStream_t st = current_stream();
  Mat a(A, false, st);
  Mat b(Q_basis, st), f(Q_coeff, st), r(R, st);
  qr_inverse_f64(st, a.s.view<double>(), b.s.view<const double>(), f.s.view<const double>(), r.s.view<const double>());
  finish_all(st, {&a.s, &b.s, &f.s, &r.s});
}

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
  if (regularization.dynamic_regularization_delta)
    delta = read_scalar_f64((const FaerV0_24_Scalar*)regularization.dynamic_regularization_delta);
  if (regularization.dynamic_regularization_epsilon)
    eps = read_scalar_f64((const FaerV0_24_Scalar*)regularization.dynamic_regularization_epsilon);
  FB_ASSERT(n == 0 || is_device_pointer(A_local), "distributed entry points take device-resident local matrices");
  LltResult r = dist_llt_f64((double*)A_local, (i64)ld, (i64)n, (i64)nb, delta, eps, lookahead);
  FaerV0_24_LltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LltStatus_NonPositivePivot;
    out.non_positive_pivot.index = r.non_positive_pivot_index;
  }
  return out;
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
  const double a = read_scalar_f64(alpha);
  Mat c(C, true, st);  // scattered destinations keep the untouched entries: always stage the old contents
  Mat lhs(A, st), rhs(B, st);
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
  spicy_matmul_f64(st, c.s.view<double>(), (int)C_block, (const long long*)dri, (const long long*)dci,
                   accum == FaerV0_24_Accum_Add ? 1 : 0, lhs.s.view<const double>(), rhs.s.view<const double>(), (const double*)dd, 1, a);
  finish_all(st, {&c.s, &lhs.s, &rhs.s});
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
    if (dtype == FaerB200_GemmDType_F32) matmul_f32_impl(C, block, acc, A, 0, B, 0, a);
    else if (dtype == FaerB200_GemmDType_C64) matmul_c64_impl(C, block, acc, A, 0, B, 0, a, conj_lhs, conj_rhs);
    else matmul_c32_impl(C, block, acc, A, 0, B, 0, a, conj_lhs, conj_rhs);
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
  const double a = read_scalar_f64((const FaerV0_24_Scalar*)alpha);
  FaerV0_24_MatMut C{dst, c_rows, c_cols, dst_rs, dst_cs};
  const bool keep_old = accum != 0 || row_idx || col_idx || block != (int)FaerV0_24_Block_Rectangular;
  Mat c(C, keep_old, st);
  Mat l(A, st), r(B, st);
  if (m > 0 && n > 0)
    spicy_matmul_f64(st, c.s.view<double>(), block, (const long long*)dri, (const long long*)dci, accum ? 1 : 0,
                     l.s.view<const double>(), r.s.view<const double>(), dd, dstride, a);
  finish_all(st, {&c.s, &l.s, &r.s});  // synchronises the stream: the host vectors above may go
  if (dri) ws_free(dri);
  if (dci) ws_free(dci);
  if (dd_own) ws_free(dd_own);
}

int faer_b200_set_option(const char* name, long long value) { return set_option_by_name(name, value) ? 0 : -1; }
long long faer_b200_get_option(const char* name) { return get_option_by_name(name); }

const char* faer_b200_version(void) { return "faer_b200 0.1 (faer-ffi v0_23 ABI subset, sm_90a)"; }

}  // extern "C"
