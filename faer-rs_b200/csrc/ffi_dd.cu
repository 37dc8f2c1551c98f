// extern "C" boundary of the double-double kinds (include/faer_b200_fx128.h): fx128 = <dd, false>, cx128 = <dd, true>. Same
// conventions as ffi.cu / ffi_types.cu (by-value PODs, synchronous on return, abort() on precondition violations, host buffers
// staged, device buffers used in place, `Par` ignored). Drivers: gemm_dd.cu, dd_factor.cu and the <dd, CX> instantiations of the
// reconstruct_types.cu compositions, qr_dd.cu for the Householder QR (include/faer_b200_fx128_qr.h). Scratch sizes are the f64
// formulas (c64 for the QR family) with 16 / 32-byte elements.
#include "../../include/faer_b200.h"
#include "dd.cuh"
#include "ffi_common.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

#include <cstring>
#include <memory>
#include <vector>

using namespace fb;

namespace {

template <bool CX>
constexpr size_t es() {
  return CX ? 32 : 16;
}
// `n` dd values from a host or device pointer
static void read_dd(const void* p, dd* out, int n) {
  FB_ASSERT(p != nullptr, "null scalar pointer");
  if (is_device_pointer(p)) FB_CUDA_CHECK(cudaMemcpy(out, p, 16 * (size_t)n, cudaMemcpyDeviceToHost));
  else memcpy(out, p, 16 * (size_t)n);
}
template <bool CX>
StagedMat stage(FaerV0_24_MatRef m, cudaStream_t st) {
  return StagedMat(m.ptr, (i64)m.nrows, (i64)m.ncols, (i64)m.row_stride, (i64)m.col_stride, es<CX>(), true, false, st);
}
template <bool CX>
StagedMat stage(FaerV0_24_MatMut m, bool copy_in, cudaStream_t st) {
  return StagedMat(m.ptr, (i64)m.nrows, (i64)m.ncols, (i64)m.row_stride, (i64)m.col_stride, es<CX>(), copy_in, true, st);
}

template <bool CX>
void matmul_dd(FaerV0_24_MatMut C, int C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, int A_block, FaerV0_24_MatRef B, int B_block,
               const FaerV0_24_Scalar* alpha) {
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  dd a[2] = {dd(0.0), dd(0.0)};
  read_dd(alpha, a, CX ? 2 : 1);
  const bool copy_in = accum == FaerV0_24_Accum_Add || C_block != FaerV0_24_Block_Rectangular;
  StagedMat c = stage<CX>(C, copy_in, st), l = stage<CX>(A, st), r = stage<CX>(B, st);
  gemm_dd(st, c.view<dd>(), C_block, accum == FaerV0_24_Accum_Add ? 1 : 0, l.view<const dd>(), A_block, false, r.view<const dd>(),
          B_block, false, CX, a[0], a[1]);
  finish_all(st, {&c, &l, &r});
}

template <bool CX>
void solve_tri_dd(FaerV0_24_MatRef T, FaerV0_24_Conj conj, FaerV0_24_MatMut rhs, bool lower, bool unit) {
  FB_ENTRY();
  FB_ASSERT(T.nrows == T.ncols && rhs.nrows == T.nrows, "triangular solve shape mismatch");
  cudaStream_t st = current_stream();
  StagedMat t = stage<CX>(T, st), r = stage<CX>(rhs, true, st);
  const bool cj = CX && conj == FaerV0_24_Conj_Yes;
  if (lower) solve_lower_t<dd, CX>(st, t.view<const dd>(), unit, cj, r.view<dd>());
  else solve_upper_t<dd, CX>(st, t.view<const dd>(), unit, cj, r.view<dd>());
  finish_all(st, {&t, &r});
}

template <bool CX>
void inverse_tri_dd(FaerV0_24_MatMut dst, FaerV0_24_MatRef src, bool lower, bool unit) {
  FB_ENTRY();
  FB_ASSERT(dst.nrows == dst.ncols && src.nrows == dst.nrows && src.ncols == dst.ncols, "inverse_triangular shape mismatch");
  if (dst.nrows == 0) return;
  cudaStream_t st = current_stream();
  // only the triangle is written: the rest of dst must survive the round trip
  StagedMat d = stage<CX>(dst, true, st), s = stage<CX>(src, st);
  inverse_triangular_t<dd, CX>(st, d.view<dd>(), s.view<const dd>(), lower, unit);
  finish_all(st, {&d, &s});
}

template <bool CX>
FaerV0_24_LltStatus llt_factor_dd(FaerV0_24_MatMut A, FaerV0_24_LltRegularization reg, FaerV0_24_LltParams params) {
  FB_ENTRY();
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  cudaStream_t st = current_stream();
  dd delta(0.0), eps(0.0);  // the regularisation parameters are T::Real: one fx128 for both kinds
  if (reg.dynamic_regularization_delta) read_dd(reg.dynamic_regularization_delta, &delta, 1);
  if (reg.dynamic_regularization_epsilon) read_dd(reg.dynamic_regularization_epsilon, &eps, 1);
  StagedMat a = stage<CX>(A, true, st);
  const LltResult r = llt_dd<CX>(st, a.view<dd>(), delta, eps, params.recursion_threshold, params.block_size);
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

// rhs <- conj?(L L^H)^-1 rhs (llt/solve.rs): L y = rhs, then L^H x = y
template <bool CX>
void llt_solve_dd(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs) {
  FB_ENTRY();
  FB_ASSERT(L.nrows == L.ncols && rhs.nrows == L.nrows, "LLT solve shape mismatch");
  cudaStream_t st = current_stream();
  StagedMat l = stage<CX>(L, st), r = stage<CX>(rhs, true, st);
  const bool cj = CX && A_conj == FaerV0_24_Conj_Yes;
  solve_lower_t<dd, CX>(st, l.view<const dd>(), false, cj, r.view<dd>());
  solve_upper_t<dd, CX>(st, l.view<const dd>().t(), false, CX && !cj, r.view<dd>());
  finish_all(st, {&l, &r});
}

template <bool CX>
void llt_recon_dd(FaerV0_24_MatMut A, FaerV0_24_MatRef L, bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat a = stage<CX>(A, true, st), l = stage<CX>(L, st);  // only the lower triangle is written
  if (inverse) llt_inverse_t<dd, CX>(st, a.view<dd>(), l.view<const dd>());
  else llt_reconstruct_t<dd, CX>(st, a.view<dd>(), l.view<const dd>());
  finish_all(st, {&a, &l});
}

template <bool CX>
FaerV0_24_PartialPivLuStatus lu_factor_dd(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd,
                                          FaerV0_24_PartialPivLuParams params, int idx_bytes) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  // the permutation length is A.nrows, never the slice's `len` (ffi.cu, lu_entry)
  FB_ASSERT(A.nrows == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  StagedMat a = stage<CX>(A, true, st);
  std::vector<long long> pf(A.nrows), pb(A.nrows);
  const size_t cnt = lu_dd<CX>(st, a.view<dd>(), params.recursion_threshold, pf.data(), pb.data());
  finish_all(st, {&a});
  write_perm(perm_fwd.ptr, pf, idx_bytes);
  write_perm(perm_bwd.ptr, pb, idx_bytes);
  FaerV0_24_PartialPivLuStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_PartialPivLuStatus_Ok;
  out.ok.transposition_count = cnt;
  return out;
}

// transpose = false: conj?(A)^-1 rhs with perm_fwd (lu/partial_pivoting/solve.rs:21-54); true: conj?(A)^-T rhs with perm_bwd (55-86)
template <bool CX>
void lu_solve_dd(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj conj, FaerV0_24_SliceRef perm, FaerV0_24_MatMut rhs, int idx_bytes,
                 bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "LU solve shape mismatch");
  const std::vector<long long> p = read_perm_checked(perm, n, idx_bytes);
  if (n == 0 || rhs.ncols == 0) return;
  StagedMat l = stage<CX>(L, st), u = stage<CX>(U, st), r = stage<CX>(rhs, true, st);
  const bool cj = CX && conj == FaerV0_24_Conj_Yes;
  if (!transpose) {
    permute_rows_t<dd, CX>(st, r.view<dd>(), p.data());
    solve_lower_t<dd, CX>(st, l.view<const dd>(), true, cj, r.view<dd>());
    solve_upper_t<dd, CX>(st, u.view<const dd>(), false, cj, r.view<dd>());
  } else {
    solve_lower_t<dd, CX>(st, u.view<const dd>().t(), false, cj, r.view<dd>());
    solve_upper_t<dd, CX>(st, l.view<const dd>().t(), true, cj, r.view<dd>());
    permute_rows_t<dd, CX>(st, r.view<dd>(), p.data());
  }
  finish_all(st, {&l, &u, &r});
}

template <bool CX>
void lu_recon_dd(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_SliceRef perm, int idx_bytes, bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const std::vector<long long> p = read_perm_checked(perm, L.nrows, idx_bytes);
  StagedMat a = stage<CX>(A, false, st), l = stage<CX>(L, st), u = stage<CX>(U, st);
  if (inverse) lu_inverse_t<dd, CX>(st, a.view<dd>(), l.view<const dd>(), u.view<const dd>(), p.data());
  else lu_reconstruct_t<dd, CX>(st, a.view<dd>(), l.view<const dd>(), u.view<const dd>(), p.data());
  finish_all(st, {&a, &l, &u});
}

// QR factor (qr/no_pivoting/factor.rs:258-301): returns the rank
template <bool CX>
FaerV0_24_QrStatus qr_factor_dd(FaerV0_24_MatMut A, FaerV0_24_MatMut Q, FaerV0_24_QrParams params) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols;
  FB_ASSERT(Q.nrows > 0 && Q.ncols == size, "Q_coeff must be block_size x min(nrows, ncols)");
  StagedMat a = stage<CX>(A, true, st), q = stage<CX>(Q, true, st);
  const i64 rank = qr_dd<CX>(st, a.view<dd>(), q.view<dd>(), (i64)params.blocking_threshold);
  finish_all(st, {&a, &q});
  FaerV0_24_QrStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_QrStatus_Ok;
  out.ok.rank = (size_t)rank;
  return out;
}

// rhs <- Q rhs (transpose = false) or Q^H rhs (true), Q conjugated for cx128 under Conj::Yes (householder.rs:724-808)
template <bool CX>
void householder_seq_dd(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, FaerV0_24_MatMut rhs, bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat b = stage<CX>(basis, st), f = stage<CX>(factor, st), r = stage<CX>(rhs, true, st);
  householder_sequence_dd<CX>(st, b.view<const dd>(), f.view<const dd>(), CX && conj == FaerV0_24_Conj_Yes, r.view<dd>(), transpose);
  finish_all(st, {&b, &f, &r});
}

// qr/no_pivoting/solve.rs:38-176. mode 0: least squares (m >= n), 1: square solve, 2: transpose solve. R may alias Q_basis (the
// packed factorization), which is then staged once.
template <bool CX>
void qr_solve_dd(FaerV0_24_MatRef Qb, FaerV0_24_MatRef Qc, FaerV0_24_MatRef Rm, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, int mode) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t m = Qb.nrows, n = Qb.ncols, size = m < n ? m : n;
  FB_ASSERT(Qc.nrows > 0 && rhs.nrows == m && m >= n && Qc.ncols == size && Rm.nrows >= size && Rm.ncols == n, "QR solve shape mismatch");
  if (mode != 0) FB_ASSERT(m == n && Rm.nrows == n, "QR solve: the factorization must be square");
  if (size == 0 || rhs.ncols == 0) return;
  const bool cj = CX && A_conj == FaerV0_24_Conj_Yes;
  StagedMat b = stage<CX>(Qb, st), f = stage<CX>(Qc, st), r = stage<CX>(rhs, true, st);
  const bool alias = Rm.ptr == Qb.ptr && Rm.row_stride == Qb.row_stride && Rm.col_stride == Qb.col_stride;
  std::unique_ptr<StagedMat> rr;
  if (!alias) rr.reset(new StagedMat(Rm.ptr, (i64)size, (i64)n, (i64)Rm.row_stride, (i64)Rm.col_stride, es<CX>(), true, false, st));
  const View<const dd> Rv = sub_t<dd, CX>(alias ? b.view<const dd>() : rr->view<const dd>(), 0, 0, (i64)size, (i64)n);
  const View<dd> x = r.view<dd>();
  if (mode == 2) {
    solve_lower_t<dd, CX>(st, Rv.t(), false, cj, x);                                           // op(R)^T y = rhs
    householder_sequence_dd<CX>(st, b.view<const dd>(), f.view<const dd>(), CX && !cj, x, false);  // the forward sequence, conj composed with Yes
  } else {
    householder_sequence_dd<CX>(st, b.view<const dd>(), f.view<const dd>(), CX && !cj, x, true);   // op(Q)^H rhs
    solve_upper_t<dd, CX>(st, Rv, false, cj, sub_t<dd, CX>(x, 0, 0, (i64)size, x.ncols));
  }
  finish_all(st, {&b, &f, &r});
  if (rr) rr->finish();
}

template <bool CX>
void qr_recon_dd(FaerV0_24_MatMut A, FaerV0_24_MatRef Qb, FaerV0_24_MatRef Qc, FaerV0_24_MatRef Rm, bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat a = stage<CX>(A, false, st), b = stage<CX>(Qb, st), f = stage<CX>(Qc, st), r = stage<CX>(Rm, st);
  if (inverse) qr_inverse_t<dd, CX>(st, a.view<dd>(), b.view<const dd>(), f.view<const dd>(), r.view<const dd>());
  else qr_reconstruct_t<dd, CX>(st, a.view<dd>(), b.view<const dd>(), f.view<const dd>(), r.view<const dd>());
  finish_all(st, {&a, &b, &f, &r});
}

// self-adjoint EVD (evd/mod.rs:270-418): the f64 / c64 entries' semantics (ffi.cu, ffi_types.cu); S holds (value, 0) for cx128
template <bool CX>
FaerV0_24_EvdStatus self_adjoint_evd_entry_dd(FaerV0_24_MatRef A, FaerV0_24_MatMut U, FaerV0_24_VecMut S) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = A.nrows, e = es<CX>();
  FB_ASSERT(A.ncols == n && S.len == n && (n == 0 || S.stride >= 1), "self_adjoint_evd: square A, S of length n, positive stride");
  const bool want_u = U.ncols != 0;
  if (want_u) FB_ASSERT(U.nrows == n && U.ncols == n, "self_adjoint_evd: U must be n x n (or have no columns)");
  FaerV0_24_EvdStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_EvdStatus_Ok;
  if (n == 0) return out;
  StagedMat a = stage<CX>(A, st);
  dd* s_dev = (dd*)ws_alloc(n * e);
  bool ok;
  if (want_u) {
    StagedMat u = stage<CX>(U, false, st);
    ok = self_adjoint_evd_dd<CX>(st, a.view<const dd>(), u.view<dd>(), s_dev);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * e, s_dev, e, e, n, cudaMemcpyDefault, st));
    finish_all(st, {&a, &u});
  } else {
    ok = self_adjoint_evd_dd<CX>(st, a.view<const dd>(), View<dd>{nullptr, 0, 0, 1, 1}, s_dev);
    if (ok) FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * e, s_dev, e, e, n, cudaMemcpyDefault, st));
    finish_all(st, {&a});
  }
  ws_free(s_dev);
  if (!ok) out.tag = FaerV0_24_EvdStatus_NoConvergence;
  return out;
}

}  // namespace

extern "C" {

#define FB_DD_FFI(SUF, CX)                                                                                                       \
  void libfaer_v0_23_matmul_##SUF(FaerV0_24_MatMut C, FaerV0_24_Accum accum, FaerV0_24_MatRef A, FaerV0_24_MatRef B,            \
                                  const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {                                           \
    (void)par;                                                                                                                  \
    matmul_dd<CX>(C, 0, accum, A, 0, B, 0, alpha);                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_matmul_triangular_##SUF(FaerV0_24_MatMut C, FaerV0_24_Block C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, \
                                             FaerV0_24_Block A_block, FaerV0_24_MatRef B, FaerV0_24_Block B_block,              \
                                             const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {                                \
    (void)par;                                                                                                                  \
    matmul_dd<CX>(C, (int)C_block, accum, A, (int)A_block, B, (int)B_block, alpha);                                             \
  }                                                                                                                             \
  void libfaer_v0_23_solve_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs,     \
                                                           FaerV0_24_Par par) {                                                 \
    (void)par;                                                                                                                  \
    solve_tri_dd<CX>(L, L_conj, rhs, true, false);                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_solve_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs,     \
                                                           FaerV0_24_Par par) {                                                 \
    (void)par;                                                                                                                  \
    solve_tri_dd<CX>(U, U_conj, rhs, false, false);                                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_solve_unit_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs, \
                                                                FaerV0_24_Par par) {                                            \
    (void)par;                                                                                                                  \
    solve_tri_dd<CX>(L, L_conj, rhs, true, true);                                                                               \
  }                                                                                                                             \
  void libfaer_v0_23_solve_unit_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs, \
                                                                FaerV0_24_Par par) {                                            \
    (void)par;                                                                                                                  \
    solve_tri_dd<CX>(U, U_conj, rhs, false, true);                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_triangular_lower_in_place_##SUF(FaerV0_24_MatMut L_inv, FaerV0_24_MatRef L, FaerV0_24_Par par) {    \
    (void)par;                                                                                                                  \
    inverse_tri_dd<CX>(L_inv, L, true, false);                                                                                  \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_triangular_upper_in_place_##SUF(FaerV0_24_MatMut U_inv, FaerV0_24_MatRef U, FaerV0_24_Par par) {    \
    (void)par;                                                                                                                  \
    inverse_tri_dd<CX>(U_inv, U, false, false);                                                                                 \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_unit_triangular_lower_in_place_##SUF(FaerV0_24_MatMut L_inv, FaerV0_24_MatRef L, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    inverse_tri_dd<CX>(L_inv, L, true, true);                                                                                   \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_unit_triangular_upper_in_place_##SUF(FaerV0_24_MatMut U_inv, FaerV0_24_MatRef U, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    inverse_tri_dd<CX>(U_inv, U, false, true);                                                                                  \
  }                                                                                                                             \
  FaerV0_24_LltParams libfaer_v0_23_LltParams_##SUF(void) { return libfaer_v0_23_LltParams_f64(); }                              \
  FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_##SUF(size_t dim, FaerV0_24_Par par, FaerV0_24_LltParams params) { \
    (void)par; (void)params;                                                                                                    \
    return FaerV0_24_Layout{dim * es<CX>(), 64}; /* temp_mat_scratch::<T>(dim, 1), llt/factor.rs:58-66 */                       \
  }                                                                                                                             \
  FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_LltRegularization regularization,   \
                                                              FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                        \
                                                              FaerV0_24_LltParams params) {                                     \
    (void)par; (void)mem;                                                                                                       \
    return llt_factor_dd<CX>(A, regularization, params);                                                                        \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {            \
    (void)dim; (void)rhs_ncols; (void)par;                                                                                      \
    return FaerV0_24_Layout{0, 1};                                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_llt_solve_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par, \
                                              FaerV0_24_MemAlloc mem) {                                                         \
    (void)par; (void)mem;                                                                                                       \
    llt_solve_dd<CX>(L, A_conj, rhs);                                                                                           \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_##SUF(size_t dim, FaerV0_24_Par par) {                                 \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{0, 1};                                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_llt_reconstruct_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)par; (void)mem;                                                                                                       \
    llt_recon_dd<CX>(A, L, false);                                                                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_##SUF(size_t dim, FaerV0_24_Par par) {                                     \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * dim * es<CX>(), 64};                                                                          \
  }                                                                                                                             \
  void libfaer_v0_23_llt_inverse_##SUF(FaerV0_24_MatMut A_inv, FaerV0_24_MatRef L, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)par; (void)mem;                                                                                                       \
    llt_recon_dd<CX>(A_inv, L, true);                                                                                           \
  }                                                                                                                             \
  FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_##SUF(void) { return libfaer_v0_23_PartialPivLuParams_f64(); }
FB_DD_FFI(fx128, false)
FB_DD_FFI(cx128, true)
#undef FB_DD_FFI

#define FB_DD_LU_FFI(IT, BYTES, SUF, CX)                                                                                         \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_##IT##_##SUF(size_t nrows, size_t ncols, FaerV0_24_Par par, \
                                                                                     FaerV0_24_PartialPivLuParams params) {    \
    (void)par; (void)params;                                                                                                    \
    return lu_scratch(nrows, ncols, BYTES);                                                                                     \
  }                                                                                                                             \
  FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_##IT##_##SUF(                                       \
      FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,   \
      FaerV0_24_PartialPivLuParams params) {                                                                                    \
    (void)par; (void)mem;                                                                                                       \
    return lu_factor_dd<CX>(A, perm_fwd, perm_bwd, params, BYTES);                                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * es<CX>(), 64};                                                                    \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,  \
                                                               FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,        \
                                                               FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)perm_bwd; (void)par; (void)mem;                                                                                       \
    lu_solve_dd<CX>(L, U, A_conj, perm_fwd, rhs, BYTES, false);                                                                 \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols,     \
                                                                                              FaerV0_24_Par par) {              \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * es<CX>(), 64};                                                                    \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_##IT##_##SUF(                                                      \
      FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,   \
      FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                                        \
    (void)perm_fwd; (void)par; (void)mem;                                                                                       \
    lu_solve_dd<CX>(L, U, A_conj, perm_bwd, rhs, BYTES, true);                                                                  \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_##IT##_##SUF(size_t nrows, size_t ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{nrows * ncols * es<CX>(), 64};                                                                      \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_reconstruct_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,        \
                                                             FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,          \
                                                             FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                       \
    (void)perm_fwd; (void)par; (void)mem;                                                                                       \
    lu_recon_dd<CX>(A, L, U, perm_bwd, BYTES, false);                                                                           \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                   \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * dim * es<CX>(), 64};                                                                          \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_inverse_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,            \
                                                         FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,              \
                                                         FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                           \
    (void)perm_bwd; (void)par; (void)mem;                                                                                       \
    lu_recon_dd<CX>(A, L, U, perm_fwd, BYTES, true);                                                                            \
  }
FB_DD_LU_FFI(u32, 4, fx128, false)
FB_DD_LU_FFI(u64, 8, fx128, false)
FB_DD_LU_FFI(u32, 4, cx128, true)
FB_DD_LU_FFI(u64, 8, cx128, true)
#undef FB_DD_LU_FFI

// ---- Householder QR, block-Householder sequences and the QR solves: the c64 entries' semantics and scratch formulas ----
#define FB_DD_QR_FFI(SUF, CX)                                                                                                    \
  FaerV0_24_QrParams libfaer_v0_23_QrParams_##SUF(void) { return FaerV0_24_QrParams{48 * 48, 192 * 256}; }                      \
  size_t libfaer_v0_23_qr_recommended_block_size_##SUF(size_t nrows, size_t ncols) {                                            \
    return (size_t)qr_recommended_block_size((i64)nrows, (i64)ncols);                                                           \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,                \
                                                                  FaerV0_24_Par par, FaerV0_24_QrParams params) {               \
    (void)nrows; (void)par; (void)params;                                                                                       \
    return FaerV0_24_Layout{block_size * ncols * es<CX>(), 64};                                                                 \
  }                                                                                                                             \
  FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatMut Q_coeff, FaerV0_24_Par par,    \
                                                            FaerV0_24_MemAlloc mem, FaerV0_24_QrParams params) {                \
    (void)par; (void)mem;                                                                                                       \
    return qr_factor_dd<CX>(A, Q_coeff, params);                                                                                \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols) { \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * rhs_ncols * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_##SUF(size_t dim, size_t block_size,           \
                                                                                        size_t rhs_ncols) {                     \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * rhs_ncols * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj,  \
                                                         FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {     \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_dd<CX>(basis, factor, conj, rhs, false);                                                                    \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_transpose_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,             \
                                                                   FaerV0_24_Conj conj, FaerV0_24_MatMut rhs,                   \
                                                                   FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                 \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_dd<CX>(basis, factor, conj, rhs, true);                                                                     \
  }                                                                                                                             \
  /* on the right = the transposed sequence on the left of the transposed view, and vice versa (householder.rs:813-854) */     \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_##SUF(size_t dim, size_t block_size, size_t lhs_nrows) { \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * lhs_nrows * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_##SUF(size_t dim, size_t block_size,          \
                                                                                         size_t lhs_nrows) {                    \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * lhs_nrows * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, \
                                                          FaerV0_24_MatMut lhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {    \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_dd<CX>(basis, factor, conj, transposed(lhs), true);                                                         \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_transpose_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,            \
                                                                    FaerV0_24_Conj conj, FaerV0_24_MatMut lhs,                  \
                                                                    FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                \
    (void)par; (void)mem;                                                                                                       \
    householder_seq_dd<CX>(basis, factor, conj, transposed(lhs), false);                                                        \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,           \
                                                                       size_t rhs_ncols, FaerV0_24_Par par) {                   \
    (void)nrows; (void)ncols; (void)par;                                                                                        \
    return FaerV0_24_Layout{block_size * rhs_ncols * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols,               \
                                                                 FaerV0_24_Par par) {                                           \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{block_size * rhs_ncols * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_##SUF(size_t dim, size_t block_size,                       \
                                                                           size_t rhs_ncols, FaerV0_24_Par par) {               \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{block_size * rhs_ncols * es<CX>(), 64};                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_lstsq_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R,      \
                                                   FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,              \
                                                   FaerV0_24_MemAlloc mem) {                                                    \
    (void)par; (void)mem;                                                                                                       \
    qr_solve_dd<CX>(Q_basis, Q_coeff, R, A_conj, rhs, 0);                                                                       \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R,            \
                                             FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,                    \
                                             FaerV0_24_MemAlloc mem) {                                                          \
    (void)par; (void)mem;                                                                                                       \
    qr_solve_dd<CX>(Q_basis, Q_coeff, R, A_conj, rhs, 1);                                                                       \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_transpose_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R,  \
                                                       FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,          \
                                                       FaerV0_24_MemAlloc mem) {                                                \
    (void)par; (void)mem;                                                                                                       \
    qr_solve_dd<CX>(Q_basis, Q_coeff, R, A_conj, rhs, 2);                                                                       \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size, FaerV0_24_Par par) { \
    (void)nrows; (void)par;                                                                                                     \
    return FaerV0_24_Layout{block_size * ncols * es<CX>(), 64};                                                                 \
  }                                                                                                                             \
  void libfaer_v0_23_qr_reconstruct_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,               \
                                          FaerV0_24_MatRef R, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                      \
    (void)par; (void)mem;                                                                                                       \
    qr_recon_dd<CX>(A, Q_basis, Q_coeff, R, false);                                                                             \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_##SUF(size_t dim, size_t block_size, FaerV0_24_Par par) {                   \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{block_size * dim * es<CX>(), 64};                                                                   \
  }                                                                                                                             \
  void libfaer_v0_23_qr_inverse_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R, \
                                      FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                              \
    (void)par; (void)mem;                                                                                                       \
    qr_recon_dd<CX>(A, Q_basis, Q_coeff, R, true);                                                                              \
  }
FB_DD_QR_FFI(fx128, false)
FB_DD_QR_FFI(cx128, true)
#undef FB_DD_QR_FFI

// ---- self-adjoint EVD: faer's defaults (evd/mod.rs:82-90) and the f64 / c64 scratch formula with 16 / 32-byte elements ----
#define FB_DD_EVD_FFI(SUF, CX)                                                                                                   \
  FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_##SUF(void) { return FaerV0_24_TridiagParams{192 * 256}; }               \
  FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_##SUF(void) {                                              \
    return FaerV0_24_SelfAdjointEvdParams{FaerV0_24_TridiagParams{192 * 256}, 128};                                            \
  }                                                                                                                            \
  FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_##SUF(size_t dim, FaerV0_24_ComputeEigenvectors compute_U,           \
                                                                FaerV0_24_Par par, FaerV0_24_SelfAdjointEvdParams params) {    \
    (void)compute_U; (void)par; (void)params;                                                                                  \
    return FaerV0_24_Layout{dim * dim * es<CX>(), 64};                                                                         \
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

}  // extern "C"
