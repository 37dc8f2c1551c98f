// The extern "C" entry points that every scalar kind shares, written once over the kind <R, complex?>: <double, false> f64,
// <float, false> f32, <double, true> c64, <float, true> c32, <dd, false> fx128, <dd, true> cx128 (complex views in complex units on
// an R* base). They cover matmul, the triangular solves and inverses, LLT, partial-pivoting LU, Householder QR and the LLT / LU /
// QR reconstruct and inverse entries. Each entry mirrors the faer-ffi function of the same name (faer-ffi/src/lib.rs, cited per
// function in the headers under include/): same argument order and meaning, by-value PODs, synchronous on return, abort() on
// precondition violations. Host buffers are staged, device buffers are used in place, and `Par` / `MemAlloc` are ignored.
//
// The solves, reconstructions and inverses are the compositions of tensor_ops.cuh / reconstruct_types.cu for every kind; only the
// factorization drivers differ by kind (the `*_kind` functions). The export macros at the end are instantiated by ffi.cu (f64,
// f32, c64, c32), ffi_types.cu (the triangular inverses and the reconstruct / inverse entries of the IEEE kinds, which it builds
// for the host too) and ffi_dd.cu (fx128, cx128). Scratch layouts are faer's formulas with the kind's element size.
#pragma once
#include "ffi_common.cuh"
#include "tensor_ops.cuh"

#include <memory>
#include <type_traits>
#include <vector>

namespace fb {

template <class R>
constexpr bool is_dd_v = std::is_same_v<R, dd>;
template <class R, bool CX>
constexpr bool is_f64_v = std::is_same_v<R, double> && !CX;
template <class R, bool CX>
constexpr bool is_ieee_real_v = !CX && !is_dd_v<R>;

// f32 partial-pivoting LU computed in f64 (ffi.cu): the matrix is widened on the device, factored by the f64 drivers and rounded
// back. The factors carry one f32 rounding instead of an f32 elimination's accumulated ones. Hidden: the library exports the C ABI.
__attribute__((visibility("hidden"))) size_t lu_partial_piv_in_place_f32_via_f64(cudaStream_t st, VF A, long long* perm_fwd,
                                                                                  long long* perm_bwd);

// The hooks and bodies below are static: each translation unit instantiates the ones it exports, and they are not exported
// themselves. (Static rather than an anonymous namespace: nvcc's kernel stubs of a unit that also has a global anonymous namespace
// must stay unambiguous.)
// ---- per-kind drivers ----
template <class R, bool CX>
static LltResult llt_kind(cudaStream_t st, View<R> A, R delta, R eps, FaerV0_24_LltParams p) {
  if constexpr (is_dd_v<R>) return llt_dd<CX>(st, A, delta, eps, p.recursion_threshold, p.block_size);
  else if constexpr (CX && sizeof(R) == 8) return llt_cholesky_in_place_c64(st, A, delta, eps);
  else if constexpr (CX) return llt_cholesky_in_place_c32(st, A, delta, eps);
  else if constexpr (sizeof(R) == 8) return llt_cholesky_in_place_f64(st, A, delta, eps, LltParams{p.recursion_threshold, p.block_size});
  else return llt_cholesky_in_place_f32(st, A, delta, eps, LltParams{p.recursion_threshold, p.block_size});
}
// returns the transposition count; perm_fwd / perm_bwd: HOST int64 of A.nrows entries
template <class R, bool CX>
static size_t lu_kind(cudaStream_t st, View<R> A, FaerV0_24_PartialPivLuParams p, long long* perm_fwd, long long* perm_bwd) {
  if constexpr (is_dd_v<R>) return lu_dd<CX>(st, A, p.recursion_threshold, perm_fwd, perm_bwd);
  else if constexpr (CX && sizeof(R) == 8) return lu_partial_piv_in_place_c64(st, A, perm_fwd, perm_bwd);
  else if constexpr (CX) return lu_partial_piv_in_place_c32(st, A, perm_fwd, perm_bwd);
  else if constexpr (sizeof(R) == 8) return lu_partial_piv_in_place_f64(st, A, perm_fwd, perm_bwd);
  else return lu_partial_piv_in_place_f32_via_f64(st, A, perm_fwd, perm_bwd);
}
// Householder QR without pivoting (qr/no_pivoting/factor.rs:258-301); returns the rank. The real IEEE drivers pick their own
// blocking.
template <class R, bool CX>
static i64 qr_kind(cudaStream_t st, View<R> A, View<R> Q, i64 blocking_threshold) {
  if constexpr (is_dd_v<R>) return qr_dd<CX>(st, A, Q, blocking_threshold);
  else if constexpr (!CX) return qr_in_place<R>(st, A, Q);
  else if constexpr (sizeof(R) == 8) return qr_in_place_c64(st, A, Q, blocking_threshold);
  else return qr_in_place_c32(st, A, Q, blocking_threshold);
}
// The row permutation of the LU solves and reconstructions, of A.nrows entries (faer.hpp fills SliceRef.len with bytes, so `len`
// is never used). An entry outside [0, n) aborts. fx128 / cx128 also abort on a null slice; the IEEE kinds do not test for it.
template <class R>
static std::vector<long long> read_lu_perm(FaerV0_24_SliceRef s, size_t n, int idx_bytes) {
  if constexpr (is_dd_v<R>) {
    return read_perm_checked(s, n, idx_bytes);
  } else {
    std::vector<long long> p = read_perm(s.ptr, n, idx_bytes);
    for (size_t i = 0; i < n; ++i) FB_ASSERT(p[i] >= 0 && (size_t)p[i] < n, "invalid permutation entry");
    return p;
  }
}

// ---- entry bodies ----
template <class R, bool CX>
static void matmul_entry(FaerV0_24_MatMut C, int C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, int A_block, FaerV0_24_MatRef B,
                  int B_block, const FaerV0_24_Scalar* alpha, bool conj_a = false, bool conj_b = false) {
  FB_ENTRY();
  FB_ASSERT(C.nrows == A.nrows && C.ncols == B.ncols && A.ncols == B.nrows, "matmul shape mismatch");
  cudaStream_t st = current_stream();
  R a[2] = {R(0), R(0)};
  read_scalar<R, CX>(alpha, a);
  const bool copy_in = accum == FaerV0_24_Accum_Add || C_block != FaerV0_24_Block_Rectangular;
  StagedMat c = stage<R, CX>(C, copy_in, st), l = stage<R, CX>(A, st), r = stage<R, CX>(B, st);
  gemm_t<R, CX>(st, c.view<R>(), C_block, accum == FaerV0_24_Accum_Add ? 1 : 0, l.view<const R>(), A_block, conj_a, r.view<const R>(),
                B_block, conj_b, a[0], a[1]);
  finish_all(st, {&c, &l, &r});
}

template <class R, bool CX>
static void solve_triangular_entry(FaerV0_24_MatRef T, FaerV0_24_Conj conj, FaerV0_24_MatMut rhs, bool lower, bool unit) {
  FB_ENTRY();
  FB_ASSERT(T.nrows == T.ncols && rhs.nrows == T.nrows, "triangular solve shape mismatch");
  cudaStream_t st = current_stream();
  StagedMat t = stage<R, CX>(T, st), r = stage<R, CX>(rhs, true, st);
  const bool cj = CX && conj == FaerV0_24_Conj_Yes;
  if (lower) solve_lower_t<R, CX>(st, t.view<const R>(), unit, cj, r.view<R>());
  else solve_upper_t<R, CX>(st, t.view<const R>(), unit, cj, r.view<R>());
  finish_all(st, {&t, &r});
}

// triangular_inverse.rs; faer-ffi/src/lib.rs:938-980
template <class R, bool CX>
static void inverse_triangular_entry(FaerV0_24_MatMut dst, FaerV0_24_MatRef src, bool lower, bool unit) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  FB_ASSERT(dst.nrows == dst.ncols && src.nrows == dst.nrows && src.ncols == dst.ncols, "inverse_triangular shape mismatch");
  if (dst.nrows == 0) return;
  // only the triangle is written: the rest of dst must survive the round trip
  StagedMat d = stage<R, CX>(dst, true, st), s = stage<R, CX>(src, st);
  inverse_triangular_t<R, CX>(st, d.view<R>(), s.view<const R>(), lower, unit);
  finish_all(st, {&d, &s});
}

template <class R, bool CX>
static FaerV0_24_LltStatus llt_factor_entry(FaerV0_24_MatMut A, FaerV0_24_LltRegularization reg, FaerV0_24_LltParams params) {
  FB_ENTRY();
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  cudaStream_t st = current_stream();
  R delta(0), eps(0);  // the regularisation parameters are T::Real
  if (reg.dynamic_regularization_delta) read_scalar<R>(reg.dynamic_regularization_delta, &delta);
  if (reg.dynamic_regularization_epsilon) read_scalar<R>(reg.dynamic_regularization_epsilon, &eps);
  if constexpr (is_f64_v<R, CX>) {
    if (A.nrows > 0 && !is_device_pointer(A.ptr) && A.row_stride == 1 && A.col_stride >= (ptrdiff_t)A.nrows &&
        (i64)A.nrows >= lookahead_min_n()) {
      // a large column-major host matrix: upload / factor / download pipelined block column by block column (dist.cu)
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      const i64 nb = lookahead_block() ? lookahead_block() : 256;
      return llt_status(llt_host_pipelined_f64((double*)A.ptr, (i64)A.col_stride, (i64)A.nrows, nb, delta, eps));
    }
  }
  StagedMat a = stage<R, CX>(A, true, st);
  const LltResult r = llt_kind<R, CX>(st, a.view<R>(), delta, eps, params);
  finish_all(st, {&a});
  return llt_status(r);
}

template <class R, bool CX>
static void llt_solve_entry(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs) {
  FB_ENTRY();
  FB_ASSERT(L.nrows == L.ncols && rhs.nrows == L.nrows, "LLT solve shape mismatch");
  cudaStream_t st = current_stream();
  StagedMat l = stage<R, CX>(L, st), r = stage<R, CX>(rhs, true, st);
  llt_solve_t<R, CX>(st, l.view<const R>(), CX && A_conj == FaerV0_24_Conj_Yes, r.view<R>());
  finish_all(st, {&l, &r});
}

template <class R, bool CX>
static FaerV0_24_PartialPivLuStatus lu_factor_entry(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd,
                                             FaerV0_24_PartialPivLuParams params, int idx_bytes) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  // faer.hpp fills SliceMut.len with BYTES while the Rust side reads elements (SURVEY.md appendix A), so the permutation length
  // is taken from A.nrows, never from `len`
  FB_ASSERT(A.nrows == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  StagedMat a = stage<R, CX>(A, true, st);
  std::vector<long long> pf(A.nrows), pb(A.nrows);
  const size_t count = lu_kind<R, CX>(st, a.view<R>(), params, pf.data(), pb.data());
  finish_all(st, {&a});
  write_perm(perm_fwd.ptr, pf, idx_bytes);
  write_perm(perm_bwd.ptr, pb, idx_bytes);
  return partial_piv_lu_status(count);
}

template <class R, bool CX>
static void lu_solve_entry(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj conj, FaerV0_24_SliceRef perm, FaerV0_24_MatMut rhs,
                    int idx_bytes, bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "LU solve shape mismatch");
  const std::vector<long long> p = read_lu_perm<R>(perm, n, idx_bytes);
  if constexpr (is_dd_v<R>) {
    if (n == 0 || rhs.ncols == 0) return;  // fx128 / cx128 stage nothing for an empty solve
  }
  StagedMat l = stage<R, CX>(L, st), u = stage<R, CX>(U, st), r = stage<R, CX>(rhs, true, st);
  lu_solve_t<R, CX>(st, l.view<const R>(), u.view<const R>(), CX && conj == FaerV0_24_Conj_Yes, p.data(), r.view<R>(), transpose);
  finish_all(st, {&l, &u, &r});
}

template <class R, bool CX>
static FaerV0_24_QrStatus qr_factor_entry(FaerV0_24_MatMut A, FaerV0_24_MatMut Q, FaerV0_24_QrParams params) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols;
  FB_ASSERT(Q.nrows > 0 && Q.ncols == size, "Q_coeff must be block_size x min(nrows, ncols)");
  StagedMat a = stage<R, CX>(A, true, st), q = stage<R, CX>(Q, true, st);
  const i64 rank = qr_kind<R, CX>(st, a.view<R>(), q.view<R>(), (i64)params.blocking_threshold);
  finish_all(st, {&a, &q});
  // the real IEEE kinds report a negative rank as QrStatus::Unknown; the complex and dd kinds pass the rank on as it is
  return qr_status(rank, is_ieee_real_v<R, CX>);
}

template <class R, bool CX>
static void householder_entry(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, FaerV0_24_MatMut rhs, bool transpose) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat b = stage<R, CX>(basis, st), f = stage<R, CX>(factor, st), r = stage<R, CX>(rhs, true, st);
  householder_sequence_t<R, CX>(st, b.view<const R>(), f.view<const R>(), conj == FaerV0_24_Conj_Yes, r.view<R>(), transpose);
  finish_all(st, {&b, &f, &r});
}

// qr/no_pivoting/solve.rs:38-176. mode 0: solve_lstsq_in_place_with_conj (m >= n): rhs <- op(Q)^H rhs, then
// op(R)[..size, ..] x = rhs[..size, ..]; mode 1: solve_in_place_with_conj, the same on a square factorization; mode 2:
// solve_transpose_in_place_with_conj: op(R)^T y = rhs (a lower solve on the transposed view), then rhs <- conj(op(Q)) y
template <class R, bool CX>
static void qr_solve_entry(FaerV0_24_MatRef Qb, FaerV0_24_MatRef Qc, FaerV0_24_MatRef Rm, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs,
                    int mode) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t m = Qb.nrows, n = Qb.ncols, size = m < n ? m : n;
  FB_ASSERT(Qc.nrows > 0 && rhs.nrows == m && m >= n && Qc.ncols == size && Rm.nrows >= size && Rm.ncols == n,
            "QR solve shape mismatch");
  if (mode != 0) FB_ASSERT(m == n && Rm.nrows == n, "QR solve: the factorization must be square");
  if (size == 0 || rhs.ncols == 0) return;
  const bool cj = CX && A_conj == FaerV0_24_Conj_Yes;
  StagedMat b = stage<R, CX>(Qb, st), f = stage<R, CX>(Qc, st), r = stage<R, CX>(rhs, true, st);
  // callers normally pass the packed QR matrix for both Q_basis and R (solve.rs:232-246): it is then staged once
  const bool alias = Rm.ptr == Qb.ptr && Rm.row_stride == Qb.row_stride && Rm.col_stride == Qb.col_stride;
  std::unique_ptr<StagedMat> rr;
  if (!alias)
    rr.reset(new StagedMat(Rm.ptr, (i64)size, (i64)n, (i64)Rm.row_stride, (i64)Rm.col_stride, elem_bytes<R, CX>(), true, false, st));
  const View<const R> Rv = sub_t<R, CX>(alias ? b.view<const R>() : rr->view<const R>(), 0, 0, (i64)size, (i64)n);
  const View<R> x = r.view<R>();
  if (mode == 2) {
    solve_lower_t<R, CX>(st, Rv.t(), false, cj, x);
    householder_sequence_t<R, CX>(st, b.view<const R>(), f.view<const R>(), !cj, x, false);  // conj composed with Yes
  } else {
    householder_sequence_t<R, CX>(st, b.view<const R>(), f.view<const R>(), !cj, x, true);
    solve_upper_t<R, CX>(st, Rv, false, cj, sub_t<R, CX>(x, 0, 0, (i64)size, x.ncols));
  }
  finish_all(st, {&b, &f, &r});
  if (rr) rr->finish();
}

template <class R, bool CX>
static void llt_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef L, bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  // only the lower triangle is written: the rest of A must survive the round trip
  StagedMat a = stage<R, CX>(A, true, st), l = stage<R, CX>(L, st);
  if (inverse) llt_inverse_t<R, CX>(st, a.view<R>(), l.view<const R>());
  else llt_reconstruct_t<R, CX>(st, a.view<R>(), l.view<const R>());
  finish_all(st, {&a, &l});
}

// reconstruct: perm = perm_bwd; inverse: perm = perm_fwd
template <class R, bool CX>
static void lu_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_SliceRef perm, int idx_bytes, bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const std::vector<long long> p = read_lu_perm<R>(perm, L.nrows, idx_bytes);
  StagedMat a = stage<R, CX>(A, false, st), l = stage<R, CX>(L, st), u = stage<R, CX>(U, st);
  if (inverse) lu_inverse_t<R, CX>(st, a.view<R>(), l.view<const R>(), u.view<const R>(), p.data());
  else lu_reconstruct_t<R, CX>(st, a.view<R>(), l.view<const R>(), u.view<const R>(), p.data());
  finish_all(st, {&a, &l, &u});
}

template <class R, bool CX>
static void qr_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef Qb, FaerV0_24_MatRef Qc, FaerV0_24_MatRef Rm, bool inverse) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  StagedMat a = stage<R, CX>(A, false, st), b = stage<R, CX>(Qb, st), f = stage<R, CX>(Qc, st), r = stage<R, CX>(Rm, st);
  if (inverse) qr_inverse_t<R, CX>(st, a.view<R>(), b.view<const R>(), f.view<const R>(), r.view<const R>());
  else qr_reconstruct_t<R, CX>(st, a.view<R>(), b.view<const R>(), f.view<const R>(), r.view<const R>());
  finish_all(st, {&a, &b, &f, &r});
}

}  // namespace fb

// ---- exports, one macro per family: (SUF, R, CX) names the kind ----
#define FB_MATMUL_FFI(SUF, R, CX)                                                                                                \
  void libfaer_v0_23_matmul_##SUF(FaerV0_24_MatMut C, FaerV0_24_Accum accum, FaerV0_24_MatRef A, FaerV0_24_MatRef B,            \
                                  const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {                                           \
    (void)par;                                                                                                                  \
    fb::matmul_entry<R, CX>(C, 0, accum, A, 0, B, 0, alpha);                                                                    \
  }                                                                                                                             \
  void libfaer_v0_23_matmul_triangular_##SUF(FaerV0_24_MatMut C, FaerV0_24_Block C_block, FaerV0_24_Accum accum, FaerV0_24_MatRef A, \
                                             FaerV0_24_Block A_block, FaerV0_24_MatRef B, FaerV0_24_Block B_block,              \
                                             const FaerV0_24_Scalar* alpha, FaerV0_24_Par par) {                                \
    (void)par;                                                                                                                  \
    fb::matmul_entry<R, CX>(C, (int)C_block, accum, A, (int)A_block, B, (int)B_block, alpha);                                   \
  }

#define FB_TRSM_FFI(SUF, R, CX)                                                                                                  \
  void libfaer_v0_23_solve_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs,     \
                                                           FaerV0_24_Par par) {                                                 \
    (void)par;                                                                                                                  \
    fb::solve_triangular_entry<R, CX>(L, L_conj, rhs, true, false);                                                             \
  }                                                                                                                             \
  void libfaer_v0_23_solve_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs,     \
                                                           FaerV0_24_Par par) {                                                 \
    (void)par;                                                                                                                  \
    fb::solve_triangular_entry<R, CX>(U, U_conj, rhs, false, false);                                                            \
  }                                                                                                                             \
  void libfaer_v0_23_solve_unit_triangular_lower_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj L_conj, FaerV0_24_MatMut rhs, \
                                                                FaerV0_24_Par par) {                                            \
    (void)par;                                                                                                                  \
    fb::solve_triangular_entry<R, CX>(L, L_conj, rhs, true, true);                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_solve_unit_triangular_upper_in_place_##SUF(FaerV0_24_MatRef U, FaerV0_24_Conj U_conj, FaerV0_24_MatMut rhs, \
                                                                FaerV0_24_Par par) {                                            \
    (void)par;                                                                                                                  \
    fb::solve_triangular_entry<R, CX>(U, U_conj, rhs, false, true);                                                             \
  }

#define FB_TRI_INV_FFI(SUF, R, CX)                                                                                               \
  void libfaer_v0_23_inverse_triangular_lower_in_place_##SUF(FaerV0_24_MatMut L_inv, FaerV0_24_MatRef L, FaerV0_24_Par par) {    \
    (void)par;                                                                                                                  \
    fb::inverse_triangular_entry<R, CX>(L_inv, L, true, false);                                                                 \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_triangular_upper_in_place_##SUF(FaerV0_24_MatMut U_inv, FaerV0_24_MatRef U, FaerV0_24_Par par) {    \
    (void)par;                                                                                                                  \
    fb::inverse_triangular_entry<R, CX>(U_inv, U, false, false);                                                                \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_unit_triangular_lower_in_place_##SUF(FaerV0_24_MatMut L_inv, FaerV0_24_MatRef L, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    fb::inverse_triangular_entry<R, CX>(L_inv, L, true, true);                                                                  \
  }                                                                                                                             \
  void libfaer_v0_23_inverse_unit_triangular_upper_in_place_##SUF(FaerV0_24_MatMut U_inv, FaerV0_24_MatRef U, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    fb::inverse_triangular_entry<R, CX>(U_inv, U, false, true);                                                                 \
  }

// faer's defaults: ldlt/factor.rs:705-714; scratch: temp_mat_scratch::<T>(dim, 1) (llt/factor.rs:58-66) and StackReq::EMPTY
// (llt/solve.rs:3-10). The GPU paths keep their workspace in the device pool but report faer's requirement.
#define FB_LLT_FFI(SUF, R, CX)                                                                                                   \
  FaerV0_24_LltParams libfaer_v0_23_LltParams_##SUF(void) { return FaerV0_24_LltParams{64, 128}; }                              \
  FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_##SUF(size_t dim, FaerV0_24_Par par, FaerV0_24_LltParams params) { \
    (void)par; (void)params;                                                                                                    \
    return FaerV0_24_Layout{dim * fb::elem_bytes<R, CX>(), 64};                                                                 \
  }                                                                                                                             \
  FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_LltRegularization regularization,   \
                                                              FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                        \
                                                              FaerV0_24_LltParams params) {                                     \
    (void)par; (void)mem;                                                                                                       \
    return fb::llt_factor_entry<R, CX>(A, regularization, params);                                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {            \
    (void)dim; (void)rhs_ncols; (void)par;                                                                                      \
    return FaerV0_24_Layout{0, 1};                                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_llt_solve_in_place_##SUF(FaerV0_24_MatRef L, FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par, \
                                              FaerV0_24_MemAlloc mem) {                                                         \
    (void)par; (void)mem;                                                                                                       \
    fb::llt_solve_entry<R, CX>(L, A_conj, rhs);                                                                                 \
  }

// scratch: StackReq::EMPTY (llt/reconstruct.rs:3-6) and temp_mat_scratch(dim, dim) (llt/inverse.rs:3-8)
#define FB_LLT_RECON_FFI(SUF, R, CX)                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_##SUF(size_t dim, FaerV0_24_Par par) {                                 \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{0, 1};                                                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_llt_reconstruct_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)par; (void)mem;                                                                                                       \
    fb::llt_recon_entry<R, CX>(A, L, false);                                                                                    \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_##SUF(size_t dim, FaerV0_24_Par par) {                                     \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * dim * fb::elem_bytes<R, CX>(), 64};                                                           \
  }                                                                                                                             \
  void libfaer_v0_23_llt_inverse_##SUF(FaerV0_24_MatMut A_inv, FaerV0_24_MatRef L, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)par; (void)mem;                                                                                                       \
    fb::llt_recon_entry<R, CX>(A_inv, L, true);                                                                                 \
  }

// faer's defaults: lu/partial_pivoting/factor.rs:212-222; factor scratch: lu_scratch; solve scratch: permute_rows_in_place_scratch
// (perm/mod.rs)
#define FB_LU_IDX_FFI(IT, BYTES, SUF, R, CX)                                                                                     \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_##IT##_##SUF(size_t nrows, size_t ncols, FaerV0_24_Par par, \
                                                                                     FaerV0_24_PartialPivLuParams params) {    \
    (void)par; (void)params;                                                                                                    \
    return fb::lu_scratch(nrows, ncols, BYTES);                                                                                 \
  }                                                                                                                             \
  FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_##IT##_##SUF(                                       \
      FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,   \
      FaerV0_24_PartialPivLuParams params) {                                                                                    \
    (void)par; (void)mem;                                                                                                       \
    return fb::lu_factor_entry<R, CX>(A, perm_fwd, perm_bwd, params, BYTES);                                                    \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                                     \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,  \
                                                               FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,        \
                                                               FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) { \
    (void)perm_bwd; (void)par; (void)mem;                                                                                       \
    fb::lu_solve_entry<R, CX>(L, U, A_conj, perm_fwd, rhs, BYTES, false);                                                       \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols,     \
                                                                                              FaerV0_24_Par par) {              \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                                     \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_##IT##_##SUF(                                                      \
      FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,   \
      FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                                        \
    (void)perm_fwd; (void)par; (void)mem;                                                                                       \
    fb::lu_solve_entry<R, CX>(L, U, A_conj, perm_bwd, rhs, BYTES, true);                                                        \
  }
#define FB_LU_FFI(SUF, R, CX)                                                                                                    \
  FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_##SUF(void) {                                                   \
    return FaerV0_24_PartialPivLuParams{16, 64, 128 * 128};                                                                     \
  }                                                                                                                             \
  FB_LU_IDX_FFI(u32, 4, SUF, R, CX)                                                                                             \
  FB_LU_IDX_FFI(u64, 8, SUF, R, CX)

#define FB_LU_RECON_IDX_FFI(IT, BYTES, SUF, R, CX)                                                                               \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_##IT##_##SUF(size_t nrows, size_t ncols, FaerV0_24_Par par) { \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{nrows * ncols * fb::elem_bytes<R, CX>(), 64};                                                       \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_reconstruct_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,        \
                                                             FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,          \
                                                             FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                       \
    (void)perm_fwd; (void)par; (void)mem;                                                                                       \
    fb::lu_recon_entry<R, CX>(A, L, U, perm_bwd, BYTES, false);                                                                 \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                   \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{dim * dim * fb::elem_bytes<R, CX>(), 64};                                                           \
  }                                                                                                                             \
  void libfaer_v0_23_partial_piv_lu_inverse_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,            \
                                                         FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,              \
                                                         FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                           \
    (void)perm_bwd; (void)par; (void)mem;                                                                                       \
    fb::lu_recon_entry<R, CX>(A, L, U, perm_fwd, BYTES, true);                                                                  \
  }
#define FB_LU_RECON_FFI(SUF, R, CX)                                                                                              \
  FB_LU_RECON_IDX_FFI(u32, 4, SUF, R, CX)                                                                                       \
  FB_LU_RECON_IDX_FFI(u64, 8, SUF, R, CX)

// every QR scratch is a block_size x (columns) temporary (temp_mat_scratch, and
// apply_block_householder_sequence_[transpose_]on_the_left_in_place_scratch for the sequences and the solves, solve.rs:3-37).
// On the right = the transposed sequence on the left of the transposed view, and vice versa (householder.rs:813-854).
#define FB_QR_FFI(SUF, R, CX)                                                                                                    \
  FaerV0_24_QrParams libfaer_v0_23_QrParams_##SUF(void) { return FaerV0_24_QrParams{48 * 48, 192 * 256}; }                      \
  size_t libfaer_v0_23_qr_recommended_block_size_##SUF(size_t nrows, size_t ncols) {                                            \
    return (size_t)fb::qr_recommended_block_size((fb::i64)nrows, (fb::i64)ncols);                                               \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,                \
                                                                  FaerV0_24_Par par, FaerV0_24_QrParams params) {               \
    (void)nrows; (void)par; (void)params;                                                                                       \
    return FaerV0_24_Layout{block_size * ncols * fb::elem_bytes<R, CX>(), 64};                                                  \
  }                                                                                                                             \
  FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatMut Q_coeff, FaerV0_24_Par par,    \
                                                            FaerV0_24_MemAlloc mem, FaerV0_24_QrParams params) {                \
    (void)par; (void)mem;                                                                                                       \
    return fb::qr_factor_entry<R, CX>(A, Q_coeff, params);                                                                      \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols) { \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_##SUF(size_t dim, size_t block_size,           \
                                                                                        size_t rhs_ncols) {                     \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj,  \
                                                         FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {     \
    (void)par; (void)mem;                                                                                                       \
    fb::householder_entry<R, CX>(basis, factor, conj, rhs, false);                                                              \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_transpose_on_the_left_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,             \
                                                                   FaerV0_24_Conj conj, FaerV0_24_MatMut rhs,                   \
                                                                   FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                 \
    (void)par; (void)mem;                                                                                                       \
    fb::householder_entry<R, CX>(basis, factor, conj, rhs, true);                                                               \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_##SUF(size_t dim, size_t block_size, size_t lhs_nrows) { \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * lhs_nrows * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_##SUF(size_t dim, size_t block_size,          \
                                                                                         size_t lhs_nrows) {                    \
    (void)dim;                                                                                                                  \
    return FaerV0_24_Layout{block_size * lhs_nrows * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor, FaerV0_24_Conj conj, \
                                                          FaerV0_24_MatMut lhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {    \
    (void)par; (void)mem;                                                                                                       \
    fb::householder_entry<R, CX>(basis, factor, conj, fb::transposed(lhs), true);                                               \
  }                                                                                                                             \
  void libfaer_v0_23_apply_householder_transpose_on_the_right_##SUF(FaerV0_24_MatRef basis, FaerV0_24_MatRef factor,            \
                                                                    FaerV0_24_Conj conj, FaerV0_24_MatMut lhs,                  \
                                                                    FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                \
    (void)par; (void)mem;                                                                                                       \
    fb::householder_entry<R, CX>(basis, factor, conj, fb::transposed(lhs), false);                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size,           \
                                                                       size_t rhs_ncols, FaerV0_24_Par par) {                   \
    (void)nrows; (void)ncols; (void)par;                                                                                        \
    return FaerV0_24_Layout{block_size * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_##SUF(size_t dim, size_t block_size, size_t rhs_ncols,               \
                                                                 FaerV0_24_Par par) {                                           \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{block_size * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_##SUF(size_t dim, size_t block_size,                       \
                                                                           size_t rhs_ncols, FaerV0_24_Par par) {               \
    (void)dim; (void)par;                                                                                                       \
    return FaerV0_24_Layout{block_size * rhs_ncols * fb::elem_bytes<R, CX>(), 64};                                              \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_lstsq_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R_,     \
                                                   FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,              \
                                                   FaerV0_24_MemAlloc mem) {                                                    \
    (void)par; (void)mem;                                                                                                       \
    fb::qr_solve_entry<R, CX>(Q_basis, Q_coeff, R_, A_conj, rhs, 0);                                                            \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R_,           \
                                             FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,                    \
                                             FaerV0_24_MemAlloc mem) {                                                          \
    (void)par; (void)mem;                                                                                                       \
    fb::qr_solve_entry<R, CX>(Q_basis, Q_coeff, R_, A_conj, rhs, 1);                                                            \
  }                                                                                                                             \
  void libfaer_v0_23_qr_solve_transpose_in_place_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R_, \
                                                       FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,          \
                                                       FaerV0_24_MemAlloc mem) {                                                \
    (void)par; (void)mem;                                                                                                       \
    fb::qr_solve_entry<R, CX>(Q_basis, Q_coeff, R_, A_conj, rhs, 2);                                                            \
  }

#define FB_QR_RECON_FFI(SUF, R, CX)                                                                                              \
  FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_##SUF(size_t nrows, size_t ncols, size_t block_size, FaerV0_24_Par par) { \
    (void)nrows; (void)par;                                                                                                     \
    return FaerV0_24_Layout{block_size * ncols * fb::elem_bytes<R, CX>(), 64};                                                  \
  }                                                                                                                             \
  void libfaer_v0_23_qr_reconstruct_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,               \
                                          FaerV0_24_MatRef R_, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                     \
    (void)par; (void)mem;                                                                                                       \
    fb::qr_recon_entry<R, CX>(A, Q_basis, Q_coeff, R_, false);                                                                  \
  }
#define FB_QR_INV_FFI(SUF, R, CX)                                                                                                \
  FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_##SUF(size_t dim, size_t block_size, FaerV0_24_Par par) {                   \
    (void)par;                                                                                                                  \
    return FaerV0_24_Layout{block_size * dim * fb::elem_bytes<R, CX>(), 64};                                                    \
  }                                                                                                                             \
  void libfaer_v0_23_qr_inverse_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R_, \
                                      FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                              \
    (void)par; (void)mem;                                                                                                       \
    fb::qr_recon_entry<R, CX>(A, Q_basis, Q_coeff, R_, true);                                                                   \
  }
