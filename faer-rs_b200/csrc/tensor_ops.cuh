// Type-generic spellings (f32 / f64, and every scalar kind <R, complex?>) of the tensor-core building blocks, so that the drivers
// are written once. f64 -> DMMA GEMM (gemm_f64.cu), f32 -> 3xTF32 GEMM (gemm_f32.cu), c64 / c32 on those (gemm_c64.cu,
// gemm_c32.cu); triangular solves from trsm.cu and cplx.cu.
#pragma once
#include <type_traits>

#include "gemm_f32.cuh"
#include "linalg_f64.cuh"

namespace fb {

// ---- double-double kinds <dd, false> (fx128) and <dd, true> (cx128); dd.cuh, gemm_dd.cu, dd_factor.cu. Complex views are in
// complex units on a dd* base. `alpha_im` is ignored by the real kind. ----
struct dd;
void gemm_dd(cudaStream_t st, View<dd> dst, int ds, int accum, View<const dd> lhs, int ls, bool conj_lhs, View<const dd> rhs, int rs,
             bool conj_rhs, bool cx, dd alpha_re, dd alpha_im);
void solve_lower_dd(cudaStream_t st, View<const dd> t, bool unit, bool conj, View<dd> rhs, bool cx);
void solve_upper_dd(cudaStream_t st, View<const dd> t, bool unit, bool conj, View<dd> rhs, bool cx);
// LLT / partial-pivoting LU drivers (dd_factor.cu); perm arrays: HOST int64 of A.nrows entries
template <bool CX>
LltResult llt_dd(cudaStream_t st, View<dd> A, dd delta, dd eps, size_t recursion_threshold, size_t block_size);
template <bool CX>
size_t lu_dd(cudaStream_t st, View<dd> A, size_t recursion_threshold, long long* perm_fwd, long long* perm_bwd);
// Householder QR (qr/no_pivoting/factor.rs:258-301; returns the rank) and block-Householder sequences (householder.rs:724-808:
// rhs <- Q rhs, or Q^H rhs with `transpose`; `conj` conjugates Q) (qr_dd.cu)
template <bool CX>
i64 qr_dd(cudaStream_t st, View<dd> A, View<dd> Q_coeff, i64 blocking_threshold);
template <bool CX>
void householder_sequence_dd(cudaStream_t st, View<const dd> basis, View<const dd> factor, bool conj, View<dd> rhs, bool transpose);
// self-adjoint EVD (evd/mod.rs:270-418) of the matrix whose lower triangle is A; U with no columns: values only; S: n entries in
// element units; false for non-finite input (evd_dd.cu)
template <bool CX>
bool self_adjoint_evd_dd(cudaStream_t st, View<const dd> A, View<dd> U, dd* S);
// divide and conquer of the real symmetric tridiagonal (d, e) of order n (device arrays): lam ascending, Z (n x n, ld n) its
// eigenvectors; false if a leaf did not converge (evd_dd.cu). Hidden, like svd_dd: the library exports only its C ABI additions.
__attribute__((visibility("hidden"))) bool tridiag_dc_dd(cudaStream_t st, const dd* d, const dd* e, i64 n, dd* lam, dd* Z);
// SVD (svd/mod.rs:530-672); U / V with ptr == nullptr or no columns: not computed (neither: values by bisection); U is
// nrows x {size, nrows}, V is ncols x {size, ncols}; S: min(m, n) entries in element units, non-increasing; false for non-finite
// input (svd_dd.cu)
template <bool CX>
__attribute__((visibility("hidden"))) bool svd_dd(cudaStream_t st, View<const dd> A, View<dd> U, dd* S, View<dd> V, double qr_ratio_threshold);

inline void gemm(cudaStream_t st, VD dst, int ds, int accum, VCD lhs, int ls, VCD rhs, int rs, double alpha) {
  gemm_f64(st, dst, ds, accum, lhs, ls, rhs, rs, alpha);
}
inline void gemm(cudaStream_t st, VF dst, int ds, int accum, VCF lhs, int ls, VCF rhs, int rs, float alpha) {
  gemm_f32(st, dst, ds, accum, lhs, ls, rhs, rs, alpha);
}
inline void solve_lower(cudaStream_t st, VCD t, bool unit, VD rhs) { solve_lower_triangular_in_place_f64(st, t, unit, rhs); }
inline void solve_lower(cudaStream_t st, VCF t, bool unit, VF rhs) { solve_lower_triangular_in_place_f32(st, t, unit, rhs); }
inline void solve_upper(cudaStream_t st, VCD t, bool unit, VD rhs) { solve_upper_triangular_in_place_f64(st, t, unit, rhs); }
inline void solve_upper(cudaStream_t st, VCF t, bool unit, VF rhs) { solve_upper_triangular_in_place_f32(st, t, unit, rhs); }

template <class T>
inline View<const T> cview(const View<T>& v) { return View<const T>{v.ptr, v.nrows, v.ncols, v.rs, v.cs}; }

// The same building blocks over the scalar kind <R, complex?>: <double, false> f64, <float, false> f32, <double, true> c64,
// <float, true> c32 (complex views in COMPLEX element units on an R* base). Real kinds ignore the conjugation flags and
// `alpha_im`.
template <class R, bool CX>
inline void gemm_t(cudaStream_t st, View<R> dst, int ds, int accum, View<const R> lhs, int ls, bool conj_lhs, View<const R> rhs,
                   int rs, bool conj_rhs, R alpha, R alpha_im = R(0)) {
  if constexpr (std::is_same_v<R, dd>) gemm_dd(st, dst, ds, accum, lhs, ls, conj_lhs, rhs, rs, conj_rhs, CX, alpha, alpha_im);
  else if constexpr (!CX) gemm(st, dst, ds, accum, lhs, ls, rhs, rs, alpha);
  else if constexpr (sizeof(R) == 8) gemm_c64(st, dst, ds, accum, lhs, ls, conj_lhs, rhs, rs, conj_rhs, alpha, alpha_im);
  else gemm_c32(st, dst, ds, accum, lhs, ls, conj_lhs, rhs, rs, conj_rhs, alpha, alpha_im);
}
template <class R, bool CX>
inline void solve_lower_t(cudaStream_t st, View<const R> t, bool unit, bool conj, View<R> rhs) {
  if constexpr (std::is_same_v<R, dd>) solve_lower_dd(st, t, unit, conj, rhs, CX);
  else if constexpr (!CX) solve_lower(st, t, unit, rhs);
  else if constexpr (sizeof(R) == 8) solve_lower_triangular_in_place_c64(st, t, unit, conj, rhs);
  else solve_lower_triangular_in_place_c32(st, t, unit, conj, rhs);
}
template <class R, bool CX>
inline void solve_upper_t(cudaStream_t st, View<const R> t, bool unit, bool conj, View<R> rhs) {
  if constexpr (std::is_same_v<R, dd>) solve_upper_dd(st, t, unit, conj, rhs, CX);
  else if constexpr (!CX) solve_upper(st, t, unit, rhs);
  else if constexpr (sizeof(R) == 8) solve_upper_triangular_in_place_c64(st, t, unit, conj, rhs);
  else solve_upper_triangular_in_place_c32(st, t, unit, conj, rhs);
}
// the m x n block at (i, j)
template <class R, bool CX>
inline View<R> sub_t(View<R> v, i64 i, i64 j, i64 m, i64 n) { return View<R>{v.ptr + (CX ? 2 : 1) * (i * v.rs + j * v.cs), m, n, v.rs, v.cs}; }
template <class R, bool CX>
inline View<const R> sub_t(View<const R> v, i64 i, i64 j, i64 m, i64 n) {
  return View<const R>{v.ptr + (CX ? 2 : 1) * (i * v.rs + j * v.cs), m, n, v.rs, v.cs};
}

// ---- householder.cu ----
// T(strict upper) <- V^H V for the N reflectors stored in V (m x N, implicit unit diagonal, R above it is ignored);
// the diagonal of Tf (the taus) is left untouched.  Reference: householder.rs:132-272 (upgrade_householder_factor)
template <class T>
void householder_build_t(cudaStream_t st, View<const T> V, View<T> Tf);
// M <- (I - V T^-1 V^H) M  (forward = false)   or   M <- (I - V T^-H V^H) M  (forward = true)
// Reference: householder.rs:370-620 (apply_block_householder_on_the_left_in_place_generic)
template <class T>
void apply_block_householder_on_the_left(cudaStream_t st, View<const T> V, View<const T> Tf, View<T> M, bool forward,
                                         T* tmp_buf = nullptr);

// sequences of block reflectors stored as (basis = V below the diagonal, factor = block_size x size T blocks)
// Reference: householder.rs:724-808
template <class T>
void apply_block_householder_sequence_on_the_left(cudaStream_t st, View<const T> basis, View<const T> factor, View<T> M);
template <class T>
void apply_block_householder_sequence_transpose_on_the_left(cudaStream_t st, View<const T> basis, View<const T> factor,
                                                            View<T> M);
// cplx.cu: T(strict upper) <- V^H V for complex reflectors (upgrade_householder_factor with prev_block_size 1; views in COMPLEX
// element units on an R* base), the twin of householder_build_t
template <class R>
void householder_build_t_cx(cudaStream_t st, View<const R> V, View<R> Tf);
// rhs[i, :] <- rhs[perm[i], :] for every scalar kind (perm: HOST int64 of rhs.nrows entries; reconstruct_types.cu); a column
// permutation is this on the transposed view
template <class R, bool CX>
void permute_rows_t(cudaStream_t st, View<R> rhs, const long long* perm);

// ---- the compositions on the factors, over the scalar kind <R, CX> ----
// rhs <- conj?(L L^H)^-1 rhs (llt/solve.rs:12-35): L y = rhs, then L^H x = y
template <class R, bool CX>
inline void llt_solve_t(cudaStream_t st, View<const R> L, bool conj, View<R> rhs) {
  solve_lower_t<R, CX>(st, L, false, conj, rhs);
  solve_upper_t<R, CX>(st, L.t(), false, CX && !conj, rhs);
}
// transpose = false: rhs <- conj?(A)^-1 rhs with perm = perm_fwd (lu/partial_pivoting/solve.rs:21-54); true: conj?(A)^-T rhs with
// perm = perm_bwd (solve.rs:55-86). perm: HOST int64 of rhs.nrows entries
template <class R, bool CX>
inline void lu_solve_t(cudaStream_t st, View<const R> L, View<const R> U, bool conj, const long long* perm, View<R> rhs, bool transpose) {
  if (!transpose) {
    permute_rows_t<R, CX>(st, rhs, perm);
    solve_lower_t<R, CX>(st, L, true, conj, rhs);
    solve_upper_t<R, CX>(st, U, false, conj, rhs);
  } else {
    solve_lower_t<R, CX>(st, U.t(), false, conj, rhs);
    solve_upper_t<R, CX>(st, L.t(), true, conj, rhs);
    permute_rows_t<R, CX>(st, rhs, perm);
  }
}
// rhs <- Q rhs (transpose = false) or Q^H rhs (true), Q conjugated under `conj` (householder.rs:724-808); real kinds ignore `conj`
template <class R, bool CX>
inline void householder_sequence_t(cudaStream_t st, View<const R> basis, View<const R> factor, bool conj, View<R> rhs, bool transpose) {
  if constexpr (std::is_same_v<R, dd>) householder_sequence_dd<CX>(st, basis, factor, CX && conj, rhs, transpose);
  else if constexpr (!CX) {
    if (transpose) apply_block_householder_sequence_transpose_on_the_left<R>(st, basis, factor, rhs);
    else apply_block_householder_sequence_on_the_left<R>(st, basis, factor, rhs);
  } else if constexpr (sizeof(R) == 8) apply_householder_sequence_left_c64(st, basis, factor, conj, rhs, transpose);
  else apply_householder_sequence_left_c32(st, basis, factor, conj, rhs, transpose);
}
// T(strict upper) <- V^H V for the reflectors stored in V, for the IEEE kinds
template <class R, bool CX>
inline void householder_factor_t(cudaStream_t st, View<const R> V, View<R> Tf) {
  if constexpr (CX) householder_build_t_cx<R>(st, V, Tf);
  else householder_build_t<R>(st, V, Tf);
}

// ---- qr.cu ----
// Householder QR without pivoting, reference qr/no_pivoting/factor.rs:258-301. H: block_size x min(m, n).
// Returns the rank (dependent columns are skipped and the reflectors compacted as factor.rs:40-83 does).
template <class T>
i64 qr_in_place(cudaStream_t st, View<T> A, View<T> H);
i64 qr_recommended_block_size(i64 nrows, i64 ncols);

// ---- bidiag.cu ----
// A = U B V^H, m >= n, column-major A. Reference: svd/bidiag.rs:47-256. Hl: bl x n, Hr: br x (n-1) (T blocks).
template <class T>
void bidiag_in_place(cudaStream_t st, View<T> A, View<T> Hl, View<T> Hr);
// ---- evd.cu ----
// S (device, compact, n entries) <- eigenvalues (nondecreasing) of the self-adjoint matrix whose lower triangle is in A
// (evd/mod.rs:270-353 with u = None)
// returns false if the tridiagonal form is not finite (EvdError::NoConvergence in the reference)
template <class T>
bool self_adjoint_eigenvalues(cudaStream_t st, View<const T> A, T* S);
// ---- svd.cu ----
// S (device, compact, min(m, n) entries) <- the singular values of A, non-increasing (svd/mod.rs:530-648 with u = v = None)
// qr_ratio_threshold: SvdParams::qr_ratio_threshold (11/6): taller inputs go through QR first
// returns false if the bidiagonal form is not finite (SvdError::NoConvergence, svd/mod.rs:282-286)
template <class T>
bool singular_values(cudaStream_t st, View<const T> A, T* S, double qr_ratio_threshold);
// ---- svd_vectors.cu: decompositions WITH vectors (f64 arithmetic), false on non-finite input ----
template <class TA>
bool svd_with_vectors(cudaStream_t st, View<const TA> A, View<TA> U, TA* S, i64 sstride, View<TA> V, double qr_ratio_threshold);
template <class TA>
bool self_adjoint_evd_with_vectors(cudaStream_t st, View<const TA> A, View<TA> U, TA* S, i64 sstride);
template <class T>
bool device_all_finite(cudaStream_t st, const T* x, i64 n);
// SVD of the real upper-bidiagonal (d, e) of order n (device arrays; e has n entries, the last one unused): S_sorted
// non-increasing, UB / VB n x n column-major (ld n) with B = UB diag(S) VB^T. False on non-finite input.
bool bidiag_svd_vectors_f64(cudaStream_t st, const double* d, const double* e, i64 n, double* S_sorted, double* UB, double* VB);
// ---- cplx_condensed.cu: `svd` / `self_adjoint_evd` for complex T (TO = double: c64, float: c32 computed in c64); views in
// COMPLEX element units on a TO* base; U / V with ptr == nullptr or ncols == 0: not computed; S: (value, 0) pairs `sstride`
// complex elements apart (device). False on non-finite input. ----
template <class TO>
bool svd_cx(cudaStream_t st, View<const TO> A, View<TO> U, TO* S, i64 sstride, View<TO> V);
template <class TO>
bool self_adjoint_evd_cx(cudaStream_t st, View<const TO> A, View<TO> U, TO* S, i64 sstride);
// complex bidiagonalization / tridiagonalization with T blocks (TO = double: c64, float: c32 computed in c64; complex-unit views)
template <class TO>
void bidiag_in_place_cx(cudaStream_t st, View<TO> A, View<TO> Hl, View<TO> Hr);
template <class TO>
void tridiag_in_place_cx(cudaStream_t st, View<TO> A, View<TO> H);
// A <- upper Hessenberg form + reflectors, Hf (bs x (n - 1)) <- T blocks (evd/hessenberg.rs:549-567); <TO, complex?>: <double, false> f64,
// <float, false> f32, <double, true> c64, <float, true> c32 (complex views in complex units)
template <class TO, bool CX>
void hessenberg_in_place_t(cudaStream_t st, View<TO> A, View<TO> Hf);
// ---- schur.cu: general eigendecomposition (evd/mod.rs:1007-1246). <TO, complex?> as above; UL / UR with ptr == nullptr: not
// computed; S / S_im: device, compact, n entries of TO's kind (S_im: real kinds only). ns_limit bounds the shifts of a sweep. False
// on a non-finite input (nothing written) or when the iteration cap is reached. ----
template <class TO, bool CX>
bool evd_general(cudaStream_t st, View<const TO> A, View<TO> UL, View<TO> UR, TO* S, TO* S_im, size_t ns_limit);
// sweeps and chased windows of the last evd_general call (tools/time_evd.py)
extern long long g_evd_last_sweeps, g_evd_last_windows;
// ---- tridiag_dc.cu: divide-and-conquer eigensolver of a symmetric tridiagonal matrix (device arrays) ----
bool tridiag_dc_f64(cudaStream_t st, const double* d, const double* e, i64 n, double* lam, double* Q, i64 ldq);
// ---- tridiag.cu ----
// A = Q T Q^H, self-adjoint A (lower triangle), column-major. Reference: evd/tridiag.rs:274-529. H: b x (n-1).
template <class T>
void tridiag_in_place(cudaStream_t st, View<T> A, View<T> H);

// ---- reconstruct_types.cu: `*_reconstruct` / `*_inverse` on the factors for every scalar kind; complex views in COMPLEX element
// units on an R* base; perm arrays HOST int64 ----
template <class R, bool CX>
void llt_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L);
template <class R, bool CX>
void llt_inverse_t(cudaStream_t st, View<R> out, View<const R> L);
template <class R, bool CX>
void lu_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L, View<const R> U, const long long* perm_bwd_host);
template <class R, bool CX>
void lu_inverse_t(cudaStream_t st, View<R> out, View<const R> L, View<const R> U, const long long* perm_fwd_host);
template <class R, bool CX>
void qr_reconstruct_t(cudaStream_t st, View<R> out, View<const R> Q_basis, View<const R> Q_coeff, View<const R> Rm);
template <class R, bool CX>
void qr_inverse_t(cudaStream_t st, View<R> out, View<const R> Q_basis, View<const R> Q_coeff, View<const R> Rm);

// out[i, j] <- src[p[i], q[j]] for every scalar kind (p, q: HOST int64 of out.nrows / out.ncols entries; out and src must not
// overlap); the permuted 2-D gather of the full-pivoting LU reconstruct / inverse
template <class R, bool CX>
void gather_2d_t(cudaStream_t st, View<R> out, View<const R> src, const long long* p, const long long* q);

// dst(triangle) <- src(triangle)^-1 (triangular_inverse.rs), every scalar kind; only the triangle is written (not the diagonal if unit)
template <class R, bool CX>
void inverse_triangular_t(cudaStream_t st, View<R> dst, View<const R> src, bool lower, bool unit);
// ---- ldlt_types.cu: LDLT beyond the f64 factorization, over the scalar kind <R, complex?> (complex views in COMPLEX element units
// on an R* base). Factor / solve: <float, false>, <double, true>, <float, true>; reconstruct / inverse: also <double, false>.
// D: DEVICE pointer to T-typed entries `dstride` elements apart; d_signs: device int8[n] or null ----
template <class R, bool CX>
LdltResult ldlt_in_place_t(cudaStream_t st, View<R> A, R delta, R eps, const signed char* d_signs);
template <class R, bool CX>
void ldlt_solve_in_place_t(cudaStream_t st, View<const R> L, const R* D, i64 dstride, bool conj, View<R> rhs);
template <class R, bool CX>
void ldlt_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L, const R* D, i64 dstride);
template <class R, bool CX>
void ldlt_inverse_t(cudaStream_t st, View<R> out, View<const R> L, const R* D, i64 dstride);

}  // namespace fb
