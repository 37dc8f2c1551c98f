// `*_reconstruct` / `*_inverse` on the factors for every scalar kind, written once over the scalar kind <R, CX> (R = real type,
// CX = interleaved complex): the structured product, the triangular solves, the LU solve, the row permutation and the
// block-Householder sequence of that scalar kind — every one of them already on the hot path and validated on its own.
// Complex views are in COMPLEX element units on an R* base (the convention of gemm_c64 / cplx.cu).
// Reference:
//   cholesky/llt/reconstruct.rs:12-33   out(lower) = L(lower) * L^H(upper)            (only the lower triangle is written)
//   cholesky/llt/inverse.rs:10-39       L_inv = L^-1 (lower), out(lower) = L_inv^H(upper) * L_inv(lower)
//   lu/partial_pivoting/reconstruct.rs:12-80   tmp = L U by structured products (square / tall / wide parts), out = P^-1 tmp
//   lu/partial_pivoting/inverse.rs:11-49       A^-1 from the factors; here as the LU solve applied to the identity
//   qr/no_pivoting/reconstruct.rs:13-39 out = [R; 0], then out <- Q out (sequence on the left, Conj::No)
//   qr/no_pivoting/inverse.rs:11-43     A^-1 = R^-1 Q^H; here as the QR solve applied to the identity (Q^H first, then R^-1)
// Tests: tests/test_gpu_zz4_reconstruct_inverse.py (f64), tests/test_gpu_zzzzzzzzz_2_reconstruct_types.py.
#include <algorithm>

#if defined(__CUDACC__)
#include "dd.cuh"
#endif
#include "flat_map.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

// Flat-map bodies (flat_map.cuh). W = 1 (real) or 2 (interleaved complex) R values per element; strides in elements.
#if defined(__CUDACC__)
#define RT_HD __host__ __device__ __forceinline__
#else
#define RT_HD inline
#endif
template <class R, int W>
struct RtSetIdentity {
  R* A; i64 rs, cs, n;
  RT_HD void operator()(i64 i, i64 j) const {
    if (i >= n || j >= n) return;
    R* p = A + W * (i * rs + j * cs);
    p[0] = i == j ? R(1) : R(0);
    if (W == 2) p[W - 1] = R(0);
  }
};
// out (m x n) <- upper trapezoid of Rm (size x n) in its first `size` rows, zero elsewhere
template <class R, int W>
struct RtSetUpperTrapezoid {
  R* out; i64 o_rs, o_cs, m, n; const R* Rm; i64 r_rs, r_cs, size;
  RT_HD void operator()(i64 i, i64 j) const {
    if (i >= m || j >= n) return;
    R* p = out + W * (i * o_rs + j * o_cs);
    const bool take = i < size && i <= j;
    const R* q = Rm + W * (i * r_rs + j * r_cs);
    p[0] = take ? q[0] : R(0);
    if (W == 2) p[W - 1] = take ? q[W - 1] : R(0);
  }
};
// tmp (compact column-major, ld = nrows) [i, c] = src[perm[i], c]
template <class R, int W>
struct RtGatherRows {
  R* tmp; const R* src; i64 rs, cs, nrows, ncols; const long long* perm;
  RT_HD void operator()(i64 i, i64 c) const {
    if (i >= nrows || c >= ncols) return;
    const R* q = src + W * (perm[i] * rs + c * cs);
    R* p = tmp + W * (c * nrows + i);
    p[0] = q[0];
    if (W == 2) p[W - 1] = q[W - 1];
  }
};
template <class R, int W>
struct RtScatterBack {
  R* dst; i64 rs, cs; const R* tmp; i64 nrows, ncols;
  RT_HD void operator()(i64 i, i64 c) const {
    if (i >= nrows || c >= ncols) return;
    const R* q = tmp + W * (c * nrows + i);
    R* p = dst + W * (i * rs + c * cs);
    p[0] = q[0];
    if (W == 2) p[W - 1] = q[W - 1];
  }
};

// out[i, j] = src[p[i], q[j]]
template <class R, int W>
struct RtGather2d {
  R* out; i64 o_rs, o_cs; const R* src; i64 s_rs, s_cs, m, n; const long long* p; const long long* q;
  RT_HD void operator()(i64 i, i64 j) const {
    if (i >= m || j >= n) return;
    const R* s = src + W * (p[i] * s_rs + q[j] * s_cs);
    R* d = out + W * (i * o_rs + j * o_cs);
    d[0] = s[0];
    if (W == 2) d[W - 1] = s[W - 1];
  }
};

// dst(i, j) = src(i, j) on the triangle `lower` selects — diagonal included unless `unit` — and nothing elsewhere
template <class R, int W>
struct RtCopyTriangle {
  R* dst; i64 d_rs, d_cs; const R* src; i64 s_rs, s_cs, n; int lower, unit;
  RT_HD void operator()(i64 i, i64 j) const {
    if (i >= n || j >= n) return;
    const bool in = lower ? (unit ? i > j : i >= j) : (unit ? i < j : i <= j);
    if (!in) return;
    const R* q = src + W * (i * s_rs + j * s_cs);
    R* p = dst + W * (i * d_rs + j * d_cs);
    p[0] = q[0];
    if (W == 2) p[W - 1] = q[W - 1];
  }
};

// A <- the n x n identity
template <class R, bool CX>
void set_identity(cudaStream_t st, View<R> A) {
  const i64 n = A.nrows;
  DevRun run{st};
  run(RtSetIdentity<R, CX ? 2 : 1>{A.ptr, A.rs, A.cs, n}, n, n);
}

}  // namespace

template <class R, bool CX>
void llt_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L) {
  const i64 n = out.nrows;
  FB_ASSERT(out.ncols == n && L.nrows == n && L.ncols == n, "llt_reconstruct shape mismatch");
  if (n == 0) return;
  gemm_t<R, CX>(st, out, TRI_LOWER, 0, L, TRI_LOWER, false, L.t(), TRI_UPPER, true, R(1));  // L * adjoint(L)
}

template <class R, bool CX>
void llt_inverse_t(cudaStream_t st, View<R> out, View<const R> L) {
  const i64 n = out.nrows;
  FB_ASSERT(out.ncols == n && L.nrows == n && L.ncols == n, "llt_inverse shape mismatch");
  if (n == 0) return;
  constexpr int W = CX ? 2 : 1;
  R* buf = (R*)ws_alloc((size_t)n * (size_t)n * W * sizeof(R));
  View<R> Li{buf, n, n, 1, n};
  set_identity<R, CX>(st, Li);
  solve_lower_t<R, CX>(st, L, false, false, Li);  // L_inv: lower triangular, exact zeros above the diagonal
  gemm_t<R, CX>(st, out, TRI_LOWER, 0, cview(Li).t(), TRI_UPPER, true, cview(Li), TRI_LOWER, false, R(1));  // adjoint(L_inv) * L_inv
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(buf);
}

// perm_bwd: HOST int64[m], the inverse row permutation
template <class R, bool CX>
void lu_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L, View<const R> U, const long long* perm_bwd) {
  const i64 m = L.nrows, n = U.ncols, size = std::min(m, n);
  FB_ASSERT(out.nrows == m && out.ncols == n && L.ncols >= size && U.nrows >= size, "lu_reconstruct shape mismatch");
  if (m == 0 || n == 0) return;
  const View<const R> Ls = sub_t<R, CX>(L, 0, 0, size, size), Us = sub_t<R, CX>(U, 0, 0, size, size);
  gemm_t<R, CX>(st, sub_t<R, CX>(out, 0, 0, size, size), RECT, 0, Ls, UNIT_LOWER, false, Us, TRI_UPPER, false, R(1));
  if (m > n)
    gemm_t<R, CX>(st, sub_t<R, CX>(out, size, 0, m - size, size), RECT, 0, sub_t<R, CX>(L, size, 0, m - size, size), RECT, false, Us,
                  TRI_UPPER, false, R(1));
  if (m < n)
    gemm_t<R, CX>(st, sub_t<R, CX>(out, 0, size, size, n - size), RECT, 0, Ls, UNIT_LOWER, false, sub_t<R, CX>(U, 0, size, size, n - size),
                  RECT, false, R(1));
  // (P A)[i, :] = A[perm_fwd[i], :]  =>  A[j, :] = (L U)[perm_bwd[j], :]
  permute_rows_t<R, CX>(st, out, perm_bwd);
}

template <class R, bool CX>
void lu_inverse_t(cudaStream_t st, View<R> out, View<const R> L, View<const R> U, const long long* perm_fwd) {
  const i64 n = out.nrows;
  FB_ASSERT(out.ncols == n && L.nrows == n && L.ncols == n && U.nrows == n && U.ncols == n, "lu_inverse shape mismatch");
  if (n == 0) return;
  set_identity<R, CX>(st, out);
  lu_solve_t<R, CX>(st, L, U, false, perm_fwd, out, false);
}

template <class R, bool CX>
void qr_reconstruct_t(cudaStream_t st, View<R> out, View<const R> Qb, View<const R> Qc, View<const R> Rm) {
  const i64 m = Qb.nrows, n = Rm.ncols, size = std::min(m, n);
  FB_ASSERT(out.nrows == m && out.ncols == n && Qb.ncols == size && Qc.nrows > 0 && Qc.ncols == size && Rm.nrows == size,
            "qr_reconstruct shape mismatch");
  if (m == 0 || n == 0) return;
  DevRun run{st};
  run(RtSetUpperTrapezoid<R, CX ? 2 : 1>{out.ptr, out.rs, out.cs, m, n, Rm.ptr, Rm.rs, Rm.cs, size}, m, n);
  if (size > 0) householder_sequence_t<R, CX>(st, Qb, Qc, false, out, false);
}

template <class R, bool CX>
void qr_inverse_t(cudaStream_t st, View<R> out, View<const R> Qb, View<const R> Qc, View<const R> Rm) {
  const i64 n = out.nrows;
  FB_ASSERT(out.ncols == n && Qb.nrows == n && Qb.ncols == n && Qc.nrows > 0 && Qc.ncols == n && Rm.nrows == n && Rm.ncols == n,
            "qr_inverse shape mismatch");
  if (n == 0) return;
  set_identity<R, CX>(st, out);
  householder_sequence_t<R, CX>(st, Qb, Qc, true, out, true);  // Q^H
  solve_upper_t<R, CX>(st, Rm, false, false, out);  // R^-1 Q^H
}

// linalg::triangular_inverse::invert_[unit_]{lower,upper}_triangular (triangular_inverse.rs): dst(triangle) <- src(triangle)^-1;
// only the triangle is written (the diagonal too unless `unit`). Here as the triangular solve applied to the identity.
template <class R, bool CX>
void inverse_triangular_t(cudaStream_t st, View<R> dst, View<const R> src, bool lower, bool unit) {
  const i64 n = dst.nrows;
  FB_ASSERT(dst.ncols == n && src.nrows == n && src.ncols == n, "inverse_triangular shape mismatch");
  if (n == 0) return;
  constexpr int W = CX ? 2 : 1;
  R* buf = (R*)ws_alloc((size_t)n * (size_t)n * W * sizeof(R));
  View<R> X{buf, n, n, 1, n};
  set_identity<R, CX>(st, X);
  if (lower) solve_lower_t<R, CX>(st, src, unit, false, X);
  else solve_upper_t<R, CX>(st, src, unit, false, X);
  DevRun run{st};
  run(RtCopyTriangle<R, W>{dst.ptr, dst.rs, dst.cs, buf, 1, n, n, lower ? 1 : 0, unit ? 1 : 0}, n, n);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(buf);
}
template void inverse_triangular_t<double, false>(cudaStream_t, View<double>, View<const double>, bool, bool);
template void inverse_triangular_t<float, false>(cudaStream_t, View<float>, View<const float>, bool, bool);
template void inverse_triangular_t<double, true>(cudaStream_t, View<double>, View<const double>, bool, bool);
template void inverse_triangular_t<float, true>(cudaStream_t, View<float>, View<const float>, bool, bool);
#if defined(__CUDACC__)  // the host builds of this file (tools/emul) provide building blocks for the four other kinds only
template void inverse_triangular_t<dd, false>(cudaStream_t, View<dd>, View<const dd>, bool, bool);
template void inverse_triangular_t<dd, true>(cudaStream_t, View<dd>, View<const dd>, bool, bool);
#endif

#define FB_RECON_INST(R, CX)                                                                                                     \
  template void llt_reconstruct_t<R, CX>(cudaStream_t, View<R>, View<const R>);                                                  \
  template void llt_inverse_t<R, CX>(cudaStream_t, View<R>, View<const R>);                                                      \
  template void lu_reconstruct_t<R, CX>(cudaStream_t, View<R>, View<const R>, View<const R>, const long long*);                  \
  template void lu_inverse_t<R, CX>(cudaStream_t, View<R>, View<const R>, View<const R>, const long long*);                      \
  template void qr_reconstruct_t<R, CX>(cudaStream_t, View<R>, View<const R>, View<const R>, View<const R>);                     \
  template void qr_inverse_t<R, CX>(cudaStream_t, View<R>, View<const R>, View<const R>, View<const R>);
FB_RECON_INST(double, false)
FB_RECON_INST(float, false)
FB_RECON_INST(double, true)
FB_RECON_INST(float, true)
#undef FB_RECON_INST
#if defined(__CUDACC__)  // double-double: the LLT, LU and QR compositions
#define FB_RECON_INST_DD(CX)                                                                                                     \
  template void llt_reconstruct_t<dd, CX>(cudaStream_t, View<dd>, View<const dd>);                                               \
  template void llt_inverse_t<dd, CX>(cudaStream_t, View<dd>, View<const dd>);                                                   \
  template void lu_reconstruct_t<dd, CX>(cudaStream_t, View<dd>, View<const dd>, View<const dd>, const long long*);              \
  template void lu_inverse_t<dd, CX>(cudaStream_t, View<dd>, View<const dd>, View<const dd>, const long long*);                  \
  template void qr_reconstruct_t<dd, CX>(cudaStream_t, View<dd>, View<const dd>, View<const dd>, View<const dd>);                \
  template void qr_inverse_t<dd, CX>(cudaStream_t, View<dd>, View<const dd>, View<const dd>, View<const dd>);
FB_RECON_INST_DD(false)
FB_RECON_INST_DD(true)
#undef FB_RECON_INST_DD
#endif

template <class R, bool CX>
void permute_rows_t(cudaStream_t st, View<R> rhs, const long long* perm) {
  constexpr int W = CX ? 2 : 1;
  const i64 n = rhs.nrows, k = rhs.ncols;
  if (n == 0 || k == 0) return;
  long long* d_perm = (long long*)ws_alloc((size_t)n * 8);
  R* tmp = (R*)ws_alloc((size_t)n * (size_t)k * W * sizeof(R));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_perm, perm, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  DevRun run{st};
  run(RtGatherRows<R, W>{tmp, rhs.ptr, rhs.rs, rhs.cs, n, k, d_perm}, n, k);
  run(RtScatterBack<R, W>{rhs.ptr, rhs.rs, rhs.cs, tmp, n, k}, n, k);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));  // perm (host, pageable) and the pool buffers are released below
  ws_free(tmp);
  ws_free(d_perm);
}
template void permute_rows_t<double, false>(cudaStream_t, View<double>, const long long*);
template void permute_rows_t<float, false>(cudaStream_t, View<float>, const long long*);
template void permute_rows_t<double, true>(cudaStream_t, View<double>, const long long*);
template void permute_rows_t<float, true>(cudaStream_t, View<float>, const long long*);
#if defined(__CUDACC__)
template void permute_rows_t<dd, false>(cudaStream_t, View<dd>, const long long*);
template void permute_rows_t<dd, true>(cudaStream_t, View<dd>, const long long*);
#endif

template <class R, bool CX>
void gather_2d_t(cudaStream_t st, View<R> out, View<const R> src, const long long* p, const long long* q) {
  constexpr int W = CX ? 2 : 1;
  const i64 m = out.nrows, n = out.ncols;
  if (m == 0 || n == 0) return;
  long long* d_p = (long long*)ws_alloc((size_t)(m + n) * 8);
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p, p, (size_t)m * 8, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p + m, q, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  DevRun run{st};
  run(RtGather2d<R, W>{out.ptr, out.rs, out.cs, src.ptr, src.rs, src.cs, m, n, d_p, d_p + m}, m, n);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));  // p / q (host, pageable) and the pool buffer are released by the caller / below
  ws_free(d_p);
}
template void gather_2d_t<double, false>(cudaStream_t, View<double>, View<const double>, const long long*, const long long*);
template void gather_2d_t<float, false>(cudaStream_t, View<float>, View<const float>, const long long*, const long long*);
template void gather_2d_t<double, true>(cudaStream_t, View<double>, View<const double>, const long long*, const long long*);
template void gather_2d_t<float, true>(cudaStream_t, View<float>, View<const float>, const long long*, const long long*);

}  // namespace fb
