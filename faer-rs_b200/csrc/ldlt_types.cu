// LDLT without pivoting beyond the f64 factorization (which stays on the tuned kernels of ldlt_f64.cu): factor / solve for f32, c64
// and c32, `reconstruct` / `inverse` for all four dtypes, written once over the scalar kind <R, CX>.
//
// Reference:
//   cholesky/ldlt/factor.rs:725-767      driver (D on the diagonal, unit-lower L strictly below, strict upper triangle untouched,
//                                        ZeroPivot { index }), leaf recurrence 299-366, dynamic regularisation 122-144
//   cholesky/ldlt/solve.rs:11-49         unit-lower solve with conj?(L), rows scaled by 1 / Re d_i, unit-upper solve with L^T under the
//                                        conjugation composed with Yes
//   cholesky/ldlt/reconstruct.rs:9-55    out(lower) = (L D)(lower) * L^H(unit upper)
//   cholesky/ldlt/inverse.rs:9-60        M = L^-1; the upper triangle filled with conj(M(i, j)) / d_i and the diagonal with 1 / d_j;
//                                        out(lower) = M(upper) * M(unit lower)
// The factorization is the unblocked right-looking launch sequence of ldlt_core.cuh (flat maps; the same source runs thread by thread
// on the host in tests/test_ldlt_types_emul_cpu.py): functional, not tuned — three launches per column, the trailing update one
// thread per element instead of a GEMM. Solve / reconstruct / inverse are compositions of the structured products and triangular
// solves of each scalar kind with the small bodies of ldlt_core.cuh in between.
#include "flat_map.cuh"
#include "ldlt_core.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

// In-place LDLT of the lower triangle of A (device view, strides in elements). d_signs: device int8[n] or null.
template <class R, bool CX>
LdltResult ldlt_in_place_t(cudaStream_t st, View<R> A, R delta, R eps, const signed char* d_signs) {
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n, "LDLT needs a square matrix");
  LdltResult res{true, 0, 0};
  if (n == 0) return res;
  constexpr int W = CX ? 2 : 1;
  i64* info = (i64*)ws_alloc(2 * sizeof(i64));
  R* D = (R*)ws_alloc((size_t)n * sizeof(R));
  R* sc = (R*)ws_alloc(4 * sizeof(R));
  R* w = (R*)ws_alloc((size_t)n * W * sizeof(R));
  const i64 init[2] = {-1, 0};
  FB_CUDA_CHECK(cudaMemcpyAsync(info, init, sizeof(init), cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemsetAsync(D, 0, (size_t)n * sizeof(R), st));
  DevRun run{st};
  ldl::factor_unblocked<R, CX>(run, A.ptr, A.rs, A.cs, n, D, d_signs, delta, eps, info, sc, w);
  i64 h[2] = {-1, 0};
  FB_CUDA_CHECK(cudaMemcpyAsync(h, info, sizeof(h), cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(w);
  ws_free(sc);
  ws_free(D);
  ws_free(info);
  if (h[0] >= 0) {
    res.ok = false;
    res.zero_pivot_index = (size_t)h[0];
  } else {
    res.dynamic_regularization_count = (size_t)h[1];
  }
  return res;
}

// rhs <- conj?(A)^-1 rhs from the factors; D: device pointer to T-typed entries `dstride` elements apart (the real parts are used)
template <class R, bool CX>
void ldlt_solve_in_place_t(cudaStream_t st, View<const R> L, const R* D, i64 dstride, bool conj, View<R> rhs) {
  const i64 n = L.nrows, k = rhs.ncols;
  FB_ASSERT(L.ncols == n && rhs.nrows == n, "LDLT solve shape mismatch");
  if (n == 0 || k == 0) return;
  DevRun run{st};
  R* dinv = (R*)ws_alloc((size_t)n * sizeof(R));
  run(ldl::RecipDiag<R, CX>{D, dstride, n, dinv}, n, 1);
  solve_lower_t<R, CX>(st, L, true, conj, rhs);
  run(ldl::ScaleRows<R, CX>{rhs.ptr, rhs.rs, rhs.cs, n, k, dinv}, n, k);
  solve_upper_t<R, CX>(st, L.t(), true, !conj, rhs);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(dinv);
}

template <class R, bool CX>
void ldlt_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L, const R* D, i64 dstride) {
  const i64 n = out.nrows;
  FB_ASSERT(out.ncols == n && L.nrows == n && L.ncols == n, "ldlt_reconstruct shape mismatch");
  if (n == 0) return;
  constexpr int W = CX ? 2 : 1;
  DevRun run{st};
  R* buf = (R*)ws_alloc((size_t)n * (size_t)n * W * sizeof(R));
  run(ldl::BuildLxD<R, CX>{L.ptr, L.rs, L.cs, D, dstride, buf, n, n}, n, n);
  gemm_t<R, CX>(st, out, TRI_LOWER, 0, View<const R>{buf, n, n, 1, n}, TRI_LOWER, false, L.t(), UNIT_UPPER, true, R(1));  // (L D) * adjoint(L)
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(buf);
}

template <class R, bool CX>
void ldlt_inverse_t(cudaStream_t st, View<R> out, View<const R> L, const R* D, i64 dstride) {
  const i64 n = out.nrows;
  FB_ASSERT(out.ncols == n && L.nrows == n && L.ncols == n, "ldlt_inverse shape mismatch");
  if (n == 0) return;
  constexpr int W = CX ? 2 : 1;
  DevRun run{st};
  R* buf = (R*)ws_alloc((size_t)n * (size_t)n * W * sizeof(R));
  R* dinv = (R*)ws_alloc((size_t)n * sizeof(R));
  View<R> M{buf, n, n, 1, n};
  run(ldl::SetIdentity<R, CX>{buf, n, n}, n, n);
  solve_lower_t<R, CX>(st, L, true, false, M);  // M = L^-1: unit lower, exact zeros above the diagonal
  run(ldl::RecipDiag<R, CX>{D, dstride, n, dinv}, n, 1);
  run(ldl::FillUpperAdjoint<R, CX>{buf, n, n, dinv}, n, n);
  const View<const R> Mc{buf, n, n, 1, n};
  gemm_t<R, CX>(st, out, TRI_LOWER, 0, Mc, TRI_UPPER, false, Mc, UNIT_LOWER, false, R(1));  // (M^H D^-1) * M
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(dinv);
  ws_free(buf);
}

#define FB_LDLT_INST_FS(R, CX)                                                                                  \
  template LdltResult ldlt_in_place_t<R, CX>(cudaStream_t, View<R>, R, R, const signed char*);                   \
  template void ldlt_solve_in_place_t<R, CX>(cudaStream_t, View<const R>, const R*, i64, bool, View<R>);
#define FB_LDLT_INST_RI(R, CX)                                                                                  \
  template void ldlt_reconstruct_t<R, CX>(cudaStream_t, View<R>, View<const R>, const R*, i64);                  \
  template void ldlt_inverse_t<R, CX>(cudaStream_t, View<R>, View<const R>, const R*, i64);
FB_LDLT_INST_FS(float, false)
FB_LDLT_INST_FS(double, true)
FB_LDLT_INST_FS(float, true)
FB_LDLT_INST_RI(double, false)
FB_LDLT_INST_RI(float, false)
FB_LDLT_INST_RI(double, true)
FB_LDLT_INST_RI(float, true)
#undef FB_LDLT_INST_FS
#undef FB_LDLT_INST_RI

}  // namespace fb
