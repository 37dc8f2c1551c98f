// Double-double (fx128 / cx128) triangular solves, LLT and partial-pivoting LU: the reference's recursions on the host with every
// off-diagonal product on the dd GEMM (gemm_dd.cu), and single-CTA leaf kernels for the diagonal blocks. Views are in elements
// (complex units on a dd* base for cx128); CX selects the kind.
//   triangular_solve.rs      split in halves down to DL_LEAF rows; leaf: one thread per right-hand side column
//   cholesky/llt/factor.rs   cholesky_recursion_right_looking (ldlt/factor.rs:367-498) with the params' recursion_threshold /
//                            block_size; leaf (ldlt/factor.rs:7-177): regularisation, !(d > 0) and the sqrt test decide failure,
//                            the whole column, diagonal included, is scaled by recip(sqrt(d))
//   lu/partial_pivoting      lu_in_place_recursion (factor.rs:68-187) with the params' recursion_threshold; leaf
//                            (lu_in_place_unblocked 19-67): first row attaining the maximum abs1, row swap, scaling by recip
// The leaves perform the scalar operations of the reference's loops in the reference's order, in dd arithmetic (dd.cuh); the row
// swaps of the LU are applied to every column of the matrix as soon as they are chosen, which is the reference's end state (the
// columns a level does not touch receive the same swaps in the same order when that level ends).
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "dd.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

constexpr int DL_LEAF = 32;
constexpr int DL_THREADS = 1024;

template <bool CX>
__device__ __forceinline__ cdd dl_ld(const dd* p, i64 off) {
  return CX ? cdd{p[2 * off], p[2 * off + 1]} : cdd{p[off], dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ void dl_st(dd* p, i64 off, cdd v) {
  if (CX) {
    p[2 * off] = v.re;
    p[2 * off + 1] = v.im;
  } else {
    p[off] = v.re;
  }
}
template <bool CX>
__device__ __forceinline__ cdd dl_mul(cdd a, cdd b) {
  return CX ? a * b : cdd{a.re * b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd dl_add(cdd a, cdd b) {
  return CX ? a + b : cdd{a.re + b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd dl_recip(cdd a) {
  return CX ? cdd_recip(a) : cdd{dd_recip(a.re), dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ dd dl_abs1(cdd a) {
  return CX ? cdd_abs1(a) : fabs(a.re);
}

// ---- triangular solve leaf: rhs <- conj?(L)^-1 rhs for a lower L of at most DL_LEAF rows; one thread per rhs column ----
template <bool CX>
__global__ void __launch_bounds__(128) dd_trsm_leaf_kernel(View<const dd> L, bool unit, bool conj, View<dd> rhs) {
  __shared__ cdd Ls[DL_LEAF][DL_LEAF];
  const int n = (int)L.nrows;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e % n, k = e / n;
    if (k > i) continue;
    cdd v = dl_ld<CX>(L.ptr, i * L.rs + k * L.cs);
    if (conj) v = cdd_conj(v);
    // the complex reciprocal keeps both limbs for diagonals of modulus <= 1 (dd.cuh, cdd_recip_scaled)
    if (k == i) v = unit ? cdd{dd(1.0), dd(0.0)} : (CX ? cdd_recip_scaled(v) : dl_recip<CX>(v));
    else v = -v;
    Ls[i][k] = v;
  }
  __syncthreads();
  const i64 j = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= rhs.ncols) return;
  dd* col = rhs.ptr + (CX ? 2 : 1) * j * rhs.cs;
  for (int i = 0; i < n; ++i) {
    cdd acc = dl_ld<CX>(col, i * rhs.rs);
    for (int k = 0; k < i; ++k) acc = dl_add<CX>(dl_mul<CX>(Ls[i][k], dl_ld<CX>(col, k * rhs.rs)), acc);
    if (!unit) acc = dl_mul<CX>(acc, Ls[i][i]);
    dl_st<CX>(col, i * rhs.rs, acc);
  }
}

template <bool CX>
void trsm_lower_rec(cudaStream_t st, View<const dd> L, bool unit, bool conj, View<dd> rhs) {
  const i64 n = L.nrows, k = rhs.ncols;
  if (n == 0 || k == 0) return;
  if (n <= DL_LEAF) {
    dd_trsm_leaf_kernel<CX><<<(unsigned)((k + 127) / 128), 128, 0, st>>>(L, unit, conj, rhs);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    return;
  }
  const i64 n1 = n / 2;
  trsm_lower_rec<CX>(st, sub_t<dd, CX>(L, 0, 0, n1, n1), unit, conj, sub_t<dd, CX>(rhs, 0, 0, n1, k));
  const View<dd> top = sub_t<dd, CX>(rhs, 0, 0, n1, k);
  gemm_dd(st, sub_t<dd, CX>(rhs, n1, 0, n - n1, k), RECT, 1, sub_t<dd, CX>(L, n1, 0, n - n1, n1), RECT, conj,
          View<const dd>{top.ptr, top.nrows, top.ncols, top.rs, top.cs}, RECT, false, CX, dd(-1.0), dd(0.0));
  trsm_lower_rec<CX>(st, sub_t<dd, CX>(L, n1, n1, n - n1, n - n1), unit, conj, sub_t<dd, CX>(rhs, n1, 0, n - n1, k));
}

// ---- LLT leaf: right-looking over one diagonal block in global memory, one CTA. status[0] = failing column or -1,
// status[1] += regularisation count ----
template <bool CX>
__global__ void __launch_bounds__(DL_THREADS) dd_llt_leaf_kernel(View<dd> A, dd delta, dd eps, bool regularize, long long* status) {
  __shared__ cdd s_inv;
  __shared__ int s_fail;
  const i64 n = A.nrows;
  const int tid = threadIdx.x;
  long long cnt = 0;
  for (i64 j = 0; j < n; ++j) {
    if (tid == 0) {
      dd d = dl_ld<CX>(A.ptr, j * A.rs + j * A.cs).re;
      if (regularize && d <= eps) {
        d = delta;
        ++cnt;
      }
      int fail = !(d > dd(0.0));
      if (!fail) {
        d = sqrt(d);
        fail = d == dd(0.0) || !dd_is_finite(d);
      }
      if (fail) status[0] = j;
      else s_inv = cdd{dd_recip(d), dd(0.0)};
      s_fail = fail;
    }
    __syncthreads();
    if (s_fail) break;
    const dd inv = s_inv.re;
    for (i64 i = j + tid; i < n; i += blockDim.x) {
      const cdd v = dl_ld<CX>(A.ptr, i * A.rs + j * A.cs);
      dl_st<CX>(A.ptr, i * A.rs + j * A.cs, cdd{v.re * inv, CX ? v.im * inv : dd(0.0)});
    }
    __syncthreads();
    // a_ic <- -conj(a_cj) * a_ij + a_ic for j < c <= i: the k = j term of the reference's left-looking sum for column c
    const i64 r = n - j - 1;
    for (i64 e = tid; e < r * r; e += blockDim.x) {
      const i64 i = j + 1 + e % r, c = j + 1 + e / r;
      if (c > i) continue;
      const cdd acj = dl_ld<CX>(A.ptr, c * A.rs + j * A.cs), aij = dl_ld<CX>(A.ptr, i * A.rs + j * A.cs);
      const cdd aic = dl_ld<CX>(A.ptr, i * A.rs + c * A.cs);
      dl_st<CX>(A.ptr, i * A.rs + c * A.cs, dl_add<CX>(dl_mul<CX>(-cdd_conj(acj), aij), aic));
    }
    __syncthreads();
  }
  if (tid == 0) status[1] += cnt;
}

i64 next_pow2(i64 n) {
  i64 p = 1;
  while (p < n) p <<= 1;
  return p;
}

template <bool CX>
i64 llt_rec(cudaStream_t st, View<dd> A, dd delta, dd eps, bool regularize, i64 rt, i64 bsz, long long* d_status) {
  const i64 n = A.nrows;
  if (n <= rt) {
    dd_llt_leaf_kernel<CX><<<1, DL_THREADS, 0, st>>>(A, delta, eps, regularize, d_status);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    long long s0;
    FB_CUDA_CHECK(cudaMemcpyAsync(&s0, d_status, 8, cudaMemcpyDeviceToHost, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    return s0;
  }
  const i64 bs0 = std::min(next_pow2(n) / 2, bsz);
  for (i64 j = 0; j < n;) {
    const i64 bs = std::min(bs0, n - j);
    const View<dd> A00 = sub_t<dd, CX>(A, j, j, bs, bs);
    const i64 fail = llt_rec<CX>(st, A00, delta, eps, regularize, rt, bs, d_status);
    if (fail >= 0) return j + fail;
    const i64 rem = n - j - bs;
    if (rem > 0) {
      const View<dd> A10 = sub_t<dd, CX>(A, j + bs, j, rem, bs), A11 = sub_t<dd, CX>(A, j + bs, j + bs, rem, rem);
      trsm_lower_rec<CX>(st, cview(A00), false, true, A10.t());
      gemm_dd(st, A11, TRI_LOWER, 1, cview(A10), RECT, false, cview(A10).t(), RECT, true, CX, dd(-1.0), dd(0.0));
    }
    j += bs;
  }
  return -1;
}

// ---- LU leaf: columns [c0, c0 + w) over rows [r0, m) of the full matrix A (all columns swapped). trans[row] = pivot - row,
// status[0] += transpositions ----
template <bool CX>
__global__ void __launch_bounds__(DL_THREADS) dd_lu_leaf_kernel(View<dd> A, i64 r0, i64 c0, i64 w, long long* trans, long long* status) {
  __shared__ dd s_val[DL_THREADS];
  __shared__ long long s_idx[DL_THREADS];
  const i64 m = A.nrows, N = A.ncols;
  const int tid = threadIdx.x;
  for (i64 jj = 0; jj < w; ++jj) {
    const i64 row = r0 + jj, col = c0 + jj;
    // first row attaining the maximum abs1 (strict `>` from max = 0): per-thread scan in row order, then the smaller index
    // among equal values
    dd best(0.0);
    long long bi = row;
    for (i64 i = row + tid; i < m; i += blockDim.x) {
      const dd a = dl_abs1<CX>(dl_ld<CX>(A.ptr, i * A.rs + col * A.cs));
      if (a > best) {
        best = a;
        bi = i;
      }
    }
    s_val[tid] = best;
    s_idx[tid] = bi;
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
      if (tid < h) {
        const dd v = s_val[tid + h];
        const long long ix = s_idx[tid + h];
        if (v > s_val[tid] || (v == s_val[tid] && ix < s_idx[tid])) {
          s_val[tid] = v;
          s_idx[tid] = ix;
        }
      }
      __syncthreads();
    }
    const long long piv = s_idx[0];
    if (tid == 0) {
      trans[row] = piv - row;
      if (piv != row) status[0] += 1;
    }
    if (piv != row)
      for (i64 c = tid; c < N; c += blockDim.x) {
        const cdd a = dl_ld<CX>(A.ptr, row * A.rs + c * A.cs), b = dl_ld<CX>(A.ptr, piv * A.rs + c * A.cs);
        dl_st<CX>(A.ptr, row * A.rs + c * A.cs, b);
        dl_st<CX>(A.ptr, piv * A.rs + c * A.cs, a);
      }
    __syncthreads();
    const cdd inv = dl_recip<CX>(dl_ld<CX>(A.ptr, row * A.rs + col * A.cs));
    for (i64 i = row + 1 + tid; i < m; i += blockDim.x)
      dl_st<CX>(A.ptr, i * A.rs + col * A.cs, dl_mul<CX>(dl_ld<CX>(A.ptr, i * A.rs + col * A.cs), inv));
    __syncthreads();
    // rank-1 update of the rest of the panel: a_ic <- a_ic + -(a_i,col * a_row,c)
    const i64 rr = m - row - 1, rc = w - jj - 1;
    for (i64 e = tid; e < rr * rc; e += blockDim.x) {
      const i64 i = row + 1 + e % rr, c = col + 1 + e / rr;
      const cdd l = dl_ld<CX>(A.ptr, i * A.rs + col * A.cs), u = dl_ld<CX>(A.ptr, row * A.rs + c * A.cs);
      const cdd a = dl_ld<CX>(A.ptr, i * A.rs + c * A.cs);
      dl_st<CX>(A.ptr, i * A.rs + c * A.cs, dl_add<CX>(a, -dl_mul<CX>(l, u)));
    }
    __syncthreads();
  }
}

i64 next_multiple_of(i64 x, i64 m) { return (x + m - 1) / m * m; }

// columns [c0, c0 + n) over rows [r0, m): lu_in_place_recursion
template <bool CX>
void lu_rec(cudaStream_t st, View<dd> A, i64 r0, i64 c0, i64 n, i64 rt, long long* d_trans, long long* d_status) {
  const i64 m = A.nrows;
  if (n <= rt) {
    dd_lu_leaf_kernel<CX><<<1, DL_THREADS, 0, st>>>(A, r0, c0, n, d_trans, d_status);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    return;
  }
  const i64 half = n / 2, bs = next_multiple_of(half, std::min<i64>(16, next_pow2(half)));
  lu_rec<CX>(st, A, r0, c0, bs, rt, d_trans, d_status);
  const View<dd> A00 = sub_t<dd, CX>(A, r0, c0, bs, bs), A01 = sub_t<dd, CX>(A, r0, c0 + bs, bs, n - bs);
  const View<dd> A10 = sub_t<dd, CX>(A, r0 + bs, c0, m - r0 - bs, bs), A11 = sub_t<dd, CX>(A, r0 + bs, c0 + bs, m - r0 - bs, n - bs);
  trsm_lower_rec<CX>(st, cview(A00), true, false, A01);
  gemm_dd(st, A11, RECT, 1, cview(A10), RECT, false, cview(A01), RECT, false, CX, dd(-1.0), dd(0.0));
  lu_rec<CX>(st, A, r0 + bs, c0 + bs, n - bs, rt, d_trans, d_status);
}

}  // namespace

void solve_lower_dd(cudaStream_t st, View<const dd> t, bool unit, bool conj, View<dd> rhs, bool cx) {
  FB_ASSERT(t.nrows == t.ncols && rhs.nrows == t.nrows, "triangular solve shape mismatch");
  if (cx) trsm_lower_rec<true>(st, t, unit, conj, rhs);
  else trsm_lower_rec<false>(st, t, unit, conj, rhs);
}
// reverse_rows_and_cols of the upper factor is lower (triangular_solve.rs:577-604)
void solve_upper_dd(cudaStream_t st, View<const dd> t, bool unit, bool conj, View<dd> rhs, bool cx) {
  FB_ASSERT(t.nrows == t.ncols && rhs.nrows == t.nrows, "triangular solve shape mismatch");
  if (t.nrows == 0 || rhs.ncols == 0) return;
  const i64 w = cx ? 2 : 1;
  const View<const dd> tr{t.ptr + w * ((t.nrows - 1) * t.rs + (t.ncols - 1) * t.cs), t.nrows, t.ncols, -t.rs, -t.cs};
  const View<dd> rr{rhs.ptr + w * (rhs.nrows - 1) * rhs.rs, rhs.nrows, rhs.ncols, -rhs.rs, rhs.cs};
  solve_lower_dd(st, tr, unit, conj, rr, cx);
}

template <bool CX>
LltResult llt_dd(cudaStream_t st, View<dd> A, dd delta, dd eps, size_t recursion_threshold, size_t block_size) {
  LltResult out{true, 0, 0};
  const i64 n = A.nrows;
  if (n == 0) return out;
  long long* d_status = (long long*)ws_alloc(16);
  const long long init[2] = {-1, 0};
  FB_CUDA_CHECK(cudaMemcpyAsync(d_status, init, 16, cudaMemcpyHostToDevice, st));
  const bool regularize = delta > dd(0.0) && eps > dd(0.0);  // llt/factor.rs:85-87
  const i64 fail = llt_rec<CX>(st, A, delta, eps, regularize, std::max<i64>(1, (i64)recursion_threshold),
                               std::max<i64>(1, (i64)block_size), d_status);
  long long h[2];
  FB_CUDA_CHECK(cudaMemcpyAsync(h, d_status, 16, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(d_status);
  if (fail >= 0) {
    out.ok = false;
    out.non_positive_pivot_index = (size_t)fail;
  } else {
    out.dynamic_regularization_count = (size_t)h[1];
  }
  return out;
}
template LltResult llt_dd<false>(cudaStream_t, View<dd>, dd, dd, size_t, size_t);
template LltResult llt_dd<true>(cudaStream_t, View<dd>, dd, dd, size_t, size_t);

// P A = L U in place; perm_fwd / perm_bwd: HOST int64[m]; returns the transposition count (lu_in_place, factor.rs:234-295)
template <bool CX>
size_t lu_dd(cudaStream_t st, View<dd> A, size_t recursion_threshold, long long* perm_fwd, long long* perm_bwd) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n);
  for (i64 i = 0; i < m; ++i) perm_fwd[i] = i;
  size_t cnt = 0;
  if (size > 0) {
    long long* d_buf = (long long*)ws_alloc((size_t)(size + 1) * 8);
    FB_CUDA_CHECK(cudaMemsetAsync(d_buf, 0, (size_t)(size + 1) * 8, st));
    lu_rec<CX>(st, A, 0, 0, size, std::max<i64>(1, (i64)recursion_threshold), d_buf + 1, d_buf);
    std::vector<long long> h((size_t)size + 1);
    FB_CUDA_CHECK(cudaMemcpyAsync(h.data(), d_buf, (size_t)(size + 1) * 8, cudaMemcpyDeviceToHost, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    ws_free(d_buf);
    cnt = (size_t)h[0];
    for (i64 i = 0; i < size; ++i) std::swap(perm_fwd[i], perm_fwd[i + h[(size_t)i + 1]]);
    if (m < n) {  // factor.rs:278-285
      solve_lower_dd(st, cview(sub_t<dd, CX>(A, 0, 0, m, size)), true, false, sub_t<dd, CX>(A, 0, size, m, n - size), CX);
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
    }
  }
  for (i64 i = 0; i < m; ++i) perm_bwd[perm_fwd[i]] = i;
  return cnt;
}
template size_t lu_dd<false>(cudaStream_t, View<dd>, size_t, long long*, long long*);
template size_t lu_dd<true>(cudaStream_t, View<dd>, size_t, long long*, long long*);

}  // namespace fb
