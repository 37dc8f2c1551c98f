// c64 / c32 (complex<f64> / complex<f32>) triangular solves, Cholesky LLT, partial-pivoting LU and Householder QR (+ block-Householder
// sequences): faer's recursions on the complex GEMMs (gemm_c64.cu, gemm_c32.cu) with small scalar complex leaf kernels, one source
// templated over the real type R. (The comment blocks at the LU and QR sections cite their reference lines.) The blocked QR driver
// and the Householder sequences are qr_blocked.cuh's, shared with the double-double kinds; this file supplies their c64 / c32 leaf.
//
// Reference:
//   triangular_solve::solve_[unit_]{lower,upper}_triangular_in_place_with_conj   faer/src/linalg/triangular_solve.rs:220-604
//       recursive split (block_size 200-211): top solve, rhs_bot -= conj?(T10) * rhs_top, bottom solve; leaves multiply by the
//       reciprocal of the diagonal (16-198); upper = lower on reversed views (577-604)
//   cholesky::llt::factor::cholesky_in_place for complex T   cholesky/llt/factor.rs:68-97 -> ldlt/factor.rs:367-498
//       A00 = L00 L00^H (recursion / leaf), conj(L00) X = A10^T, A11(lower) -= A10 A10^H; leaf recurrence
//       a_ij <- a_ij - conj(a_jk) a_ik, d = Re(a_jj), [regularise], fail if !(d > 0), l = sqrt(d), column j (diagonal included)
//       multiplied by recip(l)  (ldlt/factor.rs:7-177, 299-366)
//
// All views are in COMPLEX element units (pointer to the first complex element as R*, strides in complex elements), as in
// gemm_c64.cu / gemm_c32.cu. The leaves are plain scalar kernels (a 32 x 32 block per CTA / one thread per right-hand-side column): O(n^2 leaf)
// work next to the O(n^3) that runs on the DMMA GEMM.
#include <algorithm>
#include <vector>

#include "gemm_f32.cuh"
#include "linalg_f64.cuh"
#include "qr_blocked.cuh"
#include "runtime.cuh"

namespace fb {

namespace {

constexpr int CL = 32;  // leaf order of both recursions

template <class R>
struct CxT {
  R re, im;
};
template <class R>
__device__ __forceinline__ CxT<R> cmul(CxT<R> a, CxT<R> b) {
  return CxT<R>{fma(a.re, b.re, -a.im * b.im), fma(a.re, b.im, a.im * b.re)};
}
template <class R>
__device__ __forceinline__ CxT<R> cld(const R* p, i64 off) {
  return CxT<R>{p[2 * off], p[2 * off + 1]};
}
template <class R>
__device__ __forceinline__ void cst(R* p, i64 off, CxT<R> v) {
  p[2 * off] = v.re;
  p[2 * off + 1] = v.im;
}
// 1 / d without spurious overflow; an infinite d (the +inf diagonal of a skipped reflector, qr factor.rs:287-299) gives 0
template <class R>
__device__ __forceinline__ CxT<R> crecip(CxT<R> d) {
  if (isinf(d.re) || isinf(d.im)) return CxT<R>{R(0), R(0)};
  const R mx = fmax(fabs(d.re), fabs(d.im));
  if (mx == R(0)) {
    const R s = R(1) / fma(d.re, d.re, d.im * d.im);
    return CxT<R>{d.re * s, -d.im * s};
  }
  const R sc = R(1) / mx;
  const R a = d.re * sc, b = d.im * sc;
  const R s = sc / fma(a, a, b * b);
  return CxT<R>{a * s, -b * s};
}

// complex products of the recursions, by scalar type
inline void cgemm(cudaStream_t st, VD dst, int ds, int accum, VCD a, int as, bool ca, VCD b, int bs, bool cb, double ar, double ai) {
  gemm_c64(st, dst, ds, accum, a, as, ca, b, bs, cb, ar, ai);
}
inline void cgemm(cudaStream_t st, VF dst, int ds, int accum, VCF a, int as, bool ca, VCF b, int bs, bool cb, float ar, float ai) {
  gemm_c32(st, dst, ds, accum, a, as, ca, b, bs, cb, ar, ai);
}

// conj?(T) X = B for a lower-triangular leaf T (n <= CL): one thread per column of B, the column in registers
template <class R>
__global__ void __launch_bounds__(64) trsm_leaf_lower_cx_kernel(const R* __restrict__ T, i64 t_rs, i64 t_cs, int n, int unit,
                                                                  int conj, R* __restrict__ B, i64 b_rs, i64 b_cs, i64 ncols) {
  __shared__ R nlr[CL][CL + 1], nli[CL][CL + 1];  // -(conj? l_ik) * inv_i below the diagonal, inv_i on it
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, k = e - i * n;
    if (k > i) continue;
    CxT<R> inv{R(1), R(0)};
    if (!unit) {
      inv = crecip(cld(T, (i64)i * t_rs + (i64)i * t_cs));  // 1 / d; 0 for the +inf diagonal of a skipped reflector
      if (conj) inv.im = -inv.im;           // conj(1 / d) = 1 / conj(d)
    }
    CxT<R> v = inv;
    if (k < i) {
      CxT<R> l = cld(T, (i64)i * t_rs + (i64)k * t_cs);
      if (conj) l.im = -l.im;
      v = cmul(CxT<R>{-l.re, -l.im}, inv);
    }
    nlr[i][k] = v.re;
    nli[i][k] = v.im;
  }
  __syncthreads();
  const i64 col = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= ncols) return;
  R yr[CL], yi[CL];
#pragma unroll
  for (int i = 0; i < CL; ++i) {
    if (i < n) {
      CxT<R> v = cld(B, (i64)i * b_rs + col * b_cs);
      v = cmul(v, CxT<R>{nlr[i][i], nli[i][i]});  // * inv_i (1 for a unit diagonal)
#pragma unroll
      for (int k = 0; k < CL; ++k) {
        if (k < i) {
          const CxT<R> t = cmul(CxT<R>{nlr[i][k], nli[i][k]}, CxT<R>{yr[k], yi[k]});
          v.re += t.re;
          v.im += t.im;
        }
      }
      yr[i] = v.re;
      yi[i] = v.im;
      cst(B, (i64)i * b_rs + col * b_cs, v);
    }
  }
}

// in-place lower Cholesky of a <= CL x CL Hermitian block (lower triangle read / written), one CTA, block in shared memory
template <class R>
__global__ void __launch_bounds__(CL * CL) potf2_cx_kernel(R* __restrict__ A, i64 rs, i64 cs, int n, i64 j0, int regularize,
                                                            R eps, R delta, long long* __restrict__ info) {
  __shared__ R Sr[CL][CL + 1], Si[CL][CL + 1];
  __shared__ R s_inv;
  __shared__ int s_fail, s_count;
  if (info[0] >= 0) return;  // an earlier block already failed
  const int i = threadIdx.x % CL, c = threadIdx.x / CL;
  const bool on = i < n && c <= i;
  if (on) {
    const CxT<R> v = cld(A, (i64)i * rs + (i64)c * cs);
    Sr[i][c] = v.re;
    Si[i][c] = v.im;
  }
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    if (threadIdx.x == 0) {
      R d = Sr[j][j];
      int fail = 0;
      if (regularize && d <= eps) {
        d = delta;
        s_count += 1;
      }
      R inv = R(0);
      if (!(d > R(0))) fail = 1;
      else {
        const R sd = sqrt(d);
        if (sd == R(0) || !isfinite(sd)) fail = 1;
        else inv = R(1) / sd;
      }
      s_inv = inv;
      s_fail = fail;
    }
    __syncthreads();
    if (s_fail) {
      if (threadIdx.x == 0) info[0] = j0 + j;
      return;
    }
    const R inv = s_inv;
    // column j (diagonal included) * recip(l_jj)
    if (c == j && i >= j && i < n) {
      Sr[i][j] *= inv;
      Si[i][j] *= inv;
    }
    __syncthreads();
    // a_ic <- a_ic - conj(l_cj) l_ij for j < c <= i
    if (on && c > j) {
      const CxT<R> lc{Sr[c][j], -Si[c][j]}, li{Sr[i][j], Si[i][j]};
      const CxT<R> t = cmul(lc, li);
      Sr[i][c] -= t.re;
      Si[i][c] -= t.im;
    }
    __syncthreads();
  }
  if (on) cst(A, (i64)i * rs + (i64)c * cs, CxT<R>{Sr[i][c], Si[i][c]});
  if (threadIdx.x == 0 && s_count) info[1] += s_count;
}

template <class R>
inline View<R> csub(View<R> v, i64 i, i64 j, i64 m, i64 n) { return View<R>{v.ptr + 2 * (i * v.rs + j * v.cs), m, n, v.rs, v.cs}; }
template <class R>
inline View<const R> csub(View<const R> v, i64 i, i64 j, i64 m, i64 n) { return View<const R>{v.ptr + 2 * (i * v.rs + j * v.cs), m, n, v.rs, v.cs}; }

template <class R>
void solve_lower_rec_cx(cudaStream_t st, View<const R> T, bool unit, bool conj, View<R> rhs) {
  const i64 n = T.nrows, k = rhs.ncols;
  if (n == 0 || k == 0) return;
  if (n <= CL) {
    trsm_leaf_lower_cx_kernel<R><<<(unsigned)((k + 63) / 64), 64, 0, st>>>(T.ptr, T.rs, T.cs, (int)n, unit ? 1 : 0, conj ? 1 : 0, rhs.ptr,
                                                                         rhs.rs, rhs.cs, k);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    return;
  }
  const i64 n1 = ((n / 2 + CL - 1) / CL) * CL;
  solve_lower_rec_cx(st, csub(T, 0, 0, n1, n1), unit, conj, csub(rhs, 0, 0, n1, k));
  // rhs_bot -= conj?(T10) * rhs_top
  cgemm(st, csub(rhs, n1, 0, n - n1, k), RECT, 1, csub(T, n1, 0, n - n1, n1), RECT, conj, cv(csub(rhs, 0, 0, n1, k)), RECT, false,
           R(-1), R(0));
  solve_lower_rec_cx(st, csub(T, n1, n1, n - n1, n - n1), unit, conj, csub(rhs, n1, 0, n - n1, k));
}

template <class R>
struct LltCtxC {
  cudaStream_t st;
  int regularize;
  R eps, delta;
  long long* d_info;
};

template <class R>
void llt_rec_cx(const LltCtxC<R>& ctx, View<R> A, i64 j0) {
  const i64 n = A.nrows;
  if (n <= CL) {
    potf2_cx_kernel<R><<<1, CL * CL, 0, ctx.st>>>(A.ptr, A.rs, A.cs, (int)n, j0, ctx.regularize, ctx.eps, ctx.delta, ctx.d_info);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    return;
  }
  const i64 n1 = ((n / 2 + CL - 1) / CL) * CL, n2 = n - n1;
  View<R> A11 = csub(A, 0, 0, n1, n1), A21 = csub(A, n1, 0, n2, n1), A22 = csub(A, n1, n1, n2, n2);
  llt_rec_cx(ctx, A11, j0);
  // conj(L11) X = A21^T   (ldlt/factor.rs:421-426)
  solve_lower_rec_cx(ctx.st, cv(A11), false, true, A21.t());
  // A22(lower) -= A21 A21^H   (435-446)
  cgemm(ctx.st, A22, TRI_LOWER, 1, cv(A21), RECT, false, cv(A21).t(), RECT, true, R(-1), R(0));
  llt_rec_cx(ctx, A22, j0 + n1);
}


// ---- partial-pivoting LU (lu/partial_pivoting/factor.rs:19-295 for complex T) ---------------------------------------------
constexpr int LU_CW = 16;         // leaf width
constexpr int LU_CT = 1024;       // leaf threads (one CTA walks the panel's rows in global memory)

// Unblocked leaf on the view A (m rows, `ncols_view` columns; local row 0 = first diagonal row of the window [start, start + w)):
// pivot = first row attaining the largest abs1 = |re| + |im| (strict `>` from 0: an all-zero column keeps the diagonal row),
// the swap covers the whole row of the view (factor.rs:46), multipliers by reciprocal-multiply, rank-1 update of the window.
template <class R>
__global__ void __launch_bounds__(LU_CT) lu_leaf_cx_kernel(R* __restrict__ A, i64 rs, i64 cs, int m, int ncols_view, int start,
                                                            int w, int* __restrict__ trans) {
  __shared__ R red_v[LU_CT / 32];
  __shared__ int red_i[LU_CT / 32];
  __shared__ int s_piv;
  __shared__ R s_inv[2];
  __shared__ R s_row[LU_CW][2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int j = 0; j < w && j < m; ++j) {
    const int col = start + j;
    // ---- pivot search over rows >= j ----
    R bv = R(0);
    int bi = j;
    for (int i = j + tid; i < m; i += LU_CT) {
      const CxT<R> a = cld(A, (i64)i * rs + (i64)col * cs);
      const R v = fabs(a.re) + fabs(a.im);
      if (v > bv) {  // rows ascend within a thread: the first maximum is kept
        bv = v;
        bi = i;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const R ov = __shfl_xor_sync(0xffffffffu, bv, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ov > bv || (ov == bv && oi < bi)) {
        bv = ov;
        bi = oi;
      }
    }
    if (lane == 0) {
      red_v[warp] = bv;
      red_i[warp] = bi;
    }
    __syncthreads();
    if (warp == 0) {
      bv = red_v[lane];
      bi = red_i[lane];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const R ov = __shfl_xor_sync(0xffffffffu, bv, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (ov > bv || (ov == bv && oi < bi)) {
          bv = ov;
          bi = oi;
        }
      }
      if (lane == 0) {
        s_piv = (bv > R(0)) ? bi : j;
        trans[j] = s_piv - j;
      }
    }
    __syncthreads();
    const int piv = s_piv;
    // ---- swap rows j <-> piv over the whole view ----
    if (piv != j) {
      for (int c = tid; c < ncols_view; c += LU_CT) {
        const CxT<R> a = cld(A, (i64)j * rs + (i64)c * cs), b = cld(A, (i64)piv * rs + (i64)c * cs);
        cst(A, (i64)j * rs + (i64)c * cs, b);
        cst(A, (i64)piv * rs + (i64)c * cs, a);
      }
    }
    __syncthreads();
    if (tid == 0) {
      const CxT<R> d = cld(A, (i64)j * rs + (i64)col * cs);
      const R sc = R(1) / fma(d.re, d.re, d.im * d.im);
      s_inv[0] = d.re * sc;
      s_inv[1] = -d.im * sc;
    }
    if (tid < w - j - 1) {
      const CxT<R> u = cld(A, (i64)j * rs + (i64)(col + 1 + tid) * cs);
      s_row[tid][0] = u.re;
      s_row[tid][1] = u.im;
    }
    __syncthreads();
    const CxT<R> inv{s_inv[0], s_inv[1]};
    // ---- multipliers and rank-1 update: one row per thread and iteration ----
    for (int i = j + 1 + tid; i < m; i += LU_CT) {
      const CxT<R> l = cmul(cld(A, (i64)i * rs + (i64)col * cs), inv);
      cst(A, (i64)i * rs + (i64)col * cs, l);
      for (int c = 0; c < w - j - 1; ++c) {
        const CxT<R> t = cmul(l, CxT<R>{s_row[c][0], s_row[c][1]});
        CxT<R> a = cld(A, (i64)i * rs + (i64)(col + 1 + c) * cs);
        a.re -= t.re;
        a.im -= t.im;
        cst(A, (i64)i * rs + (i64)(col + 1 + c) * cs, a);
      }
    }
    __syncthreads();
  }
}

// apply n transpositions (row j <-> row j + trans[j], in order) to every column of the view: one thread per column
template <class R>
__global__ void laswp_cx_kernel(R* __restrict__ A, i64 rs, i64 cs, i64 ncols, const int* __restrict__ trans, int n) {
  const i64 c = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncols) return;
  for (int j = 0; j < n; ++j) {
    const int t = trans[j];
    if (t == 0) continue;
    const CxT<R> a = cld(A, (i64)j * rs + c * cs), b = cld(A, (i64)(j + t) * rs + c * cs);
    cst(A, (i64)j * rs + c * cs, b);
    cst(A, (i64)(j + t) * rs + c * cs, a);
  }
}

inline i64 next_pow2_c(i64 n) {
  i64 p = 1;
  while (p < n) p <<= 1;
  return p;
}

// the reference's recursion (factor.rs:68-187): A = current view (all m rows, ncols columns), window [start, end)
template <class R>
void lu_rec_cx(cudaStream_t st, View<R> A, i64 start, i64 end, int* trans) {
  const i64 m = A.nrows, ncols = A.ncols, n = end - start;
  if (n == 0) return;
  if (n <= LU_CW) {
    lu_leaf_cx_kernel<R><<<1, LU_CT, 0, st>>>(A.ptr, A.rs, A.cs, (int)m, (int)ncols, (int)start, (int)n, trans);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    return;
  }
  const i64 half = n / 2;
  const i64 pw = std::min<i64>(16, next_pow2_c(half));
  const i64 bs = (half + pw - 1) / pw * pw;
  View<R> W = csub(A, 0, start, m, n);
  lu_rec_cx(st, W, 0, bs, trans);
  {
    View<R> A00 = csub(W, 0, 0, bs, bs), A01 = csub(W, 0, bs, bs, n - bs), A10 = csub(W, bs, 0, m - bs, bs), A11 = csub(W, bs, bs, m - bs, n - bs);
    solve_lower_rec_cx(st, cv(A00), true, false, A01);
    cgemm(st, A11, RECT, 1, cv(A10), RECT, false, cv(A01), RECT, false, R(-1), R(0));
    lu_rec_cx(st, csub(W, bs, 0, m - bs, n), bs, n, trans + bs);
  }
  auto swap_cols = [&](View<R> M) {
    if (M.ncols == 0) return;
    laswp_cx_kernel<R><<<(unsigned)((M.ncols + 127) / 128), 128, 0, st>>>(M.ptr, M.rs, M.cs, M.ncols, trans, (int)n);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  };
  swap_cols(csub(A, 0, 0, m, start));
  swap_cols(csub(A, 0, end, m, ncols - end));
}

// conj?(T) X = rhs, T lower / upper triangular (unit diagonal or not); views in complex units
template <class R>
void solve_lower_triangular_in_place_cx(cudaStream_t st, View<const R> tril, bool unit, bool conj, View<R> rhs) {
  FB_ASSERT(tril.nrows == tril.ncols && rhs.nrows == tril.nrows, "triangular solve shape mismatch");
  solve_lower_rec_cx(st, tril, unit, conj, rhs);
}
template <class R>
void solve_upper_triangular_in_place_cx(cudaStream_t st, View<const R> triu, bool unit, bool conj, View<R> rhs) {
  FB_ASSERT(triu.nrows == triu.ncols && rhs.nrows == triu.nrows, "triangular solve shape mismatch");
  const i64 n = triu.nrows;
  if (n == 0 || rhs.ncols == 0) return;
  // upper = lower on the views with rows and columns reversed (triangular_solve.rs:577-604)
  View<const R> t{triu.ptr + 2 * ((n - 1) * triu.rs + (n - 1) * triu.cs), n, n, -triu.rs, -triu.cs};
  View<R> r{rhs.ptr + 2 * ((n - 1) * rhs.rs), n, rhs.ncols, -rhs.rs, rhs.cs};
  solve_lower_rec_cx(st, t, unit, conj, r);
}

template <class R>
LltResult llt_cholesky_in_place_cx(cudaStream_t st, View<R> A, R reg_delta, R reg_eps) {
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  LltResult res{true, 0, 0};
  if (A.nrows == 0) return res;
  long long* d_info = (long long*)ws_alloc(2 * sizeof(long long));
  long long h_info[2] = {-1, 0};
  FB_CUDA_CHECK(cudaMemcpyAsync(d_info, h_info, sizeof(h_info), cudaMemcpyHostToDevice, st));
  LltCtxC<R> ctx{st, (reg_delta > R(0) && reg_eps > R(0)) ? 1 : 0, reg_eps, reg_delta, d_info};
  llt_rec_cx(ctx, A, 0);
  FB_CUDA_CHECK(cudaMemcpyAsync(h_info, d_info, sizeof(h_info), cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(d_info);
  if (h_info[0] >= 0) {
    res.ok = false;
    res.non_positive_pivot_index = (size_t)h_info[0];
  } else {
    res.dynamic_regularization_count = (size_t)h_info[1];
  }
  return res;
}

// In-place P A = L U of an m x n c64 matrix (views in complex units); perm arrays: HOST int64 of length m. Returns the
// transposition count (lu_in_place, factor.rs:234-295).
template <class R>
size_t lu_partial_piv_in_place_cx(cudaStream_t st, View<R> A, long long* perm_fwd, long long* perm_inv) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n);
  for (i64 i = 0; i < m; ++i) perm_fwd[i] = i;
  size_t n_trans = 0;
  if (size > 0) {
    int* d_trans = (int*)ws_alloc((size_t)size * sizeof(int));
    FB_CUDA_CHECK(cudaMemsetAsync(d_trans, 0, (size_t)size * sizeof(int), st));
    lu_rec_cx(st, A, 0, size, d_trans);
    std::vector<int> h_trans((size_t)size);
    FB_CUDA_CHECK(cudaMemcpyAsync(h_trans.data(), d_trans, (size_t)size * sizeof(int), cudaMemcpyDeviceToHost, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    ws_free(d_trans);
    for (i64 i = 0; i < size; ++i) {
      const int t = h_trans[(size_t)i];
      if (t != 0) {
        std::swap(perm_fwd[i], perm_fwd[i + t]);
        ++n_trans;
      }
    }
    if (m < n) {  // factor.rs:278-285
      solve_lower_rec_cx(st, cv(csub(A, 0, 0, m, size)), true, false, csub(A, 0, size, m, n - size));
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
    }
  }
  for (i64 i = 0; i < m; ++i) perm_inv[perm_fwd[i]] = i;
  return n_trans;
}

// ---- Householder QR without pivoting for complex T: the unblocked leaf (qr/no_pivoting/factor.rs:11-86; householder.rs:59-107).
// One CTA carries the column-skipping rank logic; the blocked recursion above it is the shared driver of qr_blocked.cuh, which
// hands it blocks of <= QR_LEAF columns (whole blocks under the reference's `m * n < blocking_threshold` branch). Functional, not
// tuned: the panels run on a single SM.
constexpr int QR_CT = 1024;

template <class R>
struct RealTraits;
template <>
struct RealTraits<double> {
  static constexpr double min_pos = 2.2250738585072014e-308, eps = 2.220446049250313e-16, sml = 0x1p-511, big = 0x1p511;
};
template <>
struct RealTraits<float> {
  static constexpr float min_pos = 1.17549435e-38f, eps = 1.1920929e-7f, sml = 0x1p-63f, big = 0x1p63f;
};

// norm_l2.rs:161-172: selection between the three scaled accumulators
template <class R>
__device__ __forceinline__ R norm_select(R acc_sml, R acc_med, R acc_big) {
  if (acc_sml >= R(1)) return sqrt(acc_sml) * RealTraits<R>::big;
  if (acc_med >= R(1)) return sqrt(acc_med);
  return sqrt(acc_big) * RealTraits<R>::sml;
}

// qr_in_place_unblocked (factor.rs:11-86) on the view A (m x n), reflector coefficients into H[row * h_stride] (complex units),
// starting at (row_start, col_start); the new row index comes back in out_row[0].
template <class R>
__global__ void __launch_bounds__(QR_CT) qr_unblocked_cx_kernel(R* __restrict__ A, i64 rs, i64 cs, int m, int n, R* __restrict__ H,
                                                                i64 h_stride, int h_len, int row_start, int col_start,
                                                                int* __restrict__ out_row) {
  using Tr = RealTraits<R>;
  using Cx = CxT<R>;
  __shared__ R red[6][QR_CT / 32];
  __shared__ R s_inv[2];
  __shared__ R s_tau_inv;
  __shared__ int s_scale, s_action;  // action: 0 = column skipped, 1 = row advances without an update, 2 = update + advance
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int row = row_start, col = col_start;
  const int row_end = h_len < m ? h_len : m;
  while (row < row_end && col < n) {
    const int len = m - row - 1;
    // ---- norm of the column above `row` and of the tail below it (three scaled accumulators each, norm_l2.rs:6-172) ----
    R a0 = 0, a1 = 0, a2 = 0, t0 = 0, t1 = 0, t2 = 0;
    for (int i = tid; i < m; i += QR_CT) {
      if (i == row) continue;
      const Cx x = cld(A, (i64)i * rs + (i64)col * cs);
      const R xs = x.re * Tr::sml, ys = x.im * Tr::sml, xb = x.re * Tr::big, yb = x.im * Tr::big;
      const R q0 = fma(xs, xs, ys * ys), q1 = fma(x.re, x.re, x.im * x.im), q2 = fma(xb, xb, yb * yb);
      if (i < row) {
        a0 += q0; a1 += q1; a2 += q2;
      } else {
        t0 += q0; t1 += q1; t2 += q2;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, off);
      a1 += __shfl_xor_sync(0xffffffffu, a1, off);
      a2 += __shfl_xor_sync(0xffffffffu, a2, off);
      t0 += __shfl_xor_sync(0xffffffffu, t0, off);
      t1 += __shfl_xor_sync(0xffffffffu, t1, off);
      t2 += __shfl_xor_sync(0xffffffffu, t2, off);
    }
    if (lane == 0) {
      red[0][warp] = a0; red[1][warp] = a1; red[2][warp] = a2;
      red[3][warp] = t0; red[4][warp] = t1; red[5][warp] = t2;
    }
    __syncthreads();
    if (tid == 0) {
      R acc[6];
      for (int q = 0; q < 6; ++q) {
        R v = 0;
        for (int w = 0; w < QR_CT / 32; ++w) v += red[q][w];
        acc[q] = v;
      }
      const R norm_above = norm_select(acc[0], acc[1], acc[2]);
      const R tail_norm = norm_select(acc[3], acc[4], acc[5]);
      // make_householder_imp (householder.rs:59-107)
      Cx head = cld(A, (i64)row * rs + (i64)col * cs);
      R head_norm = hypot(head.re, head.im);
      if (head_norm < Tr::min_pos) {
        head = Cx{R(0), R(0)};
        head_norm = R(0);
        cst(A, (i64)row * rs + (i64)col * cs, head);
      }
      R tau, info_norm;
      int scale = 0;
      if (tail_norm < Tr::min_pos) {
        tau = R(INFINITY);
        info_norm = head_norm;
      } else {
        const R norm = hypot(head_norm, tail_norm);
        Cx sign{R(1), R(0)};
        if (head_norm != R(0)) {
          const R hi = R(1) / head_norm;
          sign = Cx{head.re * hi, head.im * hi};
        }
        const Cx signed_norm{sign.re * norm, sign.im * norm};
        const Cx inv = crecip(Cx{head.re + signed_norm.re, head.im + signed_norm.im});
        cst(A, (i64)row * rs + (i64)col * cs, Cx{-signed_norm.re, -signed_norm.im});
        const R t = tail_norm * hypot(inv.re, inv.im);
        tau = R(0.5) * (R(1) + t * t);
        info_norm = norm;
        s_inv[0] = inv.re;
        s_inv[1] = inv.im;
        scale = 1;
      }
      // rank test (factor.rs:41-53)
      const R nrm = hypot(info_norm, norm_above);
      const R threshold = Tr::eps * (R)((double)(m - row) * 16.0) * nrm;
      const R tau_inv = R(1) / tau;
      cst(H, (i64)row * h_stride, Cx{tau, R(0)});
      int action = 0;
      if (tau_inv < Tr::min_pos) {
        if (info_norm > R(0)) action = 1;
      } else if (info_norm > threshold) {
        action = 2;
      }
      s_tau_inv = tau_inv;
      s_scale = scale;
      s_action = action;
    }
    __syncthreads();
    const int action = s_action, scale = s_scale;
    const int vcol = row;  // the essential part always lives below the diagonal of column `row` (== col when nothing was skipped)
    {
      const Cx inv{s_inv[0], s_inv[1]};
      const int z = (col - row) < len ? (col - row) : len;  // rows of column `col` to clear when row != col (factor.rs:33-38)
      for (int i = tid; i < len; i += QR_CT) {
        const i64 r_ = (i64)(row + 1 + i) * rs;
        if (scale) cst(A, r_ + (i64)vcol * cs, cmul(cld(A, r_ + (i64)col * cs), inv));
        if (row != col && i < z) cst(A, r_ + (i64)col * cs, Cx{R(0), R(0)});
      }
    }
    __syncthreads();
    if (action == 2) {
      const R tau_inv = s_tau_inv;
      for (int c = col + 1 + warp; c < n; c += QR_CT / 32) {
        R dr = 0, di = 0;
        for (int i = lane; i < len; i += 32) {
          const i64 r_ = (i64)(row + 1 + i) * rs;
          const Cx v = cld(A, r_ + (i64)vcol * cs), a = cld(A, r_ + (i64)c * cs);
          dr += fma(v.re, a.re, v.im * a.im);   // conj(v) * a
          di += fma(v.re, a.im, -v.im * a.re);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          dr += __shfl_xor_sync(0xffffffffu, dr, off);
          di += __shfl_xor_sync(0xffffffffu, di, off);
        }
        const Cx a0c = cld(A, (i64)row * rs + (i64)c * cs);
        const Cx k{-(a0c.re + dr) * tau_inv, -(a0c.im + di) * tau_inv};
        if (lane == 0) cst(A, (i64)row * rs + (i64)c * cs, Cx{a0c.re + k.re, a0c.im + k.im});
        for (int i = lane; i < len; i += 32) {
          const i64 r_ = (i64)(row + 1 + i) * rs;
          const Cx t = cmul(k, cld(A, r_ + (i64)vcol * cs));
          Cx a = cld(A, r_ + (i64)c * cs);
          a.re += t.re;
          a.im += t.im;
          cst(A, r_ + (i64)c * cs, a);
        }
      }
    }
    __syncthreads();
    if (action != 0) row += 1;
    col += 1;
  }
  if (tid == 0) out_row[0] = row;
}

// the reference's unblocked leaf on one CTA; one host read-back of the new row index per leaf
template <class R>
i64 qr_unblocked_cx(const QrCtx<R>& cx, View<R> A, View<R> Hrow, i64 row_start, i64 col_start) {
  if (!(row_start < std::min(Hrow.ncols, A.nrows) && col_start < A.ncols)) return row_start;
  qr_unblocked_cx_kernel<R><<<1, QR_CT, 0, cx.st>>>(A.ptr, A.rs, A.cs, (int)A.nrows, (int)A.ncols, Hrow.ptr, Hrow.cs, (int)Hrow.ncols,
                                                    (int)row_start, (int)col_start, cx.d_row);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  int h_row = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(&h_row, cx.d_row, sizeof(int), cudaMemcpyDeviceToHost, cx.st));
  FB_CUDA_CHECK(cudaStreamSynchronize(cx.st));
  return h_row;
}

}  // namespace

// the leaves of the blocked driver (qr_blocked.cuh) for c64 / c32
template <>
i64 qr_unblocked_t<double, true>(const QrCtx<double>& cx, View<double> A, View<double> Hrow, i64 row_start, i64 col_start) {
  return qr_unblocked_cx<double>(cx, A, Hrow, row_start, col_start);
}
template <>
i64 qr_unblocked_t<float, true>(const QrCtx<float>& cx, View<float> A, View<float> Hrow, i64 row_start, i64 col_start) {
  return qr_unblocked_cx<float>(cx, A, Hrow, row_start, col_start);
}

// ---- exported entry points (linalg_f64.cuh / gemm_f32.cuh) ------------------------------------------------------------------
#define FB_CPLX_EXPORTS(SUF, R)                                                                                                   \
  void solve_lower_triangular_in_place_##SUF(cudaStream_t st, View<const R> t, bool unit, bool conj, View<R> rhs) {              \
    solve_lower_triangular_in_place_cx<R>(st, t, unit, conj, rhs);                                                               \
  }                                                                                                                               \
  void solve_upper_triangular_in_place_##SUF(cudaStream_t st, View<const R> t, bool unit, bool conj, View<R> rhs) {              \
    solve_upper_triangular_in_place_cx<R>(st, t, unit, conj, rhs);                                                               \
  }                                                                                                                               \
  LltResult llt_cholesky_in_place_##SUF(cudaStream_t st, View<R> A, R reg_delta, R reg_eps) {                                    \
    return llt_cholesky_in_place_cx<R>(st, A, reg_delta, reg_eps);                                                               \
  }                                                                                                                               \
  size_t lu_partial_piv_in_place_##SUF(cudaStream_t st, View<R> A, long long* perm_fwd, long long* perm_inv) {                   \
    return lu_partial_piv_in_place_cx<R>(st, A, perm_fwd, perm_inv);                                                             \
  }                                                                                                                               \
  i64 qr_in_place_##SUF(cudaStream_t st, View<R> A, View<R> Q_coeff, i64 blocking_threshold) {                                   \
    return qr_in_place_t<R, true>(st, A, Q_coeff, blocking_threshold);                                                           \
  }                                                                                                                               \
  void apply_householder_sequence_left_##SUF(cudaStream_t st, View<const R> basis, View<const R> factor, bool conj, View<R> rhs, \
                                             bool transpose) {                                                                    \
    apply_householder_sequence_left_t<R, true>(st, basis, factor, conj, rhs, transpose);                                            \
  }
FB_CPLX_EXPORTS(c64, double)
FB_CPLX_EXPORTS(c32, float)
#undef FB_CPLX_EXPORTS

template <class R>
void householder_build_t_cx(cudaStream_t st, View<const R> V, View<R> Tf) {
  upgrade_householder_factor_t<R, true>(st, Tf, V, Tf.nrows, 1);
}
template void householder_build_t_cx<double>(cudaStream_t, View<const double>, View<double>);
template void householder_build_t_cx<float>(cudaStream_t, View<const float>, View<float>);

}  // namespace fb
