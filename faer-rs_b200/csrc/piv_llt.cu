// Pivoted Cholesky (faer's `llt_pivoting`) for f64 / f32 / c64 / c32: factor, solve, reconstruct, inverse, and their C ABI
// (include/faer_b200_piv_llt.h, included by include/faer_b200.h: `libfaer_v0_23_piv_llt_*`).
//
// Reference: faer/src/linalg/cholesky/llt_pivoting/factor.rs:47-199 (factor), solve.rs:13-41, reconstruct.rs:12-52,
// inverse.rs:12-54. The factorization reproduces the reference's operation sequence, so its integer outputs (status, rank,
// transposition count, permutation) match it exactly:
//   * initial scan: a negative or NaN Re a_ii fails with index 0 (A untouched); tol = eps * n * max Re a_ii;
//   * blocks of bs = min(n - k, block_size) columns; per column j: dot[i] += |a(i, j-1)|^2 and diag[i] = Re a(i,i) - dot[i]
//     (unfused, as the reference's Rust), NaN check, first maximum of diag[j..] from (pvt = j, ajj = 0) with strict `>`,
//     rank exit if ajj < tol (a(j,j) = ajj), symmetric swap of j and pvt, a(j,j) = sqrt(ajj), left-looking GEMV of column j,
//     scale by recip(sqrt(ajj));
//   * after each block the lower trailing matrix -= P P^H (P = the block's columns below it).
//
// GPU mapping, per block (one stream, no host synchronisation inside the block loop):
//   piv_llt_panel_kernel  one cooperative launch over the trailing rows. Thread t owns rows k + t, k + t + T, ... (T = grid
//                         threads), so a warp reads 32 consecutive rows of a panel column in one coalesced access. Per column
//                         two grid barriers: [GEMV + scale of column j-1, residual update, CTA argmax, per-CTA record]
//                         -> barrier -> [every CTA reduces the records in the same order, symmetric swap spread over the grid]
//                         -> barrier. dot and the running diagonal live in a small workspace (the swap exchanges two entries).
//   piv_llt_laswp_kernel  the block's transpositions applied in order to columns 0..k (nothing in the block reads them).
//   trailing update       the structured GEMM of that dtype (TRI_LOWER destination), as the unpivoted LLT does.
// A device record holds the status (0 running, 1 NonPositivePivot, 2 rank exit), its index, the transposition count and the
// pivot history; once it is set, later panel launches return at once. It is read back once, after the block loop. The initial
// scan's verdict is read back before the loop, so that an indefinite input is returned untouched.
#include <algorithm>
#include <climits>
#include <vector>

#include "ffi_common.cuh"
#include "panel_common.cuh"
#include "piv_common.cuh"
#include "runtime.cuh"
#include "scalar.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

constexpr int PIV_THREADS = 256;
constexpr int PIV_WARPS = PIV_THREADS / 32;
// Widest panel the kernel takes: larger block sizes are clamped to it (the pivots depend on the block size only through the
// rounding of the trailing updates).
constexpr int PIV_MAX_BS = 256;

// per-CTA argmax record, read by every CTA after the barrier
template <class R>
struct PivRec {
  R val;
  int idx;
  int nan;
};

template <class R>
struct PivWs {
  R* dot;                   // [n] running sum of |a(i, k..j)|^2 within the block
  R* dg;                    // [n] Re a(i, i) of the trailing rows (kept through the swaps)
  PivRec<R>* rec;           // [grid]
  unsigned long long* bar;  // grid barrier counter (zeroed before each launch)
  long long* status;        // [3]: state (0 running, 1 NonPositivePivot, 2 rank exit), index, transposition count
  long long* hist;          // [n] pivot row chosen at column j (j itself when no swap was made)
  R* tol;                   // eps * n * max Re a_ii
};

// (v2, i2) is the better candidate than (v1, i1): larger value, then smaller row. Candidates are positive; "none" is (0, INT_MAX),
// so the first maximum with strict `>` from (pvt = j, ajj = 0) is the reduction's result whatever the combination order.
template <class R>
__device__ __forceinline__ bool piv_better(R v2, int i2, R v1, int i1) { return v2 > v1 || (v2 == v1 && i2 < i1); }

template <class R>
__device__ __forceinline__ void piv_warp_reduce(R& v, int& i, int& nan) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const R v2 = __shfl_xor_sync(0xffffffffu, v, off);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, off);
    nan |= __shfl_xor_sync(0xffffffffu, nan, off);
    if (piv_better(v2, i2, v, i)) {
      v = v2;
      i = i2;
    }
  }
}

// Initial scan (factor.rs:86-101) and reset of the device record. One CTA.
template <class R, bool CX>
__global__ void __launch_bounds__(1024) piv_llt_init_kernel(const R* __restrict__ A, i64 rs, i64 cs, int n, PivWs<R> w) {
  constexpr int W = CX ? 2 : 1;
  __shared__ R s_max[32];
  __shared__ int s_bad[32];
  R mx = R(0);
  int bad = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const R v = A[W * ((i64)i * rs + (i64)i * cs)];
    if (v < R(0) || v != v) bad = 1;
    else if (v > mx) mx = v;
    w.hist[i] = i;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    bad |= __shfl_xor_sync(0xffffffffu, bad, off);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_max[warp] = mx;
    s_bad[warp] = bad;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < (int)(blockDim.x >> 5); ++q) {
      mx = fmax(mx, s_max[q]);
      bad |= s_bad[q];
    }
    w.status[0] = bad ? 1 : 0;
    w.status[1] = 0;
    w.status[2] = 0;
    *w.tol = mul_rn(mul_rn(TLim<R>::eps(), (R)n), mx);  // eps * n * max, left to right
  }
}

// One block of columns [k, k + bs) of the factorization; see the file comment for the per-column schedule.
template <class R, bool CX>
__global__ void __launch_bounds__(PIV_THREADS) piv_llt_panel_kernel(R* __restrict__ A, i64 rs, i64 cs, int n, int k, int bs,
                                                                    PivWs<R> w) {
  constexpr int W = CX ? 2 : 1;
  __shared__ R srow[W * PIV_MAX_BS];  // row j-1 of the panel, columns k..j-2
  __shared__ R red_v[PIV_WARPS];
  __shared__ int red_i[PIV_WARPS], red_nan[PIV_WARPS];
  __shared__ R s_ajj;
  __shared__ int s_pvt, s_nan;
  if (__ldcg(&w.status[0]) != 0) return;  // an earlier block failed or exited at its rank (uniform across the grid)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool leader = blockIdx.x == 0 && tid == 0;
  const i64 T = (i64)gridDim.x * PIV_THREADS;
  const i64 gt = (i64)blockIdx.x * PIV_THREADS + tid;
  const i64 g0 = (i64)k + gt;
  const R tol = __ldcg(w.tol);
  auto at = [&](i64 i, i64 j) { return A + W * (i * rs + j * cs); };
  unsigned long long target = 0;

  for (i64 i = g0; i < n; i += T) {
    w.dot[i] = R(0);
    w.dg[i] = __ldcg(at(i, i));
  }

  R ajj = R(0);  // pivot value of column j-1 (identical in every thread)
  for (int c = 0; c <= bs; ++c) {
    const int j = k + c;
    // ---- phase A: GEMV + scale of column j-1 (c > 0), residual update and argmax of column j (c < bs) ----
    if (c > 1) {
      for (int t = tid; t < c - 1; t += PIV_THREADS) {
        const R* p = at(j - 1, (i64)k + t);
        srow[W * t] = __ldcg(p);
        if (CX) srow[W * t + 1] = __ldcg(p + 1);
      }
      __syncthreads();
    }
    const R rinv = c > 0 ? R(1) / sqrt(ajj) : R(0);  // recip(sqrt(ajj)), factor.rs:172-185
    R bv = R(0);
    int bi = INT_MAX, nan = 0;
    for (i64 i = g0; i < n; i += T) {
      if (i < j) continue;
      R d;
      if (c > 0) {
        // a(i, j-1) -= a(i, k..j-1) * a(j-1, k..j-1)^H, then * recip(sqrt(ajj))
        R* x = at(i, j - 1);
        R xr = __ldcg(x), xi = CX ? __ldcg(x + 1) : R(0);
        R ar = R(0), ai = R(0);
        const R* Ai = at(i, k);
        for (int t = 0; t < c - 1; ++t) {
          const R* p = Ai + W * (i64)t * cs;
          const R pr = __ldcg(p);
          const R br = srow[W * t];
          ar = fma(pr, br, ar);
          if (CX) {
            const R pi = __ldcg(p + 1), bim = srow[W * t + 1];
            ar = fma(pi, bim, ar);
            ai = fma(pi, br, ai);
            ai = fma(-pr, bim, ai);
          }
        }
        xr = (xr - ar) * rinv;
        x[0] = xr;
        if (CX) {
          xi = (xi - ai) * rinv;
          x[1] = xi;
        }
        if (c == bs) continue;
        // dot[i] += |a(i, j-1)|^2; diag[i] = Re a(i,i) - dot[i]   (unfused, abs2 = re*re + im*im)
        const R a2 = CX ? add_rn(mul_rn(xr, xr), mul_rn(xi, xi)) : mul_rn(xr, xr);
        const R dd = add_rn(__ldcg(w.dot + i), a2);
        w.dot[i] = dd;
        d = sub_rn(__ldcg(w.dg + i), dd);
      } else {
        d = __ldcg(w.dg + i);
      }
      if (d != d) nan = 1;
      else if (d > bv) {  // rows ascend within a thread: strict `>` keeps the first maximum
        bv = d;
        bi = (int)i;
      }
    }
    if (c == bs) break;
    piv_warp_reduce(bv, bi, nan);
    if (lane == 0) {
      red_v[warp] = bv;
      red_i[warp] = bi;
      red_nan[warp] = nan;
    }
    __syncthreads();
    if (tid == 0) {
      for (int q = 1; q < PIV_WARPS; ++q) {
        nan |= red_nan[q];
        if (piv_better(red_v[q], red_i[q], bv, bi)) {
          bv = red_v[q];
          bi = red_i[q];
        }
      }
      PivRec<R>* r = w.rec + blockIdx.x;
      r->val = bv;
      r->idx = bi;
      r->nan = nan;
    }
    target += gridDim.x;
    grid_barrier(w.bar, target);

    // ---- phase B: the same reduction of the records in every CTA, then the symmetric swap ----
    if (warp == 0) {
      R v = R(0);
      int ix = INT_MAX, nn = 0;
      for (int b = lane; b < (int)gridDim.x; b += 32) {
        const PivRec<R>* r = w.rec + b;
        const R v2 = __ldcg(&r->val);
        const int i2 = __ldcg(&r->idx);
        nn |= __ldcg(&r->nan);
        if (piv_better(v2, i2, v, ix)) {
          v = v2;
          ix = i2;
        }
      }
      piv_warp_reduce(v, ix, nn);
      if (lane == 0) {
        s_ajj = v;
        s_pvt = ix == INT_MAX ? j : ix;
        s_nan = nn;
      }
    }
    __syncthreads();
    const int pvt = s_pvt;
    const R pj = s_ajj;
    if (s_nan) {  // factor.rs:110-115
      if (leader) {
        w.status[0] = 1;
        w.status[1] = j;
      }
      return;
    }
    if (j > 0 && pj < tol) {  // rank exit, factor.rs:121-125: the residual itself is stored
      if (leader) {
        R* p = at(j, j);
        p[0] = pj;
        if (CX) p[1] = R(0);
        w.status[0] = 2;
        w.status[1] = j;
      }
      return;
    }
    if (pvt != j) {
      // factor.rs:126-154. Rows j / pvt over columns k..j (columns 0..k: piv_llt_laswp_kernel), rows below pvt over columns
      // j / pvt, and the middle segment a(j+1..pvt, j) <-> conj(a(pvt, j+1..pvt)); one element pair per index.
      const i64 n_row = c, n_below = (i64)n - 1 - pvt, n_mid = (i64)pvt - j - 1;
      for (i64 e = gt; e < n_row + n_below + n_mid; e += T) {
        R *p, *q;
        bool cj = false;
        if (e < n_row) {
          p = at(j, (i64)k + e);
          q = at(pvt, (i64)k + e);
        } else if (e < n_row + n_below) {
          const i64 i = (i64)pvt + 1 + (e - n_row);
          p = at(i, j);
          q = at(i, pvt);
        } else {
          const i64 i = (i64)j + 1 + (e - n_row - n_below);
          p = at(i, j);
          q = at(pvt, i);
          cj = true;
        }
        const R pr = __ldcg(p), qr = __ldcg(q);
        p[0] = qr;
        q[0] = pr;
        if (CX) {
          const R pi = __ldcg(p + 1), qi = __ldcg(q + 1);
          p[1] = cj ? -qi : qi;
          q[1] = cj ? -pi : pi;
        }
      }
      if (leader) {
        R* d_j = at(j, j);
        R* d_p = at(pvt, pvt);
        d_p[0] = __ldcg(d_j);  // a(pvt, pvt) = a(j, j), in that direction only
        if (CX) {
          d_p[1] = __ldcg(d_j + 1);
          R* o = at(pvt, j);
          o[1] = -__ldcg(o + 1);  // a(pvt, j) = conj(a(pvt, j))
        }
        const R t = __ldcg(w.dot + j);
        w.dot[j] = __ldcg(w.dot + pvt);
        w.dot[pvt] = t;
        w.dg[pvt] = __ldcg(w.dg + j);
        w.hist[j] = pvt;
        w.status[2] += 1;
      }
    }
    if (leader) {
      R* p = at(j, j);
      p[0] = sqrt(pj);
      if (CX) p[1] = R(0);
    }
    ajj = pj;
    target += gridDim.x;
    grid_barrier(w.bar, target);
  }
}

// Rows swapped at columns k..k+bs, applied in order to columns 0..k (one thread per column).
template <class R, bool CX>
__global__ void __launch_bounds__(256) piv_llt_laswp_kernel(R* __restrict__ A, i64 rs, i64 cs, int k, int bs,
                                                            const long long* __restrict__ hist) {
  constexpr int W = CX ? 2 : 1;
  const i64 c = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= k) return;
  for (int t = k; t < k + bs; ++t) {
    const i64 p = hist[t];
    if (p == t) continue;
    R* a = A + W * ((i64)t * rs + c * cs);
    R* b = A + W * (p * rs + c * cs);
#pragma unroll
    for (int e = 0; e < W; ++e) {
      const R x = a[e];
      a[e] = b[e];
      b[e] = x;
    }
  }
}

// dst[i, :] = src[perm[i], :]
template <class R, bool CX>
__global__ void piv_gather_rows_kernel(R* __restrict__ dst, i64 drs, i64 dcs, const R* __restrict__ src, i64 srs, i64 scs, i64 n,
                                       i64 ncols, const long long* __restrict__ perm) {
  constexpr int W = CX ? 2 : 1;
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * ncols) return;
  const i64 i = e % n, c = e / n;
  const R* q = src + W * (perm[i] * srs + c * scs);
  R* p = dst + W * (i * drs + c * dcs);
#pragma unroll
  for (int t = 0; t < W; ++t) p[t] = q[t];
}

// out(i, j), i >= j: tmp(p[i], p[j]) if p[i] >= p[j], else conj(tmp(p[j], p[i]))  (reconstruct.rs:40-51, inverse.rs:42-53).
// Only the lower triangle of tmp is read and only the lower triangle of out is written.
template <class R, bool CX>
__global__ void piv_sym_gather_kernel(R* __restrict__ out, i64 ors, i64 ocs, const R* __restrict__ tmp, i64 ld, i64 n,
                                      const long long* __restrict__ p) {
  constexpr int W = CX ? 2 : 1;
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * n) return;
  const i64 i = e % n, j = e / n;
  if (i < j) return;
  const i64 ii = p[i], jj = p[j];
  const bool direct = ii >= jj;
  const R* q = direct ? tmp + W * (ii + jj * ld) : tmp + W * (jj + ii * ld);
  R* o = out + W * (i * ors + j * ocs);
  o[0] = q[0];
  if (CX) o[1] = direct ? q[1] : -q[1];
}

// dst(i, j) = src(i, j) over an m x n block (strided views in units of the scalar kind)
template <class R, bool CX>
__global__ void piv_copy_kernel(R* __restrict__ dst, i64 drs, i64 dcs, const R* __restrict__ src, i64 srs, i64 scs, i64 m, i64 n) {
  constexpr int W = CX ? 2 : 1;
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m * n) return;
  const i64 i = e % m, j = e / m;
  const R* q = src + W * (i * srs + j * scs);
  R* p = dst + W * (i * drs + j * dcs);
  p[0] = q[0];
  if (CX) p[1] = q[1];
}

// tmp(lower) = L L^H (reconstruct) or L^-H L^-1 (inverse): the unpivoted compositions
template <class R, bool CX>
void piv_llt_product(cudaStream_t st, View<R> tmp, View<const R> L, bool inverse) {
  if (inverse) llt_inverse_t<R, CX>(st, tmp, L);
  else llt_reconstruct_t<R, CX>(st, tmp, L);
}

}  // namespace

// ---- piv_common.cuh: the one entry to the kernels above, for this file and the other pivoted factorizations ----
template <class R, bool CX>
void piv_laswp_t(cudaStream_t st, View<R> A, i64 k, i64 nt, const long long* hist) {
  if (k == 0 || nt == 0) return;
  piv_llt_laswp_kernel<R, CX><<<grid_1d(k), 256, 0, st>>>(A.ptr, A.rs, A.cs, (int)k, (int)nt, hist);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}
template <class R, bool CX>
void piv_gather_rows_t(cudaStream_t st, View<R> dst, View<const R> src, const long long* perm) {
  const i64 n = dst.nrows, k = dst.ncols;
  if (n == 0 || k == 0) return;
  piv_gather_rows_kernel<R, CX><<<grid_1d(n * k), 256, 0, st>>>(dst.ptr, dst.rs, dst.cs, src.ptr, src.rs, src.cs, n, k, perm);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}
template <class R, bool CX>
void piv_sym_gather_t(cudaStream_t st, View<R> out, const R* tmp, i64 ld, const long long* p) {
  const i64 n = out.nrows;
  if (n == 0) return;
  piv_sym_gather_kernel<R, CX><<<grid_1d(n * n), 256, 0, st>>>(out.ptr, out.rs, out.cs, tmp, ld, n, p);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}
template <class R, bool CX>
void piv_copy_t(cudaStream_t st, View<R> dst, View<const R> src) {
  const i64 m = dst.nrows, n = dst.ncols;
  if (m == 0 || n == 0) return;
  piv_copy_kernel<R, CX><<<grid_1d(m * n), 256, 0, st>>>(dst.ptr, dst.rs, dst.cs, src.ptr, src.rs, src.cs, m, n);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}
#define FB_PIV_COMMON_INST(R, CX)                                                                          \
  template void piv_laswp_t<R, CX>(cudaStream_t, View<R>, i64, i64, const long long*);                      \
  template void piv_gather_rows_t<R, CX>(cudaStream_t, View<R>, View<const R>, const long long*);           \
  template void piv_sym_gather_t<R, CX>(cudaStream_t, View<R>, const R*, i64, const long long*);            \
  template void piv_copy_t<R, CX>(cudaStream_t, View<R>, View<const R>);
FB_PIV_COMMON_INST(double, false)
FB_PIV_COMMON_INST(float, false)
FB_PIV_COMMON_INST(double, true)
FB_PIV_COMMON_INST(float, true)
#undef FB_PIV_COMMON_INST

struct PivLltResult {
  int state;  // 0 Ok, 1 NonPositivePivot
  i64 index;  // the failing column, or the rank
  i64 transposition_count;
};

// In-place pivoted Cholesky of the lower triangle of A (views in element units of the scalar kind; complex: COMPLEX units on an
// R* base). trans (host) receives the transpositions made: n entries, or none on a NonPositivePivot { index: 0 }.
template <class R, bool CX>
PivLltResult piv_llt_in_place_t(cudaStream_t st, View<R> A, i64 block_size, std::vector<long long>& trans) {
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n, "pivoted LLT needs a square matrix");
  FB_ASSERT(block_size > 0, "PivLltParams.block_size must be positive");
  FB_ASSERT(n < (i64)INT_MAX, "pivoted LLT: dimension too large");
  trans.clear();
  PivLltResult res{0, n, 0};
  if (n == 0) return res;
  const int bs = (int)std::min<i64>(block_size, PIV_MAX_BS);
  const int sms = stream_sms(st);
  int occ = 0;
  FB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, piv_llt_panel_kernel<R, CX>, PIV_THREADS, 0));
  FB_ASSERT(occ > 0, "pivoted LLT panel kernel cannot be resident");
  const int gmax = std::min(sms, sms * occ);

  const size_t rec_bytes = (size_t)gmax * sizeof(PivRec<R>);
  const size_t bytes = 2 * (size_t)n * sizeof(R) + rec_bytes + (size_t)(n + 4) * 8 + 2 * sizeof(R) + 256;
  char* buf = (char*)ws_alloc(bytes);
  PivWs<R> w;
  w.hist = (long long*)buf;
  w.status = w.hist + n;
  w.bar = (unsigned long long*)(w.status + 3);
  w.rec = (PivRec<R>*)(((uintptr_t)(w.bar + 1) + 15) & ~(uintptr_t)15);
  w.dot = (R*)((char*)w.rec + rec_bytes);
  w.dg = w.dot + n;
  w.tol = w.dg + n;

  piv_llt_init_kernel<R, CX><<<1, 1024, 0, st>>>(A.ptr, A.rs, A.cs, (int)n, w);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  long long h_status[3];
  FB_CUDA_CHECK(cudaMemcpyAsync(h_status, w.status, sizeof(h_status), cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (h_status[0] != 0) {  // a negative or NaN diagonal entry: NonPositivePivot { index: 0 }, A untouched
    ws_free(buf);
    return PivLltResult{1, 0, 0};
  }

  for (i64 k = 0; k < n; k += bs) {
    const int b = (int)std::min<i64>(bs, n - k);
    const int G = (int)std::min<i64>(gmax, (n - k + PIV_THREADS - 1) / PIV_THREADS);
    FB_CUDA_CHECK(cudaMemsetAsync(w.bar, 0, sizeof(unsigned long long), st));
    {
      R* Ap = A.ptr;
      i64 rs = A.rs, cs = A.cs;
      int ni = (int)n, ki = (int)k, bi = b;
      void* args[] = {&Ap, &rs, &cs, &ni, &ki, &bi, &w};
      FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)piv_llt_panel_kernel<R, CX>, dim3(G), dim3(PIV_THREADS), args, 0, st));
      note_launch();
    }
    piv_laswp_t<R, CX>(st, A, k, b, w.hist);
    if (k + b < n) {
      const i64 m = n - k - b;
      const View<const R> P = cview(sub_t<R, CX>(A, k + b, k, m, b));  // A22(lower) -= P P^H
      gemm_t<R, CX>(st, sub_t<R, CX>(A, k + b, k + b, m, m), TRI_LOWER, 1, P, RECT, false, P.t(), RECT, true, R(-1));
    }
  }

  trans.resize((size_t)n);
  FB_CUDA_CHECK(cudaMemcpyAsync(h_status, w.status, sizeof(h_status), cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(trans.data(), w.hist, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(buf);
  res.transposition_count = h_status[2];
  if (h_status[0] == 1) {
    res.state = 1;
    res.index = h_status[1];
  } else if (h_status[0] == 2) {
    res.index = h_status[1];
  }
  return res;
}

// rhs <- A^-1 rhs from the factor: rows permuted by perm_fwd, L and L^H solves under A_conj, rows permuted back (solve.rs:13-41).
// perm / perm_inv: host int64[n].
template <class R, bool CX>
void piv_llt_solve_t(cudaStream_t st, View<const R> L, const long long* perm, const long long* perm_inv, bool conj, View<R> rhs) {
  constexpr int W = CX ? 2 : 1;
  const i64 n = L.nrows, k = rhs.ncols;
  FB_ASSERT(L.ncols == n && rhs.nrows == n, "pivoted LLT solve shape mismatch");
  if (n == 0 || k == 0) return;
  long long* d_p = (long long*)ws_alloc((size_t)n * 16);
  R* tmp = (R*)ws_alloc((size_t)n * (size_t)k * W * sizeof(R));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p, perm, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p + n, perm_inv, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  View<R> X{tmp, n, k, 1, n};
  piv_gather_rows_t<R, CX>(st, X, View<const R>{rhs.ptr, n, k, rhs.rs, rhs.cs}, d_p);
  llt_solve_t<R, CX>(st, L, conj, X);
  piv_gather_rows_t<R, CX>(st, rhs, View<const R>{tmp, n, k, 1, n}, d_p + n);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));  // the host permutations and the pool buffers are released below
  ws_free(tmp);
  ws_free(d_p);
}

// out(lower) <- P^T (L L^H) P (reconstruct) or P^T (L^-H L^-1) P (inverse), the strict upper triangle untouched.
// perm_inv: host int64[n].
template <class R, bool CX>
void piv_llt_recon_t(cudaStream_t st, View<R> out, View<const R> L, const long long* perm_inv, bool inverse) {
  constexpr int W = CX ? 2 : 1;
  const i64 n = L.nrows;
  FB_ASSERT(L.ncols == n && out.nrows == n && out.ncols == n, "pivoted LLT reconstruct / inverse shape mismatch");
  if (n == 0) return;
  long long* d_p = (long long*)ws_alloc((size_t)n * 8);
  R* tmp = (R*)ws_alloc((size_t)n * (size_t)n * W * sizeof(R));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p, perm_inv, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  piv_llt_product<R, CX>(st, View<R>{tmp, n, n, 1, n}, L, inverse);
  piv_sym_gather_t<R, CX>(st, out, tmp, n, d_p);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(tmp);
  ws_free(d_p);
}

}  // namespace fb

// ---- C ABI (faer-ffi/src/lib.rs:1076-1186; declarations in include/faer_b200_piv_llt.h) ----
using namespace fb;

namespace {

template <class R, bool CX>
FaerV0_24_PivLltStatus piv_llt_factor_entry(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd,
                                            FaerV0_24_PivLltParams params, int idx_bytes) {
  FB_ENTRY();
  FB_ASSERT(params.block_size > 0, "PivLltParams.block_size must be positive (the reference would not terminate)");
  FB_ASSERT(A.nrows == A.ncols, "pivoted LLT needs a square matrix");
  // the permutation length is A.nrows, never SliceMut.len (see lu_entry in ffi.cu)
  FB_ASSERT(A.nrows == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  cudaStream_t st = current_stream();
  StagedMat a = stage<R, CX>(A, true, st);
  std::vector<long long> trans, fwd, bwd;
  const PivLltResult r = piv_llt_in_place_t<R, CX>(st, a.view<R>(), (i64)params.block_size, trans);
  finish_all(st, {&a});
  perm_from_transpositions(A.nrows, trans, fwd, bwd);
  FaerV0_24_PivLltStatus out;
  memset(&out, 0, sizeof(out));
  write_perm(perm_fwd.ptr, fwd, idx_bytes);
  if (r.state == 1) {
    out.tag = FaerV0_24_PivLltStatus_NonPositivePivot;
    out.non_positive_pivot.index = (size_t)r.index;
    return out;
  }
  write_perm(perm_bwd.ptr, bwd, idx_bytes);
  out.tag = FaerV0_24_PivLltStatus_Ok;
  out.ok.rank = (size_t)r.index;
  out.ok.transposition_count = (size_t)r.transposition_count;
  return out;
}

template <class R, bool CX>
void piv_llt_solve_entry(FaerV0_24_MatRef L, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd, FaerV0_24_Conj A_conj,
                         FaerV0_24_MatMut rhs, int idx_bytes) {
  FB_ENTRY();
  FB_ASSERT(L.nrows == L.ncols && rhs.nrows == L.nrows, "pivoted LLT solve shape mismatch");
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  std::vector<long long> pf = read_perm_checked(perm_fwd, n, idx_bytes), pb = read_perm_checked(perm_bwd, n, idx_bytes);
  StagedMat l = stage<R, CX>(L, st);
  StagedMat r = stage<R, CX>(rhs, true, st);
  piv_llt_solve_t<R, CX>(st, l.view<const R>(), pf.data(), pb.data(), A_conj == FaerV0_24_Conj_Yes, r.view<R>());
  finish_all(st, {&l, &r});
}

template <class R, bool CX>
void piv_llt_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_SliceRef perm_bwd, int idx_bytes, bool inverse) {
  FB_ENTRY();
  FB_ASSERT(L.nrows == L.ncols && A.nrows == L.nrows && A.ncols == L.nrows, "pivoted LLT reconstruct / inverse shape mismatch");
  cudaStream_t st = current_stream();
  const size_t n = L.nrows;
  std::vector<long long> pb = read_perm_checked(perm_bwd, n, idx_bytes);
  // only the lower triangle is written: the rest of A must survive the round trip
  StagedMat a = stage<R, CX>(A, true, st);
  StagedMat l = stage<R, CX>(L, st);
  piv_llt_recon_t<R, CX>(st, a.view<R>(), l.view<const R>(), pb.data(), inverse);
  finish_all(st, {&a, &l});
}

}  // namespace

extern "C" {

// Scratch layouts are the reference's (factor.rs:36-45, solve.rs:4-11, reconstruct.rs:4-10, inverse.rs:4-11); the GPU paths
// keep their workspace in the device pool and ignore `mem`.
#define FB_PIV_LLT_FFI(SUF, R, CX, IT, BYTES)                                                                                        \
  FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par,                          \
                                                                              FaerV0_24_PivLltParams params) {                        \
    (void)par; (void)params;                                                                                                         \
    return FaerV0_24_Layout{dim * 2 * sizeof(R), 64}; /* temp_mat_scratch::<Real>(dim, 2) */                                          \
  }                                                                                                                                  \
  FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_SliceMut perm_fwd,          \
                                                                            FaerV0_24_SliceMut perm_bwd, FaerV0_24_Par par,          \
                                                                            FaerV0_24_MemAlloc mem, FaerV0_24_PivLltParams params) { \
    (void)par; (void)mem;                                                                                                            \
    return piv_llt_factor_entry<R, CX>(A, perm_fwd, perm_bwd, params, BYTES);                                                        \
  }                                                                                                                                  \
  FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {       \
    (void)par;                                                                                                                       \
    return FaerV0_24_Layout{dim * rhs_ncols * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, rhs_ncols) */              \
  }                                                                                                                                  \
  void libfaer_v0_23_piv_llt_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef L, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd, \
                                                         FaerV0_24_Conj A_conj, FaerV0_24_MatMut rhs, FaerV0_24_Par par,               \
                                                         FaerV0_24_MemAlloc mem) {                                                   \
    (void)par; (void)mem;                                                                                                            \
    piv_llt_solve_entry<R, CX>(L, perm_fwd, perm_bwd, A_conj, rhs, BYTES);                                                           \
  }                                                                                                                                  \
  FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                           \
    (void)par;                                                                                                                       \
    return FaerV0_24_Layout{dim * dim * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, dim) */                          \
  }                                                                                                                                  \
  void libfaer_v0_23_piv_llt_reconstruct_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_SliceRef perm_fwd,            \
                                                      FaerV0_24_SliceRef perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {        \
    (void)perm_fwd; (void)par; (void)mem;                                                                                            \
    piv_llt_recon_entry<R, CX>(A, L, perm_bwd, BYTES, false);                                                                        \
  }                                                                                                                                  \
  FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                               \
    (void)par;                                                                                                                       \
    return FaerV0_24_Layout{dim * dim * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, dim) */                          \
  }                                                                                                                                  \
  void libfaer_v0_23_piv_llt_inverse_##IT##_##SUF(FaerV0_24_MatMut A_inv, FaerV0_24_MatRef L, FaerV0_24_SliceRef perm_fwd,           \
                                                  FaerV0_24_SliceRef perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {            \
    (void)perm_fwd; (void)par; (void)mem;                                                                                            \
    piv_llt_recon_entry<R, CX>(A_inv, L, perm_bwd, BYTES, true);                                                                     \
  }
#define FB_PIV_LLT_DTYPE(SUF, R, CX)                                                                             \
  FaerV0_24_PivLltParams libfaer_v0_23_PivLltParams_##SUF(void) { return FaerV0_24_PivLltParams{128}; } /* factor.rs:12-20 */ \
  FB_PIV_LLT_FFI(SUF, R, CX, u32, 4)                                                                             \
  FB_PIV_LLT_FFI(SUF, R, CX, u64, 8)
FB_PIV_LLT_DTYPE(f64, double, false)
FB_PIV_LLT_DTYPE(f32, float, false)
FB_PIV_LLT_DTYPE(c64, double, true)
FB_PIV_LLT_DTYPE(c32, float, true)
#undef FB_PIV_LLT_DTYPE
#undef FB_PIV_LLT_FFI

}  // extern "C"
