// Column-pivoted Householder QR (faer's `qr::col_pivoting`) for f64 / f32 / c64 / c32: factor, solves, reconstruct, inverse,
// and their C ABI (include/faer_b200_colpiv_qr.h, included by include/faer_b200.h: `libfaer_v0_23_colpiv_qr_*`).
//
// Reference: faer/src/linalg/qr/col_pivoting/factor.rs:112-388 (factor), solve.rs:52-184, reconstruct.rs:16-45,
// inverse.rs:16-50. The factorization follows the reference's operation sequence, so the permutation and the transposition
// count match it wherever the pivots are separated by more than rounding:
//   * column norms (faer's scaled three-accumulator norm_l2), A scaled by recip(best) (an all-zero A becomes NaN, as in the
//     reference), the upper trapezoid scaled back by best at the end;
//   * per column k: pivot = first maximum of the downdated norms (strict `>`); the update of the previous reflector is delayed
//     iff k > 0, the CALLER's row stride is 1 and the pivot norm is >= sqrt(eps) * (the maximum of the last recompute);
//     otherwise that update is applied to the whole trailing block and the norms are recomputed (factor.rs:170-195);
//   * column swap; the pending update of the pivot column; make_householder_in_place (tau = (1 + |v|^2) / 2, +inf for a
//     zero tail);
//   * delayed step (update_mat_and_dot_simd, factor.rs:7-90): one pass over the trailing block that applies the previous
//     reflector's pending update, accumulates v_k^H dst and writes dst back; then per column d0 = -(a_kj + l dot_j + acc) / tau,
//     a_kj += ..., dot_j = d0, norm_j = sqrt(norm_j^2 - |a_kj|^2). Otherwise the GEMV form (factor.rs:286-303).
// Afterwards the T blocks of Q_coeff (block_size = Q_coeff.nrows) are built as qr_factor_in_place lays them out
// (factor.rs:367-386).
//
// GPU mapping: the whole column loop is ONE persistent cooperative kernel (colpiv_qr_kernel). The trailing block is walked by
// warps, a warp on 32 consecutive rows of one column at a time (coalesced); when fewer trailing columns remain than warps
// (tall inputs, the last columns) every column is also split into row segments. Partial sums go to per-(column, segment)
// records and are combined in segment order, so the result is the same bits from run to run. Per column:
//   [pivot choice in every CTA from the same norms -> uniform branch; recompute pass + barrier if not delayed]
//   P1 swap + pending update of the pivot column + partial tail norms   -> barrier
//   P2 reflector scalars (every CTA, same records, same order), tail scaling -> barrier
//   T  fused trailing pass (delayed) or v_k^H B11 (GEMV form)            -> barrier
//   F  per-column finish: a_kj, dot_j, norm_j                              -> barrier
// The algorithm is BLAS-2: each column reads and writes the trailing block once, so the kernel is HBM-bound.
#include <algorithm>
#include <climits>
#include <vector>

#include "ffi_common.cuh"
#include "panel_common.cuh"
#include "piv_common.cuh"
#include "pivot_record.cuh"
#include "runtime.cuh"
#include "scalar.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

constexpr int CPQ_THREADS = 256;
constexpr int CPQ_WARPS = CPQ_THREADS / 32;
constexpr int CPQ_MIN_SEG = 256;  // shortest row segment of a split column
constexpr int CPQ_REC = 4;        // stride of a partial record (3 norm accumulators, or one scalar)

template <class R, bool CX>
__device__ __forceinline__ void acc_norm(NormAcc<R>& a, Sc<R> x) {
  a.add(x.re, TLim<R>::sqrt_min(), TLim<R>::sqrt_max());
  if (CX) a.add(x.im, TLim<R>::sqrt_min(), TLim<R>::sqrt_max());
}
template <class R>
__device__ __forceinline__ R acc_value(R s, R m, R b) {
  return norm_from_acc(s, m, b, TLim<R>::sqrt_min(), TLim<R>::sqrt_max());
}

template <class R>
struct CpqWs {
  R* norm;                  // [n]
  R* dot;                   // [W n]
  R* tau;                   // [size]
  int* hist;                // [size] pivot column chosen at step k
  R* part;                  // [(n + warps) * CPQ_REC] per-(column, segment) partial records
  R* rec;                   // [grid * PANEL_NV] per-CTA records of the pivot column's tail norm
  unsigned long long* bar;  // grid barrier counter (zeroed before the launch)
};

// work split of a column pass over `nc` columns of `nr` rows: S row segments per column, `seg` rows each (a multiple of 32)
struct Split {
  int S;
  i64 seg;
};
__device__ __forceinline__ Split make_split(i64 nc, i64 nr, int warps) {
  Split s;
  s.S = 1;
  if (nc > 0 && nc < warps) s.S = (int)min((i64)(warps / nc), max((i64)1, nr / CPQ_MIN_SEG));
  s.seg = ((nr + s.S - 1) / s.S + 31) / 32 * 32;
  return s;
}

// CTA-wide first maximum by pivot_record.cuh's `better` on (norm, column), "none" = (0, INT_MAX): the reference's first maximum
// with strict `>` from 0 (factor.rs:161-169, 186-193); a norm of exactly 0 or NaN is never chosen, and "none" leaves the caller's
// default. Every thread gets the result.
template <class R>
__device__ __forceinline__ void cta_argmax(R& v, int& i, R* sv, int* si) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const R v2 = __shfl_xor_sync(0xffffffffu, v, off);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, off);
    if (better(v2, i2, v, i)) {
      v = v2;
      i = i2;
    }
  }
  __syncthreads();  // sv / si may still be read by a previous call
  if (lane == 0) {
    sv[warp] = v;
    si[warp] = i;
  }
  __syncthreads();
  v = sv[0];
  i = si[0];
  for (int q = 1; q < CPQ_WARPS; ++q)
    if (better(sv[q], si[q], v, i)) {
      v = sv[q];
      i = si[q];
    }
}

// the norm of column j from its S partial records
template <class R>
__device__ __forceinline__ R combine_norm(const R* part, i64 u0, int S) {
  R s = R(0), m = R(0), b = R(0);
  for (int q = 0; q < S; ++q) {
    const R* p = part + (u0 + q) * CPQ_REC;
    s += __ldcg(p);
    m += __ldcg(p + 1);
    b += __ldcg(p + 2);
  }
  return acc_value(s, m, b);
}

// The whole factorization of the (scaled, column-major, leading dimension ld) m x n matrix; see the file comment.
template <class R, bool CX>
__global__ void __launch_bounds__(CPQ_THREADS) colpiv_qr_kernel(R* __restrict__ A, i64 ld, int m, int n, int rs1, CpqWs<R> w) {
  constexpr int W = CX ? 2 : 1;
  __shared__ R s_v[CPQ_WARPS];
  __shared__ int s_i[CPQ_WARPS];
  __shared__ R s_fin[CPQ_WARPS * PANEL_NV];
  __shared__ R s_tail[PANEL_NV];
  const int size = min(m, n);
  const int tid = threadIdx.x, lane = tid & 31;
  const int G = gridDim.x;
  const int warps = G * CPQ_WARPS;
  const int gw = blockIdx.x * CPQ_WARPS + (tid >> 5);
  const i64 T = (i64)G * CPQ_THREADS;
  const i64 gt = (i64)blockIdx.x * CPQ_THREADS + tid;
  const bool leader = blockIdx.x == 0 && tid == 0;
  auto at = [&](i64 i, i64 j) { return A + W * (i + j * ld); };
  unsigned long long target = 0;
  auto barrier = [&]() {
    target += G;
    grid_barrier(w.bar, target);
  };

  // ---- initial norms (factor.rs:142-150) and scaling (151-158) ----
  {
    const Split sp = make_split(n, m, warps);
    for (i64 u = gw; u < (i64)n * sp.S; u += warps) {
      const i64 j = u / sp.S, lo = (u % sp.S) * sp.seg, hi = min((i64)m, lo + sp.seg);
      NormAcc<R> a{R(0), R(0), R(0)};
      for (i64 i = lo + lane; i < hi; i += 32) acc_norm<R, CX>(a, sc_ld<R, CX>(at(i, j)));
      a.s = warp_sum(a.s);
      a.m = warp_sum(a.m);
      a.b = warp_sum(a.b);
      if (lane == 0) {
        R* p = w.part + u * CPQ_REC;
        p[0] = a.s;
        p[1] = a.m;
        p[2] = a.b;
      }
    }
  }
  barrier();
  R best;
  {
    const Split sp = make_split(n, m, warps);
    R v = R(0);
    int ix = INT_MAX;
    for (int j = tid; j < n; j += CPQ_THREADS) {
      const R val = combine_norm(w.part, (i64)j * sp.S, sp.S);
      if (better(val, j, v, ix)) {
        v = val;
        ix = j;
      }
    }
    cta_argmax(v, ix, s_v, s_i);
    best = v;  // the maximum (0 if every norm is 0 or NaN)
  }
  const R scale_fwd = best;
  const R scale_bwd = R(1) / best;
  if (blockIdx.x == 0) {
    const Split sp = make_split(n, m, warps);
    for (int j = tid; j < n; j += CPQ_THREADS) w.norm[j] = combine_norm(w.part, (i64)j * sp.S, sp.S) * scale_bwd;
  }
  for (i64 j = gw; j < n; j += warps)
    for (i64 i = lane; i < m; i += 32) {
      R* p = at(i, j);
      p[0] *= scale_bwd;
      if (CX) p[1] *= scale_bwd;
    }
  best = best * scale_bwd;
  const R threshold = sqrt(TLim<R>::eps());
  R best_threshold = best * threshold;
  barrier();

  for (int k = 0; k < size; ++k) {
    // ---- pivot choice (factor.rs:161-172), identical in every CTA ----
    R new_best = R(0);
    int best_col = INT_MAX;
    for (int j = k + tid; j < n; j += CPQ_THREADS) {
      const R val = __ldcg(w.norm + j);
      if (better(val, j, new_best, best_col)) {
        new_best = val;
        best_col = j;
      }
    }
    cta_argmax(new_best, best_col, s_v, s_i);
    if (best_col == INT_MAX) best_col = k;
    const bool delayed = rs1 && k > 0 && new_best >= best_threshold;

    if (k > 0 && !delayed) {
      // ---- A11 += v_{k-1} dot[k..], exact norms of the trailing columns (factor.rs:173-195) ----
      const i64 nc = n - k, nr = m - k;
      const Split sp = make_split(nc, nr, warps);
      for (i64 u = gw; u < nc * sp.S; u += warps) {
        const i64 j = k + u / sp.S, lo = k + (u % sp.S) * sp.seg, hi = min((i64)m, lo + sp.seg);
        const Sc<R> d = sc_ld<R, CX>(w.dot + W * j);
        NormAcc<R> a{R(0), R(0), R(0)};
        for (i64 i = lo + lane; i < hi; i += 32) {
          R* p = at(i, j);
          const Sc<R> x = mul_add<R, CX>(sc_ld<R, CX>(at(i, k - 1)), d, sc_ld<R, CX>(p));
          sc_st<R, CX>(p, x);
          acc_norm<R, CX>(a, x);
        }
        a.s = warp_sum(a.s);
        a.m = warp_sum(a.m);
        a.b = warp_sum(a.b);
        if (lane == 0) {
          R* p = w.part + u * CPQ_REC;
          p[0] = a.s;
          p[1] = a.m;
          p[2] = a.b;
        }
      }
      barrier();
      R v = R(0);
      int ix = INT_MAX;
      for (int j = k + tid; j < n; j += CPQ_THREADS) {
        const R val = combine_norm(w.part, (i64)(j - k) * sp.S, sp.S);
        if (blockIdx.x == 0) w.norm[j] = val;
        if (better(val, j, v, ix)) {
          v = val;
          ix = j;
        }
      }
      cta_argmax(v, ix, s_v, s_i);
      best = v;
      if (ix != INT_MAX) best_col = ix;  // no exact norm > 0: best_col keeps the first scan's choice (factor.rs:185-193)
      best_threshold = best * threshold;
    }

    // ---- P1: swap columns k / best_col, pending update of the pivot column, partial tail norms ----
    const Sc<R> r = sc_ld<R, CX>(w.dot + W * best_col);  // dot[k] after the swap
    NormAcc<R> a{R(0), R(0), R(0)};
    for (i64 i = gt; i < m; i += T) {
      R* pk = at(i, k);
      Sc<R> x = sc_ld<R, CX>(pk);
      if (best_col != k) {
        R* pb = at(i, best_col);
        const Sc<R> y = sc_ld<R, CX>(pb);
        sc_st<R, CX>(pb, x);
        x = y;
      }
      if (i >= k && delayed) x = mul_add<R, CX>(r, sc_ld<R, CX>(at(i, k - 1)), x);
      sc_st<R, CX>(pk, x);
      if (i > k) acc_norm<R, CX>(a, x);
    }
    {
      const R vals[3] = {a.s, a.m, a.b};
      block_publish_n<R, 3, CPQ_WARPS>(vals, s_fin, w.rec + (i64)blockIdx.x * PANEL_NV);
    }
    barrier();

    // ---- P2: make_householder_in_place (householder.rs:59-107) from the same records in every CTA ----
    if (tid < 32) {
      R out[3];
      reduce_partials<R, 3>(w.rec, G, out);
      if (tid == 0) s_tail[0] = acc_value(out[0], out[1], out[2]);
    }
    __syncthreads();
    const R tail_norm = s_tail[0];
    Sc<R> head = sc_ld<R, CX>(at(k, k));
    R head_norm = CX ? hypot(head.re, head.im) : fabs(head.re);
    if (head_norm < TLim<R>::min_pos()) {
      head = Sc<R>{R(0), R(0)};
      head_norm = R(0);
    }
    R tau;
    Sc<R> inv{R(0), R(0)}, new_head = head;
    const bool no_tail = tail_norm < TLim<R>::min_pos();
    if (no_tail) {
      tau = TLim<R>::inf();
    } else {
      const R nrm = hypot(head_norm, tail_norm);
      const Sc<R> sign = head_norm != R(0) ? scale<R, CX>(head, R(1) / head_norm) : Sc<R>{R(1), R(0)};
      const Sc<R> sn = scale<R, CX>(sign, nrm);
      const Sc<R> hb = cadd<R, CX>(head, sn);
      if (CX) {
        const R den = hb.re * hb.re + hb.im * hb.im;
        inv = Sc<R>{hb.re / den, -hb.im / den};
      } else {
        inv = Sc<R>{R(1) / hb.re, R(0)};
      }
      new_head = Sc<R>{-sn.re, -sn.im};
      const R t = tail_norm * (CX ? hypot(inv.re, inv.im) : fabs(inv.re));
      tau = R(0.5) * (R(1) + t * t);
    }
    if (!no_tail)
      for (i64 i = gt; i < m; i += T)
        if (i > k) sc_st<R, CX>(at(i, k), cmul<R, CX>(sc_ld<R, CX>(at(i, k)), inv));
    if (leader) {
      w.tau[k] = tau;
      w.hist[k] = best_col;
      if (best_col != k) {
        for (int e = 0; e < W; ++e) {
          const R t0 = w.dot[W * k + e];
          w.dot[W * k + e] = w.dot[W * best_col + e];
          w.dot[W * best_col + e] = t0;
        }
        const R t1 = w.norm[k];
        w.norm[k] = w.norm[best_col];
        w.norm[best_col] = t1;
      }
    }
    const R tau_inv = R(1) / tau;
    const Sc<R> l = delayed ? sc_ld<R, CX>(at(k, k - 1)) : Sc<R>{R(0), R(0)};  // row k of column k-1: not written in P1 / P2
    barrier();
    if (leader) sc_st<R, CX>(at(k, k), new_head);  // beta; every CTA has read the old head before the barrier

    if (k + 1 == size) {
      // factor.rs:231-240: the last reflector; the pending update reaches row k of the remaining columns only
      if (delayed)
        for (i64 j = k + 1 + gt; j < n; j += T) {
          R* p = at(k, j);
          sc_st<R, CX>(p, mul_add<R, CX>(l, sc_ld<R, CX>(w.dot + W * j), sc_ld<R, CX>(p)));
        }
      break;
    }

    // ---- T: one pass over B11 = A[k+1.., k+1..] ----
    const i64 nc = n - k - 1, nr = m - k - 1;
    const Split sp = make_split(nc, nr, warps);
    for (i64 u = gw; u < nc * sp.S; u += warps) {
      const i64 j = k + 1 + u / sp.S, lo = k + 1 + (u % sp.S) * sp.seg, hi = min((i64)m, lo + sp.seg);
      Sc<R> acc{R(0), R(0)};
      if (delayed) {
        // update_mat_and_dot_simd: dst += v_{k-1} dot[j]; acc += v_k^H dst; dst written back
        const Sc<R> b0 = sc_ld<R, CX>(w.dot + W * j);
        i64 i = lo + lane;
        for (; i + 96 < hi; i += 128) {
          Sc<R> y[4], v[4], d[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            y[q] = sc_ld<R, CX>(at(i + 32 * q, k - 1));
            v[q] = sc_ld<R, CX>(at(i + 32 * q, k));
            d[q] = sc_ld<R, CX>(at(i + 32 * q, j));
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            d[q] = mul_add<R, CX>(y[q], b0, d[q]);
            acc = conj_mul_add<R, CX>(v[q], d[q], acc);
            sc_st<R, CX>(at(i + 32 * q, j), d[q]);
          }
        }
        for (; i < hi; i += 32) {
          const Sc<R> d = mul_add<R, CX>(sc_ld<R, CX>(at(i, k - 1)), b0, sc_ld<R, CX>(at(i, j)));
          acc = conj_mul_add<R, CX>(sc_ld<R, CX>(at(i, k)), d, acc);
          sc_st<R, CX>(at(i, j), d);
        }
      } else {
        // the GEMV form: acc = v_k^H B11[:, j]
        i64 i = lo + lane;
        for (; i + 96 < hi; i += 128) {
          Sc<R> v[4], d[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            v[q] = sc_ld<R, CX>(at(i + 32 * q, k));
            d[q] = sc_ld<R, CX>(at(i + 32 * q, j));
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) acc = conj_mul_add<R, CX>(v[q], d[q], acc);
        }
        for (; i < hi; i += 32) acc = conj_mul_add<R, CX>(sc_ld<R, CX>(at(i, k)), sc_ld<R, CX>(at(i, j)), acc);
      }
      acc.re = warp_sum(acc.re);
      if (CX) acc.im = warp_sum(acc.im);
      if (lane == 0) {
        R* p = w.part + u * CPQ_REC;
        p[0] = acc.re;
        p[1] = acc.im;
      }
    }
    barrier();

    // ---- F: row k of the trailing columns, dot and the downdated norms (factor.rs:63-69, 296-302) ----
    for (i64 j = k + 1 + gt; j < n; j += T) {
      Sc<R> acc{R(0), R(0)};
      const i64 u0 = (j - k - 1) * sp.S;
      for (int q = 0; q < sp.S; ++q) {
        const R* p = w.part + (u0 + q) * CPQ_REC;
        acc.re += __ldcg(p);
        if (CX) acc.im += __ldcg(p + 1);
      }
      R* pu = at(k, j);
      Sc<R> u = sc_ld<R, CX>(pu);
      Sc<R> d0;
      if (delayed) {
        const Sc<R> tmp = mul_add<R, CX>(l, sc_ld<R, CX>(w.dot + W * j), u);
        d0 = scale<R, CX>(cadd<R, CX>(tmp, acc), -tau_inv);
        u = cadd<R, CX>(tmp, d0);
      } else {
        const Sc<R> s = scale<R, CX>(cadd<R, CX>(u, acc), tau_inv);
        d0 = Sc<R>{-s.re, -s.im};
        u = cadd<R, CX>(u, d0);
      }
      sc_st<R, CX>(pu, u);
      sc_st<R, CX>(w.dot + W * j, d0);
      const R nj = __ldcg(w.norm + j);
      w.norm[j] = sqrt(nj * nj - abs2<R, CX>(u));
    }
    barrier();
  }

  // ---- factor.rs:306-309: the upper trapezoid scaled back ----
  barrier();
  for (i64 j = gw; j < n; j += warps) {
    const i64 hi = min(j + 1, (i64)m);
    for (i64 i = lane; i < hi; i += 32) {
      R* p = at(i, j);
      p[0] *= scale_fwd;
      if (CX) p[1] *= scale_fwd;
    }
  }
}

// Q_coeff[0, j] = Q_coeff[j % bs, j] = tau_j (factor.rs:374-376; the diagonal of every T block is its taus)
template <class R, bool CX>
__global__ void cpq_tau_kernel(R* __restrict__ H, i64 rs, i64 cs, const R* __restrict__ tau, i64 size, i64 bs) {
  constexpr int W = CX ? 2 : 1;
  const i64 j = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= size) return;
  const i64 jj = j % bs;
  R* p0 = H + W * (j * cs);
  R* pd = H + W * (jj * rs + j * cs);
  p0[0] = tau[j];
  pd[0] = tau[j];
  if (CX) {
    p0[1] = R(0);
    pd[1] = R(0);
  }
}

}  // namespace

// In-place column-pivoted QR (views in element units of the scalar kind; complex: COMPLEX units on an R* base). H: block_size x
// min(m, n). rs1: the caller's row stride is 1 (the reference's delayed-update condition). trans (host, min(m, n) entries) receives
// the column transpositions. Returns the transposition count.
template <class R, bool CX>
i64 colpiv_qr_in_place_t(cudaStream_t st, View<R> A, View<R> H, bool rs1, std::vector<long long>& trans) {
  constexpr int W = CX ? 2 : 1;
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n);
  FB_ASSERT(m < (i64)INT_MAX && n < (i64)INT_MAX, "column-pivoted QR: dimension too large");
  trans.assign((size_t)size, 0);
  if (size == 0) return 0;
  FB_ASSERT(H.nrows > 0 && H.ncols == size, "Q_coeff must be block_size x min(nrows, ncols) with block_size > 0");

  // the kernel works on a column-major matrix; other layouts go through a compact copy
  const bool compact = A.rs == 1 && A.cs >= m;
  R* work = A.ptr;
  i64 ld = A.cs;
  if (!compact) {
    work = (R*)ws_alloc((size_t)m * (size_t)n * W * sizeof(R));
    ld = m;
    piv_copy_t<R, CX>(st, View<R>{work, m, n, 1, m}, cview(A));
  }

  const int sms = stream_sms(st);
  int occ = 0;
  FB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, colpiv_qr_kernel<R, CX>, CPQ_THREADS, 0));
  FB_ASSERT(occ > 0, "column-pivoted QR kernel cannot be resident");
  const int G = sms * std::min(occ, 4);  // 4 CTAs per SM keep enough loads in flight; more only lengthen the barriers
  const i64 warps = (i64)G * CPQ_WARPS;

  const size_t b_norm = (size_t)n * sizeof(R), b_dot = (size_t)W * n * sizeof(R), b_tau = (size_t)size * sizeof(R);
  const size_t b_hist = (size_t)size * sizeof(int), b_part = (size_t)(n + warps) * CPQ_REC * sizeof(R);
  const size_t b_rec = (size_t)G * PANEL_NV * sizeof(R);
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  char* buf = (char*)ws_alloc(up(b_norm) + up(b_dot) + up(b_tau) + up(b_hist) + up(b_part) + up(b_rec) + 256);
  CpqWs<R> w;
  char* p = buf;
  w.norm = (R*)p; p += up(b_norm);
  w.dot = (R*)p; p += up(b_dot);
  w.tau = (R*)p; p += up(b_tau);
  w.hist = (int*)p; p += up(b_hist);
  w.part = (R*)p; p += up(b_part);
  w.rec = (R*)p; p += up(b_rec);
  w.bar = (unsigned long long*)p;
  FB_CUDA_CHECK(cudaMemsetAsync(w.dot, 0, b_dot, st));
  FB_CUDA_CHECK(cudaMemsetAsync(w.bar, 0, sizeof(unsigned long long), st));
  {
    int mi = (int)m, ni = (int)n, r1 = rs1 ? 1 : 0;
    void* args[] = {&work, &ld, &mi, &ni, &r1, &w};
    FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)colpiv_qr_kernel<R, CX>, dim3(G), dim3(CPQ_THREADS), args, 0, st));
    note_launch();
  }
  if (!compact) {
    piv_copy_t<R, CX>(st, A, View<const R>{work, m, n, 1, m});
  }

  // T blocks (factor.rs:367-386)
  const i64 bs = H.nrows;
  cpq_tau_kernel<R, CX><<<grid_1d(size), 256, 0, st>>>(H.ptr, H.rs, H.cs, w.tau, size, bs);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  for (i64 j = 0; j < size; j += bs) {
    const i64 b = std::min(bs, size - j);
    View<const R> V{A.ptr + W * (j * A.rs + j * A.cs), m - j, b, A.rs, A.cs};
    View<R> Tf{H.ptr + W * (j * H.cs), b, b, H.rs, H.cs};
    householder_factor_t<R, CX>(st, V, Tf);
  }

  std::vector<int> hist((size_t)size);
  FB_CUDA_CHECK(cudaMemcpyAsync(hist.data(), w.hist, b_hist, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(buf);
  if (!compact) ws_free(work);
  i64 count = 0;
  for (i64 k = 0; k < size; ++k) {
    trans[(size_t)k] = hist[(size_t)k];
    count += hist[(size_t)k] != k;
  }
  return count;
}

}  // namespace fb

// ---- C ABI (faer-ffi/src/lib.rs:1721-1940; declarations in include/faer_b200_colpiv_qr.h) ----
using namespace fb;

namespace {

template <class R, bool CX>
FaerV0_24_ColPivQrStatus colpiv_qr_factor_entry(FaerV0_24_MatMut A, FaerV0_24_MatMut Q_coeff, FaerV0_24_SliceMut perm_fwd,
                                                FaerV0_24_SliceMut perm_bwd, int idx_bytes) {
  FB_ENTRY();
  const size_t size = A.nrows < A.ncols ? A.nrows : A.ncols;
  FB_ASSERT(Q_coeff.ncols == size, "Q_coeff must have min(nrows, ncols) columns");
  FB_ASSERT(size == 0 || Q_coeff.nrows > 0, "Q_coeff.nrows (the block size) must be positive (the reference would not terminate)");
  FB_ASSERT(A.ncols == 0 || (perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr), "null permutation slice");
  cudaStream_t st = current_stream();
  std::vector<long long> trans, fwd, bwd;
  i64 count = 0;
  if (size > 0) {
    StagedMat a = stage<R, CX>(A, true, st);
    StagedMat q = stage<R, CX>(Q_coeff, true, st);
    count = colpiv_qr_in_place_t<R, CX>(st, a.view<R>(), q.view<R>(), A.row_stride == 1, trans);
    finish_all(st, {&a, &q});
  }
  perm_from_transpositions(A.ncols, trans, fwd, bwd);
  write_perm(perm_fwd.ptr, fwd, idx_bytes);
  write_perm(perm_bwd.ptr, bwd, idx_bytes);
  FaerV0_24_ColPivQrStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_ColPivQrStatus_Ok;
  out.ok.transposition_count = (size_t)count;
  return out;
}

// M (host or device) is staged once; `unpivoted` (an unpivoted QR entry point) runs on the device mirror, and rows [0, nrows) of
// the mirror get rows perm[i] (`cols`: columns instead, the rows of the transposed view) before it (`perm_first`) or after it.
// A host M thus crosses the bus once each way, as for the other entry points.
template <class R, bool CX, class F>
void cpq_staged(FaerV0_24_MatMut M, size_t nrows, const std::vector<long long>& perm, bool cols, bool perm_first, F&& unpivoted) {
  cudaStream_t st = current_stream();
  StagedMat s = stage<R, CX>(M, true, st);
  View<R> v = s.view<R>();
  const FaerV0_24_MatMut dm{(void*)v.ptr, M.nrows, M.ncols, (ptrdiff_t)v.rs, (ptrdiff_t)v.cs};
  View<R> pv = cols ? View<R>{v.ptr, v.ncols, v.nrows, v.cs, v.rs} : v;
  pv.nrows = (i64)nrows;
  const bool permute = nrows > 0 && pv.ncols > 0;
  if (permute && perm_first) permute_rows_t<R, CX>(st, pv, perm.data());
  unpivoted(dm);
  if (permute && !perm_first) permute_rows_t<R, CX>(st, pv, perm.data());
  finish_all(st, {&s});
}

}  // namespace

// The unpivoted QR entry points these compose (include/faer_b200.h), by scalar kind
#define FB_CPQ_FFI(SUF, R, CX, IT, BYTES)                                                                                                 \
  FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_##IT##_##SUF(size_t nrows, size_t ncols, size_t block_size,            \
                                                                                FaerV0_24_Par par, FaerV0_24_ColPivQrParams params) {    \
    (void)nrows; (void)block_size; (void)par; (void)params;                                                                               \
    return FaerV0_24_Layout{ncols * 2 * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(ncols, 2) */                                \
  }                                                                                                                                       \
  FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatMut Q_coeff,             \
                                                                                FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd, \
                                                                                FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                \
                                                                                FaerV0_24_ColPivQrParams params) {                        \
    (void)par; (void)mem; (void)params;                                                                                                   \
    return colpiv_qr_factor_entry<R, CX>(A, Q_coeff, perm_fwd, perm_bwd, BYTES);                                                          \
  }                                                                                                                                       \
  FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_##IT##_##SUF(size_t nrows, size_t ncols, size_t block_size,       \
                                                                                     size_t rhs_ncols, FaerV0_24_Par par) {              \
    /* StackReq::and(the unpivoted lstsq scratch, permute_rows_in_place_scratch::<I, T>(ncols, rhs_ncols)) */                              \
    const FaerV0_24_Layout a = libfaer_v0_23_qr_solve_lstsq_in_place_scratch_##SUF(nrows, ncols, block_size, rhs_ncols, par);             \
    return layout_and(a, ncols * rhs_ncols * (CX ? 2 : 1) * sizeof(R));                                                                   \
  }                                                                                                                                       \
  FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t block_size, size_t rhs_ncols,           \
                                                                               FaerV0_24_Par par) {                                      \
    return libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_##IT##_##SUF(dim, dim, block_size, rhs_ncols, par);                       \
  }                                                                                                                                       \
  FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_##IT##_##SUF(size_t dim, size_t block_size,                   \
                                                                                         size_t rhs_ncols, FaerV0_24_Par par) {          \
    const FaerV0_24_Layout a = libfaer_v0_23_qr_solve_transpose_in_place_scratch_##SUF(dim, block_size, rhs_ncols, par);                  \
    return layout_and(a, dim * rhs_ncols * (CX ? 2 : 1) * sizeof(R));                                                                     \
  }                                                                                                                                       \
  void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_##IT##_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R_, \
                                                                 FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd,                      \
                                                                 FaerV0_24_SliceRef perm_bwd, FaerV0_24_MatMut rhs, FaerV0_24_Par par,    \
                                                                 FaerV0_24_MemAlloc mem) {                                                \
    FB_ENTRY();                                                                                                                           \
    (void)perm_fwd;                                                                                                                       \
    const size_t n = Q_basis.ncols;                                                                                                       \
    const std::vector<long long> pb = read_perm_checked(perm_bwd, n, BYTES);                                                                  \
    /* the unpivoted lstsq, then rows ..size <- perm^-1 (solve.rs:66-79) */                                                             \
    cpq_staged<R, CX>(rhs, n, pb, false, false, [&](FaerV0_24_MatMut d) {                                                                 \
      libfaer_v0_23_qr_solve_lstsq_in_place_##SUF(Q_basis, Q_coeff, R_, A_conj, d, par, mem);                                            \
    });                                                                                                                                   \
  }                                                                                                                                       \
  void libfaer_v0_23_colpiv_qr_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff, FaerV0_24_MatRef R_,       \
                                                           FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd, \
                                                           FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {             \
    FB_ENTRY();                                                                                                                           \
    FB_ASSERT(Q_coeff.nrows > 0 && Q_basis.nrows == Q_basis.ncols && rhs.nrows == Q_basis.nrows && Q_coeff.ncols == Q_basis.ncols &&      \
                  R_.nrows == Q_basis.nrows && R_.ncols == Q_basis.ncols,                                                                 \
              "column-pivoted QR solve shape mismatch");                                                                                  \
    libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_##IT##_##SUF(Q_basis, Q_coeff, R_, A_conj, perm_fwd, perm_bwd, rhs, par, mem);            \
  }                                                                                                                                       \
  void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_##IT##_##SUF(FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,                  \
                                                                     FaerV0_24_MatRef R_, FaerV0_24_Conj A_conj,                          \
                                                                     FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,            \
                                                                     FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {   \
    FB_ENTRY();                                                                                                                           \
    (void)perm_bwd;                                                                                                                       \
    const size_t n = Q_basis.nrows;                                                                                                       \
    FB_ASSERT(Q_coeff.nrows > 0 && Q_basis.ncols == n && rhs.nrows == n && Q_coeff.ncols == n && R_.nrows == n && R_.ncols == n,        \
              "column-pivoted QR solve shape mismatch");                                                                                  \
    const std::vector<long long> pf = read_perm_checked(perm_fwd, n, BYTES);                                                                  \
    /* rhs <- P rhs (solve.rs:180), then the unpivoted transpose solve */                                                               \
    cpq_staged<R, CX>(rhs, n, pf, false, true, [&](FaerV0_24_MatMut d) {                                                                  \
      libfaer_v0_23_qr_solve_transpose_in_place_##SUF(Q_basis, Q_coeff, R_, A_conj, d, par, mem);                                        \
    });                                                                                                                                   \
  }                                                                                                                                       \
  FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_##IT##_##SUF(size_t nrows, size_t ncols, size_t block_size,                \
                                                                            FaerV0_24_Par par) {                                         \
    (void)par;                                                                                                                            \
    /* StackReq::or(apply_block_householder_sequence_on_the_left_in_place_scratch(nrows, bs, ncols), permute_cols(nrows, ncols)) */      \
    const size_t a = block_size * ncols * (CX ? 2 : 1) * sizeof(R), b = nrows * ncols * (CX ? 2 : 1) * sizeof(R);                         \
    return FaerV0_24_Layout{a > b ? a : b, 64};                                                                                           \
  }                                                                                                                                       \
  void libfaer_v0_23_colpiv_qr_reconstruct_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,           \
                                                        FaerV0_24_MatRef R_, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,    \
                                                        FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                      \
    FB_ENTRY();                                                                                                                           \
    (void)perm_fwd;                                                                                                                       \
    const size_t n = R_.ncols;                                                                                                            \
    FB_ASSERT(A.ncols == n, "column-pivoted QR reconstruct shape mismatch");                                                              \
    const std::vector<long long> pb = read_perm_checked(perm_bwd, n, BYTES);                                                                  \
    /* Q R, then columns <- perm^-1 (reconstruct.rs:38-44) */                                                                          \
    cpq_staged<R, CX>(A, n, pb, true, false, [&](FaerV0_24_MatMut d) {                                                                    \
      libfaer_v0_23_qr_reconstruct_##SUF(d, Q_basis, Q_coeff, R_, par, mem);                                                             \
    });                                                                                                                                   \
  }                                                                                                                                       \
  FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_##IT##_##SUF(size_t dim, size_t block_size, FaerV0_24_Par par) {               \
    (void)par;                                                                                                                            \
    /* StackReq::or(apply_block_householder_sequence_transpose_on_the_right_in_place_scratch(dim, bs, dim), permute_cols(dim, dim)) */    \
    const size_t a = block_size * dim * (CX ? 2 : 1) * sizeof(R), b = dim * dim * (CX ? 2 : 1) * sizeof(R);                               \
    return FaerV0_24_Layout{a > b ? a : b, 64};                                                                                           \
  }                                                                                                                                       \
  void libfaer_v0_23_colpiv_qr_inverse_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef Q_basis, FaerV0_24_MatRef Q_coeff,               \
                                                    FaerV0_24_MatRef R_, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,        \
                                                    FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                          \
    FB_ENTRY();                                                                                                                           \
    (void)perm_fwd;                                                                                                                       \
    const size_t n = Q_basis.ncols;                                                                                                       \
    FB_ASSERT(Q_coeff.nrows > 0 && A.nrows == n, "column-pivoted QR inverse shape mismatch");                                             \
    const std::vector<long long> pb = read_perm_checked(perm_bwd, n, BYTES);                                                                  \
    /* R^-1 Q^H, then rows <- perm^-1 (inverse.rs:38-49) */                                                                            \
    cpq_staged<R, CX>(A, n, pb, false, false, [&](FaerV0_24_MatMut d) {                                                                   \
      libfaer_v0_23_qr_inverse_##SUF(d, Q_basis, Q_coeff, R_, par, mem);                                                                 \
    });                                                                                                                                   \
  }
#define FB_CPQ_DTYPE(SUF, R, CX)                                                                                    \
  FaerV0_24_ColPivQrParams libfaer_v0_23_ColPivQrParams_##SUF(void) {                                              \
    return FaerV0_24_ColPivQrParams{48 * 48, 192 * 256}; /* factor.rs:101-110 */                                    \
  }                                                                                                                 \
  FB_CPQ_FFI(SUF, R, CX, u32, 4)                                                                                    \
  FB_CPQ_FFI(SUF, R, CX, u64, 8)

extern "C" {
FB_CPQ_DTYPE(f64, double, false)
FB_CPQ_DTYPE(f32, float, false)
FB_CPQ_DTYPE(c64, double, true)
FB_CPQ_DTYPE(c32, float, true)
}  // extern "C"
#undef FB_CPQ_DTYPE
#undef FB_CPQ_FFI
