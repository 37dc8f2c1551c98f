// Householder QR without pivoting (f32 / f64): cooperative panel kernel + blocked driver.
//
// Reference: faer/src/linalg/qr/no_pivoting/factor.rs
//   qr_in_place 258-301, qr_in_place_blocked 137-256 (panel -> T factor -> block apply to the trailing columns),
//   qr_in_place_unblocked 11-86 (per column: make_householder, rank test, dot + axpy on the rest of the panel),
//   householder::make_householder_imp (householder.rs:59-107): tail norm, beta = -sign(head) * norm stored in the
//   head, v_tail = tail / (head + sign * norm), tau = (1 + (|tail| * |1/(head + sign*norm)|)^2) / 2, tau = +inf when
//   the tail vanishes.
//
// GPU mapping. The reference recurses 256 -> 128 -> ... -> 1 with a GEMM-based T upgrade at every level; on the GPU
// that is ~10^5 tiny launches, so the blocking is different while the mathematics (and the output format: V below the
// diagonal, R above, Q_coeff = one block_size x block_size T block per block of columns, T = striu(V^H V) + diag(tau))
// is the same:
//   * a block of `block_size` columns is factored as sub-panels of <= 32 columns; each sub-panel is ONE cooperative
//     kernel (`qr_panel_kernel`): the panel is sliced by rows over <= one CTA per SM and stays in shared memory; per column
//     there is exactly one grid-wide exchange: every CTA publishes its partial tail norm (three scaled accumulators,
//     as reductions/norm_l2.rs) and its partial dot products of the tail with the remaining panel columns, the owner
//     of the diagonal row publishes that row; after the barrier every CTA reduces the partials in a fixed order
//     (deterministic), forms (beta, tau, 1/(head+beta)) and the coefficients k_c = -(head_c + v^H a_c) / tau, and updates
//     its slice (v in place, a_c += k_c v);
//   * the sub-panel's T block and the block's full T are tall-skinny V^H V products (split-K DMMA / 3xTF32 GEMM);
//   * reflector blocks are applied to the rest of the block and to the trailing matrix with the block-Householder
//     GEMM composition (householder.cu).
// Rank deficiency: the reference skips columns whose norm falls below eps*16*(m-row)*norm, keeps `row` where it is and
// writes later reflectors out of place into column `row` (factor.rs:40-83), so the reflectors stay compacted in the
// first `rank` columns and R becomes a staircase. Two drivers produce exactly that:
//   * the fast driver assumes row == col (full rank so far). Its panel kernel runs the same rank test and only REPORTS
//     the first failing column; the driver checks that flag once per block of `block_size` columns, before the block's
//     reflector is applied to the trailing matrix. The block's columns are saved before they are touched, so on a report
//     they are restored and
//   * the general driver (`qr_general_from`) takes over from (row, col) = the start of that block: sub-panels of <= 16
//     columns through `qr_panel_general_kernel` (separate pivot row and column counters, reflectors written to their own
//     shared-memory columns and stored in column `row` of A, the zero fill of factor.rs:46-48), one host read-back of
//     the number of reflectors per sub-panel, T blocks indexed by reflector (= row) number as in factor.rs:184-239.
//   Q_coeff's columns >= rank are zero-filled with +inf on the block diagonals (factor.rs:287-299).
#include <algorithm>
#include <limits>
#include <vector>

#include "panel_common.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

constexpr int QR_PW = 32;       // sub-panel width (columns per cooperative launch)
// 32 row groups x 32 column lanes: the per-column dot and update loops walk the CTA's rows (443 at 65536 rows) one row
// per warp and iteration with a dependent shared-memory chain, so their latency divides by the number of warps
//
constexpr int QR_THREADS = 1024;
constexpr int QR_NV = QR_PW + 4; // published values per CTA and column: dots[PW], sml, med, big, above

template <class T>
struct QrScratch {
  T* part;   // [2][G][QR_NV]
  T* rowv;   // [2][QR_PW]
  unsigned long long* bar;
};

__device__ __forceinline__ void qr_grid_barrier(unsigned long long* bar, unsigned long long target) {
  grid_barrier(bar, target);  // panel_common.cuh
}

// A: panel top-left (local row 0 = the diagonal row of panel column 0); mp rows, w <= QR_PW columns.
// taus: pointer to the T-block diagonal entry of column 0, `tau_stride` elements between consecutive diagonal entries.
// above2[c]: sum of squares of the w panel columns over the matrix rows ABOVE the panel (rank test only).
// flag: set to 1 if a rank-deficient column is met.
template <class T>
__global__ void __launch_bounds__(QR_THREADS) qr_panel_kernel(T* __restrict__ A, i64 rs, i64 cs, int mp, int w,
                                                               int rows_per_cta, T* __restrict__ taus, i64 tau_stride,
                                                               QrScratch<T> sc, unsigned long long bar_base,
                                                               const T* __restrict__ above2, long long rows_below0,
                                                               int* __restrict__ flag) {
  extern __shared__ unsigned char qr_smem_raw[];
  T* S = reinterpret_cast<T*>(qr_smem_raw);  // [rows_per_cta][LD]
  const int LD = w | 1;
  __shared__ T red[QR_THREADS / 32][QR_NV];
  __shared__ T tot[QR_NV];
  __shared__ T rowj[QR_PW];
  __shared__ T kc[QR_PW];

  const int tid = threadIdx.x, lane = tid & 31, rg = tid >> 5;  // lane = panel column, rg = row group
  const int G = gridDim.x, bid = blockIdx.x;
  const int r0 = bid * rows_per_cta;
  const int nloc = max(0, min(rows_per_cta, mp - r0));
  const int ncol = min(w, mp);

  const T min_pos = TLim<T>::min_pos();
  const T sml = t_sqrt(min_pos), big = t_sqrt(T(1) / min_pos);
  const T eps = TLim<T>::eps();

  for (int r = tid; r < nloc; r += QR_THREADS) {
    const T* src = A + (i64)(r0 + r) * rs;
    T* dst = S + r * LD;
#pragma unroll 8
    for (int c = 0; c < w; ++c) dst[c] = src[(i64)c * cs];
  }
  __syncthreads();

  unsigned long long nbar = 0;
  for (int j = 0; j < ncol; ++j) {
    const int par = j & 1;
    // ---- phase A: partial dots of the tail of column j with columns c > j, and partial norms ----
    T acc = T(0), a_sml = T(0), a_big = T(0), a_above = T(0);
    for (int r = rg; r < nloc; r += QR_THREADS / 32) {
      const int il = r0 + r;
      const T x = S[r * LD + j];
      if (il > j) {
        if (lane >= j && lane < w) acc = fma(x, S[r * LD + lane], acc);
        if (lane == j) {
          const T xs = x * sml, xb = x * big;
          a_sml = fma(xs, xs, a_sml);
          a_big = fma(xb, xb, a_big);
        }
      } else if (il < j && lane == j) {
        a_above = fma(x, x, a_above);
      }
    }
    red[rg][lane] = acc;  // lane == j carries the unscaled sum of squares ("med")
    if (lane == j) {
      red[rg][QR_PW + 0] = a_sml;
      red[rg][QR_PW + 1] = a_big;
      red[rg][QR_PW + 2] = a_above;
    }
    __syncthreads();
    if (tid < QR_NV - 1) {
      T s = T(0);
#pragma unroll
      for (int q = 0; q < QR_THREADS / 32; ++q) s += red[q][tid];
      sc.part[((i64)par * G + bid) * QR_NV + tid] = s;
    }
    if (j >= r0 && j < r0 + nloc) {
      if (tid < w) sc.rowv[par * QR_PW + tid] = S[(j - r0) * LD + tid];
    }
    ++nbar;
    qr_grid_barrier(sc.bar, bar_base + nbar * (unsigned long long)G);

    // ---- phase B: deterministic reduction over the CTAs (fixed order), then the reflector scalars ----
    {
      // warp `rg` reduces the values v = rg, rg + 8, ... (QR_NV - 1 = 35 <= 40 values over 8 warps); every lane loads
      // the records of the CTAs lane, lane + 32, ... (G <= 160, checked on the host): all 25 loads of a lane are issued
      // before the first use, i.e. ONE L2 round trip per column instead of a chain of G / 4 dependent ones.
      // The records are read as 16-byte vectors: every CTA reads every CTA's record, i.e. G^2 * QR_NV values per column
      // grid-wide — as scalar loads that is ~0.8 M L2 requests per column and the L2 request rate, not latency, bounds
      // the panel; vectors cut the requests by 4x (f32) / 2x (f64).
      typedef typename Vec16<T>::type V;
      constexpr int NWARP = QR_THREADS / 32, VEC = Vec16<T>::N, NVV = QR_NV / VEC, NCH = (NVV + NWARP - 1) / NWARP;
      static_assert(QR_NV % VEC == 0, "record length must be a multiple of the vector width");
      const V* pv = reinterpret_cast<const V*>(sc.part) + (i64)par * G * NVV;
      V rec[NCH][5];
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const int c = rg + NWARP * i;
#pragma unroll
        for (int u = 0; u < 5; ++u) {
          const int b = lane + 32 * u;
          rec[i][u] = (c < NVV && b < G) ? __ldcg(&pv[(i64)b * NVV + c]) : Vec16<T>::zero();
        }
      }
      if (tid < w) rowj[tid] = t_ldcg(&sc.rowv[par * QR_PW + tid]);
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const int c = rg + NWARP * i;
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
          T s = ((Vec16<T>::get(rec[i][0], e) + Vec16<T>::get(rec[i][1], e)) +
                 (Vec16<T>::get(rec[i][2], e) + Vec16<T>::get(rec[i][3], e))) + Vec16<T>::get(rec[i][4], e);
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
          const int v = c * VEC + e;
          if (lane == 0 && c < NVV && v < QR_NV - 1) tot[v] = s;
        }
      }
      __syncthreads();
    }
    // make_householder (householder.rs:59-107), evaluated redundantly by every thread
    const T acc_med = tot[j], acc_sml = tot[QR_PW + 0], acc_big = tot[QR_PW + 1];
    T tail_norm;
    if (acc_sml >= T(1)) tail_norm = t_sqrt(acc_sml) * big;
    else if (acc_med >= T(1)) tail_norm = t_sqrt(acc_med);
    else tail_norm = t_sqrt(acc_big) * sml;
    T head = rowj[j];
    T head_norm = t_abs(head);
    if (head_norm < min_pos) {
      head = T(0);
      head_norm = T(0);
    }
    T tau, inv = T(0), norm, new_head = head;
    const bool no_tail = tail_norm < min_pos;
    if (no_tail) {
      tau = TLim<T>::inf();
      norm = head_norm;
    } else {
      norm = t_hypot(head_norm, tail_norm);
      const T sign = head_norm != T(0) ? head * (T(1) / head_norm) : T(1);
      const T signed_norm = sign * norm;
      inv = T(1) / (head + signed_norm);
      new_head = -signed_norm;
      const T tt = tail_norm * t_abs(inv);
      tau = T(0.5) * (T(1) + tt * tt);
    }
    // rank test (factor.rs:52-64)
    const T norm_above = t_sqrt(above2[j] + tot[QR_PW + 2]);
    const T total = t_hypot(norm, norm_above);
    const T threshold = eps * T((double)(rows_below0 - j) * 16.0) * total;
    const T tau_inv = T(1) / tau;
    bool apply = false;
    if (tau_inv < min_pos) {
      if (!(norm > T(0))) {
        if (bid == 0 && tid == 0) *flag = 1;  // exactly zero column: the reference would not advance `row`
      }
    } else if (norm > threshold) {
      apply = true;
    } else {
      if (bid == 0 && tid == 0) *flag = 1;    // numerically dependent column: reference skips it
    }
    if (bid == 0 && tid == 0) taus[(i64)j * tau_stride] = tau;
    if (tid < w) {
      // k_c = -(head_c + v^H a_c) / tau   (factor.rs:65-80)
      const T dot = rowj[tid] + inv * tot[tid];
      kc[tid] = (apply && tid > j) ? -(dot * tau_inv) : T(0);
    }
    __syncthreads();
    // ---- phase C: write v (scaled tail), beta, and update the remaining panel columns ----
    if (j >= r0 && j < r0 + nloc && rg == ((j - r0) & (QR_THREADS / 32 - 1))) {
      T* row = S + (j - r0) * LD;
      if (lane == j && !no_tail) row[j] = new_head;
      else if (lane == j && no_tail && head_norm == T(0)) row[j] = T(0);
      if (lane > j && lane < w) row[lane] += kc[lane];
    }
    if (!no_tail) {
      for (int r = rg; r < nloc; r += QR_THREADS / 32) {
        const int il = r0 + r;
        if (il > j) {
          const T vi = S[r * LD + j] * inv;
          __syncwarp();
          if (lane == j) S[r * LD + j] = vi;
          else if (lane > j && lane < w) S[r * LD + lane] = fma(kc[lane], vi, S[r * LD + lane]);
        }
      }
    }
    // rows are owned by warps (row r -> warp r mod 8) in phases A and C alike; the next phase A needs no CTA barrier
    // for S, and red/tot/rowj/kc are protected by the barriers of the next iteration
    __syncthreads();
  }
  for (int r = tid; r < nloc; r += QR_THREADS) {
    T* dstg = A + (i64)(r0 + r) * rs;
    const T* srcs = S + r * LD;
#pragma unroll 8
    for (int c = 0; c < w; ++c) dstg[(i64)c * cs] = srcs[c];
  }
}

// ---- general (column-skipping) sub-panel: reference qr_in_place_unblocked (factor.rs:11-86) with row != col ----------
constexpr int QRG_PW = 16;        // panel columns per launch
constexpr int QRG_THREADS = 512;  // 16 warps: lane = panel column (lanes >= w idle), warp = row group
constexpr int QRG_NV = QRG_PW + 4;  // published per CTA and column: dots[16], sml, big, above, (pad)

// A: at (row0, col0) — local row 0 is the first pivot row, panel column 0 is global column col0 = row0 + d0.
// Vout: at (row0, row0) — reflector l (pivot row row0 + l) is stored in column l of Vout, rows > l.
// max_refl: reflectors this launch may produce (<= w). taus[l * tau_stride]: tau of reflector l.
// info[0] <- number of reflectors produced (`new_row - row`).
template <class T>
__global__ void __launch_bounds__(QRG_THREADS) qr_panel_general_kernel(T* __restrict__ A, T* __restrict__ Vout, i64 rs, i64 cs,
                                                                        int mp, int w, int d0, int max_refl, int rows_per_cta,
                                                                        T* __restrict__ taus, i64 tau_stride, QrScratch<T> sc,
                                                                        const T* __restrict__ above2, int* __restrict__ info) {
  extern __shared__ unsigned char qr_smem_raw[];
  T* S = reinterpret_cast<T*>(qr_smem_raw);  // [rows_per_cta][LD]: columns 0..w-1 = panel, w..2w-1 = reflectors
  const int LD = (2 * w) | 1;
  constexpr int NWARP = QRG_THREADS / 32;
  __shared__ T red[NWARP][QRG_NV];
  __shared__ T tot[QRG_NV];
  __shared__ T rowj[QRG_PW];
  __shared__ T kc[QRG_PW];

  const int tid = threadIdx.x, lane = tid & 31, rg = tid >> 5;
  const int G = gridDim.x, bid = blockIdx.x;
  const int r0 = bid * rows_per_cta;
  const int nloc = max(0, min(rows_per_cta, mp - r0));

  const T min_pos = TLim<T>::min_pos();
  const T sml = t_sqrt(min_pos), big = t_sqrt(T(1) / min_pos);
  const T eps = TLim<T>::eps();

  for (int r = tid; r < nloc; r += QRG_THREADS) {
    const T* src = A + (i64)(r0 + r) * rs;
    T* dst = S + r * LD;
    for (int c = 0; c < w; ++c) dst[c] = src[(i64)c * cs];
    for (int c = 0; c < w; ++c) dst[w + c] = T(0);
  }
  __syncthreads();

  unsigned long long nbar = 0;
  int lr = 0, jend = 0;  // pivot row (local), first unprocessed panel column
  for (int j = 0; j < w && lr < max_refl; ++j) {
    jend = j + 1;
    const int par = j & 1;
    // ---- phase A: partial dots of the tail (rows > lr) of column j with columns c >= j, partial norms ----
    T acc = T(0), a_sml = T(0), a_big = T(0), a_above = T(0);
    for (int r = rg; r < nloc; r += NWARP) {
      const int il = r0 + r;
      const T x = S[r * LD + j];
      if (il > lr) {
        if (lane >= j && lane < w) acc = fma(x, S[r * LD + lane], acc);
        if (lane == j) {
          const T xs = x * sml, xb = x * big;
          a_sml = fma(xs, xs, a_sml);
          a_big = fma(xb, xb, a_big);
        }
      } else if (il < lr && lane == j) {
        a_above = fma(x, x, a_above);
      }
    }
    if (lane < QRG_PW) red[rg][lane] = acc;
    if (lane == j) {
      red[rg][QRG_PW + 0] = a_sml;
      red[rg][QRG_PW + 1] = a_big;
      red[rg][QRG_PW + 2] = a_above;
    }
    __syncthreads();
    if (tid < QRG_NV - 1) {
      T s = T(0);
#pragma unroll
      for (int q = 0; q < NWARP; ++q) s += red[q][tid];
      sc.part[((i64)par * G + bid) * QRG_NV + tid] = s;
    }
    if (lr >= r0 && lr < r0 + nloc) {
      if (tid < w) sc.rowv[par * QR_PW + tid] = S[(lr - r0) * LD + tid];
    }
    ++nbar;
    qr_grid_barrier(sc.bar, nbar * (unsigned long long)G);

    // ---- phase B: fixed-order reduction over the CTAs, identical in every CTA ----
    for (int v = rg; v < QRG_NV - 1; v += NWARP) {
      T s = T(0);
      for (int b = lane; b < G; b += 32) s += t_ldcg(&sc.part[((i64)par * G + b) * QRG_NV + v]);
      s = warp_sum(s);
      if (lane == 0) tot[v] = s;
    }
    if (rg == NWARP - 1 && lane < w) rowj[lane] = t_ldcg(&sc.rowv[par * QR_PW + lane]);
    __syncthreads();
    const T acc_med = tot[j], acc_sml = tot[QRG_PW + 0], acc_big = tot[QRG_PW + 1];
    const T tail_norm = norm_from_acc(acc_sml, acc_med, acc_big, sml, big);
    T head = rowj[j];
    T head_norm = t_abs(head);
    if (head_norm < min_pos) {
      head = T(0);
      head_norm = T(0);
    }
    T tau, inv = T(0), norm, new_head = head;
    const bool no_tail = tail_norm < min_pos;
    if (no_tail) {
      tau = TLim<T>::inf();
      norm = head_norm;
    } else {
      norm = t_hypot(head_norm, tail_norm);
      const T sign = head_norm != T(0) ? head * (T(1) / head_norm) : T(1);
      const T signed_norm = sign * norm;
      inv = T(1) / (head + signed_norm);
      new_head = -signed_norm;
      const T tt = tail_norm * t_abs(inv);
      tau = T(0.5) * (T(1) + tt * tt);
    }
    // rank test (factor.rs:52-83)
    const T norm_above = t_sqrt(above2[j] + tot[QRG_PW + 2]);
    const T total = t_hypot(norm, norm_above);
    const T threshold = eps * T((double)(mp - lr) * 16.0) * total;
    const T tau_inv = T(1) / tau;
    bool apply = false, advance = false;
    if (tau_inv < min_pos) {
      advance = norm > T(0);
    } else if (norm > threshold) {
      apply = true;
      advance = true;
    }
    if (bid == 0 && tid == 0) taus[(i64)lr * tau_stride] = tau;
    if (tid < w) {
      const T dot = rowj[tid] + inv * tot[tid];  // head_c + v^H a_c
      kc[tid] = (apply && tid > j) ? -(dot * tau_inv) : T(0);
    }
    __syncthreads();
    // ---- phase C: head, zero fill, reflector, update of the remaining panel columns ----
    const int gap = d0 + j - lr;  // col - row
    if (lr >= r0 && lr < r0 + nloc && rg == ((lr - r0) & (NWARP - 1))) {
      T* row = S + (lr - r0) * LD;
      if (lane == j) row[j] = no_tail ? head : new_head;
      if (lane > j && lane < w) row[lane] += kc[lane];
    }
    for (int r = rg; r < nloc; r += NWARP) {
      const int il = r0 + r;
      if (il > lr) {
        const T x = S[r * LD + j];
        const T vi = no_tail ? T(0) : x * inv;
        __syncwarp();
        if (lane == j) {
          S[r * LD + w + lr] = vi;                // reflector lr (overwrites a skipped attempt at the same pivot row)
          if (il <= lr + gap) S[r * LD + j] = T(0);  // factor.rs:46-48
        } else if (lane > j && lane < w) {
          S[r * LD + lane] = fma(kc[lane], vi, S[r * LD + lane]);
        }
      }
    }
    if (advance) ++lr;
    __syncthreads();
  }
  if (bid == 0 && tid == 0) info[0] = lr;
  const int local = lr;
  for (int r = tid; r < nloc; r += QRG_THREADS) {
    const int il = r0 + r;
    T* dstg = A + (i64)il * rs;
    const T* srcs = S + r * LD;
    for (int c = 0; c < w; ++c)
      if (c >= jend || il <= d0 + c) dstg[(i64)c * cs] = srcs[c];
    T* dstv = Vout + (i64)il * rs;
    for (int l = 0; l < local; ++l)
      if (il > l) dstv[(i64)l * cs] = srcs[w + l];
  }
}

// Q_coeff columns >= rank: zero, +inf on the diagonal of their T block (factor.rs:287-299)
template <class T>
__global__ void qr_coeff_fixup_kernel(T* __restrict__ H, i64 rs, i64 cs, int bs, i64 rank, i64 size) {
  const i64 c = rank + blockIdx.x;
  if (c >= size) return;
  for (int i = threadIdx.x; i < bs; i += blockDim.x) H[(i64)i * rs + c * cs] = (i == (int)(c % bs)) ? TLim<T>::inf() : T(0);
}

// dst (compact column-major, ld = nrows) <-> src view
template <class T>
__global__ void qr_save_kernel(T* __restrict__ buf, T* __restrict__ A, i64 rs, i64 cs, i64 nrows, bool restore) {
  const i64 c = blockIdx.y;
  for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (i64)gridDim.x * blockDim.x) {
    if (restore) A[i * rs + c * cs] = buf[c * nrows + i];
    else buf[c * nrows + i] = A[i * rs + c * cs];
  }
}

// above2[c] = sum_{i < nrows} A[i, c]^2 for c < w  (one CTA per column; only feeds the rank test)
template <class T>
__global__ void __launch_bounds__(256) col_sumsq_kernel(const T* __restrict__ A, i64 rs, i64 cs, i64 nrows, T* out) {
  __shared__ T red[256];
  const T* col = A + (i64)blockIdx.x * cs;
  T s = T(0);
  for (i64 i = threadIdx.x; i < nrows; i += 256) {
    const T x = col[i * rs];
    s = fma(x, x, s);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if ((int)threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = red[0];
}

}  // namespace

i64 qr_recommended_block_size(i64 nrows, i64 ncols) {
  // reference qr/no_pivoting/factor.rs:91-116
  const i64 prod = nrows * ncols, size = std::min(nrows, ncols);
  i64 bs;
  if (prod > 8192ll * 8192) bs = 256;
  else if (prod > 2048 * 2048) bs = 128;
  else if (prod > 1024 * 1024) bs = 64;
  else if (prod > 512 * 512) bs = 48;
  else if (prod > 128 * 128) bs = 32;
  else if (prod > 32 * 32) bs = 8;
  else if (prod > 16 * 16) bs = 4;
  else bs = 1;
  return std::max<i64>(1, std::min(bs, size));
}

// General driver: continues the factorization from the state (row, col) with the reference's column-skipping logic
// (factor.rs:137-256 on sub-panels of <= QRG_PW columns; every sub-panel's reflector is applied to all the columns to its
// right at once). `row` must be a multiple of the block size. Synchronous: one read-back per sub-panel. Returns the rank.
template <class T>
static i64 qr_general_from(cudaStream_t st, View<T> A, View<T> H, i64 row, i64 col, QrScratch<T> sc, T* above2, int* d_info,
                           T* apply_tmp, int Gmax) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n), bs = H.nrows;
  static bool configured = false;
  if (!configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(qr_panel_general_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  while (row < size && col < n) {
    const i64 start = row;
    i64 offset = 0, pieces = 0;
    const i64 blk = std::min(bs, std::min(size - row, n - col));
    while (offset < blk && col < n) {
      const i64 w = std::min<i64>(QRG_PW, std::min(blk - offset, n - col));
      const i64 mp = m - row;
      if (row > 0) {
        col_sumsq_kernel<T><<<(unsigned)w, 256, 0, st>>>(A.at(0, col), A.rs, A.cs, row, above2);
        FB_CUDA_CHECK(cudaGetLastError());
        note_launch();
      } else {
        FB_CUDA_CHECK(cudaMemsetAsync(above2, 0, QR_PW * sizeof(T), st));
      }
      int G = (int)std::min<i64>(Gmax, (mp + 63) / 64);
      if (G < 1) G = 1;
      int rows_per_cta = (int)((mp + G - 1) / G);
      const size_t smem = (size_t)rows_per_cta * (size_t)((2 * (int)w) | 1) * sizeof(T);
      FB_ASSERT(smem <= 200 * 1024, "QR panel too tall for the shared-memory slices");
      FB_CUDA_CHECK(cudaMemsetAsync(sc.bar, 0, 8, st));
      T* Ap = A.at(row, col);
      T* Vp = A.at(row, row);
      i64 rs = A.rs, cs = A.cs;
      int mpi = (int)mp, wi = (int)w, d0 = (int)(col - row), max_refl = (int)std::min<i64>(w, size - row);
      T* taus = H.at(offset, row);
      i64 tau_stride = H.rs + H.cs;
      const T* ab = above2;
      void* args[] = {&Ap, &Vp, &rs, &cs, &mpi, &wi, &d0, &max_refl, &rows_per_cta, &taus, &tau_stride, &sc, &ab, &d_info};
      FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)qr_panel_general_kernel<T>, dim3(G), dim3(QRG_THREADS), args, smem, st));
      note_launch();
      int local_i = 0;
      FB_CUDA_CHECK(cudaMemcpyAsync(&local_i, d_info, sizeof(int), cudaMemcpyDeviceToHost, st));
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      const i64 local = local_i;
      FB_ASSERT(local >= 0 && local <= w, "QR panel returned an impossible reflector count");
      if (local > 0) {
        View<const T> Vs = cview(A.sub(row, row, mp, local));
        View<T> Tss = H.sub(offset, row, local, local);
        householder_build_t<T>(st, Vs, Tss);
        const i64 rest = n - (col + w);
        if (rest > 0) apply_block_householder_on_the_left<T>(st, Vs, cview(Tss), A.sub(row, col + w, mp, rest), true, apply_tmp);
        ++pieces;
      }
      offset += local;
      row += local;
      col += w;
    }
    // full T of the block of reflectors [start, start + offset)
    if (pieces > 1) householder_build_t<T>(st, cview(A.sub(start, start, m - start, offset)), H.sub(0, start, offset, offset));
  }
  return row;
}

template <class T>
static void qr_coeff_fixup(cudaStream_t st, View<T> H, i64 rank) {
  const i64 size = H.ncols;
  if (rank >= size) return;
  qr_coeff_fixup_kernel<T><<<(unsigned)(size - rank), 64, 0, st>>>(H.ptr, H.rs, H.cs, (int)H.nrows, rank, size);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

template <class T>
static void qr_save_block(cudaStream_t st, T* buf, View<T> blk, bool restore) {
  if (blk.nrows == 0 || blk.ncols == 0) return;
  dim3 grid((unsigned)std::min<i64>((blk.nrows + 255) / 256, 1024), (unsigned)blk.ncols);
  qr_save_kernel<T><<<grid, 256, 0, st>>>(buf, blk.ptr, blk.rs, blk.cs, blk.nrows, restore);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

template <class T>
i64 qr_in_place(cudaStream_t st, View<T> A, View<T> H) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n), bs = H.nrows;
  FB_ASSERT(bs > 0 && H.ncols == size, "Q_coeff must be block_size x min(nrows, ncols)");
  if (size == 0) return 0;
  FB_ASSERT(m < (1ll << 31) && n < (1ll << 31), "dimension too large");
  int dev = 0, num_sms = 0;
  FB_CUDA_CHECK(cudaGetDevice(&dev));
  FB_CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  const int Gmax = std::min(num_sms, 160);  // the panel kernel's record reduction covers <= 160 CTAs
  // scratch
  const size_t part_elems = (size_t)2 * Gmax * QR_NV, rowv_elems = (size_t)2 * QR_PW;
  char* scb = (char*)ws_alloc((part_elems + rowv_elems + QR_PW) * sizeof(T) + 64);
  QrScratch<T> sc;
  sc.part = (T*)scb;
  sc.rowv = sc.part + part_elems;
  T* above2 = sc.rowv + rowv_elems;
  sc.bar = (unsigned long long*)(((uintptr_t)(above2 + QR_PW) + 15) & ~(uintptr_t)15);
  int* d_flag = (int*)ws_alloc(sizeof(int) * 4);
  FB_CUDA_CHECK(cudaMemsetAsync(sc.bar, 0, 8, st));
  FB_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
  unsigned long long bar_count = 0;
  static bool configured = false;
  if (!configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(qr_panel_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  // one W = V^H M buffer for every block-reflector application of this factorization (no per-apply pool round trip and
  // no host synchronisation inside the column loop)
  T* apply_tmp = (T*)ws_alloc((size_t)std::min(bs, size) * (size_t)n * sizeof(T));
  // the current block's columns as they were before its sub-panels touched them (restart point of the general driver)
  T* saved = (T*)ws_alloc((size_t)m * (size_t)std::min(bs, size) * sizeof(T));
  i64 rank = size;
  bool general = false;

  for (i64 j0 = 0; j0 < size; j0 += bs) {
    const i64 jb = std::min(bs, size - j0);
    qr_save_block<T>(st, saved, A.sub(j0, j0, m - j0, jb), false);
    for (i64 s0 = 0; s0 < jb; s0 += QR_PW) {
      const i64 sw = std::min<i64>(QR_PW, jb - s0), c0 = j0 + s0;
      const i64 mp = m - c0;
      // sums of squares above the panel (rank test)
      if (c0 > 0) {
        col_sumsq_kernel<T><<<(unsigned)sw, 256, 0, st>>>(A.at(0, c0), A.rs, A.cs, c0, above2);
        FB_CUDA_CHECK(cudaGetLastError());
        note_launch();
      } else {
        FB_CUDA_CHECK(cudaMemsetAsync(above2, 0, QR_PW * sizeof(T), st));
      }
      int G = (int)std::min<i64>(Gmax, (mp + 63) / 64);
      if (G < 1) G = 1;
      int rows_per_cta = (int)((mp + G - 1) / G);
      const size_t smem = (size_t)rows_per_cta * (size_t)((int)sw | 1) * sizeof(T);
      FB_ASSERT(smem <= 200 * 1024, "QR panel too tall for the shared-memory slices");
      T* Ap = A.at(c0, c0);
      i64 rs = A.rs, cs = A.cs;
      int mpi = (int)mp, wi = (int)sw;
      T* taus = H.at(s0, c0);
      i64 tau_stride = H.rs + H.cs;
      unsigned long long base = bar_count;
      const T* ab = above2;
      long long rows_below0 = (long long)(m - c0);
      void* args[] = {&Ap, &rs, &cs, &mpi, &wi, &rows_per_cta, &taus, &tau_stride, &sc, &base, &ab, &rows_below0, &d_flag};
      FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)qr_panel_kernel<T>, dim3(G), dim3(QR_THREADS), args, smem, st));
      note_launch();
      bar_count += (unsigned long long)std::min<i64>(sw, mp) * G;
      // T block of this sub-panel, then apply it to the rest of the block
      View<const T> Vs = cview(A.sub(c0, c0, mp, sw));
      View<T> Tss = H.sub(s0, c0, sw, sw);
      householder_build_t<T>(st, Vs, Tss);
      const i64 rest = j0 + jb - (c0 + sw);
      if (rest > 0)
        apply_block_householder_on_the_left<T>(st, Vs, cview(Tss), A.sub(c0, c0 + sw, mp, rest), true, apply_tmp);
    }
    // one status read per block, before the block's reflector touches the trailing matrix
    int h_flag = 0;
    FB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (h_flag) {
      qr_save_block<T>(st, saved, A.sub(j0, j0, m - j0, jb), true);
      rank = qr_general_from<T>(st, A, H, j0, j0, sc, above2, d_flag, apply_tmp, Gmax);
      general = true;
      break;
    }
    // full T of the block (off-diagonal sub-blocks V_i^H V_j; the diagonal sub-blocks are recomputed identically)
    View<const T> Vb = cview(A.sub(j0, j0, m - j0, jb));
    View<T> Tb = H.sub(0, j0, jb, jb);
    if (jb > QR_PW) householder_build_t<T>(st, Vb, Tb);
    if (j0 + jb < n)
      apply_block_householder_on_the_left<T>(st, Vb, cview(Tb), A.sub(j0, j0 + jb, m - j0, n - (j0 + jb)), true, apply_tmp);
  }
  if (general) qr_coeff_fixup<T>(st, H, rank);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(saved);
  ws_free(apply_tmp);
  ws_free(d_flag);
  ws_free(scb);
  return rank;
}

template i64 qr_in_place<double>(cudaStream_t, View<double>, View<double>);
template i64 qr_in_place<float>(cudaStream_t, View<float>, View<float>);

}  // namespace fb
