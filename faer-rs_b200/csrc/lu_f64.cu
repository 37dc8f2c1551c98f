// P2/P3 + driver: in-place LU with partial pivoting (f64).
//
// Reference: faer/src/linalg/lu/partial_pivoting/factor.rs
//   lu_in_place 234-295, lu_in_place_recursion 68-187 (split bs = round_up(n/2, min(16, next_pow2(n/2))),
//   recurse left, A01 <- unit_lower(A00)^-1 A01, A11 -= A10 A01, recurse right, then apply the level's
//   transpositions to the columns outside the window), lu_in_place_unblocked 19-67 (pivot = FIRST row attaining
//   max abs1 with strict `>` from 0; whole-row swap; multipliers by reciprocal-multiply; rank-1 update).
//
// GPU mapping (same recursion as the reference, so every GEMM is as large as the reference's):
//   * the recursion runs on the host stream; TRSM = G3, trailing update = G1 (DMMA GEMM);
//   * windows of <= 64 columns are factored by ONE cooperative kernel (`lu_panel_kernel`): the tall panel is
//     sliced by rows across up to one CTA per SM, each slice lives in shared memory for the whole panel, and each
//     column costs exactly one grid-wide barrier: every CTA publishes its best pivot candidate (value, row
//     index, the candidate row itself) and the owner of the diagonal row publishes that row; after the barrier
//     every CTA reduces the candidates redundantly (ties -> lowest row index, zeros/NaNs never selected, exactly
//     the reference's scan), the two owners exchange rows in shared memory and everybody applies the rank-1
//     update to its slice while tracking the next column's local arg-max (warp-shuffle reduction);
//   * inside the SM-partitioned look-ahead driver (dist.cu) the leaves run as ONE thread-block cluster instead
//     (`lu_panel_cluster_kernel`): candidates are exchanged through distributed shared memory with one hardware
//     cluster barrier per column — no L2 round trips on the per-column critical path;
//   * row interchanges outside the window (P3) are applied group-wise: a tiny planning kernel turns each group
//     of 64 transpositions into a net gather list (<= 128 affected rows), and the apply kernel moves all
//     affected rows of a 32-column strip through shared memory with independent loads (full memory-level
//     parallelism instead of a dependent swap chain).
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "linalg_f64.cuh"

namespace fb {

namespace {

constexpr int PANEL_W = 64;         // max panel width handled by the cooperative kernel
constexpr int PANEL_THREADS = 256;
constexpr int SWAP_GROUP = 64;      // transpositions per plan group
constexpr int SWAP_CW = 32;         // columns per CTA in the apply kernel
constexpr int SWAP_THREADS = 256;

struct Cand {
  double val;
  long long idx;
};

__device__ __forceinline__ bool cand_better(double v1, long long i1, double v2, long long i2) {
  // reference scan: `if abs > max { max = abs; imax = i }` over ascending i  => largest value, lowest index
  return v1 > v2 || (v1 == v2 && i1 < i2);
}

__device__ __forceinline__ void grid_barrier(unsigned long long* bar, unsigned long long target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1ull);
    while (*((volatile unsigned long long*)bar) < target) {
    }
    __threadfence();
  }
  __syncthreads();
}

// Net effect of transpositions [t0, t1) (rows relative to the view) as a gather list (dst row <- src row), built
// by ONE WARP. Slots 0..63 are the group's own rows t0..t0+63, pivot rows outside are appended (warp-parallel search).
template <bool TRANS_IN_SMEM = false>
__device__ __forceinline__ void build_plan_warp(const int* trans, int t0, int t1, int* ids, int* cur,
                                                int* __restrict__ out_rows, int* __restrict__ out_src,
                                                int* __restrict__ out_cnt, int lane) {
  for (int q = lane; q < 2 * SWAP_GROUP; q += 32) {
    ids[q] = q < SWAP_GROUP ? t0 + q : -1;
    cur[q] = q < SWAP_GROUP ? t0 + q : -1;
  }
  __syncwarp();
  int cnt = SWAP_GROUP;
  for (int t = t0; t < t1; ++t) {
    // global list: L2 read (it may have been written earlier in this kernel)
    const int a = t, b = t + (TRANS_IN_SMEM ? trans[t] : __ldcg(trans + t));
    if (a == b) continue;  // uniform
    const int qa = a - t0;
    int qb;
    if (b < t0 + SWAP_GROUP) {
      qb = b - t0;
    } else {
      const int q1 = SWAP_GROUP + lane, q2 = SWAP_GROUP + 32 + lane;
      const bool h1 = q1 < cnt && ids[q1] == b, h2 = q2 < cnt && ids[q2] == b;
      const unsigned m1 = __ballot_sync(0xffffffffu, h1), m2 = __ballot_sync(0xffffffffu, h2);
      if (m1) qb = SWAP_GROUP + __ffs(m1) - 1;
      else if (m2) qb = SWAP_GROUP + 32 + __ffs(m2) - 1;
      else {
        qb = cnt;
        if (lane == 0) {
          ids[cnt] = b;
          cur[cnt] = b;
        }
        ++cnt;
      }
    }
    __syncwarp();
    if (lane == 0) {
      const int tmp = cur[qa];
      cur[qa] = cur[qb];
      cur[qb] = tmp;
    }
    __syncwarp();
  }
  int out = 0;
  for (int base = 0; base < cnt; base += 32) {
    const int q = base + lane;
    const bool mv = q < cnt && ids[q] != cur[q];
    const unsigned m = __ballot_sync(0xffffffffu, mv);
    if (mv) {
      const int pos = out + __popc(m & ((1u << lane) - 1u));
      out_rows[pos] = ids[q];
      out_src[pos] = cur[q];
    }
    out += __popc(m);
  }
  if (lane == 0) *out_cnt = out;
}

// Scratch layout (doubles): for parity p in {0,1}:
//   cand_val[p][G], cand_idx[p][G] (as long long), cand_row[p][G][PANEL_W], diag_row[p][PANEL_W]
struct PanelScratch {
  double* cand_val;      // [2][G]
  long long* cand_idx;   // [2][G]
  double* cand_row;      // [2][G][PANEL_W]
  double* diag_row;      // [2][PANEL_W]
  unsigned long long* bar;
};

__global__ void __launch_bounds__(PANEL_THREADS) lu_panel_kernel(double* __restrict__ A, i64 rs, i64 cs, int m, int w,
                                                                  int rows_per_cta, int* __restrict__ trans,
                                                                  PanelScratch sc, unsigned long long bar_base,
                                                                  int* __restrict__ plan_rows, int* __restrict__ plan_src,
                                                                  int* __restrict__ plan_cnt) {
  extern __shared__ double S[];  // [rows_per_cta][LD], LD odd => conflict-free row-per-thread access
  const int LD = w | 1;
  __shared__ double pr[PANEL_W];  // pivot row
  __shared__ double dr[PANEL_W];  // old diagonal row
  __shared__ double red_val[PANEL_THREADS / 32];
  __shared__ long long red_idx[PANEL_THREADS / 32];
  __shared__ long long s_piv;
  __shared__ int s_wincta;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x, bid = blockIdx.x;
  const int r0 = bid * rows_per_cta;
  const int nloc = max(0, min(rows_per_cta, m - r0));
  const int ncol = min(w, m);  // columns to eliminate

  // ---- load slice (coalesced along rows for column-major A) ----
  // (each thread owns rows r = tid, tid+256, ...; the column loop is unrolled so 8 independent loads are in flight)
  for (int r = tid; r < nloc; r += PANEL_THREADS) {
    const double* src = A + (i64)(r0 + r) * rs;
    double* dst = S + r * LD;
#pragma unroll 8
    for (int c = 0; c < w; ++c) dst[c] = src[(i64)c * cs];
  }
  __syncthreads();

  // local arg-max of column 0 over rows >= 0
  double my_val = 0.0;
  long long my_idx = -1;
  for (int r = tid; r < nloc; r += PANEL_THREADS) {
    double v = fabs(S[r * LD + 0]);
    if (v > 0.0 && cand_better(v, r0 + r, my_val, my_idx < 0 ? (1ll << 62) : my_idx)) {
      my_val = v;
      my_idx = r0 + r;
    }
  }

  unsigned long long nbar = 0;
  for (int j = 0; j < ncol; ++j) {
    const int par = j & 1;
    // ---- (1) block-reduce the local candidate ----
    {
      double v = my_val;
      long long ix = my_idx < 0 ? (1ll << 62) : my_idx;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        double ov = __shfl_xor_sync(0xffffffffu, v, off);
        long long oi = __shfl_xor_sync(0xffffffffu, ix, off);
        if (cand_better(ov, oi, v, ix)) {
          v = ov;
          ix = oi;
        }
      }
      if (lane == 0) {
        red_val[warp] = v;
        red_idx[warp] = ix;
      }
      __syncthreads();
      if (warp == 0) {
        v = lane < PANEL_THREADS / 32 ? red_val[lane] : 0.0;
        ix = lane < PANEL_THREADS / 32 ? red_idx[lane] : (1ll << 62);
#pragma unroll
        for (int off = 4; off > 0; off >>= 1) {
          double ov = __shfl_xor_sync(0xffffffffu, v, off);
          long long oi = __shfl_xor_sync(0xffffffffu, ix, off);
          if (cand_better(ov, oi, v, ix)) {
            v = ov;
            ix = oi;
          }
        }
        if (lane == 0) {
          red_val[0] = v;
          red_idx[0] = ix;
        }
      }
      __syncthreads();
    }
    {
      const double bv = red_val[0];
      const long long bi = red_idx[0];
      if (tid == 0) {
        sc.cand_val[par * G + bid] = bv;
        sc.cand_idx[par * G + bid] = bi;
      }
      if (bv > 0.0) {
        const int lr = (int)(bi - r0);
        for (int c = tid; c < w; c += PANEL_THREADS) sc.cand_row[((i64)par * G + bid) * PANEL_W + c] = S[lr * LD + c];
      }
      if (j >= r0 && j < r0 + nloc) {
        const int lr = j - r0;
        for (int c = tid; c < w; c += PANEL_THREADS) sc.diag_row[par * PANEL_W + c] = S[lr * LD + c];
      }
    }
    ++nbar;
    grid_barrier(sc.bar, bar_base + nbar * (unsigned long long)G);

    // ---- (2) global winner (computed redundantly by every CTA) ----
    if (warp == 0) {
      double v = 0.0;
      long long ix = (1ll << 62);
      int wc = -1;
      // G <= 160: five predicated, independent (value, index) loads per lane, all in flight together
      double ovs[5];
      long long ois[5];
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        const int b = lane + 32 * u;
        ovs[u] = b < G ? __ldcg(&sc.cand_val[par * G + b]) : 0.0;
        ois[u] = b < G ? __ldcg(&sc.cand_idx[par * G + b]) : (1ll << 62);
      }
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        if (ovs[u] > 0.0 && cand_better(ovs[u], ois[u], v, ix)) {
          v = ovs[u];
          ix = ois[u];
          wc = lane + 32 * u;
        }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        double ov = __shfl_xor_sync(0xffffffffu, v, off);
        long long oi = __shfl_xor_sync(0xffffffffu, ix, off);
        int oc = __shfl_xor_sync(0xffffffffu, wc, off);
        if (cand_better(ov, oi, v, ix)) {
          v = ov;
          ix = oi;
          wc = oc;
        }
      }
      if (lane == 0) {
        // an all-zero / all-NaN column keeps imax = row (reference factor.rs:35-44)
        s_piv = (v > 0.0) ? ix : (long long)j;
        s_wincta = (v > 0.0) ? wc : -1;
      }
    }
    __syncthreads();
    const int piv = (int)s_piv;
    const int wincta = s_wincta;
    for (int c = tid; c < w; c += PANEL_THREADS) {
      const double d = __ldcg(&sc.diag_row[par * PANEL_W + c]);
      dr[c] = d;
      pr[c] = (piv != j) ? __ldcg(&sc.cand_row[((i64)par * G + wincta) * PANEL_W + c]) : d;
    }
    __syncthreads();
    if (piv != j) {
      if (piv >= r0 && piv < r0 + nloc)
        for (int c = tid; c < w; c += PANEL_THREADS) S[(piv - r0) * LD + c] = dr[c];
      if (j >= r0 && j < r0 + nloc)
        for (int c = tid; c < w; c += PANEL_THREADS) S[(j - r0) * LD + c] = pr[c];
    }
    if (bid == 0 && tid == 0) trans[j] = piv - j;
    __syncthreads();

    // ---- (3) multipliers + rank-1 update of the slice; track next column's local arg-max ----
    const double inv = 1.0 / pr[j];
    my_val = 0.0;
    my_idx = -1;
    for (int r = tid; r < nloc; r += PANEL_THREADS) {
      if (r0 + r > j) {
        double* row = S + r * LD;
        const double l = row[j] * inv;
        row[j] = l;
        for (int c = j + 1; c < w; ++c) row[c] = fma(-l, pr[c], row[c]);
        if (j + 1 < w) {
          const double v = fabs(row[j + 1]);
          if (v > 0.0 && cand_better(v, r0 + r, my_val, my_idx < 0 ? (1ll << 62) : my_idx)) {
            my_val = v;
            my_idx = r0 + r;
          }
        }
      }
    }
    // (the block reduction at the top of the next iteration starts with __syncthreads-protected smem)
  }
  __syncthreads();
  // ---- store slice ----
  for (int r = tid; r < nloc; r += PANEL_THREADS) {
    double* dstg = A + (i64)(r0 + r) * rs;
    const double* srcs = S + r * LD;
#pragma unroll 8
    for (int c = 0; c < w; ++c) dstg[(i64)c * cs] = srcs[c];
  }
  // ---- swap plan for this window (one group) so that the caller can permute the outside columns ----
  if (plan_rows != nullptr && bid == 0) {
    __shared__ int p_ids[2 * SWAP_GROUP], p_cur[2 * SWAP_GROUP];
    __syncthreads();  // thread 0's `trans` writes (global) are ordered before the reads below
    __threadfence_block();
    if (warp == 0) build_plan_warp(trans, 0, ncol, p_ids, p_cur, plan_rows, plan_src, plan_cnt, lane);
  }
}

// ---- cluster variant of the panel kernel --------------------------------------------------------------------------
// Same algorithm, but the CTAs form ONE thread-block cluster (8 portable, 16 opt-in) and the per-column exchange goes
// through distributed shared memory: every CTA stores its candidate (value, row index, the row itself) into the
// exchange buffer of EVERY CTA of the cluster, one hardware cluster barrier makes the stores visible, and the scan /
// pivot-row fetch are local shared-memory reads. The grid-barrier version pays three dependent L2 round trips per
// column (arrival counter, candidate records, winner row); here the exchange costs one cluster barrier.
// The slices live in shared memory as before (<= ~190 KB per CTA), so the panel is narrower for tall matrices
// (w in {64, 32, 16, 8} by height) and the host recursion supplies the rest (lu_rec).
constexpr int CL_THREADS = 512;
constexpr int CL_MAXC = 16;

struct ClExchange {
  double val[2][CL_MAXC];
  long long idx[2][CL_MAXC];
  double row[2][CL_MAXC][PANEL_W];
  double diag[2][PANEL_W];
};

__global__ void __launch_bounds__(CL_THREADS) lu_panel_cluster_kernel(double* __restrict__ A, i64 rs, i64 cs, int m, int w,
                                                                       int rows_per_cta, int* __restrict__ trans,
                                                                       int* __restrict__ plan_rows,
                                                                       int* __restrict__ plan_src,
                                                                       int* __restrict__ plan_cnt) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  extern __shared__ double S[];  // [rows_per_cta][LD]
  const int LD = w | 1;
  __shared__ ClExchange X;
  __shared__ double pr[PANEL_W];
  __shared__ double dr[PANEL_W];
  __shared__ double red_val[CL_THREADS / 32];
  __shared__ long long red_idx[CL_THREADS / 32];
  __shared__ long long s_piv;
  __shared__ int s_wincta;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = rank * rows_per_cta;
  const int nloc = max(0, min(rows_per_cta, m - r0));
  const int ncol = min(w, m);

  for (int r = tid; r < nloc; r += CL_THREADS) {
    const double* src = A + (i64)(r0 + r) * rs;
    double* dst = S + r * LD;
#pragma unroll 8
    for (int c = 0; c < w; ++c) dst[c] = src[(i64)c * cs];
  }
  double my_val = 0.0;
  long long my_idx = -1;
  __syncthreads();
  for (int r = tid; r < nloc; r += CL_THREADS) {
    const double v = fabs(S[r * LD + 0]);
    if (v > 0.0 && cand_better(v, r0 + r, my_val, my_idx < 0 ? (1ll << 62) : my_idx)) {
      my_val = v;
      my_idx = r0 + r;
    }
  }
  cluster.sync();  // every CTA of the cluster is resident and its exchange buffer may be written

  for (int j = 0; j < ncol; ++j) {
    const int par = j & 1;
    // ---- (1) CTA-wide candidate ----
    {
      double v = my_val;
      long long ix = my_idx < 0 ? (1ll << 62) : my_idx;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, off);
        const long long oi = __shfl_xor_sync(0xffffffffu, ix, off);
        if (cand_better(ov, oi, v, ix)) {
          v = ov;
          ix = oi;
        }
      }
      if (lane == 0) {
        red_val[warp] = v;
        red_idx[warp] = ix;
      }
      __syncthreads();
      if (warp == 0) {
        v = lane < CL_THREADS / 32 ? red_val[lane] : 0.0;
        ix = lane < CL_THREADS / 32 ? red_idx[lane] : (1ll << 62);
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) {
          const double ov = __shfl_xor_sync(0xffffffffu, v, off);
          const long long oi = __shfl_xor_sync(0xffffffffu, ix, off);
          if (cand_better(ov, oi, v, ix)) {
            v = ov;
            ix = oi;
          }
        }
        if (lane == 0) {
          red_val[0] = v;
          red_idx[0] = ix;
        }
      }
      __syncthreads();
    }
    // ---- (2) publish to every CTA of the cluster: warp `warp` serves destination rank `warp` ----
    {
      const double bv = red_val[0];
      const long long bi = red_idx[0];
      if (warp < C) {
        ClExchange* Xr = cluster.map_shared_rank(&X, warp);
        if (lane == 0) {
          Xr->val[par][rank] = bv;
          Xr->idx[par][rank] = bi;
        }
        if (bv > 0.0) {
          const int lr = (int)(bi - r0);
          for (int c = lane; c < w; c += 32) Xr->row[par][rank][c] = S[lr * LD + c];
        }
        if (j >= r0 && j < r0 + nloc) {
          const int lr = j - r0;
          for (int c = lane; c < w; c += 32) Xr->diag[par][c] = S[lr * LD + c];
        }
      }
    }
    cluster.sync();
    // ---- (3) winner (local scan of the C candidates), pivot row, old diagonal row ----
    if (warp == 0) {
      double v = lane < C ? X.val[par][lane] : 0.0;
      long long ix = lane < C ? X.idx[par][lane] : (1ll << 62);
      int wc = lane;
      if (!(v > 0.0)) {
        v = 0.0;
        ix = (1ll << 62);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, off);
        const long long oi = __shfl_xor_sync(0xffffffffu, ix, off);
        const int oc = __shfl_xor_sync(0xffffffffu, wc, off);
        if (cand_better(ov, oi, v, ix)) {
          v = ov;
          ix = oi;
          wc = oc;
        }
      }
      if (lane == 0) {
        s_piv = (v > 0.0) ? ix : (long long)j;  // all-zero / all-NaN column keeps imax = row (factor.rs:35-44)
        s_wincta = (v > 0.0) ? wc : -1;
      }
    }
    __syncthreads();
    const int piv = (int)s_piv;
    const int wincta = s_wincta;
    for (int c = tid; c < w; c += CL_THREADS) {
      const double d = X.diag[par][c];
      dr[c] = d;
      pr[c] = (piv != j) ? X.row[par][wincta][c] : d;
    }
    __syncthreads();
    if (piv != j) {
      if (piv >= r0 && piv < r0 + nloc)
        for (int c = tid; c < w; c += CL_THREADS) S[(piv - r0) * LD + c] = dr[c];
      if (j >= r0 && j < r0 + nloc)
        for (int c = tid; c < w; c += CL_THREADS) S[(j - r0) * LD + c] = pr[c];
    }
    if (rank == 0 && tid == 0) trans[j] = piv - j;
    __syncthreads();
    // ---- (4) multipliers + rank-1 update; next column's local arg-max ----
    const double inv = 1.0 / pr[j];
    my_val = 0.0;
    my_idx = -1;
    for (int r = tid; r < nloc; r += CL_THREADS) {
      if (r0 + r > j) {
        double* row = S + r * LD;
        const double l = row[j] * inv;
        row[j] = l;
        for (int c = j + 1; c < w; ++c) row[c] = fma(-l, pr[c], row[c]);
        if (j + 1 < w) {
          const double v = fabs(row[j + 1]);
          if (v > 0.0 && cand_better(v, r0 + r, my_val, my_idx < 0 ? (1ll << 62) : my_idx)) {
            my_val = v;
            my_idx = r0 + r;
          }
        }
      }
    }
  }
  __syncthreads();
  for (int r = tid; r < nloc; r += CL_THREADS) {
    double* dstg = A + (i64)(r0 + r) * rs;
    const double* srcs = S + r * LD;
#pragma unroll 8
    for (int c = 0; c < w; ++c) dstg[(i64)c * cs] = srcs[c];
  }
  if (plan_rows != nullptr && rank == 0) {
    __shared__ int p_ids[2 * SWAP_GROUP], p_cur[2 * SWAP_GROUP];
    __syncthreads();
    __threadfence_block();
    if (warp == 0) build_plan_warp(trans, 0, ncol, p_ids, p_cur, plan_rows, plan_src, plan_cnt, lane);
  }
  cluster.sync();  // no CTA may exit while its shared memory can still be addressed by the others
}

// ---- fused sub-panel kernel (one cluster, one launch for up to SP_MAXW columns) -----------------------------------
// The cluster panel above keeps every row slice in shared memory, so for tall panels its windows are narrow (8 columns
// at 32768 rows) and the host recursion over them costs more in small launches (row swaps, TRSM leaves, thin GEMMs)
// than the pivot chain itself. This kernel factors
// a whole W-column sub-panel (W <= 256) in ONE launch: the sub-panel stays in global memory (L2-resident: 32768 x 128
// doubles = 33 MB), the current window of WW columns lives in REGISTERS (thread t of a CTA owns the rows t, t + 512, ...
// of the CTA's slice: R rows x WW columns, R * WW = 32 doubles), and the steps the recursion did with separate launches
// are done in place, Crout order (each entry is written once):
//   S1  window columns  -= L[:, 0:j0] * U[0:j0, window]          (R x WW accumulators per thread, U block in shared memory)
//   S2  pivot search / swap / rank-1 update of the window, one hardware cluster barrier per column, candidates and rows
//       exchanged through distributed shared memory; the column loop is fully unrolled so the window stays in registers
//   S3  the window's transpositions applied to the other columns of the sub-panel (gather plan, columns dealt to CTAs)
//   S4  rows of U to the right of the window: (A[j0:j0+ww, c] - L[j0:j0+ww, 0:j0] U[0:j0, c]), then the unit-lower
//       solve with the window's top block (columns dealt to CTAs)
// An earlier version kept the window in shared memory; the rank-1 update there and a Crout pass with 4 loads in flight
// per thread were the largest costs per column.
// Same pivot rule as the reference's scan (largest |a|, lowest row, zeros / NaNs never chosen), same swaps, multipliers
// by reciprocal-multiply; the floating-point operation ORDER differs from the recursive formulation (as any blocked LU
// does), which the parity tests cover by comparing permutations exactly and factors to tolerance.
constexpr int SP_THREADS = 512;
constexpr int SP_MAXW = 256;  // widest fused sub-panel
constexpr int SP_MAXWW = 32;  // widest window
constexpr int SP_CG = 8;      // right-hand columns per S4 chunk

// One candidate record as it travels between CTAs: 16-byte header + the candidate row (always SP_MAXWW slots, WW sent)
struct alignas(16) SpRec {
  double val;
  long long idx;
  double row[SP_MAXWW];
};

// ---- cluster exchange primitives: bulk shared -> remote-shared copies that signal the DESTINATION's mbarrier ----
__device__ __forceinline__ uint32_t sp_mapa(uint32_t cta_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(cta_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void sp_bulk_to_cluster(uint32_t dst_cluster, uint32_t src_cta, uint32_t bytes, uint32_t mbar_cluster) {
  asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_cluster),
               "r"(src_cta), "r"(bytes), "r"(mbar_cluster)
               : "memory");
}
__device__ __forceinline__ void sp_mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void sp_mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sp_mbar_wait(unsigned long long* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}

// Warp-wide (value, row) arg-max with the reference's tie rule (largest value, lowest row), result in every lane.
// v >= 0 and not NaN (0 = "no candidate"); the bit pattern of a non-negative double orders like the value, so the maximum is
// found with two 32-bit integer reductions and the lowest row among the lanes that hold it with a third.
__device__ __forceinline__ void warp_argmax(double& v, int& ix) {
  const unsigned long long key = (unsigned long long)__double_as_longlong(v);
  const unsigned hi = (unsigned)(key >> 32), lo = (unsigned)key;
  const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
  const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
  const bool top = hi == mh && lo == ml;
  const unsigned mi = __reduce_min_sync(0xffffffffu, top ? (unsigned)ix : 0xffffffffu);
  v = __longlong_as_double((long long)(((unsigned long long)mh << 32) | ml));
  ix = (int)mi;
}

template <int WW, int R>
__global__ void __launch_bounds__(SP_THREADS) lu_subpanel_cluster_kernel(double* __restrict__ A, i64 rs, i64 cs, int m,
                                                                          int W, int rows_per_cta,
                                                                          int* __restrict__ trans,
                                                                          int* __restrict__ plan_rows,
                                                                          int* __restrict__ plan_src,
                                                                          int* __restrict__ plan_cnt,
                                                                          long long* __restrict__ prof) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  // Cycle counts per phase, accumulated by thread 0 of CTA 0 when prof != nullptr. The host always passes nullptr; the
  // counters stay because the branches they add shape ptxas's register allocation: without them the <32, 1> instantiation
  // spills ~44 KB and f64 LU at n = 8192 takes 145 ms instead of 50 ms (H100 80GB HBM3, 700 W).
  __shared__ long long pt[9];  // [8] = time of the last tick
  const bool profiling = prof != nullptr && rank == 0 && threadIdx.x == 0;
  if (profiling)
    for (int i = 0; i < 9; ++i) pt[i] = 0;
  auto tick = [&](int slot) {
    if (profiling) {
      const long long now = clock64();
      pt[slot] += now - pt[8];
      pt[8] = now;
    }
  };
  extern __shared__ double smem_sp[];
  double* R1 = smem_sp;                  // [W][WW]: S1: U[0:j0, window] (k-major); S4: L rows [ww][j0]
  double* R2 = R1 + (size_t)W * WW;      // [W][SP_CG]   S4: U[0:j0, chunk]
  __shared__ SpRec Xrec[2][CL_MAXC];                 // received candidate records [parity][source CTA]
  __shared__ alignas(16) double Xdiag[2][SP_MAXWW];  // received diagonal row [parity]
  __shared__ SpRec rec_s[2];                         // send staging [parity]
  __shared__ alignas(16) double diag_s[2][SP_MAXWW];
  __shared__ alignas(8) unsigned long long xbar[2];  // one mbarrier per parity: all of a column's records have landed
  __shared__ double L11s[SP_MAXWW][SP_MAXWW + 1];
  __shared__ double X4[SP_MAXWW][SP_CG];
  __shared__ double red_val[SP_THREADS / 32];
  __shared__ int red_idx[SP_THREADS / 32];
  __shared__ int trans_s[SP_MAXW];
  __shared__ int p_rows[2 * SWAP_GROUP], p_src[2 * SWAP_GROUP];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = rank * rows_per_cta;
  const int nloc = max(0, min(rows_per_cta, m - r0));
  // this thread's rows: local tid + 512 q, global gr[q]
  int gr[R];
  bool have[R];
#pragma unroll
  for (int q = 0; q < R; ++q) {
    gr[q] = r0 + tid + SP_THREADS * q;
    have[q] = tid + SP_THREADS * q < nloc;
  }

  if (tid == 0) {
    sp_mbar_init(&xbar[0], 1);
    sp_mbar_init(&xbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster.sync();  // every CTA of the cluster is resident and its barriers are initialised: records may be sent to it
  if (profiling) pt[8] = clock64();
  // per column every CTA receives one record from each CTA (itself included) and the diagonal row
  constexpr uint32_t REC_BYTES = 16 + WW * 8, DIAG_BYTES = WW * 8;
  const uint32_t col_bytes = (uint32_t)C * REC_BYTES + DIAG_BYTES;
  uint32_t ccount = 0;  // columns done: parity = ccount & 1, barrier phase = (ccount >> 1) & 1

  for (int j0 = 0; j0 < W; j0 += WW) {
    const int ww = min(WW, W - j0);
    // ================= S1: the window into registers, minus the sub-panel's earlier columns (Crout) =================
    for (int e = tid; e < j0 * WW; e += SP_THREADS) {
      const int k = e / WW, c = e - k * WW;
      R1[e] = c < ww ? __ldcg(A + (i64)k * rs + (i64)(j0 + c) * cs) : 0.0;
    }
    double a[R][WW];
    bool act[R];  // rows on / below the window's diagonal block (rows above hold finished U entries: not ours)
#pragma unroll
    for (int q = 0; q < R; ++q) {
      act[q] = have[q] && gr[q] >= j0;
#pragma unroll
      for (int c = 0; c < WW; ++c) a[q][c] = (act[q] && c < ww) ? __ldcg(A + (i64)gr[q] * rs + (i64)(j0 + c) * cs) : 0.0;
    }
    __syncthreads();
    {
      constexpr int KU = (R >= 8) ? 2 : (R == 4 ? 4 : 8);  // R * KU = 8 or 16 loads in flight per thread
      int k = 0;
      for (; k + KU <= j0; k += KU) {
        double l[R][KU];
#pragma unroll
        for (int q = 0; q < R; ++q)
#pragma unroll
          for (int u = 0; u < KU; ++u) l[q][u] = act[q] ? __ldcg(A + (i64)gr[q] * rs + (i64)(k + u) * cs) : 0.0;
#pragma unroll
        for (int u = 0; u < KU; ++u) {
          const double* uu = R1 + (size_t)(k + u) * WW;
#pragma unroll
          for (int c = 0; c < WW; ++c) {
            const double uv = uu[c];
#pragma unroll
            for (int q = 0; q < R; ++q) a[q][c] = fma(-l[q][u], uv, a[q][c]);
          }
        }
      }
      for (; k < j0; ++k) {
        const double* uu = R1 + (size_t)k * WW;
#pragma unroll
        for (int q = 0; q < R; ++q) {
          const double lv = act[q] ? __ldcg(A + (i64)gr[q] * rs + (i64)k * cs) : 0.0;
#pragma unroll
          for (int c = 0; c < WW; ++c) a[q][c] = fma(-lv, uu[c], a[q][c]);
        }
      }
    }
    tick(0);
    // ================= S2: the window's columns (fully unrolled: a[][] stays in registers) =================
    // Per column the critical path is: thread candidate -> warp arg-max -> CTA arg-max -> candidate / diagonal row into the
    // exchange buffers of all CTAs -> cluster barrier -> cluster arg-max -> reciprocal -> rank-1 update. The arg-max steps
    // use three integer warp reductions (redux.sync) on the bit pattern of |a| (monotone for non-negative doubles) and on
    // the row index instead of 64-bit shuffle butterflies, and the rows are pushed by the owner's own warp (no second CTA
    // barrier).
#pragma unroll
    for (int j = 0; j < WW; ++j) {
      if (j < ww) {  // uniform
        const int par = (int)(ccount & 1u);
        const uint32_t phase = (ccount >> 1) & 1u;
        ++ccount;
        const int dj = j0 + j;  // global row of the diagonal
        // ---- candidate of this thread, warp, CTA ----
        double v = 0.0;
        int ix = 0x7fffffff;
#pragma unroll
        for (int q = 0; q < R; ++q) {
          const double t = fabs(a[q][j]);
          if (have[q] && gr[q] >= dj && t > 0.0 && (t > v || (t == v && gr[q] < ix))) {
            v = t;
            ix = gr[q];
          }
        }
        warp_argmax(v, ix);
        if (lane == 0) {
          red_val[warp] = v;
          red_idx[warp] = ix;
        }
        __syncthreads();
        v = lane < SP_THREADS / 32 ? red_val[lane] : 0.0;
        ix = lane < SP_THREADS / 32 ? red_idx[lane] : 0x7fffffff;
        warp_argmax(v, ix);  // every warp holds the CTA's candidate (v, ix) in all lanes
        if (tid == 0) sp_mbar_expect_tx(&xbar[par], col_bytes);
        // ---- the warp that owns the candidate row sends the record to every CTA of the cluster (one bulk copy per
        // destination, completing on the destination's barrier); the warp that owns the diagonal row sends that one ----
        {
          const int lr = (v > 0.0) ? ix - r0 : 0;
          const int o_warp = (lr & (SP_THREADS - 1)) >> 5;
          if (warp == o_warp) {
            if (lane == 0) {
              rec_s[par].val = v;
              rec_s[par].idx = ix;
            }
#pragma unroll
            for (int q = 0; q < R; ++q) {
              if (v > 0.0 && have[q] && gr[q] == ix) {
#pragma unroll
                for (int c = 0; c < WW; ++c) rec_s[par].row[c] = a[q][c];
              }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> async-proxy reads
            __syncwarp();
            if (lane < C)
              sp_bulk_to_cluster(sp_mapa(smem_u32(&Xrec[par][rank]), (uint32_t)lane), smem_u32(&rec_s[par]), REC_BYTES,
                                 sp_mapa(smem_u32(&xbar[par]), (uint32_t)lane));
          }
          const bool diag_here = dj >= r0 && dj < r0 + nloc;
          if (diag_here && warp == (((dj - r0) & (SP_THREADS - 1)) >> 5)) {
#pragma unroll
            for (int q = 0; q < R; ++q) {
              if (have[q] && gr[q] == dj) {
#pragma unroll
                for (int c = 0; c < WW; ++c) diag_s[par][c] = a[q][c];
              }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane < C)
              sp_bulk_to_cluster(sp_mapa(smem_u32(&Xdiag[par][0]), (uint32_t)lane), smem_u32(&diag_s[par][0]), DIAG_BYTES,
                                 sp_mapa(smem_u32(&xbar[par]), (uint32_t)lane));
          }
        }
        tick(1);
        sp_mbar_wait(&xbar[par], phase);
        tick(2);
        // ---- winner: every warp scans the C candidates redundantly ----
        int piv, wincta;
        {
          double gv = lane < C ? Xrec[par][lane].val : 0.0;
          int gi = lane < C ? (int)Xrec[par][lane].idx : 0x7fffffff;
          if (!(gv > 0.0)) {
            gv = 0.0;
            gi = 0x7fffffff;
          }
          const double mv = gv;
          const int mi = gi;
          warp_argmax(gv, gi);
          const unsigned who = __ballot_sync(0xffffffffu, mv == gv && mi == gi && lane < C);
          // an all-zero / all-NaN column keeps imax = row (reference factor.rs:35-44)
          piv = (gv > 0.0) ? gi : dj;
          wincta = (gv > 0.0) ? (__ffs(who) - 1) : -1;
        }
        const double* prow = (piv != dj) ? Xrec[par][wincta].row : Xdiag[par];
        const double* drow = Xdiag[par];
        if (tid == 0) {
          trans_s[dj] = piv - dj;
          if (rank == 0) trans[dj] = piv - dj;
        }
        // ---- swap (in registers), multipliers (reciprocal-multiply, as the reference), rank-1 update ----
        // the pivot row from column j on, read once per thread with 16-byte loads (the rows are 16-byte aligned)
        // (narrow windows only: 32 extra doubles would not fit next to a 32-column window)
        constexpr int PRN = WW <= 16 ? WW : 1;
        double pr[PRN];
        if constexpr (WW <= 16) {
#pragma unroll
          for (int c = (j & ~1); c < WW; c += 2) {
            const double2 t2 = *reinterpret_cast<const double2*>(prow + c);
            pr[c] = t2.x;
            pr[c + 1] = t2.y;
          }
        }
        const double inv = __drcp_rn(prow[j]);
#pragma unroll
        for (int q = 0; q < R; ++q) {
          if (have[q] && piv != dj) {
            if (gr[q] == piv) {
#pragma unroll
              for (int c = 0; c < WW; ++c)
                if (c < ww) a[q][c] = drow[c];
            } else if (gr[q] == dj) {
#pragma unroll
              for (int c = 0; c < WW; ++c)
                if (c < ww) a[q][c] = prow[c];
            }
          }
          if (have[q] && gr[q] > dj) {
            const double l = a[q][j] * inv;
            a[q][j] = l;
#pragma unroll
            for (int c = j + 1; c < WW; ++c)
              if (c < ww) a[q][c] = fma(-l, (WW <= 16 ? pr[c < PRN ? c : 0] : prow[c]), a[q][c]);
          }
        }
        tick(3);
      }
    }
    // store the window (rows above j0 hold finished U entries written in S4: not ours to touch)
#pragma unroll
    for (int q = 0; q < R; ++q) {
      if (act[q]) {
        double* dstg = A + (i64)gr[q] * rs + (i64)j0 * cs;
#pragma unroll
        for (int c = 0; c < WW; ++c)
          if (c < ww) dstg[(i64)c * cs] = a[q][c];
      }
    }
    const int nother = W - ww;  // columns of the sub-panel outside the window
    if (nother == 0) break;     // uniform
    // ================= S3: the window's transpositions on the other columns =================
    __syncthreads();  // trans_s
    // gather plan of the window's transpositions, one candidate row per slot (slots 0..ww-1: the diagonal rows, ww..2ww-1: the
    // pivot rows), each followed independently through the ww transpositions: dst = final position of original row src
    if (tid < 2 * WW) {
      const int sl = tid;
      int src = -1;
      if (sl < ww) src = j0 + sl;
      else if (sl < 2 * ww) {
        const int t = sl - ww;
        src = j0 + t + trans_s[j0 + t];
        bool dup = src < j0 + ww;  // a diagonal row: already has a slot
        for (int t2 = 0; t2 < t; ++t2) dup = dup || (j0 + t2 + trans_s[j0 + t2] == src);
        if (dup) src = -1;
      }
      int pos = src;
      for (int t = 0; t < ww; ++t) {
        const int ra = j0 + t, rb = ra + trans_s[ra];
        pos = (pos == ra) ? rb : ((pos == rb) ? ra : pos);
      }
      p_src[sl] = src;
      p_rows[sl] = (src >= 0 && pos != src) ? pos : -1;
    }
    cluster.sync();  // (A) window stores visible cluster-wide; plan visible CTA-wide
    tick(4);
    {
      const int qs = tid & (2 * SWAP_GROUP - 1), cb = tid >> 7;  // 128 plan slots x 4 columns in flight
      const bool on_slot = qs < 2 * ww && p_rows[qs] >= 0;
      const i64 srow = on_slot ? (i64)p_src[qs] : 0, drw = on_slot ? (i64)p_rows[qs] : 0;
      // my columns: oc = rank, rank + C, ... over the nother other columns
      for (int base = rank; base < nother; base += 4 * C) {
        const int oc = base + cb * C;
        const bool on = on_slot && oc < nother;
        const int col = oc < j0 ? oc : oc + ww;
        double v = 0.0;
        if (on) v = __ldcg(A + srow * rs + (i64)col * cs);
        __syncthreads();
        if (on) A[drw * rs + (i64)col * cs] = v;
        __syncthreads();
      }
    }
    const int nright = W - j0 - ww;
    tick(5);
    if (nright > 0) {
      cluster.sync();  // (B) swapped rows visible
      // ================= S4: rows j0 .. j0+ww of U to the right of the window =================
      // L rows of the window's diagonal block rows against the earlier columns, and the block itself
      for (int e = tid; e < ww * j0; e += SP_THREADS) {
        const int i = e / j0, k = e - i * j0;
        R1[e] = __ldcg(A + (i64)(j0 + i) * rs + (i64)k * cs);  // [i][k], leading dimension j0
      }
      for (int e = tid; e < ww * ww; e += SP_THREADS) {
        const int i = e / ww, i2 = e - i * ww;
        L11s[i][i2] = __ldcg(A + (i64)(j0 + i) * rs + (i64)(j0 + i2) * cs);
      }
      // my right-hand columns: rc = rank, rank + C, ...; SP_CG at a time
      for (int cbase = rank; cbase < nright; cbase += SP_CG * C) {
        __syncthreads();
        for (int e = tid; e < j0 * SP_CG; e += SP_THREADS) {
          const int cl = e / j0, k = e - cl * j0;  // k fastest: coalesced along the column
          const int rc = cbase + cl * C;
          R2[k * SP_CG + cl] = rc < nright ? __ldcg(A + (i64)k * rs + (i64)(j0 + ww + rc) * cs) : 0.0;
        }
        __syncthreads();
        if (tid < ww * SP_CG) {
          const int i = tid / SP_CG, cl = tid - i * SP_CG;
          const int rc = cbase + cl * C;
          double x = 0.0;
          if (rc < nright) {
            x = __ldcg(A + (i64)(j0 + i) * rs + (i64)(j0 + ww + rc) * cs);
            const double* lr = R1 + (size_t)i * j0;
            // four partial sums: the dot product is a latency chain otherwise
            double x0 = 0.0, x1 = 0.0, x2 = 0.0, x3 = 0.0;
            int k = 0;
            for (; k + 4 <= j0; k += 4) {
              x0 = fma(lr[k], R2[k * SP_CG + cl], x0);
              x1 = fma(lr[k + 1], R2[(k + 1) * SP_CG + cl], x1);
              x2 = fma(lr[k + 2], R2[(k + 2) * SP_CG + cl], x2);
              x3 = fma(lr[k + 3], R2[(k + 3) * SP_CG + cl], x3);
            }
            for (; k < j0; ++k) x0 = fma(lr[k], R2[k * SP_CG + cl], x0);
            x -= (x0 + x1) + (x2 + x3);
          }
          X4[i][cl] = x;
        }
        __syncthreads();
        if (tid < SP_CG) {
          const int cl = tid;
          const int rc = cbase + cl * C;
          if (rc < nright) {
            double xs[SP_MAXWW];
#pragma unroll
            for (int i = 0; i < SP_MAXWW; ++i) {
              if (i < ww) {
                double x = X4[i][cl];
#pragma unroll
                for (int i2 = 0; i2 < SP_MAXWW; ++i2)
                  if (i2 < i) x = fma(-L11s[i][i2], xs[i2], x);
                xs[i] = x;
                A[(i64)(j0 + i) * rs + (i64)(j0 + ww + rc) * cs] = x;
              }
            }
          }
        }
      }
    }
    cluster.sync();  // (C) U rows / swapped columns visible before the next window reads them
    tick(6);
  }
  // gather plans of the sub-panel's transpositions (groups of 64) for the caller's row swaps on the outside columns: built
  // here by CTA 0 (every CTA holds all of trans_s) instead of by a separate one-warp launch
  if (plan_rows != nullptr && rank == 0) {
    __syncthreads();  // trans_s of the last window
    const int ngroups = (W + SWAP_GROUP - 1) / SWAP_GROUP;
    __shared__ int g_ids[SP_MAXW / SWAP_GROUP][2 * SWAP_GROUP], g_cur[SP_MAXW / SWAP_GROUP][2 * SWAP_GROUP];
    if (warp < ngroups)
      build_plan_warp<true>(trans_s, warp * SWAP_GROUP, min(W, (warp + 1) * SWAP_GROUP), g_ids[warp], g_cur[warp],
                            plan_rows + (i64)warp * 2 * SWAP_GROUP, plan_src + (i64)warp * 2 * SWAP_GROUP, plan_cnt + warp, lane);
  }
  if (profiling)
    for (int i = 0; i < 8; ++i) atomicAdd((unsigned long long*)prof + i, (unsigned long long)pt[i]);
  cluster.sync();  // no CTA may exit while its shared memory can still be addressed by the others
}

__global__ void __launch_bounds__(32) laswp_plan_kernel(const int* __restrict__ trans, int n, int* __restrict__ plan_rows,
                                                        int* __restrict__ plan_src, int* __restrict__ plan_cnt,
                                                        int ngroups) {
  __shared__ int ids[2 * SWAP_GROUP], cur[2 * SWAP_GROUP];
  const int gi = blockIdx.x;
  if (gi >= ngroups) return;
  const int t0 = gi * SWAP_GROUP, t1 = min(n, t0 + SWAP_GROUP);
  build_plan_warp(trans, t0, t1, ids, cur, plan_rows + (i64)gi * 2 * SWAP_GROUP, plan_src + (i64)gi * 2 * SWAP_GROUP,
                  plan_cnt + gi, threadIdx.x);
}

// Apply the gather lists of all groups (in order) to a strip of SWAP_CW columns per CTA.
__global__ void __launch_bounds__(SWAP_THREADS) laswp_apply_kernel(double* __restrict__ A, i64 rs, i64 cs, i64 ncols,
                                                                    const int* __restrict__ plan_rows,
                                                                    const int* __restrict__ plan_src,
                                                                    const int* __restrict__ plan_cnt, int ngroups) {
  __shared__ double tile[2 * SWAP_GROUP][SWAP_CW + 1];
  const i64 c0 = (i64)blockIdx.x * SWAP_CW;
  const int nc = (int)min((i64)SWAP_CW, ncols - c0);
  const int tid = threadIdx.x;
  const int q = tid & (2 * SWAP_GROUP - 1), cb = tid >> 7;  // 256 threads = 128 rows x 2 column phases
  for (int gi = 0; gi < ngroups; ++gi) {
    const int cnt = plan_cnt[gi];
    if (cnt == 0) continue;
    const bool act = q < cnt;
    const i64 srow = act ? (i64)plan_src[(i64)gi * 2 * SWAP_GROUP + q] : 0;
    const i64 drow = act ? (i64)plan_rows[(i64)gi * 2 * SWAP_GROUP + q] : 0;
    // independent loads, unrolled => full memory-level parallelism
#pragma unroll 8
    for (int cc = 0; cc < SWAP_CW / 2; ++cc) {
      const int c = cb + 2 * cc;
      if (act && c < nc) tile[q][c] = A[srow * rs + (c0 + c) * cs];
    }
    __syncthreads();
#pragma unroll 8
    for (int cc = 0; cc < SWAP_CW / 2; ++cc) {
      const int c = cb + 2 * cc;
      if (act && c < nc) A[drow * rs + (c0 + c) * cs] = tile[q][c];
    }
    __syncthreads();
  }
}

inline i64 next_pow2(i64 n) {
  i64 p = 1;
  while (p < n) p <<= 1;
  return p;
}

struct LuCtx {
  cudaStream_t st;
  int num_sms;
  int* d_trans;          // [size]
  int* plan_rows;        // [ngroups_max][2*SWAP_GROUP]
  int* plan_src;
  int* plan_cnt;         // [ngroups_max]
  PanelScratch sc;
  unsigned long long bar_count;  // host mirror of the barrier counter
  int cluster_ctas = 0;           // > 0: factor leaves with the cluster (DSMEM) panel kernel on this many CTAs
  cudaStream_t st_big = nullptr;  // optional: stream of a larger SM partition for the recursion's big TRSM / GEMM nodes
  cudaEvent_t ev_to_big = nullptr, ev_from_big = nullptr;
};

constexpr i64 PANEL_SMEM_BUDGET = 200 * 1024;

// widest window (<= PANEL_W) whose row slices (ceil(m / #CTAs) rows x (w|1) doubles) fit in shared memory
constexpr i64 CL_SMEM_BUDGET = 200 * 1024;
int cluster_width_for(int C, i64 m) {
  const i64 rows = std::max<i64>(1, (m + C - 1) / C);
  for (int w = PANEL_W; w >= 1; w >>= 1)
    if (rows * (i64)(w | 1) * 8 <= CL_SMEM_BUDGET) return w;
  return 0;
}

int panel_width_for(const LuCtx& ctx, i64 m) {
  if (ctx.cluster_ctas > 0) {
    const int wc = cluster_width_for(ctx.cluster_ctas, m);
    if (wc >= 4) return wc;
  }
  const i64 rows = std::max<i64>(1, (m + ctx.num_sms - 1) / ctx.num_sms);
  i64 w = PANEL_SMEM_BUDGET / (8 * rows) - 1;
  if (w > PANEL_W) w = PANEL_W;
  if (w >= 16) w = w / 16 * 16;
  return (int)std::max<i64>(1, w);
}

// Cluster (DSMEM) panel; returns false when the launch is not possible here (the caller falls back).
bool launch_panel_cluster(LuCtx& ctx, VD P, int* trans, bool want_plan) {
  const int m = (int)P.nrows, w = (int)P.ncols, C = ctx.cluster_ctas;
  if (C <= 0 || w > PANEL_W) return false;
  int rows_per_cta = (m + C - 1) / C;
  const size_t smem = (size_t)rows_per_cta * (size_t)(w | 1) * sizeof(double);
  if (smem > (size_t)CL_SMEM_BUDGET) return false;
  static bool configured = false;
  if (!configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(lu_panel_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CL_SMEM_BUDGET));
    if (C > 8) FB_CUDA_CHECK(cudaFuncSetAttribute(lu_panel_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)C);
  cfg.blockDim = dim3(CL_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx.st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)C;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  double* Aptr = P.ptr;
  i64 rs = P.rs, cs = P.cs;
  int* pr = want_plan ? ctx.plan_rows : nullptr;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, lu_panel_cluster_kernel, Aptr, rs, cs, m, w, rows_per_cta, trans, pr,
                                           ctx.plan_src, ctx.plan_cnt);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    fprintf(stderr, "faer_b200: cluster panel launch failed (%s, %d CTAs); using the grid-barrier panel\n",
            cudaGetErrorString(e), C);
    ctx.cluster_ctas = 0;
    return false;
  }
  note_launch();
  return true;
}

// Fused sub-panel (one cluster launch for the whole window): the widest sub-panel it takes, and the rows above which that
// width is halved
constexpr i64 SUBPANEL_MAX_W = 128, SUBPANEL_TALL_ROWS = 16384;

template <int WW, int R>
cudaError_t launch_subpanel_t(LuCtx& ctx, VD P, int* trans, int rows_per_cta, size_t smem, bool want_plan) {
  const int C = ctx.cluster_ctas;
  static bool configured = false;
  if (!configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(lu_subpanel_cluster_kernel<WW, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    FB_CUDA_CHECK(cudaFuncSetAttribute(lu_subpanel_cluster_kernel<WW, R>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)C);
  cfg.blockDim = dim3(SP_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx.st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)C;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  double* Aptr = P.ptr;
  i64 rs = P.rs, cs = P.cs;
  int m = (int)P.nrows, W = (int)P.ncols;
  int* pr = want_plan ? ctx.plan_rows : nullptr;
  long long* prof = nullptr;
  return cudaLaunchKernelEx(&cfg, lu_subpanel_cluster_kernel<WW, R>, Aptr, rs, cs, m, W, rows_per_cta, trans, pr, ctx.plan_src,
                            ctx.plan_cnt, prof);
}

// returns false when the fused sub-panel does not apply here
bool launch_subpanel(LuCtx& ctx, VD P, int* trans, bool want_plan) {
  const int C = ctx.cluster_ctas;
  const i64 m = P.nrows, W = P.ncols;
  // tall panels: the Crout pass streams the CTA's rows of the earlier columns from L2 once per window (8-column windows above
  // 16384 rows), a cost per column proportional to the fused width: halve it there and let the recursion's GEMM (on the large
  // partition) supply the level above
  const i64 wmax = m > SUBPANEL_TALL_ROWS ? SUBPANEL_MAX_W / 2 : SUBPANEL_MAX_W;
  if (C <= 0 || W > wmax || W > m) return false;
  const int rows_per_cta = (int)((m + C - 1) / C);
  // R rows x WW columns per thread in registers (R * WW = 32): the smallest R whose 512 R rows cover the CTA's slice
  auto bytes = [&](int ww) { return ((size_t)W * ww + (size_t)W * SP_CG) * sizeof(double); };
  cudaError_t e;
  if (rows_per_cta <= SP_THREADS) e = launch_subpanel_t<32, 1>(ctx, P, trans, rows_per_cta, bytes(32), want_plan);
  else if (rows_per_cta <= 2 * SP_THREADS) e = launch_subpanel_t<16, 2>(ctx, P, trans, rows_per_cta, bytes(16), want_plan);
  else if (rows_per_cta <= 4 * SP_THREADS) e = launch_subpanel_t<8, 4>(ctx, P, trans, rows_per_cta, bytes(8), want_plan);
  else if (rows_per_cta <= 8 * SP_THREADS) e = launch_subpanel_t<4, 8>(ctx, P, trans, rows_per_cta, bytes(4), want_plan);
  else return false;
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    fprintf(stderr, "faer_b200: fused LU sub-panel launch failed (%s, %d CTAs); using the recursion\n", cudaGetErrorString(e), C);
    return false;
  }
  note_launch();
  return true;
}

void launch_panel(LuCtx& ctx, VD P, int* trans, bool want_plan) {
  if (launch_panel_cluster(ctx, P, trans, want_plan)) return;
  const int m = (int)P.nrows, w = (int)P.ncols;
  int G = (int)std::min<i64>(ctx.num_sms, (m + 63) / 64);
  if (G < 1) G = 1;
  int rows_per_cta = (m + G - 1) / G;
  size_t smem = (size_t)rows_per_cta * (size_t)(w | 1) * sizeof(double);
  FB_ASSERT(smem <= 220 * 1024, "LU panel too tall for the shared-memory slices");
  static size_t configured = 0;
  if (smem > configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(lu_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    configured = 220 * 1024;
  }
  double* Aptr = P.ptr;
  i64 rs = P.rs, cs = P.cs;
  int mm = m, ww = w;
  unsigned long long base = ctx.bar_count;
  int* pr = want_plan ? ctx.plan_rows : nullptr;
  int* ps = ctx.plan_src;
  int* pc = ctx.plan_cnt;
  void* args[] = {&Aptr, &rs, &cs, &mm, &ww, &rows_per_cta, &trans, &ctx.sc, &base, &pr, &ps, &pc};
  FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)lu_panel_kernel, dim3(G), dim3(PANEL_THREADS), args, smem, ctx.st));
  note_launch();
  ctx.bar_count += (unsigned long long)std::min(w, m) * G;
}

void apply_plan(LuCtx& ctx, VD cols, int ngroups) {
  if (cols.ncols == 0 || cols.nrows == 0) return;
  unsigned blocks = (unsigned)((cols.ncols + SWAP_CW - 1) / SWAP_CW);
  laswp_apply_kernel<<<blocks, SWAP_THREADS, 0, ctx.st>>>(cols.ptr, cols.rs, cols.cs, cols.ncols, ctx.plan_rows,
                                                          ctx.plan_src, ctx.plan_cnt, ngroups);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

// A: current view (all m rows, ncols columns); window [start, end); trans: device pointer for this window.
void lu_rec(LuCtx& ctx, VD A, i64 start, i64 end, int* trans) {
  const i64 m = A.nrows, ncols = A.ncols, n = end - start;
  if (n == 0) return;
  const bool has_outside = start > 0 || end < ncols;
  if (n <= panel_width_for(ctx, m) || n == 1) {
    launch_panel(ctx, A.sub(0, start, m, n), trans, has_outside);
    if (has_outside) {
      apply_plan(ctx, A.sub(0, 0, m, start), 1);
      apply_plan(ctx, A.sub(0, end, m, ncols - end), 1);
    }
    return;
  }
  if (launch_subpanel(ctx, A.sub(0, start, m, n), trans, has_outside)) {
    if (has_outside) {
      const int ngroups = (int)((n + SWAP_GROUP - 1) / SWAP_GROUP);  // plans written by the kernel itself
      apply_plan(ctx, A.sub(0, 0, m, start), ngroups);
      apply_plan(ctx, A.sub(0, end, m, ncols - end), ngroups);
    }
    return;
  }
  const i64 half = n / 2;
  const i64 pw = std::min<i64>(16, next_pow2(half));
  const i64 bs = (half + pw - 1) / pw * pw;
  VD W = A.sub(0, start, m, n);
  lu_rec(ctx, W, 0, bs, trans);
  {
    VD A00 = W.sub(0, 0, bs, bs), A01 = W.sub(0, bs, bs, n - bs), A10 = W.sub(bs, 0, m - bs, bs),
       A11 = W.sub(bs, bs, m - bs, n - bs);
    // On a partitioned GPU the panel stream owns few SMs: the larger TRSM / GEMM nodes of the recursion go to the
    // update partition's urgent stream (two event fences) and come back.
    const bool offload = ctx.st_big != nullptr && n >= 128 && (double)(m - bs) * (double)(n - bs) * (double)bs >= 2e8;
    cudaStream_t sg = offload ? ctx.st_big : ctx.st;
    if (offload) {
      FB_CUDA_CHECK(cudaEventRecord(ctx.ev_to_big, ctx.st));
      FB_CUDA_CHECK(cudaStreamWaitEvent(sg, ctx.ev_to_big, 0));
    }
    solve_lower_triangular_in_place_f64(sg, cv(A00), true, A01);
    gemm_f64(sg, A11, 1, cv(A10), cv(A01), -1.0);
    if (offload) {
      FB_CUDA_CHECK(cudaEventRecord(ctx.ev_from_big, sg));
      FB_CUDA_CHECK(cudaStreamWaitEvent(ctx.st, ctx.ev_from_big, 0));
    }
    lu_rec(ctx, W.sub(bs, 0, m - bs, n), bs, n, trans + bs);
  }
  if (has_outside) {
    const int ngroups = (int)((n + SWAP_GROUP - 1) / SWAP_GROUP);
    laswp_plan_kernel<<<ngroups, 32, 0, ctx.st>>>(trans, (int)n, ctx.plan_rows, ctx.plan_src, ctx.plan_cnt, ngroups);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    apply_plan(ctx, A.sub(0, 0, m, start), ngroups);
    apply_plan(ctx, A.sub(0, end, m, ncols - end), ngroups);
  }
}

}  // namespace

size_t lu_partial_piv_in_place_f64(cudaStream_t stream, VD A, long long* perm_fwd, long long* perm_inv) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n);
  FB_ASSERT(m < (1ll << 31) && n < (1ll << 31), "dimension too large");
  for (i64 i = 0; i < m; ++i) perm_fwd[i] = i;
  size_t n_trans = 0;
  // Large square column-major problems: right-looking block-column driver with two-stream look-ahead (dist.cu on a
  // single rank; same panel kernel => same pivots).
  const bool use_lookahead = m == n && A.rs == 1 && n >= lookahead_min_n();
  if (use_lookahead) {
    // block width: 512 up to n = 20000, 1024 beyond (FAER_B200_NB overrides)
    const i64 nbl = lookahead_block() ? lookahead_block() : (n <= 20000 ? 512 : 1024);
    n_trans = dist_lu_f64(A.ptr, A.cs, n, nbl, perm_fwd, perm_inv, /*lookahead | local*/ 3);
  } else if (size > 0) {
    LuCtx ctx;
    ctx.st = stream;
    int dev = 0;
    FB_CUDA_CHECK(cudaGetDevice(&dev));
    FB_CUDA_CHECK(cudaDeviceGetAttribute(&ctx.num_sms, cudaDevAttrMultiProcessorCount, dev));
    const int G = ctx.num_sms;
    const i64 ngroups_max = (size + SWAP_GROUP - 1) / SWAP_GROUP + 1;
    ctx.d_trans = (int*)ws_alloc((size_t)size * sizeof(int));
    ctx.plan_rows = (int*)ws_alloc((size_t)ngroups_max * 2 * SWAP_GROUP * sizeof(int));
    ctx.plan_src = (int*)ws_alloc((size_t)ngroups_max * 2 * SWAP_GROUP * sizeof(int));
    ctx.plan_cnt = (int*)ws_alloc((size_t)ngroups_max * sizeof(int));
    const size_t sc_bytes = (size_t)2 * G * 8 * 2 + (size_t)2 * G * PANEL_W * 8 + (size_t)2 * PANEL_W * 8 + 64;
    char* scb = (char*)ws_alloc(sc_bytes);
    ctx.sc.cand_val = (double*)scb;
    ctx.sc.cand_idx = (long long*)(scb + (size_t)2 * G * 8);
    ctx.sc.cand_row = (double*)(scb + (size_t)4 * G * 8);
    ctx.sc.diag_row = (double*)(scb + (size_t)4 * G * 8 + (size_t)2 * G * PANEL_W * 8);
    ctx.sc.bar = (unsigned long long*)(scb + (size_t)4 * G * 8 + (size_t)2 * G * PANEL_W * 8 + (size_t)2 * PANEL_W * 8);
    FB_CUDA_CHECK(cudaMemsetAsync(ctx.sc.bar, 0, 8, stream));
    ctx.bar_count = 0;

    lu_rec(ctx, A, 0, size, ctx.d_trans);

    std::vector<int> h_trans((size_t)size);
    FB_CUDA_CHECK(cudaMemcpyAsync(h_trans.data(), ctx.d_trans, (size_t)size * sizeof(int), cudaMemcpyDeviceToHost, stream));
    FB_CUDA_CHECK(cudaStreamSynchronize(stream));
    // perm.swap(idx, idx + t)  (reference factor.rs:274-277)
    for (i64 i = 0; i < size; ++i) {
      const int t = h_trans[(size_t)i];
      if (t != 0) {
        std::swap(perm_fwd[i], perm_fwd[i + t]);
        ++n_trans;
      }
    }
    if (m < n) {
      // reference factor.rs:278-285
      solve_lower_triangular_in_place_f64(stream, cv(A.sub(0, 0, m, size)), true, A.sub(0, size, m, n - size));
      FB_CUDA_CHECK(cudaStreamSynchronize(stream));
    }
    ws_free(scb);
    ws_free(ctx.plan_cnt);
    ws_free(ctx.plan_src);
    ws_free(ctx.plan_rows);
    ws_free(ctx.d_trans);
  }
  for (i64 i = 0; i < m; ++i) perm_inv[perm_fwd[i]] = i;
  return n_trans;
}

// ---- workspace-based entry points used by the multi-GPU driver (dist.cu) --------------------------------------
struct LuWorkspace {
  LuCtx ctx;
  char* scb;
  i64 max_window;
};

LuWorkspace* lu_ws_create(cudaStream_t stream, i64 max_window, int sm_limit) {
  LuWorkspace* w = new LuWorkspace();
  LuCtx& ctx = w->ctx;
  ctx.st = stream;
  int dev = 0;
  FB_CUDA_CHECK(cudaGetDevice(&dev));
  FB_CUDA_CHECK(cudaDeviceGetAttribute(&ctx.num_sms, cudaDevAttrMultiProcessorCount, dev));
  // a stream bound to an SM partition (green context): the cooperative panel grid must fit the partition
  if (sm_limit > 0 && sm_limit < ctx.num_sms) ctx.num_sms = sm_limit;
  const int G = ctx.num_sms;
  w->max_window = max_window;
  const i64 ngroups_max = (max_window + SWAP_GROUP - 1) / SWAP_GROUP + 1;
  ctx.d_trans = nullptr;
  ctx.plan_rows = (int*)ws_alloc((size_t)ngroups_max * 2 * SWAP_GROUP * sizeof(int));
  ctx.plan_src = (int*)ws_alloc((size_t)ngroups_max * 2 * SWAP_GROUP * sizeof(int));
  ctx.plan_cnt = (int*)ws_alloc((size_t)ngroups_max * sizeof(int));
  const size_t sc_bytes = (size_t)2 * G * 8 * 2 + (size_t)2 * G * PANEL_W * 8 + (size_t)2 * PANEL_W * 8 + 64;
  w->scb = (char*)ws_alloc(sc_bytes);
  char* scb = w->scb;
  ctx.sc.cand_val = (double*)scb;
  ctx.sc.cand_idx = (long long*)(scb + (size_t)2 * G * 8);
  ctx.sc.cand_row = (double*)(scb + (size_t)4 * G * 8);
  ctx.sc.diag_row = (double*)(scb + (size_t)4 * G * 8 + (size_t)2 * G * PANEL_W * 8);
  ctx.sc.bar = (unsigned long long*)(scb + (size_t)4 * G * 8 + (size_t)2 * G * PANEL_W * 8 + (size_t)2 * PANEL_W * 8);
  FB_CUDA_CHECK(cudaMemsetAsync(ctx.sc.bar, 0, 8, stream));
  ctx.bar_count = 0;
  return w;
}

void lu_ws_set_cluster(LuWorkspace* w, int ctas) { w->ctx.cluster_ctas = ctas > CL_MAXC ? CL_MAXC : ctas; }

void lu_ws_set_big_stream(LuWorkspace* w, cudaStream_t big) {
  w->ctx.st_big = big;
  if (big && !w->ctx.ev_to_big) {
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&w->ctx.ev_to_big, cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&w->ctx.ev_from_big, cudaEventDisableTiming));
  }
}

void lu_ws_destroy(LuWorkspace* w) {
  if (!w) return;
  if (w->ctx.ev_to_big) cudaEventDestroy(w->ctx.ev_to_big);
  if (w->ctx.ev_from_big) cudaEventDestroy(w->ctx.ev_from_big);
  ws_free(w->scb);
  ws_free(w->ctx.plan_cnt);
  ws_free(w->ctx.plan_src);
  ws_free(w->ctx.plan_rows);
  delete w;
}

// Factor the window [start, end) of the view A (all rows) on the workspace's stream; relative transpositions go to
// d_trans (device, length end-start); the view's columns outside the window receive the row swaps.
void lu_factor_window_f64(LuWorkspace* w, VD A, i64 start, i64 end, int* d_trans) {
  FB_ASSERT(end - start <= w->max_window, "LU window larger than the workspace was sized for");
  lu_rec(w->ctx, A, start, end, d_trans);
}

// Apply n transpositions (device array, relative to row 0 of `cols`) to every column of `cols`.
void lu_apply_transpositions_f64(LuWorkspace* w, VD cols, const int* d_trans, i64 n) {
  if (cols.ncols == 0 || n == 0) return;
  FB_ASSERT(n <= w->max_window, "too many transpositions for this workspace");
  LuCtx& ctx = w->ctx;
  const int ngroups = (int)((n + SWAP_GROUP - 1) / SWAP_GROUP);
  laswp_plan_kernel<<<ngroups, 32, 0, ctx.st>>>(d_trans, (int)n, ctx.plan_rows, ctx.plan_src, ctx.plan_cnt, ngroups);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  apply_plan(ctx, cols, ngroups);
}

}  // namespace fb
