// f64 GEMM, TMA-fed and warp-specialised (the north-star mainloop for the f64 hot path).
//
// Replaces `private_gemm_x86::gemm(DstKind::{Full, Lower, Upper})` (reference faer/src/linalg/matmul/mod.rs:1373-1411,
// matmul/triangular.rs:641-680) for rectangular operands: `dst(struct) = [dst +] alpha * lhs * rhs`, i.e. the trailing
// updates of LLT (SYRK), LU and QR and `matmul` itself. Structured INPUTS, odd strides and tiny / tall-skinny problems
// stay on the cp.async kernel (gemm_f64.cu).
//
// wgmma has no f64 type; the f64 tensor ops of sm_90a are the warp-level mma.sync shapes m8n8k4, m16n8k4, m16n8k8 and
// m16n8k16 (SASS DMMA). Only the 16-row shapes reach the full f64 tensor rate (profiles/r03_f64_peaks.log); this kernel
// issues m16n8k8 (the 16-deep shape's fragments do not fit beside 128 accumulator registers). So "tensor-core tiles fed by
// TMA" means here:
//   * CTAs of bounded persistence (each owns `tiles_per_cta` consecutive tiles, sized so that a CTA lives ~100 us: long
//     enough to amortise its start-up and to overlap every epilogue with the next tile's loads, short enough that the SMs
//     turn over and a higher-priority stream — the panel chain of the look-ahead factorizations — gets in), 2 per SM,
//     each with a producer warpgroup (one working warp) and a consumer warpgroup of 4 warps;
//     CTA tile 128 x 64, warp tile 32 x 64 (64 accumulator doubles = 128 registers per thread), 16-deep k-steps. The
//     register file is re-divided at run time with setmaxnreg (producer warpgroup 24, consumers 232 registers per thread);
//   * producer: one elected lane issues cp.async.bulk.tensor (TMA, SASS UTMALDG) loads of both operand slabs into a
//     4-stage ring of 128B-swizzled shared-memory tiles and signals `full[s]` through the mbarrier's transaction count;
//     out-of-range rows / columns / k are zero-filled by the TMA unit (no predication in the loop);
//   * consumers: wait `full[s]`, read DMMA fragments with conflict-free 8-byte loads (see "k permutation"), issue 32
//     DMMA.16x8x8 per stage, then one lane per warp arrives on `empty[s]`. There is no CTA-wide barrier in the main loop; the
//     producer runs up to 4 stages ahead, ACROSS tile boundaries, so the next tile's operands land while the epilogue
//     of the current one runs, and the second CTA of the SM keeps the DMMA pipe busy during that epilogue;
//   * epilogue: registers -> global directly (alpha, optional accumulate with the 16 old values of a row block loaded
//     first, structure / bounds masks); every 8 lanes write 64 contiguous bytes.
//
// Shared-memory layouts (both produced by TMA with CU_TENSOR_MAP_SWIZZLE_128B, rows of 128 B):
//   MN-major operand (unit stride along m or n; e.g. column-major lhs): boxes of 16 (mn) x 16 (k): [blk][k][16 mn]
//   K-major  operand (unit stride along k; e.g. column-major rhs):      one box 16 (k) x rows:     [mn][16 k]
// k permutation: lane t = lane & 3 supplies, in fragment k slot q (k = t + 4q of the PTX layout), stage index K4(q, t)
// for both operands. Any bijection of the 16 k-indices of a stage is valid (a sum is a sum); {0,3,12,15} ^ {0,1,4,5} makes
// the 16 eight-byte fragment loads of a half-warp hit 16 distinct banks in BOTH layouts under the 128B swizzle.
#pragma once
#include <cuda.h>

#include <algorithm>

#include "gemm_f64.cuh"
#include "runtime.cuh"

namespace fb {
namespace ws64 {

constexpr int BM = 128, BN = 64, BK = 16, STAGES = 4;
constexpr int CONSUMERS = 4;                       // consumer warps (warpgroup 1), stacked along m: warp tile 32 x 64
constexpr int THREADS = 256;                       // warpgroup 0: producer (warp 0 works), warpgroup 1: consumers
constexpr int WMI = 4, WNI = 8;                    // 8 x 8 DMMA blocks per warp tile
constexpr int A_BYTES = BM * BK * 8, B_BYTES = BN * BK * 8, STAGE_BYTES = A_BYTES + B_BYTES;  // 16 KB + 8 KB
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*alignment*/ + 128 /*barriers*/;

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
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
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ double lds64(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}

struct Params {
  double* C;
  i64 c_rs, c_cs;
  int m, n, k;
  int c_struct, accum;
  double alpha;
  int tiles_m, tiles_n;
  int tiles_per_cta;
  // Stagger of the two CTAs that share an SM: both start together and their tiles take the same time, so without it they
  // reach their epilogues together and the DMMA pipe idles (ncu, k = 256: tensor pipe 78.7 % active). The second-slot CTAs of
  // the first wave (blockIdx in [sm_slots, 2 sm_slots)) start their first tile half a tile late; their successors inherit
  // the phase because a CTA is replaced when its predecessor on the same SM exits.
  int sm_slots;          // SMs the launch can use (stream's partition)
  long long stagger_cycles;  // 0 = off
  // "spicy" variant (matmul/internal/mod.rs:45-379): dst[row_idx[i], col_idx[j]] (+)= alpha (A diag(d) B)[i, j]
  const long long* row_idx;  // device, m entries, or null
  const long long* col_idx;  // device, n entries, or null
  const double* diag;        // device, k entries `diag_stride` apart, or null
  i64 diag_stride;
};

// ---- static tile schedule: tile `idx` of the launch -> (tm, tn); identical in every warp of every CTA ---------------
// RECT: grouped rasterisation (GROUP_M tile-rows share their lhs slabs through L2). Triangular dst: only the tiles that
// intersect the kept triangle are enumerated (row-major over tile-rows), so the round-robin stays balanced.
struct TileWalk {
  int tiles_m, tiles_n, c_struct;
  int row, row_first;  // triangular: current tile-row and the linear index of its first tile
  __device__ __forceinline__ int row_lo(int tm) const { return is_upper(c_struct) ? (tm * BM) / BN : 0; }
  __device__ __forceinline__ int row_hi(int tm) const {  // exclusive
    return is_lower(c_struct) ? min(tiles_n, (tm * BM + BM - 1) / BN + 1) : tiles_n;
  }
  __device__ __forceinline__ void init(int tm_, int tn_, int cs_) {
    tiles_m = tm_; tiles_n = tn_; c_struct = cs_;
    row = 0; row_first = 0;
  }
  // returns false when idx is past the last tile
  __device__ __forceinline__ bool locate(int idx, int& tm, int& tn) {
    if (c_struct == RECT) {
      constexpr int GROUP = 8;
      if (idx >= tiles_m * tiles_n) return false;
      const int width = GROUP * tiles_n;
      const int first_m = (idx / width) * GROUP;
      const int gsize = min(tiles_m - first_m, GROUP);
      tm = first_m + (idx % width) % gsize;
      tn = (idx % width) / gsize;
      return true;
    }
    while (row < tiles_m) {
      const int cnt = max(0, row_hi(row) - row_lo(row));
      if (idx < row_first + cnt) {
        tm = row;
        tn = row_lo(row) + (idx - row_first);
        return true;
      }
      row_first += cnt;
      ++row;
    }
    return false;
  }
};

// byte offset (inside one operand tile) of the 8-byte element (mn, kk), before adding i * 8 rows
// MN-major: [blk = mn / 16][kk][16 mn], 128B swizzle: 16-byte chunk ^= kk & 7
__device__ __forceinline__ uint32_t off_mn_major(int mn, int kk) {
  const int blk = mn >> 4, w = mn & 15;
  return (uint32_t)(blk * 2048 + kk * 128 + ((((w >> 1) ^ (kk & 7)) << 4) | ((w & 1) << 3)));
}
// K-major: [mn][16 kk], 128B swizzle: chunk ^= mn & 7
__device__ __forceinline__ uint32_t off_k_major(int mn, int kk) {
  return (uint32_t)(mn * 128 + ((((kk >> 1) ^ (mn & 7)) << 4) | ((kk & 1) << 3)));
}

// VAR (bring-up variants, selected by FAER_B200_WS_VAR): 0 = production; 1 = no setmaxnreg, one CTA per SM; 5 = the kernel as
// first written (no proxy fence before a stage is released, old dst values through L1), kept to reproduce the failure below.
//
// Stage release. The consumers read a stage with ld.shared (generic proxy) and the producer's next TMA load overwrites it
// through the async proxy: a write-after-read ACROSS proxies, which the mbarrier hand-over alone does not order. Without
// `fence.proxy.async` before the arrive on `empty[s]`, a warp can read B fragments the next load has already replaced. The old values of dst are read with ld.global.cg:
// they are used once, and keeping them out of L1 leaves it to nothing at all (the operands arrive by TMA).
template <bool A_KMAJOR, bool B_KMAJOR, bool SPICY, int VAR = 0>
__global__ void __launch_bounds__(THREADS, VAR == 1 ? 1 : 2)   // 128 registers per thread at launch, re-divided below
gemm_f64_ws_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const Params p) {
  extern __shared__ uint8_t ws_smem_raw[];
  const uint32_t smem_base = (smem_u32(ws_smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = ws_smem_raw + (smem_base - smem_u32(ws_smem_raw));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_gen + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMERS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int nkt = (p.k + BK - 1) / BK;
  TileWalk walk;
  walk.init(p.tiles_m, p.tiles_n, p.c_struct);

  if (warp < 4) {
    // ================= producer warpgroup =================
    if constexpr (VAR != 1) asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;  // global k-step counter: stage = it % STAGES, phase = (it / STAGES) & 1
      for (int i = 0; i < p.tiles_per_cta; ++i) {
        int tm, tn;
        if (!walk.locate((int)blockIdx.x * p.tiles_per_cta + i, tm, tn)) break;
        const int m0 = tm * BM, n0 = tn * BN;
        for (int kt = 0; kt < nkt; ++kt, ++it) {
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
          mbar_wait(&empty[s], ph ^ 1u);
          const uint32_t sa = smem_base + s * STAGE_BYTES, sb = sa + A_BYTES;
          mbar_expect_tx(&full[s], STAGE_BYTES);
          const int k0 = kt * BK;
          if constexpr (A_KMAJOR) {
            tma_load_2d(sa, &mapA, &full[s], k0, m0);
          } else {
#pragma unroll
            for (int b = 0; b < BM / 16; ++b) tma_load_2d(sa + b * 2048, &mapA, &full[s], m0 + b * 16, k0);
          }
          if constexpr (B_KMAJOR) {
            tma_load_2d(sb, &mapB, &full[s], k0, n0);
          } else {
#pragma unroll
            for (int b = 0; b < BN / 16; ++b) tma_load_2d(sb + b * 2048, &mapB, &full[s], n0 + b * 16, k0);
          }
        }
      }
    }
    return;
  }

  // ================= consumer warpgroup =================
  if constexpr (VAR != 1) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = lane >> 2, t = lane & 3;
  const int wm0 = (warp - 4) * (WMI * 8);  // warp tile rows [wm0, wm0 + 32) x all 64 columns
  // per-lane fragment offsets for the 4 k slots of a stage: k index K4(q, t) = {0,3,12,15}[t] ^ {0,1,4,5}[q]
  uint32_t offA[4][2], offB[4][2];  // [k slot][parity of the 8-row block] (MN-major) / [k slot][0] (K-major)
  {
    const int base_k = (t == 0) ? 0 : (t == 1) ? 3 : (t == 2) ? 12 : 15;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int kk = base_k ^ ((s & 1) | ((s & 2) << 1));
      if constexpr (A_KMAJOR) {
        offA[s][0] = off_k_major(wm0 + g, kk);
        offA[s][1] = 0;
      } else {
        offA[s][0] = off_mn_major(wm0 + g, kk);
        offA[s][1] = off_mn_major(wm0 + 8 + g, kk);
      }
      if constexpr (B_KMAJOR) {
        offB[s][0] = off_k_major(g, kk);
        offB[s][1] = 0;
      } else {
        offB[s][0] = off_mn_major(g, kk);
        offB[s][1] = off_mn_major(8 + g, kk);
      }
    }
  }

  const int cs_ = p.c_struct;
  const bool c_low = is_lower(cs_), c_up = is_upper(cs_);
  const bool c_nodiag = is_strict(cs_) || is_unit(cs_);
  const double alpha = p.alpha;
  const bool add = p.accum != 0;

  if (p.stagger_cycles > 0 && (int)blockIdx.x >= p.sm_slots && (int)blockIdx.x < 2 * p.sm_slots) {
    const long long t0 = clock64();
    while (clock64() - t0 < p.stagger_cycles) __nanosleep(256);
  }

  uint32_t it = 0;
  for (int ti = 0; ti < p.tiles_per_cta; ++ti) {
    int tm, tn;
    if (!walk.locate((int)blockIdx.x * p.tiles_per_cta + ti, tm, tn)) break;
    const int m0 = tm * BM, n0 = tn * BN;

    double acc[WMI][WNI][2];
#pragma unroll
    for (int i = 0; i < WMI; ++i)
#pragma unroll
      for (int j = 0; j < WNI; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    for (int kt = 0; kt < nkt; ++kt, ++it) {
      const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
      double dk[4] = {1.0, 1.0, 1.0, 1.0};
      if constexpr (SPICY) {
        if (p.diag) {  // this lane's four k indices of the stage: K4(ss, t)
          const int base_k = (t == 0) ? 0 : (t == 1) ? 3 : (t == 2) ? 12 : 15;
#pragma unroll
          for (int ss = 0; ss < 4; ++ss) {
            const int kg = kt * BK + (base_k ^ ((ss & 1) | ((ss & 2) << 1)));
            dk[ss] = kg < p.k ? p.diag[(i64)kg * p.diag_stride] : 0.0;
          }
        }
      }
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_base + s * STAGE_BYTES, sb = sa + A_BYTES;
      // two DMMA.16x8x8 per 16 x 8 block and stage (the 16-deep shape's fragments do not fit beside the 128 accumulator
      // registers): half h contracts fragment k slots q = 2h + (v >> 1) (A) / 2h + i (B), i.e. stage indices K4(q, t).
      // A fragments of the whole warp tile, B fragments one 8-column block at a time.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        double a[WMI / 2][4];
#pragma unroll
        for (int ip = 0; ip < WMI / 2; ++ip)
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            const int i = 2 * ip + (v & 1), q = 2 * h + (v >> 1);
            if constexpr (A_KMAJOR) a[ip][v] = lds64(sa + offA[q][0] + i * 8 * 128);
            else a[ip][v] = lds64(sa + offA[q][i & 1] + (i >> 1) * 2048);
            if constexpr (SPICY) a[ip][v] *= dk[q];
          }
#pragma unroll
        for (int j = 0; j < WNI; ++j) {
          double b[2];
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            const int q = 2 * h + v;
            if constexpr (B_KMAJOR) b[v] = lds64(sb + offB[q][0] + j * 8 * 128);
            else b[v] = lds64(sb + offB[q][j & 1] + (j >> 1) * 2048);
          }
#pragma unroll
          for (int ip = 0; ip < WMI / 2; ++ip)
            dmma1688(acc[2 * ip][j][0], acc[2 * ip][j][1], acc[2 * ip + 1][j][0], acc[2 * ip + 1][j][1], a[ip], b);
        }
      }
      if constexpr (VAR != 5) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }

    // ---- epilogue: dst = [dst +] alpha * acc, masked by dst structure and bounds. Add mode: the old values of row block
    // i + 1 are requested before row block i is combined and stored (two register sets), so the four row blocks cost about
    // two global-memory round trips instead of four ----
    auto coloff = [&](int col) -> i64 {
      if constexpr (SPICY) {
        if (p.col_idx) return col < p.n ? (i64)p.col_idx[col] * p.c_cs : 0;
      }
      return (i64)col * p.c_cs;
    };
    auto rowoff = [&](int row) -> i64 {
      if constexpr (SPICY) {
        if (p.row_idx) return row < p.m ? (i64)p.row_idx[row] * p.c_rs : 0;
      }
      return (i64)row * p.c_rs;
    };
    auto kept = [&](int row, int col) -> bool {
      bool v = row < p.m && col < p.n;
      if (c_low && (row < col || (row == col && c_nodiag))) v = false;
      if (c_up && (row > col || (row == col && c_nodiag))) v = false;
      return v;
    };
    double cv[2][WNI][2];
    auto load_old = [&](int i, double (&dst)[WNI][2]) {
      const int row = m0 + wm0 + i * 8 + g;
      const i64 roff = rowoff(row);
#pragma unroll
      for (int j = 0; j < WNI; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + j * 8 + 2 * t + e;
          if constexpr (VAR != 5) dst[j][e] = kept(row, col) ? __ldcg(p.C + roff + coloff(col)) : 0.0;
          else dst[j][e] = kept(row, col) ? p.C[roff + coloff(col)] : 0.0;
        }
    };
    if (add) load_old(0, cv[0]);
#pragma unroll
    for (int i = 0; i < WMI; ++i) {
      if (add && i + 1 < WMI) load_old(i + 1, cv[(i + 1) & 1]);
      const int row = m0 + wm0 + i * 8 + g;
      const i64 roff = rowoff(row);
#pragma unroll
      for (int j = 0; j < WNI; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + j * 8 + 2 * t + e;
          if (kept(row, col)) p.C[roff + coloff(col)] = add ? (alpha * acc[i][j][e] + cv[i & 1][j][e]) : alpha * acc[i][j][e];
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && f) fn = (EncodeTiledFn)f;
  }
  return fn;
}

// 2-D f64 tensor map: `inner` contiguous elements per line, `outer` lines `ld` elements apart; box 16 x box_outer
inline bool make_map(CUtensorMap* map, const double* base, i64 inner, i64 outer, i64 ld, int box_outer) {
  const cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 8};
  const cuuint32_t box[2] = {16u, (cuuint32_t)box_outer};
  const cuuint32_t estr[2] = {1, 1};
  return encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// operand (rows = m or n, contraction = k) with element strides s_mn / s_k: can TMA read it, and in which layout?
inline bool tma_layout(const double* ptr, i64 rows, i64 k, i64 s_mn, i64 s_k, bool* kmajor) {
  if ((((uintptr_t)ptr) & 15) != 0) return false;
  if (s_mn == 1 && s_k >= rows && (s_k % 2 == 0 || k == 1)) {
    *kmajor = false;
    return true;
  }
  if (s_k == 1 && s_mn >= k && (s_mn % 2 == 0 || rows == 1)) {
    *kmajor = true;
    return true;
  }
  return false;
}

// Launches the kernel if the problem qualifies; returns false otherwise (caller falls back to the cp.async kernel).
struct Spicy {
  const long long* row_idx = nullptr;
  const long long* col_idx = nullptr;
  const double* diag = nullptr;
  i64 diag_stride = 1;
};
inline bool try_gemm_f64_ws(cudaStream_t stream, const GemmF64Params& q, const Spicy* sp = nullptr) {
  if (q.a_struct != RECT || q.b_struct != RECT || q.k_split_len > 0) return false;
  if (!encode_fn()) return false;
  bool ak = false, bk = false;
  if (!tma_layout(q.A, q.m, q.k, q.a_rs, q.a_cs, &ak)) return false;
  if (!tma_layout(q.B, q.n, q.k, q.b_cs, q.b_rs, &bk)) return false;
  if (q.a_rs == 1 && q.a_cs == 1) return false;  // degenerate vectors: leave to the general kernel
  if (q.b_rs == 1 && q.b_cs == 1) return false;
  Params p;
  p.C = q.C; p.c_rs = q.c_rs; p.c_cs = q.c_cs;
  p.m = q.m; p.n = q.n; p.k = q.k;
  p.c_struct = q.c_struct; p.accum = q.accum; p.alpha = q.alpha;
  p.row_idx = sp ? sp->row_idx : nullptr;
  p.col_idx = sp ? sp->col_idx : nullptr;
  p.diag = sp ? sp->diag : nullptr;
  p.diag_stride = sp ? sp->diag_stride : 1;
  p.tiles_m = (q.m + BM - 1) / BM;
  p.tiles_n = (q.n + BN - 1) / BN;
  long long tiles = (long long)p.tiles_m * p.tiles_n;
  if (q.c_struct != RECT) {  // exactly the tiles TileWalk enumerates
    tiles = 0;
    for (int tm = 0; tm < p.tiles_m; ++tm) {
      const int lo = is_upper(q.c_struct) ? (tm * BM) / BN : 0;
      const int hi = is_lower(q.c_struct) ? std::min(p.tiles_n, (tm * BM + BM - 1) / BN + 1) : p.tiles_n;
      tiles += std::max(0, hi - lo);
    }
  }
  if (tiles == 0) return true;
  CUtensorMap mapA, mapB;
  const bool okA = ak ? make_map(&mapA, q.A, q.k, q.m, q.a_rs, BM) : make_map(&mapA, q.A, q.m, q.k, q.a_cs, 16);
  const bool okB = bk ? make_map(&mapB, q.B, q.k, q.n, q.b_cs, BN) : make_map(&mapB, q.B, q.n, q.k, q.b_rs, 16);
  if (!okA || !okB) return false;
  // tiles per CTA shrink with k so that a CTA stays short-lived (on the order of 50 us at 128 f64 FMA / clock / SM), and
  // never below two CTAs per SM while the tiles allow it (fewer would leave SMs idle in small launches)
  p.sm_slots = stream_sms(stream);
  const long long tpc_fill = std::max<long long>(1, (tiles + 2ll * p.sm_slots - 1) / (2ll * p.sm_slots));
  p.tiles_per_cta = (int)std::max<long long>(1, std::min<long long>({8, 768 / std::max(q.k, 1), tpc_fill}));
  const int grid = (int)((tiles + p.tiles_per_cta - 1) / p.tiles_per_cta);
  {
    static int stagger = -1;
    if (stagger < 0) {
      const char* e = getenv("FAER_B200_WS_STAGGER");  // 0 switches the stagger off (dev knob)
      stagger = e ? atoi(e) : 1;
    }
    // half a tile at the full rate of one SM: (k / 16) k-steps x 128 x 64 x 16 FMA / (128 FMA / clock) / 2
    p.stagger_cycles = (stagger && grid >= 2 * p.sm_slots) ? (long long)((q.k + BK - 1) / BK) * 512 : 0;
  }
  // one opt-in to > 48 KB of dynamic shared memory per kernel variant
  static bool configured[16] = {};
  static int var = -1, extra_smem = 0;
  if (var < 0) {
    const char* e = getenv("FAER_B200_WS_VAR");  // bring-up knob
    var = e ? atoi(e) : 0;
    const char* x = getenv("FAER_B200_WS_EXTRA_SMEM");  // bring-up knob: > 14 KB forces one CTA per SM
    extra_smem = x ? atoi(x) : 0;
  }
  const int smem_bytes = SMEM_BYTES + extra_smem;
  auto launch = [&](int which, void (*kern)(CUtensorMap, CUtensorMap, Params)) {
    if (!configured[which]) {
      FB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
      configured[which] = true;
    }
    kern<<<grid, THREADS, smem_bytes, stream>>>(mapA, mapB, p);
  };
  if (!sp && var != 0 && !ak) {
    if (var == 1) { if (bk) launch(8, gemm_f64_ws_kernel<false, true, false, 1>); else launch(9, gemm_f64_ws_kernel<false, false, false, 1>); }
    else { if (bk) launch(10, gemm_f64_ws_kernel<false, true, false, 5>); else launch(11, gemm_f64_ws_kernel<false, false, false, 5>); }
  } else if (!sp) {
    if (ak && bk) launch(0, gemm_f64_ws_kernel<true, true, false>);
    else if (ak && !bk) launch(1, gemm_f64_ws_kernel<true, false, false>);
    else if (!ak && bk) launch(2, gemm_f64_ws_kernel<false, true, false>);
    else launch(3, gemm_f64_ws_kernel<false, false, false>);
  } else {
    if (ak && bk) launch(4, gemm_f64_ws_kernel<true, true, true>);
    else if (ak && !bk) launch(5, gemm_f64_ws_kernel<true, false, true>);
    else if (!ak && bk) launch(6, gemm_f64_ws_kernel<false, true, true>);
    else launch(7, gemm_f64_ws_kernel<false, false, true>);
  }
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return true;
}

}  // namespace ws64
}  // namespace fb
