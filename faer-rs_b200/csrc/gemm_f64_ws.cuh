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

constexpr int BM = 128, BK = 16;
constexpr int WMI = 4, WNI = 8;                    // 8 x 8 DMMA blocks per warp tile (32 x 64)
constexpr int A_BYTES = BM * BK * 8;               // 16 KB

// Two configurations of the same kernel.
//   narrow (WIDE = false): CTA tile 128 x 64, 4 consumer warps stacked along m, 4 stages of 24 KB, two CTAs per SM, the
//     register epilogue for every tile.
//   wide (WIDE = true): CTA tile 128 x 128, 8 consumer warps (4 along m x 2 along n, two consumer warpgroups), 3 stages of
//     32 KB and a 128 KB destination buffer, one CTA per SM. Per DMMA it reads half the operand bytes of the 64 x 64
//     cp.async tile (16 instead of 32 B per clock and SM at the full DMMA rate). Tiles that lie wholly inside the kept
//     part of dst are combined in shared memory: the producer TMA-loads the old dst tile while the tile's main loop runs
//     (Add mode), the consumers write alpha * acc [+ old] into the buffer, signal `dst_ready` and go straight into the
//     next tile's main loop; a storer warp of the producer warpgroup TMA-stores the buffer and frees it once the store
//     has read it. With one CTA per SM nothing else covers a consumer stall, so no consumer waits for a store or for the
//     other consumers at a tile's end. (The tensor form of cp.reduce.async.bulk has no f64 add, so Add mode keeps the
//     TMA load of the old tile.) Tiles that straddle the diagonal of a triangular dst keep the masked
//     register epilogue (the untouched triangle must not be written, not even with its own values).
template <bool WIDE>
struct Shape {
  static constexpr int BN = WIDE ? 128 : 64;
  static constexpr int CONSUMERS = WIDE ? 8 : 4;            // consumer warps: 4 along m x BN / 64 along n
  static constexpr int THREADS = 128 + 32 * CONSUMERS;      // warpgroup 0: producer (warp 0 works), then the consumers
  static constexpr int STAGES = WIDE ? 3 : 4;
  static constexpr int B_BYTES = BN * BK * 8, STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int DST_BYTES = WIDE ? BM * BN * 8 : 0;  // 8 boxes of 16 rows x 128 columns, 128B-swizzled
  static constexpr int SMEM_BYTES = DST_BYTES + STAGES * STAGE_BYTES + 1024 /*alignment*/ + 128 /*barriers*/;
  // registers per thread after setmaxnreg; the launch gives every thread 65536 / THREADS (rounded down to a multiple of
  // 8): 128 x 24 + 128 x 232 = 256 x 128, and 128 x 40 + 256 x 232 = 384 x 168. ptxas allocates the consumer code at
  // 232 (the 128 / 168 it reports is the launch value). Dropping the idle producer warps would not give the consumers
  // more: each of the 4 SM sub-partitions has its own 16 K registers, and 10 warps per SM put 3 on some of them, which
  // caps every thread at 168.
  static constexpr int PRODUCER_REGS = WIDE ? 40 : 24, CONSUMER_REGS = 232;
};
static_assert(Shape<true>::SMEM_BYTES <= 227 * 1024, "wide configuration exceeds the shared memory of one SM");
static_assert(128 * Shape<true>::PRODUCER_REGS + 256 * Shape<true>::CONSUMER_REGS <= 384 * 168, "register file");

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
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ double lds64(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, double v) {
  asm volatile("st.shared.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}

struct Params {
  double* C;
  i64 c_rs, c_cs;
  int m, n, k;
  int c_struct, accum;
  int dst_tma;  // wide configuration: the dst tensor map is valid, tiles inside the kept part go through shared memory
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
template <int BN>
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

// Stage release. The consumers read a stage with ld.shared (generic proxy) and the producer's next TMA load overwrites it
// through the async proxy: a write-after-read ACROSS proxies, which the mbarrier hand-over alone does not order. Without
// `fence.proxy.async` before the arrive on `empty[s]`, a warp can read B fragments the next load has already replaced. The old values of dst are read with ld.global.cg:
// they are used once, and keeping them out of L1 leaves it to nothing at all (the operands arrive by TMA).
template <bool WIDE, bool A_KMAJOR, bool B_KMAJOR, bool SPICY>
__global__ void __launch_bounds__(Shape<WIDE>::THREADS, WIDE ? 1 : 2)  // re-divided below with setmaxnreg
gemm_f64_ws_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                   const __grid_constant__ CUtensorMap mapC, const Params p) {
  using S = Shape<WIDE>;
  constexpr int BN = S::BN, STAGES = S::STAGES, STAGE_BYTES = S::STAGE_BYTES, CONSUMERS = S::CONSUMERS;
  static_assert(!(WIDE && SPICY), "the wide configuration has no spicy variant");
  extern __shared__ uint8_t ws_smem_raw[];
  const uint32_t smem_base = (smem_u32(ws_smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = ws_smem_raw + (smem_base - smem_u32(ws_smem_raw));
  const uint32_t sdst = smem_base;                        // wide: destination tile buffer
  const uint32_t sstages = smem_base + S::DST_BYTES;      // operand ring
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_gen + S::DST_BYTES + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  uint64_t* dst_full = empty + STAGES;   // wide: old dst values landed (Add) / buffer free to overwrite (Replace)
  uint64_t* dst_free = dst_full + 1;     // wide: the previous TMA store has read the buffer
  uint64_t* dst_ready = dst_free + 1;    // wide: every consumer warp has written its part of the buffer

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMERS);
    }
    mbar_init(dst_full, 1);
    mbar_init(dst_free, 1);
    mbar_init(dst_ready, CONSUMERS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int nkt = (p.k + BK - 1) / BK;
  TileWalk<BN> walk;
  walk.init(p.tiles_m, p.tiles_n, p.c_struct);
  // wide: does tile (tm, tn) lie wholly inside the kept part of dst (BM == BN, so off-diagonal tiles do)?
  auto staged = [&](int tm, int tn) -> bool {
    if constexpr (!WIDE) return false;
    if (!p.dst_tma) return false;
    if (is_lower(p.c_struct)) return tm > tn;
    if (is_upper(p.c_struct)) return tn > tm;
    return true;
  };

  if (warp < 4) {
    // ================= producer warpgroup =================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(S::PRODUCER_REGS));
    if (warp == 0 && lane == 0) {
      uint32_t s = 0, ph = 0;  // ring slot of the next k-step and the parity of its pass over the ring
      uint32_t ds = 0;         // staged tiles so far
      for (int i = 0; i < p.tiles_per_cta; ++i) {
        int tm, tn;
        if (!walk.locate((int)blockIdx.x * p.tiles_per_cta + i, tm, tn)) break;
        const int m0 = tm * BM, n0 = tn * BN;
        const bool st = staged(tm, tn);
        const int dst_at = min(STAGES, nkt) - 1;
        for (int kt = 0; kt < nkt; ++kt) {
          mbar_wait(&empty[s], ph ^ 1u);
          const uint32_t sa = sstages + s * STAGE_BYTES, sb = sa + A_BYTES;
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
          // the old dst tile is requested once the ring holds this tile's first stages: waiting here for the previous
          // tile's store costs nothing, since the next stage needs the consumers back in the main loop anyway
          if (st && kt == dst_at) {
            mbar_wait(dst_free, (ds & 1u) ^ 1u);
            if (p.accum) {
              mbar_expect_tx(dst_full, S::DST_BYTES);
#pragma unroll
              for (int b = 0; b < BM / 16; ++b) tma_load_2d(sdst + b * (16 * BN * 8), &mapC, dst_full, m0 + b * 16, n0);
            } else {
              mbar_arrive(dst_full);
            }
            ++ds;
          }
          if (++s == STAGES) {
            s = 0;
            ph ^= 1u;
          }
        }
      }
    }
    if constexpr (WIDE) {
      // storer (warp 1): TMA-stores each staged tile once the consumers have filled the buffer, and frees the buffer
      // when the store has read it, so that the consumers go from one tile's epilogue straight into the next main loop
      if (warp == 1 && lane == 0) {
        uint32_t ds = 0;
        for (int i = 0; i < p.tiles_per_cta; ++i) {
          int tm, tn;
          if (!walk.locate((int)blockIdx.x * p.tiles_per_cta + i, tm, tn)) break;
          if (!staged(tm, tn)) continue;
          mbar_wait(dst_ready, ds & 1u);
          ++ds;
#pragma unroll
          for (int b = 0; b < BM / 16; ++b) tma_store_2d(&mapC, sdst + b * (16 * BN * 8), tm * BM + b * 16, tn * BN);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
          mbar_arrive(dst_free);
        }
        // the tile stores must have completed before the kernel ends
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
      }
    }
    return;
  }

  // ================= consumer warpgroups =================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(S::CONSUMER_REGS));
  const int cw = warp - 4;
  const int g = lane >> 2, t = lane & 3;
  const int wm0 = (cw & 3) * (WMI * 8), wn0 = (cw >> 2) * (WNI * 8);  // warp tile rows [wm0, wm0 + 32) x cols [wn0, wn0 + 64)
  // per-lane fragment offsets for the 4 k slots of a stage: k index K4(q, t) = {0,3,12,15}[t] ^ {0,1,4,5}[q]
  const int base_k = (t == 0) ? 0 : (t == 1) ? 3 : (t == 2) ? 12 : 15;
  uint32_t offA[4][2], offB[4][2];  // [k slot][parity of the 8-row block] (MN-major) / [k slot][0] (K-major)
  {
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
        offB[s][0] = off_k_major(wn0 + g, kk);
        offB[s][1] = 0;
      } else {
        offB[s][0] = off_mn_major(wn0 + g, kk);
        offB[s][1] = off_mn_major(wn0 + 8 + g, kk);
      }
      // opaque to the compiler, so that it keeps the offsets in registers instead of rebuilding them from the thread
      // index in every k-step (it does that when the register epilogue's accumulators and old values crowd them)
      asm volatile("" : "+r"(offA[s][0]), "+r"(offB[s][0]));
      if constexpr (!A_KMAJOR) asm volatile("" : "+r"(offA[s][1]));
      if constexpr (!B_KMAJOR) asm volatile("" : "+r"(offB[s][1]));
    }
  }

  const int cs_ = p.c_struct;
  const bool c_low = is_lower(cs_), c_up = is_upper(cs_);
  const bool c_nodiag = is_strict(cs_) || is_unit(cs_);
  const double alpha = p.alpha;
  const bool add = p.accum != 0;

  if (!WIDE && p.stagger_cycles > 0 && (int)blockIdx.x >= p.sm_slots && (int)blockIdx.x < 2 * p.sm_slots) {
    const long long t0 = clock64();
    while (clock64() - t0 < p.stagger_cycles) __nanosleep(256);
  }

  uint32_t s = 0, ph = 0;  // ring slot of the next k-step and the parity of its pass over the ring (as the producer's)
  uint32_t sa = sstages;   // the slot's A tile; its B tile follows at + A_BYTES
  uint32_t dc = 0;         // staged tiles so far
  for (int ti = 0; ti < p.tiles_per_cta; ++ti) {
    int tm, tn;
    if (!walk.locate((int)blockIdx.x * p.tiles_per_cta + ti, tm, tn)) break;
    const int m0 = tm * BM, n0 = tn * BN;

    double acc[WMI][WNI][2];
#pragma unroll
    for (int i = 0; i < WMI; ++i)
#pragma unroll
      for (int j = 0; j < WNI; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    for (int kt = 0; kt < nkt; ++kt) {
      double dk[4] = {1.0, 1.0, 1.0, 1.0};
      if constexpr (SPICY) {
        if (p.diag) {  // this lane's four k indices of the stage: K4(ss, t)
#pragma unroll
          for (int ss = 0; ss < 4; ++ss) {
            const int kg = kt * BK + (base_k ^ ((ss & 1) | ((ss & 2) << 1)));
            dk[ss] = kg < p.k ? p.diag[(i64)kg * p.diag_stride] : 0.0;
          }
        }
      }
      mbar_wait(&full[s], ph);
      const uint32_t sb = sa + A_BYTES;
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
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (++s == STAGES) {
        s = 0;
        ph ^= 1u;
        sa = sstages;
      } else {
        sa += STAGE_BYTES;
      }
    }

    if (staged(tm, tn)) {
      // ---- wide epilogue through shared memory: buffer = alpha * acc [+ old], then the storer warp's TMA store. Element
      // (r, c) of the tile sits in box r / 16 at line c, 16-byte chunk ((r & 15) / 2) ^ (c & 7): a half-warp's 8-byte
      // accesses (4 rows x 4 column pairs) hit 16 distinct banks ----
      mbar_wait(dst_full, dc & 1u);
      ++dc;
#pragma unroll
      for (int i = 0; i < WMI; ++i) {
        const int r = wm0 + i * 8 + g;
        const uint32_t rbase = sdst + (r >> 4) * (16 * BN * 8) + ((r & 1) << 3);
        const int rchunk = (r & 15) >> 1;
#pragma unroll
        for (int j = 0; j < WNI; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = wn0 + j * 8 + 2 * t + e;
            const uint32_t addr = rbase + c * 128 + ((rchunk ^ (c & 7)) << 4);
            sts64(addr, add ? (alpha * acc[i][j][e] + lds64(addr)) : alpha * acc[i][j][e]);
          }
      }
      // the generic-proxy writes above must be visible to the async proxy (the TMA store) before it reads the buffer
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(dst_ready);
      continue;
    }

    // ---- register epilogue: dst = [dst +] alpha * acc, masked by dst structure and bounds. Add mode: the old values of
    // row block i + 1 are requested before row block i is combined and stored (two register sets), so the four row blocks
    // cost about two global-memory round trips instead of four ----
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
    // wide: only the tiles on the diagonal of a triangular dst take this epilogue, so the old values of a row block are
    // loaded just before it is combined. A second register set here would push the fragment offsets out of registers,
    // and every k-step of every tile would reload them from local memory.
    constexpr int CV = WIDE ? 1 : 2;
    double cv[CV][WNI][2];
    auto load_old = [&](int i, double (&dst)[WNI][2]) {
      const int row = m0 + wm0 + i * 8 + g;
      const i64 roff = rowoff(row);
#pragma unroll
      for (int j = 0; j < WNI; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + wn0 + j * 8 + 2 * t + e;
          dst[j][e] = kept(row, col) ? __ldcg(p.C + roff + coloff(col)) : 0.0;
        }
    };
    if (add) load_old(0, cv[0]);
#pragma unroll
    for (int i = 0; i < WMI; ++i) {
      if constexpr (WIDE) {
        if (add && i > 0) load_old(i, cv[0]);
      } else {
        if (add && i + 1 < WMI) load_old(i + 1, cv[(i + 1) & 1]);
      }
      const int row = m0 + wm0 + i * 8 + g;
      const i64 roff = rowoff(row);
#pragma unroll
      for (int j = 0; j < WNI; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + wn0 + j * 8 + 2 * t + e;
          if (kept(row, col)) p.C[roff + coloff(col)] = add ? (alpha * acc[i][j][e] + cv[i % CV][j][e]) : alpha * acc[i][j][e];
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

struct Spicy {
  const long long* row_idx = nullptr;
  const long long* col_idx = nullptr;
  const double* diag = nullptr;
  i64 diag_stride = 1;
};
// tiles the kernel enumerates for an m x n dst of structure c_struct with CTA tiles BM x bn (see TileWalk)
inline long long ws_tiles(int m, int n, int c_struct, int bn) {
  const int tiles_m = (m + BM - 1) / BM, tiles_n = (n + bn - 1) / bn;
  if (c_struct == RECT) return (long long)tiles_m * tiles_n;
  long long tiles = 0;
  for (int tm = 0; tm < tiles_m; ++tm) {
    const int lo = is_upper(c_struct) ? (tm * BM) / bn : 0;
    const int hi = is_lower(c_struct) ? std::min(tiles_n, (tm * BM + BM - 1) / bn + 1) : tiles_n;
    tiles += std::max(0, hi - lo);
  }
  return tiles;
}

// Launches the kernel if the problem qualifies; returns false otherwise (caller falls back to the cp.async kernel).
// `wide` selects the 128 x 128 configuration (no spicy variant).
inline bool try_gemm_f64_ws(cudaStream_t stream, const GemmF64Params& q, const Spicy* sp = nullptr, bool wide = false) {
  if (q.a_struct != RECT || q.b_struct != RECT || q.k_split_len > 0 || q.k < 1) return false;
  if (wide && sp) return false;
  if (!encode_fn()) return false;
  bool ak = false, bk = false;
  if (!tma_layout(q.A, q.m, q.k, q.a_rs, q.a_cs, &ak)) return false;
  if (!tma_layout(q.B, q.n, q.k, q.b_cs, q.b_rs, &bk)) return false;
  if (q.a_rs == 1 && q.a_cs == 1) return false;  // degenerate vectors: leave to the general kernel
  if (q.b_rs == 1 && q.b_cs == 1) return false;
  const int bn = wide ? Shape<true>::BN : Shape<false>::BN;
  Params p;
  p.C = q.C; p.c_rs = q.c_rs; p.c_cs = q.c_cs;
  p.m = q.m; p.n = q.n; p.k = q.k;
  p.c_struct = q.c_struct; p.accum = q.accum; p.alpha = q.alpha;
  p.row_idx = sp ? sp->row_idx : nullptr;
  p.col_idx = sp ? sp->col_idx : nullptr;
  p.diag = sp ? sp->diag : nullptr;
  p.diag_stride = sp ? sp->diag_stride : 1;
  p.tiles_m = (q.m + BM - 1) / BM;
  p.tiles_n = (q.n + bn - 1) / bn;
  const long long tiles = ws_tiles(q.m, q.n, q.c_struct, bn);
  if (tiles == 0) return true;
  CUtensorMap mapA, mapB, mapC;
  const bool okA = ak ? make_map(&mapA, q.A, q.k, q.m, q.a_rs, BM) : make_map(&mapA, q.A, q.m, q.k, q.a_cs, 16);
  const bool okB = bk ? make_map(&mapB, q.B, q.k, q.n, q.b_cs, bn) : make_map(&mapB, q.B, q.n, q.k, q.b_rs, 16);
  if (!okA || !okB) return false;
  // wide: dst tiles through shared memory when TMA can address dst (column-major, 16-byte aligned base and ld); any other
  // dst takes the register epilogue for every tile
  p.dst_tma = wide && q.c_rs == 1 && q.c_cs >= q.m && q.c_cs % 2 == 0 && (((uintptr_t)q.C) & 15) == 0 &&
              make_map(&mapC, q.C, q.m, q.n, q.c_cs, 128);
  if (!p.dst_tma) mapC = mapA;  // not read
  p.sm_slots = stream_sms(stream);
  if (!wide) {
    // tiles per CTA shrink with k so that a CTA stays short-lived (on the order of 50 us at 128 f64 FMA / clock / SM), and
    // never below two CTAs per SM while the tiles allow it (fewer would leave SMs idle in small launches)
    const long long tpc_fill = std::max<long long>(1, (tiles + 2ll * p.sm_slots - 1) / (2ll * p.sm_slots));
    p.tiles_per_cta = (int)std::max<long long>(1, std::min<long long>({8, 768 / std::max(q.k, 1), tpc_fill}));
  } else {
    // one CTA per SM, so a launch takes ceil(CTAs / SMs) waves of tiles_per_cta tiles. Up to 1024 / k tiles per CTA
    // (about 70 us at k = 256 and the full DMMA rate: long enough to amortise the pipeline fill and the last tile's
    // store, short enough that the SMs turn over for the panel stream of the look-ahead factorizations); among those,
    // the count with the shortest launch, each CTA start charged 0.15 tile
    const int tpc_max = (int)std::max<long long>(1, std::min<long long>(8, 1024 / q.k));
    double best = 1e300;
    p.tiles_per_cta = 1;
    for (int tpc = 1; tpc <= tpc_max; ++tpc) {
      const long long waves = ((tiles + tpc - 1) / tpc + p.sm_slots - 1) / p.sm_slots;
      const double cost = (double)waves * (tpc + 0.15);
      if (cost < best) { best = cost; p.tiles_per_cta = tpc; }
    }
  }
  const int grid = (int)((tiles + p.tiles_per_cta - 1) / p.tiles_per_cta);
  // narrow only (two CTAs per SM): half a tile at the full rate of one SM, (k / 16) k-steps x 128 x 64 x 16 FMA /
  // (128 FMA / clock) / 2
  p.stagger_cycles = (!wide && grid >= 2 * p.sm_slots) ? (long long)((q.k + BK - 1) / BK) * 512 : 0;
  // one opt-in to > 48 KB of dynamic shared memory per kernel variant
  static bool configured[12] = {};
  auto launch = [&](int which, auto kern, int threads, int smem_bytes) {
    if (!configured[which]) {
      FB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
      configured[which] = true;
    }
    kern<<<grid, threads, smem_bytes, stream>>>(mapA, mapB, mapC, p);
  };
  using N = Shape<false>;
  using W = Shape<true>;
  const int nsm = N::SMEM_BYTES;
  if (wide) {
    if (ak && bk) launch(8, gemm_f64_ws_kernel<true, true, true, false>, W::THREADS, W::SMEM_BYTES);
    else if (ak && !bk) launch(9, gemm_f64_ws_kernel<true, true, false, false>, W::THREADS, W::SMEM_BYTES);
    else if (!ak && bk) launch(10, gemm_f64_ws_kernel<true, false, true, false>, W::THREADS, W::SMEM_BYTES);
    else launch(11, gemm_f64_ws_kernel<true, false, false, false>, W::THREADS, W::SMEM_BYTES);
  } else if (!sp) {
    if (ak && bk) launch(0, gemm_f64_ws_kernel<false, true, true, false>, N::THREADS, nsm);
    else if (ak && !bk) launch(1, gemm_f64_ws_kernel<false, true, false, false>, N::THREADS, nsm);
    else if (!ak && bk) launch(2, gemm_f64_ws_kernel<false, false, true, false>, N::THREADS, nsm);
    else launch(3, gemm_f64_ws_kernel<false, false, false, false>, N::THREADS, nsm);
  } else {
    if (ak && bk) launch(4, gemm_f64_ws_kernel<false, true, true, true>, N::THREADS, nsm);
    else if (ak && !bk) launch(5, gemm_f64_ws_kernel<false, true, false, true>, N::THREADS, nsm);
    else if (!ak && bk) launch(6, gemm_f64_ws_kernel<false, false, true, true>, N::THREADS, nsm);
    else launch(7, gemm_f64_ws_kernel<false, false, false, true>, N::THREADS, nsm);
  }
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return true;
}

}  // namespace ws64
}  // namespace fb
