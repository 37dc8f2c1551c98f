// f64 GEMM / structured GEMM kernel, see gemm_f64.cuh for the reference semantics it implements.
//
// Design (H100, sm_90a):
//   * math: mma.sync.m16n8k16.f64 -> one DMMA.16x8x16 per 16 x 8 block and 16-deep k-step (wgmma has no f64 type).
//     The m8n8k4 shape sustains only half of the H100's f64 tensor rate; the wide shapes reach ~128 f64 FMA/clk/SM
//     (profiles/r03_f64_peaks.log).
//   * operands staged with cp.async (16 B vectors when the view is aligned, 8 B otherwise => any stride,
//     any sign) into padded shared tiles; pad of 4 doubles makes every fragment load (8 rows x 4 k of
//     8-byte words per half-warp) hit 16 distinct 8-byte banks.
//   * structure handling: triangular inputs are masked in shared memory after the tile lands (only tiles
//     that intersect the diagonal pay the extra pass), fully-masked k-ranges are skipped, triangular dst
//     tiles above/below the diagonal exit immediately and diagonal tiles mask the store.
#include "gemm_f64.cuh"
#include "gemm_f64_sliced.cuh"
#include "gemm_f64_ws.cuh"
#include "runtime.cuh"

namespace fb {

namespace {

template <int WARPS_M_, int WARPS_N_, int WMI_, int WNI_, int BK_, int STAGES_>
struct TileCfg {
  static constexpr int WARPS_M = WARPS_M_, WARPS_N = WARPS_N_, WMI = WMI_, WNI = WNI_, BK = BK_, STAGES = STAGES_;
  static constexpr int BM = WARPS_M * WMI * 8;
  static constexpr int BN = WARPS_N * WNI * 8;
  static constexpr int THREADS = WARPS_M * WARPS_N * 32;
};

// One operand tile: `ROWS` indices along the non-contracted dim (mn) x BK along k.
// KMAJOR: smem[mn][k] (ld = BK+4) else smem[k][mn] (ld = ROWS+4).
template <int ROWS, int BK, bool KMAJOR>
struct OpTile {
  static constexpr int LD = KMAJOR ? BK + 4 : ROWS + 4;
  static constexpr int SIZE = KMAJOR ? ROWS * LD : BK * LD;
  __device__ static __forceinline__ int idx(int mn, int kk) {
    return KMAJOR ? mn * LD + kk : kk * LD + mn;
  }
};

// Global -> shared copy of one operand tile. Element (mn, kk) lives at g + (mn0+mn)*s_mn + (k0+kk)*s_k.
template <int ROWS, int BK, bool KMAJOR, bool VEC, int THREADS>
__device__ __forceinline__ void load_tile(double* __restrict__ s, const double* __restrict__ g, i64 s_mn, i64 s_k,
                                          int mn0, int k0, int MN, int K, int tid) {
  using T = OpTile<ROWS, BK, KMAJOR>;
  if constexpr (VEC) {
    constexpr int CHUNKS = ROWS * BK / 2;
    static_assert(CHUNKS % THREADS == 0, "tile/threads mismatch");
#pragma unroll
    for (int it = 0; it < CHUNKS / THREADS; ++it) {
      int c = it * THREADS + tid;
      int mn, kk, nvalid;
      const double* src;
      if constexpr (KMAJOR) {
        mn = c / (BK / 2);
        kk = (c % (BK / 2)) * 2;
        int rem = K - (k0 + kk);
        nvalid = (mn0 + mn < MN) ? (rem < 0 ? 0 : (rem > 2 ? 2 : rem)) : 0;
        src = g + (i64)(mn0 + mn) * s_mn + (i64)(k0 + kk);
      } else {
        kk = c / (ROWS / 2);
        mn = (c % (ROWS / 2)) * 2;
        int rem = MN - (mn0 + mn);
        nvalid = (k0 + kk < K) ? (rem < 0 ? 0 : (rem > 2 ? 2 : rem)) : 0;
        src = g + (i64)(mn0 + mn) + (i64)(k0 + kk) * s_k;
      }
      if (nvalid == 0) src = g;
      cp_async_16(s + T::idx(mn, kk), src, nvalid * 8);
    }
  } else {
    constexpr int ELEMS = ROWS * BK;
    static_assert(ELEMS % THREADS == 0, "tile/threads mismatch");
#pragma unroll
    for (int it = 0; it < ELEMS / THREADS; ++it) {
      int e = it * THREADS + tid;
      int mn, kk;
      if constexpr (KMAJOR) {
        mn = e / BK;
        kk = e % BK;
      } else {
        kk = e / ROWS;
        mn = e % ROWS;
      }
      bool ok = (mn0 + mn < MN) && (k0 + kk < K);
      const double* src = ok ? g + (i64)(mn0 + mn) * s_mn + (i64)(k0 + kk) * s_k : g;
      cp_async_8(s + T::idx(mn, kk), src, ok ? 8 : 0);
    }
  }
}

// rel > 0 : kept side of a lower-triangular operand; rel == 0 : diagonal.
// lhs (m x k): row = mn, col = k  -> rel_lower = mn - k
// rhs (k x n): row = k,  col = mn -> rel_lower = k - mn
template <int ROWS, int BK, bool KMAJOR, int THREADS>
__device__ __forceinline__ void fixup_tile(double* s, int structure, bool is_rhs, int mn0, int k0, int tid) {
  using T = OpTile<ROWS, BK, KMAJOR>;
  const bool lower = is_lower(structure);
  const double diagval = is_unit(structure) ? 1.0 : 0.0;
  const bool keepdiag = !(is_unit(structure) || is_strict(structure));
  for (int e = tid; e < ROWS * BK; e += THREADS) {
    int mn = e % ROWS, kk = e / ROWS;
    int rel = is_rhs ? (k0 + kk) - (mn0 + mn) : (mn0 + mn) - (k0 + kk);
    if (!lower) rel = -rel;
    if (rel < 0)
      s[T::idx(mn, kk)] = 0.0;
    else if (rel == 0 && !keepdiag)
      s[T::idx(mn, kk)] = diagval;
  }
}

// does the (mn0..mn0+ROWS) x (k0..k0+BK) tile of a structured operand need masking?
__device__ __forceinline__ bool tile_needs_fixup(int structure, bool is_rhs, int mn0, int rows, int k0, int bk) {
  if (structure == RECT) return false;
  // min/max of rel_lower over the tile
  int lo, hi;
  if (!is_rhs) {
    lo = mn0 - (k0 + bk - 1);
    hi = (mn0 + rows - 1) - k0;
  } else {
    lo = k0 - (mn0 + rows - 1);
    hi = (k0 + bk - 1) - mn0;
  }
  if (!is_lower(structure)) {
    int t = lo;
    lo = -hi;
    hi = -t;
  }
  (void)hi;
  // entirely strictly inside the kept region <=> lo > 0
  return lo <= 0;
}

template <class Cfg, bool AK, bool BNM, bool VEC>
__global__ void __launch_bounds__(Cfg::THREADS) gemm_f64_kernel(const GemmF64Params p) {
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES, THREADS = Cfg::THREADS;
  constexpr int WMI = Cfg::WMI, WNI = Cfg::WNI;
  static_assert(BK == 16 && WMI % 2 == 0, "the main loop issues 16 x 8 x 16 DMMAs");
  using TA = OpTile<BM, BK, AK>;
  using TB = OpTile<BN, BK, !BNM>;  // rhs: K-major when b_rs == 1
  extern __shared__ __align__(16) double smem[];
  double* As = smem;
  double* Bs = smem + STAGES * TA::SIZE;

  // ---- tile coordinates (grouped rasterisation for L2 reuse) ----
  constexpr int GROUP = 8;
  int bid = blockIdx.x;
  int width = GROUP * p.tiles_n;
  int group_id = bid / width;
  int first_m = group_id * GROUP;
  int gsize = min(p.tiles_m - first_m, GROUP);
  int tm = first_m + (bid % width) % gsize;
  int tn = (bid % width) / gsize;
  const int m0 = tm * BM, n0 = tn * BN;

  // ---- dst structure: skip tiles with nothing to write ----
  const int cs_ = p.c_struct;
  if (is_lower(cs_)) {
    if (m0 + BM - 1 < n0) return;
  } else if (is_upper(cs_)) {
    if (n0 + BN - 1 < m0) return;
  }

  // ---- contracted range after structure pruning ----
  int k_begin = 0, k_end = p.k;
  if (is_lower(p.a_struct)) k_end = min(k_end, m0 + BM);
  if (is_upper(p.a_struct)) k_begin = max(k_begin, m0);
  if (is_lower(p.b_struct)) k_begin = max(k_begin, n0);
  if (is_upper(p.b_struct)) k_end = min(k_end, n0 + BN);
  double* __restrict__ Cout = p.C;
  if (p.k_split_len > 0) {
    const int kb = (int)blockIdx.y * p.k_split_len;
    k_begin = max(k_begin, kb);
    k_end = min(k_end, kb + p.k_split_len);
    Cout += (i64)blockIdx.y * p.c_split_stride;
  }
  k_begin = (k_begin / BK) * BK;
  const int nkt = k_end > k_begin ? (k_end - k_begin + BK - 1) / BK : 0;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm0 = (warp % Cfg::WARPS_M) * (WMI * 8);
  const int wn0 = (warp / Cfg::WARPS_M) * (WNI * 8);

  double acc[WMI][WNI][2];
#pragma unroll
  for (int i = 0; i < WMI; ++i)
#pragma unroll
    for (int j = 0; j < WNI; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  auto load_stage = [&](int stage, int kt) {
    const int k0 = k_begin + kt * BK;
    load_tile<BM, BK, AK, VEC, THREADS>(As + stage * TA::SIZE, p.A, p.a_rs, p.a_cs, m0, k0, p.m, p.k, tid);
    load_tile<BN, BK, !BNM, VEC, THREADS>(Bs + stage * TB::SIZE, p.B, p.b_cs, p.b_rs, n0, k0, p.n, p.k, tid);
  };

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) load_stage(s, s);
    cp_async_commit();
  }

  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    const int stage = kt % STAGES;
    double* a_s = As + stage * TA::SIZE;
    double* b_s = Bs + stage * TB::SIZE;
    {
      const int k0 = k_begin + kt * BK;
      const bool fa = tile_needs_fixup(p.a_struct, false, m0, BM, k0, BK);
      const bool fb_ = tile_needs_fixup(p.b_struct, true, n0, BN, k0, BK);
      if (fa || fb_) {
        if (fa) fixup_tile<BM, BK, AK, THREADS>(a_s, p.a_struct, false, m0, k0, tid);
        if (fb_) fixup_tile<BN, BK, !BNM, THREADS>(b_s, p.b_struct, true, n0, k0, tid);
        __syncthreads();
      }
    }
    {
      const int nk = kt + STAGES - 1;
      if (nk < nkt) load_stage(nk % STAGES, nk);
      cp_async_commit();
    }
    // one 16-deep DMMA per 16 x 8 block (rows 8 (2 ip) .. 8 (2 ip + 2) of the warp tile x 8 columns), k = t + 4 q
    double a[WMI / 2][8], b[WNI][4];
#pragma unroll
    for (int ip = 0; ip < WMI / 2; ++ip)
#pragma unroll
      for (int v = 0; v < 8; ++v) a[ip][v] = a_s[TA::idx(wm0 + (2 * ip + (v & 1)) * 8 + g, 4 * (v >> 1) + t)];
#pragma unroll
    for (int j = 0; j < WNI; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) b[j][q] = b_s[TB::idx(wn0 + j * 8 + g, 4 * q + t)];
#pragma unroll
    for (int ip = 0; ip < WMI / 2; ++ip)
#pragma unroll
      for (int j = 0; j < WNI; ++j)
        dmma16816(acc[2 * ip][j][0], acc[2 * ip][j][1], acc[2 * ip + 1][j][0], acc[2 * ip + 1][j][1], a[ip], b[j]);
  }
  cp_async_wait<0>();

  // ---- epilogue: dst = [dst +] alpha * acc, masked by dst structure ----
  const bool c_low = is_lower(cs_), c_up = is_upper(cs_);
  const bool c_nodiag = is_strict(cs_) || is_unit(cs_);
  const double alpha = p.alpha;
  const bool add = p.accum != 0;
  // Two passes per half of the warp tile: (1) issue ALL dst loads of the half as independent predicated loads
  // (a load->add->store chain per element would expose the full memory latency 2*WMI*WNI times
  // per tile), (2) combine and store.
  constexpr int HALF = WMI > 1 ? WMI / 2 : 1;
#pragma unroll
  for (int ih = 0; ih < WMI; ih += HALF) {
    double cv[HALF][WNI][2];
    bool ok[HALF][WNI][2];
#pragma unroll
    for (int ii = 0; ii < HALF; ++ii) {
      const int row = m0 + wm0 + (ih + ii) * 8 + g;
#pragma unroll
      for (int j = 0; j < WNI; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + wn0 + j * 8 + 2 * t + e;
          bool v = row < p.m && col < p.n;
          if (c_low && (row < col || (row == col && c_nodiag))) v = false;
          if (c_up && (row > col || (row == col && c_nodiag))) v = false;
          ok[ii][j][e] = v;
          cv[ii][j][e] = (add && v) ? Cout[(i64)row * p.c_rs + (i64)col * p.c_cs] : 0.0;
        }
      }
    }
#pragma unroll
    for (int ii = 0; ii < HALF; ++ii) {
      const int row = m0 + wm0 + (ih + ii) * 8 + g;
#pragma unroll
      for (int j = 0; j < WNI; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + wn0 + j * 8 + 2 * t + e;
          if (ok[ii][j][e]) Cout[(i64)row * p.c_rs + (i64)col * p.c_cs] = alpha * acc[ih + ii][j][e] + cv[ii][j][e];
        }
      }
    }
  }
}

using CfgS3 = TileCfg<2, 2, 4, 4, 16, 3>;  // 64 x 64 x 16, 128 threads, warp tile 32 x 32, 3 stages (57 KB => 3 CTAs/SM)

template <class Cfg, bool AK, bool BNM>
constexpr size_t smem_bytes() {
  return sizeof(double) * Cfg::STAGES *
         (OpTile<Cfg::BM, Cfg::BK, AK>::SIZE + OpTile<Cfg::BN, Cfg::BK, !BNM>::SIZE);
}

template <class Cfg, bool AK, bool BNM, bool VEC>
void launch_cfg(cudaStream_t stream, GemmF64Params& p) {
  p.tiles_m = (p.m + Cfg::BM - 1) / Cfg::BM;
  p.tiles_n = (p.n + Cfg::BN - 1) / Cfg::BN;
  constexpr size_t smem = smem_bytes<Cfg, AK, BNM>();
  static bool configured = false;
  if (!configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(gemm_f64_kernel<Cfg, AK, BNM, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    configured = true;
  }
  long long tiles = (long long)p.tiles_m * p.tiles_n;
  const unsigned splits = p.k_split_len > 0 ? (unsigned)((p.k + p.k_split_len - 1) / p.k_split_len) : 1u;
  gemm_f64_kernel<Cfg, AK, BNM, VEC><<<dim3((unsigned)tiles, splits), Cfg::THREADS, smem, stream>>>(p);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

template <bool AK, bool BNM, bool VEC>
void launch_layout(cudaStream_t stream, GemmF64Params& p) {
  // the 64x64 tile with several CTAs per SM: the prologue / epilogue of one CTA overlap another CTA's main loop
  launch_cfg<CfgS3, AK, BNM, VEC>(stream, p);
}

inline int transpose_struct(int s) {
  switch (s) {
    case TRI_LOWER: return TRI_UPPER;
    case TRI_UPPER: return TRI_LOWER;
    case STRICT_LOWER: return STRICT_UPPER;
    case STRICT_UPPER: return STRICT_LOWER;
    case UNIT_LOWER: return UNIT_UPPER;
    case UNIT_UPPER: return UNIT_LOWER;
    default: return RECT;
  }
}

inline int ws_mode() { return (int)get_option(OPT_GEMM_WS); }

// per-stream grow-only workspace of the int8-sliced path (slices of both operands + exponents)
oz::Workspace* sliced_workspace(cudaStream_t stream) {
  struct Slot {
    cudaStream_t st;
    oz::Workspace ws;
    bool used;
  };
  static Slot slots[8];
  for (auto& s : slots)
    if (s.used && s.st == stream) return &s.ws;
  for (auto& s : slots)
    if (!s.used) {
      s.used = true;
      s.st = stream;
      return &s.ws;
    }
  cudaStreamSynchronize(slots[0].st);
  slots[0].st = stream;
  return &slots[0].ws;
}

inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }

// dst(struct) = [dst +] alpha * sum_z W_z  (W_z: compact column-major m x n partial products, summed in z order)
__global__ void splitk_reduce_kernel(double* __restrict__ C, i64 rs, i64 cs, int m, int n, int c_struct, int accum,
                                     double alpha, const double* __restrict__ W, int splits) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)m * n) return;
  const int row = (int)(e % m), col = (int)(e / m);
  const bool nodiag = is_strict(c_struct) || is_unit(c_struct);
  if (is_lower(c_struct) && (row < col || (row == col && nodiag))) return;
  if (is_upper(c_struct) && (row > col || (row == col && nodiag))) return;
  double s = 0.0;
  for (int z = 0; z < splits; ++z) s += W[(long long)z * m * n + e];
  double* cp = C + (i64)row * rs + (i64)col * cs;
  *cp = accum ? (*cp + alpha * s) : alpha * s;
}

}  // namespace

void gemm_f64(cudaStream_t stream, VD dst, int dst_struct, int accum, VCD lhs, int lhs_struct, VCD rhs, int rhs_struct,
              double alpha) {
  FB_ASSERT(dst.nrows == lhs.nrows && dst.ncols == rhs.ncols && lhs.ncols == rhs.nrows, "matmul shape mismatch");
  if (dst_struct != RECT) FB_ASSERT(dst.nrows == dst.ncols, "triangular dst must be square");
  if (lhs_struct != RECT) FB_ASSERT(lhs.nrows == lhs.ncols, "triangular lhs must be square");
  if (rhs_struct != RECT) FB_ASSERT(rhs.nrows == rhs.ncols, "triangular rhs must be square");
  if (dst.nrows == 0 || dst.ncols == 0) return;
  if (lhs.ncols == 0 && accum != 0) return;
  FB_ASSERT(dst.nrows < (1ll << 31) && dst.ncols < (1ll << 31) && lhs.ncols < (1ll << 31), "dimension too large");

  // Prefer a unit row stride on dst: C^T = B^T A^T.
  if (dst.rs != 1 && dst.cs == 1) {
    VD d2 = dst.t();
    VCD l2 = rhs.t(), r2 = lhs.t();
    int ls = transpose_struct(rhs_struct), rs_ = transpose_struct(lhs_struct);
    dst = d2; lhs = l2; rhs = r2;
    dst_struct = transpose_struct(dst_struct);
    lhs_struct = ls; rhs_struct = rs_;
  }

  GemmF64Params p;
  p.m = (int)dst.nrows; p.n = (int)dst.ncols; p.k = (int)lhs.ncols;
  p.A = lhs.ptr; p.a_rs = lhs.rs; p.a_cs = lhs.cs; p.a_struct = lhs_struct;
  p.B = rhs.ptr; p.b_rs = rhs.rs; p.b_cs = rhs.cs; p.b_struct = rhs_struct;
  p.C = dst.ptr; p.c_rs = dst.rs; p.c_cs = dst.cs; p.c_struct = dst_struct;
  p.alpha = alpha; p.accum = accum;
  p.k_split_len = 0; p.c_split_stride = 0;

  // split-K for tall-skinny products (few output tiles, long contraction): partial products go to workspace slices,
  // then one deterministic reduce pass applies alpha / accum / the dst structure mask.
  double* split_ws = nullptr;
  int splits = 1;
  {
    const long long tiles = (long long)((p.m + 63) / 64) * ((p.n + 63) / 64);
    const int sms = stream_sms(stream);
    if (tiles < sms && p.k >= 4096 && lhs_struct == RECT && rhs_struct == RECT) {
      splits = (int)std::min<long long>((sms * 3ll + tiles - 1) / tiles, p.k / 1024);
      if (splits >= 2) {
        int len = (p.k + splits - 1) / splits;
        len = (len + 63) / 64 * 64;
        splits = (p.k + len - 1) / len;
        split_ws = (double*)stream_scratch(stream, (size_t)splits * p.m * p.n * sizeof(double));
        p.k_split_len = len;
        p.c_split_stride = (i64)p.m * p.n;
        p.C = split_ws; p.c_rs = 1; p.c_cs = p.m; p.c_struct = RECT;
        p.alpha = 1.0; p.accum = 0;
      } else {
        splits = 1;
      }
    }
  }

  // operand layouts
  bool a_unit_m = (lhs.rs == 1) || lhs.nrows == 1;
  bool a_unit_k = (lhs.cs == 1) || lhs.ncols == 1;
  bool AK = !a_unit_m && a_unit_k;  // k contiguous
  bool a_vec = AK ? (lhs.cs == 1 && (lhs.rs % 2 == 0)) : (lhs.rs == 1 && (lhs.cs % 2 == 0));
  a_vec = a_vec && aligned16(lhs.ptr);
  bool b_unit_k = (rhs.rs == 1) || rhs.nrows == 1;
  bool b_unit_n = (rhs.cs == 1) || rhs.ncols == 1;
  bool BNM = !b_unit_k && b_unit_n;  // n contiguous
  bool b_vec = BNM ? (rhs.cs == 1 && (rhs.rs % 2 == 0)) : (rhs.rs == 1 && (rhs.cs % 2 == 0));
  b_vec = b_vec && aligned16(rhs.ptr);
  bool VEC = a_vec && b_vec;

  // algorithmic flop count of this launch (structured operands / dst count only their kept part)
  double flops = 2.0 * (double)p.m * (double)p.n * (double)p.k;
  if (dst_struct != RECT) flops *= ((double)p.m + 1.0) / (2.0 * (double)p.m);
  if (lhs_struct != RECT) flops *= 0.5;
  if (rhs_struct != RECT) flops *= 0.5;
  const bool prof = profiling_enabled();
  // opt-in (f64_gemm_mode = 1): large unstructured products as int8-sliced wgmma products (gemm_f64_sliced.cuh)
  if (get_option(OPT_F64_GEMM_MODE) == 1 && !split_ws && dst_struct == RECT && lhs_struct == RECT && rhs_struct == RECT &&
      p.m >= 256 && p.n >= 256 && p.k >= 128 && p.k <= 32768) {
    oz::Operand a{lhs.ptr, p.m, p.k, lhs.rs, lhs.cs};
    oz::Operand b{rhs.ptr, p.k, p.n, rhs.rs, rhs.cs};
    if (prof) profile_record_start(stream);
    const bool ok = oz::gemm_f64_ozaki(stream, dst.ptr, dst.rs, dst.cs, p.m, p.n, p.k, accum, a, b, alpha, sliced_workspace(stream));
    if (prof) profile_record_stop(stream, flops);
    if (ok) {
      note_launch();
      return;
    }
    (void)cudaGetLastError();
  }
  // large rectangular-operand products: the TMA-fed warp-specialised kernel (gemm_f64_ws.cuh)
  if (ws_mode() != 0 && !split_ws) {
    // Heuristic. Triangular destinations with k <= 1024 and >= 3 waves of 128 x 128 tiles (one CTA per SM) take the wide
    // configuration: the SYRK trailing updates of LLT (at n = 16128 it beat the narrow one at k = 768 and 1024 too,
    // profiles/r08_gemm_f64_shapes.log). Other products take the narrow one when their 128 x 64 tiles fill
    // >= 3 waves of two CTAs per SM and their contraction is deep enough to amortise a tile's epilogue (k >= 512: at
    // k = 256 the cp.async kernel is faster even on a full 16384 x 16384 update, profiles/r03_gemm_f64_shapes.log); the
    // cp.async kernel (64 x 64 tiles, three CTAs per SM) keeps short contractions and products with few tiles.
    // gemm_ws = 2 forces the narrow configuration, 3 the wide one.
    const int sms = stream_sms(stream);
    const bool wide = ws_mode() == 3 ||
                      (ws_mode() == 1 && dst_struct != RECT && p.k <= 1024 &&
                       ws64::ws_tiles(p.m, p.n, dst_struct, ws64::Shape<true>::BN) >= 3ll * sms);
    long long tiles_narrow = (long long)((p.m + ws64::BM - 1) / ws64::BM) * ((p.n + ws64::Shape<false>::BN - 1) / ws64::Shape<false>::BN);
    if (dst_struct != RECT) tiles_narrow = tiles_narrow / 2 + 1;
    const bool narrow = ws_mode() == 2 || (ws_mode() == 1 && tiles_narrow >= 3 * 2ll * sms && p.k >= 512);
    if (wide || narrow) {
      if (prof) profile_record_start(stream);
      const bool took = ws64::try_gemm_f64_ws(stream, p, nullptr, wide);
      if (took) {
        if (prof) profile_record_stop(stream, flops);
        return;
      }
    }
  }
#define FB_DISPATCH(ak, bnm, vec)                                   \
  if (AK == ak && BNM == bnm && VEC == vec) {                       \
    if (prof) profile_record_start(stream);                         \
    launch_layout<ak, bnm, vec>(stream, p);                         \
    if (prof) profile_record_stop(stream, flops);                   \
    launched = true;                                                \
  }
  bool launched = false;
  FB_DISPATCH(false, false, true)
  else FB_DISPATCH(false, true, true)
  else FB_DISPATCH(true, false, true)
  else FB_DISPATCH(true, true, true)
  else FB_DISPATCH(false, false, false)
  else FB_DISPATCH(false, true, false)
  else FB_DISPATCH(true, false, false)
  else FB_DISPATCH(true, true, false)
#undef FB_DISPATCH
  FB_ASSERT(launched, "no GEMM variant matched");
  if (split_ws) {
    const long long total = (long long)dst.nrows * dst.ncols;
    splitk_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dst.ptr, dst.rs, dst.cs, (int)dst.nrows,
                                                                             (int)dst.ncols, dst_struct, accum, alpha,
                                                                             split_ws, splits);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
}

// ---- "spicy" matmul (reference faer/src/linalg/matmul/internal/mod.rs:45-379): dst[row_idx[i], col_idx[j]] (+)= alpha *
// (lhs * diag(d) * rhs)[i, j] for the (i, j) the block structure of the PRODUCT keeps; used by LDLT's trailing updates
// (cholesky/ldlt/factor.rs:447-492) and the supernodal sparse Cholesky fronts. All pointers are device pointers.
// Large TMA-readable operands: ONE launch of the warp-specialised kernel with the diagonal folded into the lhs fragments
// (prologue) and the scatter folded into the store (epilogue). Otherwise the reference's own fallback composition
// (internal/mod.rs:206-379): scale, structured product into a temporary, masked scatter.
namespace {
__global__ void scale_cols_kernel(double* __restrict__ dst, i64 ld, const double* __restrict__ src, i64 rs, i64 cs, i64 m,
                                  const double* __restrict__ d, i64 dstride) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = blockIdx.y;
  if (i < m) dst[j * ld + i] = src[i * rs + j * cs] * d[j * dstride];
}
__global__ void spicy_scatter_kernel(double* __restrict__ C, i64 rs, i64 cs, const double* __restrict__ out, i64 m, i64 n,
                                     const long long* __restrict__ ri, const long long* __restrict__ ci, int c_struct, int accum,
                                     i64 j0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = j0 + blockIdx.y;
  if (i >= m || j >= n) return;
  const bool nodiag = is_strict(c_struct) || is_unit(c_struct);
  if (is_lower(c_struct) && (i < j || (i == j && nodiag))) return;
  if (is_upper(c_struct) && (i > j || (i == j && nodiag))) return;
  double* p = C + (ri ? ri[i] : i) * rs + (ci ? ci[j] : j) * cs;
  const double v = out[j * m + i];
  *p = accum ? *p + v : v;
}
}  // namespace

void spicy_matmul_f64(cudaStream_t st, VD C, int c_struct, const long long* row_idx, const long long* col_idx, int accum, VCD A,
                      VCD B, const double* diag, i64 diag_stride, double alpha) {
  const i64 m = A.nrows, n = B.ncols, k = A.ncols;
  FB_ASSERT(B.nrows == k, "spicy_matmul shape mismatch");
  if (!row_idx) FB_ASSERT(C.nrows == m, "spicy_matmul: dst rows");
  if (!col_idx) FB_ASSERT(C.ncols == n, "spicy_matmul: dst columns");
  if (m == 0 || n == 0) return;
  if (k == 0 && accum) return;
  FB_ASSERT(m < (1ll << 31) && n < (1ll << 31) && k < (1ll << 31), "dimension too large");
  if (k > 0 && ws_mode() != 0) {
    GemmF64Params p;
    p.m = (int)m; p.n = (int)n; p.k = (int)k;
    p.A = A.ptr; p.a_rs = A.rs; p.a_cs = A.cs; p.a_struct = RECT;
    p.B = B.ptr; p.b_rs = B.rs; p.b_cs = B.cs; p.b_struct = RECT;
    p.C = C.ptr; p.c_rs = C.rs; p.c_cs = C.cs; p.c_struct = c_struct;
    p.alpha = alpha; p.accum = accum; p.k_split_len = 0; p.c_split_stride = 0;
    const long long tiles = (long long)((m + ws64::BM - 1) / ws64::BM) * ((n + ws64::Shape<false>::BN - 1) / ws64::Shape<false>::BN);
    if (ws_mode() == 2 || (tiles >= 32 && k >= 16)) {
      ws64::Spicy sp;
      sp.row_idx = row_idx; sp.col_idx = col_idx; sp.diag = diag; sp.diag_stride = diag_stride;
      if (ws64::try_gemm_f64_ws(st, p, &sp)) return;
    }
  }
  // fallback composition
  double* scaled = nullptr;
  VCD lhs = A;
  if (diag && k > 0) {
    scaled = (double*)ws_alloc((size_t)m * (size_t)k * 8);
    for (i64 c0 = 0; c0 < k; c0 += 65535) {
      const i64 nc = std::min<i64>(65535, k - c0);
      scale_cols_kernel<<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(scaled + c0 * m, m, A.ptr + c0 * A.cs, A.rs, A.cs,
                                                                                        m, diag + c0 * diag_stride, diag_stride);
      note_launch();
    }
    lhs = VCD{scaled, m, k, 1, m};
  }
  const bool gather = row_idx || col_idx;
  double* outb = gather ? (double*)ws_alloc((size_t)m * (size_t)n * 8) : nullptr;
  VD out = gather ? VD{outb, m, n, 1, m} : C;
  const int acc2 = gather ? 0 : accum;
  if (c_struct == RECT) {
    gemm_f64(st, out, RECT, acc2, lhs, RECT, B, RECT, alpha);
  } else {
    const i64 size = std::min(m, n);
    gemm_f64(st, out.sub(0, 0, size, size), c_struct, acc2, lhs.sub(0, 0, size, k), RECT, B.sub(0, 0, k, size), RECT, alpha);
    if (is_lower(c_struct) && m > n)
      gemm_f64(st, out.sub(size, 0, m - size, size), RECT, acc2, lhs.sub(size, 0, m - size, k), RECT, B.sub(0, 0, k, size), RECT, alpha);
    else if (is_upper(c_struct) && n > m)
      gemm_f64(st, out.sub(0, size, size, n - size), RECT, acc2, lhs.sub(0, 0, size, k), RECT, B.sub(0, size, k, n - size), RECT, alpha);
  }
  if (gather) {
    for (i64 c0 = 0; c0 < n; c0 += 65535) {
      const i64 nc = std::min<i64>(65535, n - c0);
      spicy_scatter_kernel<<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(C.ptr, C.rs, C.cs, outb, m, n, row_idx, col_idx,
                                                                                           c_struct, accum, c0);
      note_launch();
    }
  }
  FB_CUDA_CHECK(cudaGetLastError());
  if (outb || scaled) FB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (outb) ws_free(outb);
  if (scaled) ws_free(scaled);
}

}  // namespace fb
