// f32 GEMM / structured GEMM with fp32-level accuracy on the tensor pipe: error-compensated 3xTF32.
//
// Reference semantics: the same entry points as gemm_f64.cu (faer/src/linalg/matmul/mod.rs:1617-1660,
// matmul/triangular.rs:1193-1245) for T = f32.
//
// Each fp32 operand is split in registers into a_hi = tf32(a), a_lo = tf32(a - a_hi) and every product is issued as
// three tensor-core MMAs (a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, small terms first) with fp32 accumulation: the dropped
// a_lo*b_lo term is O(2^-22) relative, i.e. the result is as accurate as an fp32 FMA chain up to summation order.
// This file holds the warp-level `mma.sync.m16n8k8.tf32` kernel with the same cp.async ring / padded-tile /
// structure-mask machinery as the f64 kernel — it serves structured (triangular) operands / destinations and small
// products — and the dispatcher: large unstructured products go to the wgmma kernel (`gemm_f32_tc.cuh`: TMA operand
// staging, `wgmma.mma_async` tf32, register accumulators).
#include <cstdlib>

#include "gemm_f32.cuh"
#include "gemm_f32_tc.cuh"
#include "runtime.cuh"

namespace fb {

namespace {

constexpr int F_WARPS_M = 2, F_WARPS_N = 2, F_WMI = 2, F_WNI = 4, F_BK = 16, F_STAGES = 3;
constexpr int F_BM = F_WARPS_M * F_WMI * 16;  // 64
constexpr int F_BN = F_WARPS_N * F_WNI * 8;   // 64
constexpr int F_THREADS = F_WARPS_M * F_WARPS_N * 32;

// KMAJOR: smem[mn][k], ld = BK + 4 (g*ld + t hits 32 distinct 4-byte banks); else smem[k][mn], ld = ROWS + 8.
template <int ROWS, bool KMAJOR>
struct FTile {
  static constexpr int LD = KMAJOR ? F_BK + 4 : ROWS + 8;
  static constexpr int SIZE = KMAJOR ? ROWS * LD : F_BK * LD;
  __device__ static __forceinline__ int idx(int mn, int kk) { return KMAJOR ? mn * LD + kk : kk * LD + mn; }
};

template <int ROWS, bool KMAJOR, bool VEC>
__device__ __forceinline__ void f_load_tile(float* __restrict__ s, const float* __restrict__ g, i64 s_mn, i64 s_k, int mn0,
                                            int k0, int MN, int K, int tid) {
  using T = FTile<ROWS, KMAJOR>;
  if constexpr (VEC) {
    constexpr int CHUNKS = ROWS * F_BK / 4;
    static_assert(CHUNKS % F_THREADS == 0, "tile/threads mismatch");
#pragma unroll
    for (int it = 0; it < CHUNKS / F_THREADS; ++it) {
      const int c = it * F_THREADS + tid;
      int mn, kk, nvalid;
      const float* src;
      if constexpr (KMAJOR) {
        mn = c / (F_BK / 4);
        kk = (c % (F_BK / 4)) * 4;
        const int rem = K - (k0 + kk);
        nvalid = (mn0 + mn < MN) ? (rem < 0 ? 0 : (rem > 4 ? 4 : rem)) : 0;
        src = g + (i64)(mn0 + mn) * s_mn + (i64)(k0 + kk);
      } else {
        kk = c / (ROWS / 4);
        mn = (c % (ROWS / 4)) * 4;
        const int rem = MN - (mn0 + mn);
        nvalid = (k0 + kk < K) ? (rem < 0 ? 0 : (rem > 4 ? 4 : rem)) : 0;
        src = g + (i64)(mn0 + mn) + (i64)(k0 + kk) * s_k;
      }
      if (nvalid == 0) src = g;
      cp_async_16(s + T::idx(mn, kk), src, nvalid * 4);
    }
  } else {
    constexpr int ELEMS = ROWS * F_BK;
    static_assert(ELEMS % F_THREADS == 0, "tile/threads mismatch");
#pragma unroll
    for (int it = 0; it < ELEMS / F_THREADS; ++it) {
      const int e = it * F_THREADS + tid;
      int mn, kk;
      if constexpr (KMAJOR) {
        mn = e / F_BK;
        kk = e % F_BK;
      } else {
        kk = e / ROWS;
        mn = e % ROWS;
      }
      const bool ok = (mn0 + mn < MN) && (k0 + kk < K);
      const float* src = ok ? g + (i64)(mn0 + mn) * s_mn + (i64)(k0 + kk) * s_k : g;
      cp_async_4(s + T::idx(mn, kk), src, ok ? 4 : 0);
    }
  }
}

template <int ROWS, bool KMAJOR>
__device__ __forceinline__ void f_fixup_tile(float* s, int structure, bool is_rhs, int mn0, int k0, int tid) {
  using T = FTile<ROWS, KMAJOR>;
  const bool lower = is_lower(structure);
  const float diagval = is_unit(structure) ? 1.0f : 0.0f;
  const bool keepdiag = !(is_unit(structure) || is_strict(structure));
  for (int e = tid; e < ROWS * F_BK; e += F_THREADS) {
    const int mn = e % ROWS, kk = e / ROWS;
    int rel = is_rhs ? (k0 + kk) - (mn0 + mn) : (mn0 + mn) - (k0 + kk);
    if (!lower) rel = -rel;
    if (rel < 0) s[T::idx(mn, kk)] = 0.0f;
    else if (rel == 0 && !keepdiag) s[T::idx(mn, kk)] = diagval;
  }
}

__device__ __forceinline__ bool f_needs_fixup(int structure, bool is_rhs, int mn0, int rows, int k0, int bk) {
  if (structure == RECT) return false;
  int lo, hi;
  if (!is_rhs) {
    lo = mn0 - (k0 + bk - 1);
    hi = (mn0 + rows - 1) - k0;
  } else {
    lo = k0 - (mn0 + rows - 1);
    hi = (k0 + bk - 1) - mn0;
  }
  if (!is_lower(structure)) lo = -hi;
  return lo <= 0;
}

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}

// D(16x8, f32) += A(16x8, tf32, row) * B(8x8, tf32, col)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <bool AK, bool BNM, bool VEC>
__global__ void __launch_bounds__(F_THREADS) gemm_f32_kernel(const GemmF32Params p) {
  using TA = FTile<F_BM, AK>;
  using TB = FTile<F_BN, !BNM>;
  extern __shared__ __align__(16) float fsmem[];
  float* As = fsmem;
  float* Bs = fsmem + F_STAGES * TA::SIZE;

  constexpr int GROUP = 8;
  const int bid = blockIdx.x;
  const int width = GROUP * p.tiles_n;
  const int first_m = (bid / width) * GROUP;
  const int gsize = min(p.tiles_m - first_m, GROUP);
  const int tm = first_m + (bid % width) % gsize;
  const int tn = (bid % width) / gsize;
  const int m0 = tm * F_BM, n0 = tn * F_BN;

  const int cs_ = p.c_struct;
  if (is_lower(cs_)) {
    if (m0 + F_BM - 1 < n0) return;
  } else if (is_upper(cs_)) {
    if (n0 + F_BN - 1 < m0) return;
  }
  int k_begin = 0, k_end = p.k;
  if (is_lower(p.a_struct)) k_end = min(k_end, m0 + F_BM);
  if (is_upper(p.a_struct)) k_begin = max(k_begin, m0);
  if (is_lower(p.b_struct)) k_begin = max(k_begin, n0);
  if (is_upper(p.b_struct)) k_end = min(k_end, n0 + F_BN);
  float* __restrict__ Cout = p.C;
  if (p.k_split_len > 0) {
    const int kb = (int)blockIdx.y * p.k_split_len;
    k_begin = max(k_begin, kb);
    k_end = min(k_end, kb + p.k_split_len);
    Cout += (i64)blockIdx.y * p.c_split_stride;
  }
  k_begin = (k_begin / F_BK) * F_BK;
  const int nkt = k_end > k_begin ? (k_end - k_begin + F_BK - 1) / F_BK : 0;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm0 = (warp % F_WARPS_M) * (F_WMI * 16);
  const int wn0 = (warp / F_WARPS_M) * (F_WNI * 8);

  float acc[F_WMI][F_WNI][4];
#pragma unroll
  for (int i = 0; i < F_WMI; ++i)
#pragma unroll
    for (int j = 0; j < F_WNI; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0f;

  auto load_stage = [&](int stage, int kt) {
    const int k0 = k_begin + kt * F_BK;
    f_load_tile<F_BM, AK, VEC>(As + stage * TA::SIZE, p.A, p.a_rs, p.a_cs, m0, k0, p.m, p.k, tid);
    f_load_tile<F_BN, !BNM, VEC>(Bs + stage * TB::SIZE, p.B, p.b_cs, p.b_rs, n0, k0, p.n, p.k, tid);
  };
#pragma unroll
  for (int s = 0; s < F_STAGES - 1; ++s) {
    if (s < nkt) load_stage(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<F_STAGES - 2>();
    __syncthreads();
    const int stage = kt % F_STAGES;
    float* a_s = As + stage * TA::SIZE;
    float* b_s = Bs + stage * TB::SIZE;
    {
      const int k0 = k_begin + kt * F_BK;
      const bool fa = f_needs_fixup(p.a_struct, false, m0, F_BM, k0, F_BK);
      const bool fb_ = f_needs_fixup(p.b_struct, true, n0, F_BN, k0, F_BK);
      if (fa || fb_) {
        if (fa) f_fixup_tile<F_BM, AK>(a_s, p.a_struct, false, m0, k0, tid);
        if (fb_) f_fixup_tile<F_BN, !BNM>(b_s, p.b_struct, true, n0, k0, tid);
        __syncthreads();
      }
    }
    {
      const int nk = kt + F_STAGES - 1;
      if (nk < nkt) load_stage(nk % F_STAGES, nk);
      cp_async_commit();
    }
#pragma unroll
    for (int kk = 0; kk < F_BK; kk += 8) {
      uint32_t ah[F_WMI][4], al[F_WMI][4], bh[F_WNI][2], bl[F_WNI][2];
#pragma unroll
      for (int i = 0; i < F_WMI; ++i) {
        const int r = wm0 + i * 16 + g;
        split_tf32(a_s[TA::idx(r, kk + t)], ah[i][0], al[i][0]);
        split_tf32(a_s[TA::idx(r + 8, kk + t)], ah[i][1], al[i][1]);
        split_tf32(a_s[TA::idx(r, kk + t + 4)], ah[i][2], al[i][2]);
        split_tf32(a_s[TA::idx(r + 8, kk + t + 4)], ah[i][3], al[i][3]);
      }
#pragma unroll
      for (int j = 0; j < F_WNI; ++j) {
        const int c = wn0 + j * 8 + g;
        split_tf32(b_s[TB::idx(c, kk + t)], bh[j][0], bl[j][0]);
        split_tf32(b_s[TB::idx(c, kk + t + 4)], bh[j][1], bl[j][1]);
      }
#pragma unroll
      for (int i = 0; i < F_WMI; ++i)
#pragma unroll
        for (int j = 0; j < F_WNI; ++j) {
          mma_tf32(acc[i][j], al[i], bh[j]);
          mma_tf32(acc[i][j], ah[i], bl[j]);
          mma_tf32(acc[i][j], ah[i], bh[j]);
        }
    }
  }
  cp_async_wait<0>();

  const bool c_low = is_lower(cs_), c_up = is_upper(cs_);
  const bool c_nodiag = is_strict(cs_) || is_unit(cs_);
  const float alpha = p.alpha;
  const bool add = p.accum != 0;
#pragma unroll
  for (int i = 0; i < F_WMI; ++i) {
    float cv[F_WNI][4];
    bool ok[F_WNI][4];
#pragma unroll
    for (int j = 0; j < F_WNI; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = m0 + wm0 + i * 16 + g + (e >= 2 ? 8 : 0);
        const int col = n0 + wn0 + j * 8 + 2 * t + (e & 1);
        bool v = row < p.m && col < p.n;
        if (c_low && (row < col || (row == col && c_nodiag))) v = false;
        if (c_up && (row > col || (row == col && c_nodiag))) v = false;
        ok[j][e] = v;
        cv[j][e] = (add && v) ? Cout[(i64)row * p.c_rs + (i64)col * p.c_cs] : 0.0f;
      }
#pragma unroll
    for (int j = 0; j < F_WNI; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = m0 + wm0 + i * 16 + g + (e >= 2 ? 8 : 0);
        const int col = n0 + wn0 + j * 8 + 2 * t + (e & 1);
        if (ok[j][e]) Cout[(i64)row * p.c_rs + (i64)col * p.c_cs] = alpha * acc[i][j][e] + cv[j][e];
      }
  }
}

template <bool AK, bool BNM>
constexpr size_t f_smem_bytes() {
  return sizeof(float) * F_STAGES * (FTile<F_BM, AK>::SIZE + FTile<F_BN, !BNM>::SIZE);
}

template <bool AK, bool BNM, bool VEC>
void f_launch(cudaStream_t stream, GemmF32Params& p) {
  p.tiles_m = (p.m + F_BM - 1) / F_BM;
  p.tiles_n = (p.n + F_BN - 1) / F_BN;
  constexpr size_t smem = f_smem_bytes<AK, BNM>();
  static bool configured = false;
  if (!configured) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(gemm_f32_kernel<AK, BNM, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  const unsigned splits = p.k_split_len > 0 ? (unsigned)((p.k + p.k_split_len - 1) / p.k_split_len) : 1u;
  gemm_f32_kernel<AK, BNM, VEC><<<dim3((unsigned)((long long)p.tiles_m * p.tiles_n), splits), F_THREADS, smem, stream>>>(p);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

inline int f_transpose_struct(int s) {
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
inline bool f_aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }

// split-K partial buffer of the mma.sync kernel: per-stream grow-only scratch (runtime.cu)
float* f32_split_workspace(cudaStream_t stream, size_t bytes) { return (float*)stream_scratch(stream, bytes); }

// per-stream packing workspace of the wgmma path (grow-only device buffers; work on one stream is ordered, so a stream's
// buffer can be reused call after call)
tc::Workspace* f32_tc_workspace(cudaStream_t stream) {
  struct Slot {
    cudaStream_t st;
    tc::Workspace ws;
    bool used;
  };
  static Slot slots[16];
  for (auto& s : slots)
    if (s.used && s.st == stream) return &s.ws;
  for (auto& s : slots)
    if (!s.used) {
      s.used = true;
      s.st = stream;
      return &s.ws;
    }
  // more than 16 distinct streams: recycle slot 0 after draining it
  cudaStreamSynchronize(slots[0].st);
  slots[0].st = stream;
  return &slots[0].ws;
}

// dst(struct) = [dst +] alpha * sum_z W_z (partial products summed in z order, in double to keep fp32-level accuracy)
__global__ void f_splitk_reduce_kernel(float* __restrict__ C, i64 rs, i64 cs, int m, int n, int c_struct, int accum,
                                       float alpha, const float* __restrict__ W, int splits) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)m * n) return;
  const int row = (int)(e % m), col = (int)(e / m);
  const bool nodiag = is_strict(c_struct) || is_unit(c_struct);
  if (is_lower(c_struct) && (row < col || (row == col && nodiag))) return;
  if (is_upper(c_struct) && (row > col || (row == col && nodiag))) return;
  double s = 0.0;
  for (int z = 0; z < splits; ++z) s += (double)W[(long long)z * m * n + e];
  float* cp = C + (i64)row * rs + (i64)col * cs;
  const float v = alpha * (float)s;
  *cp = accum ? (*cp + v) : v;
}

}  // namespace

void gemm_f32(cudaStream_t stream, VF dst, int dst_struct, int accum, VCF lhs, int lhs_struct, VCF rhs, int rhs_struct,
              float alpha) {
  FB_ASSERT(dst.nrows == lhs.nrows && dst.ncols == rhs.ncols && lhs.ncols == rhs.nrows, "matmul shape mismatch");
  if (dst_struct != RECT) FB_ASSERT(dst.nrows == dst.ncols, "triangular dst must be square");
  if (lhs_struct != RECT) FB_ASSERT(lhs.nrows == lhs.ncols, "triangular lhs must be square");
  if (rhs_struct != RECT) FB_ASSERT(rhs.nrows == rhs.ncols, "triangular rhs must be square");
  if (dst.nrows == 0 || dst.ncols == 0) return;
  if (lhs.ncols == 0 && accum != 0) return;
  FB_ASSERT(dst.nrows < (1ll << 31) && dst.ncols < (1ll << 31) && lhs.ncols < (1ll << 31), "dimension too large");
  if (dst.rs != 1 && dst.cs == 1) {
    VF d2 = dst.t();
    VCF l2 = rhs.t(), r2 = lhs.t();
    const int ls = f_transpose_struct(rhs_struct), rs_ = f_transpose_struct(lhs_struct);
    dst = d2; lhs = l2; rhs = r2;
    dst_struct = f_transpose_struct(dst_struct);
    lhs_struct = ls; rhs_struct = rs_;
  }
  // Large unstructured products go to the wgmma kernel (gemm_f32_tc.cuh: TMA + mbarrier pipeline, 3xTF32 on the Hopper
  // tensor cores). Structured operands / destinations and small products stay on the mma.sync kernel.
  if (dst_struct == RECT && lhs_struct == RECT && rhs_struct == RECT && dst.nrows >= 64 &&
      dst.ncols >= 64 && lhs.ncols >= 32 && 2.0 * (double)dst.nrows * (double)dst.ncols * (double)lhs.ncols >= 2.5e8) {
    tc::Operand a{lhs.ptr, (int)lhs.nrows, (int)lhs.ncols, lhs.rs, lhs.cs};
    tc::Operand b{rhs.ptr, (int)rhs.nrows, (int)rhs.ncols, rhs.rs, rhs.cs};
    const bool prof_tc = profiling_enabled();
    if (prof_tc) profile_record_start(stream);
    const bool ok = tc::gemm_f32_tc(stream, dst.ptr, dst.rs, dst.cs, (int)dst.nrows, (int)dst.ncols, (int)lhs.ncols, accum, a, b,
                                    alpha, f32_tc_workspace(stream));
    if (prof_tc) profile_record_stop(stream, 2.0 * (double)dst.nrows * (double)dst.ncols * (double)lhs.ncols);
    if (ok) {
      note_launch();
      return;
    }
    (void)cudaGetLastError();
  }
  GemmF32Params p;
  p.m = (int)dst.nrows; p.n = (int)dst.ncols; p.k = (int)lhs.ncols;
  p.A = lhs.ptr; p.a_rs = lhs.rs; p.a_cs = lhs.cs; p.a_struct = lhs_struct;
  p.B = rhs.ptr; p.b_rs = rhs.rs; p.b_cs = rhs.cs; p.b_struct = rhs_struct;
  p.C = dst.ptr; p.c_rs = dst.rs; p.c_cs = dst.cs; p.c_struct = dst_struct;
  p.alpha = alpha; p.accum = accum;
  p.k_split_len = 0; p.c_split_stride = 0;
  // split-K for tall-skinny products (see gemm_f64.cu)
  float* split_ws = nullptr;
  int splits = 1;
  {
    const long long tiles = (long long)((p.m + F_BM - 1) / F_BM) * ((p.n + F_BN - 1) / F_BN);
    const int sms = stream_sms(stream);
    if (tiles < sms && p.k >= 4096 && lhs_struct == RECT && rhs_struct == RECT) {
      splits = (int)std::min<long long>((sms * 4ll + tiles - 1) / tiles, p.k / 1024);
      if (splits >= 2) {
        int len = (p.k + splits - 1) / splits;
        len = (len + 63) / 64 * 64;
        splits = (p.k + len - 1) / len;
        // per-stream grow-only buffer (no host synchronisation on the steady state: work on a stream is ordered)
        split_ws = f32_split_workspace(stream, (size_t)splits * p.m * p.n * sizeof(float));
        p.k_split_len = len;
        p.c_split_stride = (i64)p.m * p.n;
        p.C = split_ws; p.c_rs = 1; p.c_cs = p.m; p.c_struct = RECT;
        p.alpha = 1.0f; p.accum = 0;
      } else {
        splits = 1;
      }
    }
  }
  const bool a_unit_m = (lhs.rs == 1) || lhs.nrows == 1;
  const bool a_unit_k = (lhs.cs == 1) || lhs.ncols == 1;
  const bool AK = !a_unit_m && a_unit_k;
  bool a_vec = AK ? (lhs.cs == 1 && (lhs.rs % 4 == 0)) : (lhs.rs == 1 && (lhs.cs % 4 == 0));
  a_vec = a_vec && f_aligned16(lhs.ptr);
  const bool b_unit_k = (rhs.rs == 1) || rhs.nrows == 1;
  const bool b_unit_n = (rhs.cs == 1) || rhs.ncols == 1;
  const bool BNM = !b_unit_k && b_unit_n;
  bool b_vec = BNM ? (rhs.cs == 1 && (rhs.rs % 4 == 0)) : (rhs.rs == 1 && (rhs.cs % 4 == 0));
  b_vec = b_vec && f_aligned16(rhs.ptr);
  const bool VEC = a_vec && b_vec;
  double flops = 2.0 * (double)p.m * (double)p.n * (double)p.k;
  if (dst_struct != RECT) flops *= ((double)p.m + 1.0) / (2.0 * (double)p.m);
  if (lhs_struct != RECT) flops *= 0.5;
  if (rhs_struct != RECT) flops *= 0.5;
  const bool prof = profiling_enabled();
#define FB_FDISPATCH(ak, bnm, vec)                    \
  if (AK == ak && BNM == bnm && VEC == vec) {         \
    if (prof) profile_record_start(stream);           \
    f_launch<ak, bnm, vec>(stream, p);                \
    if (prof) profile_record_stop(stream, flops);     \
    launched = true;                                  \
  }
  bool launched = false;
  FB_FDISPATCH(false, false, true)
  else FB_FDISPATCH(false, true, true)
  else FB_FDISPATCH(true, false, true)
  else FB_FDISPATCH(true, true, true)
  else FB_FDISPATCH(false, false, false)
  else FB_FDISPATCH(false, true, false)
  else FB_FDISPATCH(true, false, false)
  else FB_FDISPATCH(true, true, false)
#undef FB_FDISPATCH
  FB_ASSERT(launched, "no GEMM variant matched");
  if (split_ws) {
    const long long total = (long long)dst.nrows * dst.ncols;
    f_splitk_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dst.ptr, dst.rs, dst.cs, (int)dst.nrows,
                                                                               (int)dst.ncols, dst_struct, accum, alpha,
                                                                               split_ws, splits);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
}

}  // namespace fb
