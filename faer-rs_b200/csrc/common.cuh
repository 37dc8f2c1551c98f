// Shared device/host helpers for the H100 (sm_90a) dense backend.
//
// Views mirror faer's five-field strided matrix view
// (reference: faer/src/mat/mod.rs:7-13, faer-ffi/src/lib.rs:12-29): a pointer plus
// nrows/ncols and row/col strides counted in ELEMENTS (any sign).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

namespace fb {

typedef long long i64;

// Block structure of an operand; numeric values follow faer-ffi's `Block` enum
// (reference: faer-ffi/src/lib.rs:86-97), NOT Rust's BlockStructure order.
enum Structure : int {
  RECT = 0,
  TRI_LOWER = 1,
  TRI_UPPER = 2,
  STRICT_LOWER = 3,
  STRICT_UPPER = 4,
  UNIT_LOWER = 5,
  UNIT_UPPER = 6,
};

__host__ __device__ inline bool is_lower(int s) { return s == TRI_LOWER || s == STRICT_LOWER || s == UNIT_LOWER; }
__host__ __device__ inline bool is_upper(int s) { return s == TRI_UPPER || s == STRICT_UPPER || s == UNIT_UPPER; }
__host__ __device__ inline bool is_strict(int s) { return s == STRICT_LOWER || s == STRICT_UPPER; }
__host__ __device__ inline bool is_unit(int s) { return s == UNIT_LOWER || s == UNIT_UPPER; }

template <class T>
struct View {
  T* ptr;
  i64 nrows, ncols;
  i64 rs, cs;
  __host__ __device__ T* at(i64 i, i64 j) const { return ptr + i * rs + j * cs; }
  __host__ __device__ View sub(i64 i, i64 j, i64 m, i64 n) const { return View{ptr + i * rs + j * cs, m, n, rs, cs}; }
  __host__ __device__ View t() const { return View{ptr, ncols, nrows, cs, rs}; }
  // reverse_rows_and_cols (reference: triangular_solve.rs:577-604)
  __host__ __device__ View rev_rows_cols() const {
    return View{ptr + (nrows - 1) * rs + (ncols - 1) * cs, nrows, ncols, -rs, -cs};
  }
  __host__ __device__ View rev_rows() const { return View{ptr + (nrows - 1) * rs, nrows, ncols, -rs, cs}; }
  template <class U>
  __host__ __device__ View<U> as() const { return View<U>{(U*)ptr, nrows, ncols, rs, cs}; }
};
typedef View<double> VD;
typedef View<const double> VCD;

inline VCD cv(const VD& v) { return VCD{v.ptr, v.nrows, v.ncols, v.rs, v.cs}; }

#define FB_CUDA_CHECK(x)                                                                   \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      fprintf(stderr, "faer_b200: CUDA error %s at %s:%d: %s\n", cudaGetErrorName(e_), __FILE__, __LINE__, \
              cudaGetErrorString(e_));                                                     \
      abort();                                                                             \
    }                                                                                      \
  } while (0)

// Precondition violations abort (faer panics inside extern "C" => process abort;
// reference: faer/src/linalg/matmul/mod.rs:1562-1575).
#define FB_ASSERT(cond, msg)                                                       \
  do {                                                                             \
    if (!(cond)) {                                                                 \
      fprintf(stderr, "faer_b200: assertion failed: %s (%s) at %s:%d\n", #cond, msg, __FILE__, __LINE__); \
      abort();                                                                     \
    }                                                                              \
  } while (0)

// every kernel launch of this library is counted (bench.py reports it as gpu_launches). While a launch log is open
// (faer_b200_launch_log_begin / _end), each counted launch also records the phase tag current when it was issued, so that a
// profiler trace of the same launches can be split by phase (tools/time_fx128_qr.py).
extern unsigned long long g_launch_count;
extern int g_launch_tag;
extern signed char* g_launch_log;
extern size_t g_launch_log_len, g_launch_log_cap;
inline void note_launch() {
  ++g_launch_count;
  if (g_launch_log) {
    if (g_launch_log_len < g_launch_log_cap) g_launch_log[g_launch_log_len] = (signed char)g_launch_tag;
    ++g_launch_log_len;
  }
}
enum LaunchPhase { LAUNCH_OTHER = 0, LAUNCH_PANEL = 1, LAUNCH_PRODUCT = 2, LAUNCH_TBUILD = 3, LAUNCH_SOLVE = 4 };
// the phase of the launches issued while it is alive
struct LaunchTag {
  int prev;
  explicit LaunchTag(LaunchPhase t) : prev(g_launch_tag) { g_launch_tag = t; }
  ~LaunchTag() { g_launch_tag = prev; }
};

// ---- PTX helpers (device compilation only; the host build of the flat-map drivers, tools/emul/drivers_host.cpp, includes this
// header through a plain C++ compiler) -----------------------------------------------------------
#if defined(__CUDACC__)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// cp.async with zero-fill: copies `src_bytes` (<= CP) bytes and zero-fills the rest.
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_8(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// The widest f64 tensor-core op of sm_90: one SASS DMMA.16x8x16, 8x the work of the m8n8k4 shape per instruction
// (which cannot keep the H100's f64 tensor pipe full, profiles/r03_f64_peaks.log).
// Fragment layout (PTX ISA, mma.m16n8k16 f64): g = lane>>2, t = lane&3:
//   a[v] = A[g + 8 (v & 1)][t + 4 (v >> 1)]   (16x16, row), v = 0..7
//   b[i] = B[t + 4 i][g]                      (16x8, col),  i = 0..3
//   c0 = C[g][2t], c1 = C[g][2t+1], c2 = C[g+8][2t], c3 = C[g+8][2t+1]
// Any bijection of the 16 k indices is allowed as long as A and B use the same one (the product is a sum over k).
__device__ __forceinline__ void dmma16816(double& c0, double& c1, double& c2, double& c3, const double (&a)[8],
                                          const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
      "{%0,%1,%2,%3};\n"
      : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}
// The same layout truncated to k = 8 (a[0..3], b[0..1]; one SASS DMMA.16x8x8): half the fragment registers per instruction.
__device__ __forceinline__ void dmma1688(double& c0, double& c1, double& c2, double& c3, const double (&a)[4],
                                         const double (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
#endif  // __CUDACC__

}  // namespace fb
