// G1/G2: f64 GEMM on the native f64 tensor path (DMMA.16x8x16 / DMMA.16x8x8 via mma.sync.m16n8k16 / m16n8k8 .f64).
//
// Computes   dst(struct) = [dst +] alpha * lhs(struct) * rhs(struct)
// with faer's semantics:
//   * matmul            : faer/src/linalg/matmul/mod.rs:1617-1660 (Replace never reads dst, 1580-1582;
//                         K==0 => zero-fill on Replace, 1193-1198)
//   * triangular matmul : faer/src/linalg/matmul/triangular.rs:1193-1245, 906-977 — the excluded half of a
//                         triangular INPUT is never interpreted as data (masked on load, 26-52), the part
//                         of dst outside the selected triangle is left untouched, strict/unit dst also leaves
//                         the diagonal untouched.
//   * DstKind::Lower    : triangular.rs:641-680 (the SYRK-like trailing update of LLT).
//
// wgmma has no f64 type; this is the native f64 tensor-core roofline path.
#pragma once
#include "common.cuh"

namespace fb {

struct GemmF64Params {
  int m, n, k;
  const double* A; i64 a_rs, a_cs; int a_struct;
  const double* B; i64 b_rs, b_cs; int b_struct;
  double* C;       i64 c_rs, c_cs; int c_struct;
  double alpha;
  int accum;  // 0 = Replace, 1 = Add
  int tiles_m, tiles_n;
  // split-K (tall-skinny products, e.g. V^H V with k = 65536): blockIdx.y = z handles k in [z*len, (z+1)*len) and
  // writes its partial product to C + z * c_split_stride; a reduce kernel combines the slices deterministically.
  int k_split_len;       // 0 = no split; otherwise a multiple of the k-tile
  i64 c_split_stride;    // elements between consecutive partial slices
};

// Launch on `stream`. All pointers are device pointers. Views use element strides of any sign.
void gemm_f64(cudaStream_t stream, VD dst, int dst_struct, int accum, VCD lhs, int lhs_struct, VCD rhs, int rhs_struct,
              double alpha);

// "spicy" matmul (matmul/internal/mod.rs:45-379): dst[row_idx[i], col_idx[j]] (+)= alpha (lhs diag(d) rhs)[i, j], masked by the
// block structure of the product. row_idx / col_idx / diag: DEVICE pointers or null.
void spicy_matmul_f64(cudaStream_t st, VD dst, int dst_struct, const long long* row_idx, const long long* col_idx, int accum,
                      VCD lhs, VCD rhs, const double* diag, i64 diag_stride, double alpha);

inline void gemm_f64(cudaStream_t stream, VD dst, int accum, VCD lhs, VCD rhs, double alpha) {
  gemm_f64(stream, dst, RECT, accum, lhs, RECT, rhs, RECT, alpha);
}

}  // namespace fb
