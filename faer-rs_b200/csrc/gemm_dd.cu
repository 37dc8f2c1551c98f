// Double-double GEMM / structured GEMM on the CUDA cores (fx128 and cx128): dst = [dst +] alpha * op(lhs) * op(rhs), with the
// structure codes of faer-ffi's `Block` for all three operands (the semantics of matmul/triangular.rs as the other GEMMs of this
// library implement them: the half of a structured operand outside its triangle reads as 0, its diagonal as 0 (strict) or 1
// (unit); only the part of dst its structure selects is written, without the diagonal for a strict or unit dst).
//
// One CTA of 256 threads computes a BM x BN tile, each thread an RM x RN grid of entries 16 rows / 16 columns apart, from BK-deep
// slices of both operands staged in shared memory. Every product is accumulated with faer's own mul_add for the scalar
// (add(mul(a, b), acc), dd.cuh): 20 FP64 instructions per real multiply-add, no lazy renormalisation, so each entry carries
// the accuracy of faer's scalar loop (the summation order is ours, as for f64: DESIGN.md §3).
//
// cx128 runs a fused complex kernel rather than 4M on the real one. 4M would need planar copies of both operands and four real
// passes whose partial sums are combined by extra dd additions; the fused kernel applies faer's complex mul_add to each term, reads
// each operand once, and has the same FP64 instruction count per real multiply-add.
//
// Tiles that lie entirely outside dst's triangle are not launched work (the CTA returns), and the k range of a tile is cut to the
// part where a triangular lhs / rhs can be nonzero.
#include <type_traits>

#include "common.cuh"
#include "dd.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

constexpr int GD_THREADS = 256;

template <bool CX>
struct GdShape;
template <>
struct GdShape<false> {
  static constexpr int RM = 4, RN = 4, BK = 16;
};
template <>
struct GdShape<true> {
  static constexpr int RM = 4, RN = 2, BK = 8;
};

// element (i, j) of a structured operand, conjugated if asked; 0 outside the matrix
template <bool CX>
__device__ __forceinline__ cdd gd_load(const dd* p, i64 rs, i64 cs, i64 nr, i64 nc, i64 i, i64 j, int s, bool conj) {
  const cdd zero{dd(0.0), dd(0.0)};
  if (i >= nr || j >= nc) return zero;
  if (s != RECT) {
    if (i == j) {
      if (is_unit(s)) return cdd{dd(1.0), dd(0.0)};
      if (is_strict(s)) return zero;
    } else if (is_lower(s) ? i < j : i > j) {
      return zero;
    }
  }
  const dd* q = p + (CX ? 2 : 1) * (i * rs + j * cs);
  cdd v;
  v.re = q[0];
  if (CX) v.im = conj ? -q[1] : q[1];
  else v.im = dd(0.0);
  return v;
}

__device__ __forceinline__ void gd_put(dd& s, cdd v) { s = v.re; }
__device__ __forceinline__ void gd_put(cdd& s, cdd v) { s = v; }
__device__ __forceinline__ cdd gd_get(const dd& s) { return cdd{s, dd(0.0)}; }
__device__ __forceinline__ cdd gd_get(const cdd& s) { return s; }

template <bool CX>
__device__ __forceinline__ cdd gd_mul_add(cdd a, cdd b, cdd acc) {
  if (!CX) return cdd{a.re * b.re + acc.re, acc.im};
  return a * b + acc;
}

template <bool CX>
__global__ void __launch_bounds__(GD_THREADS) gemm_dd_kernel(View<dd> dst, int ds, int accum, View<const dd> lhs, int ls, bool conj_lhs,
                                                            View<const dd> rhs, int rsu, bool conj_rhs, cdd alpha) {
  typedef GdShape<CX> S;
  constexpr int RM = S::RM, RN = S::RN, BK = S::BK, BM = 16 * RM, BN = 16 * RN;
  // real operands are staged as dd, complex ones as cdd
  typedef std::conditional_t<CX, cdd, dd> E;
  __shared__ E As[BK][BM];
  __shared__ E Bs[BK][BN];
  const i64 m = dst.nrows, n = dst.ncols, K = lhs.ncols;
  const i64 m0 = (i64)blockIdx.y * BM, n0 = (i64)blockIdx.x * BN;
  if (is_lower(ds) && m0 + BM - 1 < n0) return;  // tile strictly above a lower dst's diagonal
  if (is_upper(ds) && m0 > n0 + BN - 1) return;  // tile strictly below an upper dst's diagonal
  i64 kb = 0, ke = K;
  if (is_lower(ls)) ke = min(ke, m0 + BM);  // lhs(i, k) = 0 for k > i
  if (is_upper(ls)) kb = max(kb, m0);       // lhs(i, k) = 0 for k < i
  if (is_lower(rsu)) kb = max(kb, n0);      // rhs(k, j) = 0 for k < j
  if (is_upper(rsu)) ke = min(ke, n0 + BN);  // rhs(k, j) = 0 for k > j
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  cdd acc[RM][RN];
#pragma unroll
  for (int a = 0; a < RM; ++a)
#pragma unroll
    for (int b = 0; b < RN; ++b) acc[a][b] = cdd{dd(0.0), dd(0.0)};

  for (i64 k0 = kb; k0 < ke; k0 += BK) {
    for (int e = tid; e < BM * BK; e += GD_THREADS) {
      const int r = e % BM, k = e / BM;
      const cdd v = k0 + k < ke ? gd_load<CX>(lhs.ptr, lhs.rs, lhs.cs, m, K, m0 + r, k0 + k, ls, conj_lhs) : cdd{dd(0.0), dd(0.0)};
      gd_put(As[k][r], v);
    }
    for (int e = tid; e < BK * BN; e += GD_THREADS) {
      const int k = e % BK, c = e / BK;
      const cdd v = k0 + k < ke ? gd_load<CX>(rhs.ptr, rhs.rs, rhs.cs, K, n, k0 + k, n0 + c, rsu, conj_rhs) : cdd{dd(0.0), dd(0.0)};
      gd_put(Bs[k][c], v);
    }
    __syncthreads();
#pragma unroll 2
    for (int k = 0; k < BK; ++k) {
      cdd av[RM], bv[RN];
#pragma unroll
      for (int a = 0; a < RM; ++a) av[a] = gd_get(As[k][ty + 16 * a]);
#pragma unroll
      for (int b = 0; b < RN; ++b) bv[b] = gd_get(Bs[k][tx + 16 * b]);
#pragma unroll
      for (int a = 0; a < RM; ++a)
#pragma unroll
        for (int b = 0; b < RN; ++b) acc[a][b] = gd_mul_add<CX>(av[a], bv[b], acc[a][b]);
    }
    __syncthreads();
  }

  const bool diag_too = !(is_strict(ds) || is_unit(ds));
#pragma unroll
  for (int a = 0; a < RM; ++a) {
#pragma unroll
    for (int b = 0; b < RN; ++b) {
      const i64 i = m0 + ty + 16 * a, j = n0 + tx + 16 * b;
      if (i >= m || j >= n) continue;
      if (is_lower(ds) && (i < j || (i == j && !diag_too))) continue;
      if (is_upper(ds) && (i > j || (i == j && !diag_too))) continue;
      dd* q = dst.ptr + (CX ? 2 : 1) * (i * dst.rs + j * dst.cs);
      if (!CX) {
        dd v = alpha.re * acc[a][b].re;
        if (accum) v = q[0] + v;
        q[0] = v;
      } else {
        cdd v = alpha * acc[a][b];
        if (accum) v = cdd{q[0], q[1]} + v;
        q[0] = v.re;
        q[1] = v.im;
      }
    }
  }
}

template <bool CX>
void gemm_dd_launch(cudaStream_t st, View<dd> dst, int ds, int accum, View<const dd> lhs, int ls, bool conj_lhs, View<const dd> rhs,
                    int rs, bool conj_rhs, cdd alpha) {
  typedef GdShape<CX> S;
  const i64 m = dst.nrows, n = dst.ncols;
  if (m == 0 || n == 0) return;
  const i64 gy = (m + 16 * S::RM - 1) / (16 * S::RM), gx = (n + 16 * S::RN - 1) / (16 * S::RN);
  FB_ASSERT(gy <= 65535 && gx <= 0x7fffffff, "double-double GEMM: too many rows");
  gemm_dd_kernel<CX><<<dim3((unsigned)gx, (unsigned)gy), GD_THREADS, 0, st>>>(dst, ds, accum, lhs, ls, conj_lhs, rhs, rs, conj_rhs,
                                                                              alpha);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

}  // namespace

void gemm_dd(cudaStream_t st, View<dd> dst, int ds, int accum, View<const dd> lhs, int ls, bool conj_lhs, View<const dd> rhs, int rs,
             bool conj_rhs, bool cx, dd alpha_re, dd alpha_im) {
  FB_ASSERT(dst.nrows == lhs.nrows && dst.ncols == rhs.ncols && lhs.ncols == rhs.nrows, "matmul shape mismatch");
  if (cx) gemm_dd_launch<true>(st, dst, ds, accum, lhs, ls, conj_lhs, rhs, rs, conj_rhs, cdd{alpha_re, alpha_im});
  else gemm_dd_launch<false>(st, dst, ds, accum, lhs, ls, false, rhs, rs, false, cdd{alpha_re, dd(0.0)});
}

}  // namespace fb
