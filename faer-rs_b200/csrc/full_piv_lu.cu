// Full-pivoting LU (faer's `lu::full_pivoting`) for f64 / f32 / c64 / c32: factor, solves, reconstruct, inverse, and their C ABI
// (include/faer_b200_full_piv_lu.h, included by include/faer_b200.h: `libfaer_v0_23_full_piv_lu_*`).
//
// Reference: faer/src/linalg/lu/full_pivoting/factor.rs:321-538 (factor), solve.rs:21-93, reconstruct.rs:13-82, inverse.rs:12-63.
// The factorization follows the reference's operation sequence on the working matrix X:
//   * X = A when |row_stride| < |col_stride| (the multipliers of column k are scaled), otherwise X = A^T (row k of X is scaled;
//     X's row transpositions are A's column transpositions), factor.rs:492-510;
//   * (r, c, s) = the first maximum of abs1 over X in X's column-major order, strict `>` from 0 (best_in_matrix_fallback,
//     factor.rs:255-273: a 0 or NaN entry is never chosen). The reference's SIMD search may pick another of several EXACTLY
//     equal maxima; this is the documented deviation of DESIGN.md §3;
//   * per step k: exit with identity transpositions if s < min_positive; swap rows k / r and columns k / c; inv = recip(X[k, k]);
//     scale the multipliers; X[k+1.., k+1..] -= l u^T fused with the next search (rank_one_update_and_best_in_matrix).
//
// GPU mapping: the whole step loop is ONE persistent cooperative kernel (full_piv_lu_kernel), two grid barriers per step:
//   [every CTA reduces the per-CTA records (score, column-major index) in the same order -> the same (r, c, s) and exit decision]
//   S  swap rows k / r over all columns and columns k / c over all rows (disjoint element sets, the 2 x 2 corner by one thread);
//      the swapped pivot column and pivot row are copied, unscaled, to two workspace vectors         -> barrier
//   U  the scaled side written from the workspace copy; the trailing block updated with the multiplier recomputed in registers
//      from the same copy (the same bits as the stored one); the first maximum tracked while writing -> per-CTA record -> barrier
// The workspace copy lets the readers and the writers of the pivot column / row share a phase without a race. The trailing pass
// is tiled: a warp owns 128 consecutive rows (4 per lane, so 32 consecutive rows per access) of 8 consecutive columns, keeps its
// 4 multipliers in registers across the 8 columns, reads the pivot row entry once per column and issues the loads of 4 (complex: 2)
// columns before the first use; a c64 element moves as one 16-byte access. Full pivoting is BLAS-2: every
// pivot needs the fully updated trailing block, so each step reads and writes the trailing block once and the kernel is
// HBM-bound. X is loaded through L2 (ld.cg: other CTAs wrote it in the previous phase), which keeps the last few thousand
// steps of a large factor L2-resident.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
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

constexpr int FPL_THREADS = 256;
constexpr int FPL_WARPS = FPL_THREADS / 32;
constexpr int FPL_TR = 128;  // rows of a trailing tile: 4 per lane
constexpr int FPL_TC = 8;    // columns of a trailing tile

// scalar.cuh's sc_ld / sc_st, except that a c64 element moves as one 16-byte access
template <class R, bool CX>
__device__ __forceinline__ Sc<R> fld(const R* p) {
  if (CX && sizeof(R) == 8) {  // one 16-byte access per c64 element (the working matrix is 16-byte aligned)
    const double2 v = __ldcg(reinterpret_cast<const double2*>(p));
    return Sc<R>{(R)v.x, (R)v.y};
  }
  return Sc<R>{__ldcg(p), CX ? __ldcg(p + 1) : R(0)};
}
template <class R, bool CX>
__device__ __forceinline__ void fst(R* p, Sc<R> v) {
  if (CX && sizeof(R) == 8) {
    *reinterpret_cast<double2*>(p) = make_double2((double)v.re, (double)v.im);
    return;
  }
  p[0] = v.re;
  if (CX) p[1] = v.im;
}

// per-CTA argmax record (pivot_record.cuh): the score and the column-major index i + j * m in X
template <class R>
struct FplWs {
  FplRec<R>* rec;           // [grid]
  R* col;                   // [W m] the swapped pivot column (entry k: the pivot), unscaled
  R* row;                   // [W n] the swapped pivot row, unscaled
  int* hist;                // [2 size]: row transposition, then column transposition of X at step k
  unsigned long long* bar;  // grid barrier counter (zeroed before the launch)
};

// The whole factorization of the column-major m x n working matrix X (leading dimension ld); tr: row k of X is the scaled side.
template <class R, bool CX>
__global__ void __launch_bounds__(FPL_THREADS) full_piv_lu_kernel(R* __restrict__ X, i64 ld, int m, int n, int tr, FplWs<R> w) {
  constexpr int W = CX ? 2 : 1;
  constexpr int FPL_JB = CX ? 2 : 4;  // columns whose loads are in flight together (FPL_TC is a multiple)
  __shared__ R s_pv[FPL_WARPS];
  __shared__ long long s_pi[FPL_WARPS];
  __shared__ R s_v;
  __shared__ long long s_i;
  const int size = min(m, n);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x;
  const int warps = G * FPL_WARPS;
  const int gw = blockIdx.x * FPL_WARPS + warp;
  const i64 T = (i64)G * FPL_THREADS;
  const i64 gt = (i64)blockIdx.x * FPL_THREADS + tid;
  const bool leader = blockIdx.x == 0 && tid == 0;
  auto at = [&](i64 i, i64 j) { return X + W * (i + j * ld); };
  unsigned long long target = 0;
  auto barrier = [&]() {
    target += G;
    grid_barrier(w.bar, target);
  };

  // One pass over X[k0.., k0..] in tiles of FPL_TR x FPL_TC; with `upd`, x -= l_i u_j first (l, u from the workspace copies,
  // the side `tr` selects scaled by inv). Publishes this CTA's first maximum of abs1 to w.rec.
  auto pass = [&](int k0, bool upd, Sc<R> inv) {
    R bv = R(0);
    long long bi = LLONG_MAX;
    const i64 nr = m - k0, nc = n - k0;
    const i64 tiles_r = (nr + FPL_TR - 1) / FPL_TR, tiles_c = (nc + FPL_TC - 1) / FPL_TC;
    for (i64 t = gw; t < tiles_r * tiles_c; t += warps) {
      const i64 i0 = k0 + (t % tiles_r) * FPL_TR + lane;
      const i64 j0 = k0 + (t / tiles_r) * FPL_TC, j1 = min((i64)n, j0 + FPL_TC);
      Sc<R> l[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        l[q] = Sc<R>{R(0), R(0)};
        const i64 i = i0 + 32 * q;
        if (upd && i < m) {
          l[q] = fld<R, CX>(w.col + W * i);
          if (!tr) l[q] = cmul_rn<R, CX>(l[q], inv);
        }
      }
      // JB columns at a time: all their loads are issued before the first use (4 JB accesses in flight per lane)
      for (i64 jb = j0; jb < j1; jb += FPL_JB) {
        Sc<R> u[FPL_JB], x[FPL_JB][4];
        R* base = at(i0, jb);  // the 4 JB accesses of a lane are immediate offsets of one address
#pragma unroll
        for (int c = 0; c < FPL_JB; ++c) {
          u[c] = Sc<R>{R(0), R(0)};
          if (jb + c < j1) {
            if (upd) u[c] = fld<R, CX>(w.row + W * (jb + c));
#pragma unroll
            for (int q = 0; q < 4; ++q)
              if (i0 + 32 * q < m) x[c][q] = fld<R, CX>(base + W * (c * ld + 32 * q));
          }
        }
#pragma unroll
        for (int c = 0; c < FPL_JB; ++c) {
          const i64 j = jb + c;
          if (j >= j1) continue;
          if (upd && tr) u[c] = cmul_rn<R, CX>(u[c], inv);
          const Sc<R> nu{-u[c].re, -u[c].im};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const i64 i = i0 + 32 * q;
            if (i < m) {
              if (upd) {
                x[c][q] = mul_add<R, CX>(l[q], nu, x[c][q]);
                fst<R, CX>(base + W * (c * ld + 32 * q), x[c][q]);
              }
              const R s = abs1_rn<R, CX>(x[c][q]);
              const long long ix = i + j * (i64)m;
              if (better(s, ix, bv, bi)) {
                bv = s;
                bi = ix;
              }
            }
          }
        }
      }
    }
    cta_publish<FPL_WARPS>(w.rec, bv, bi, s_pv, s_pi);
  };

  pass(0, false, Sc<R>{R(0), R(0)});  // best_in_matrix(A), factor.rs:337
  barrier();

  for (int k = 0; k < size; ++k) {
    // ---- the same reduction of the G records in every CTA ----
    __syncthreads();  // s_v / s_i may still be read from the previous step
    if (warp == 0) {
      R v = R(0);
      long long ix = LLONG_MAX;
      for (int b0 = 0; b0 < G; b0 += 128) {
        R vs[4];
        long long is[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int b = b0 + lane + 32 * u;
          vs[u] = b < G ? __ldcg(&w.rec[b].score) : R(0);
          is[u] = b < G ? __ldcg(&w.rec[b].idx) : LLONG_MAX;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (better(vs[u], is[u], v, ix)) {
            v = vs[u];
            ix = is[u];
          }
      }
      fpl_warp_argmax(v, ix);
      if (lane == 0) {
        s_v = v;
        s_i = ix;
      }
    }
    __syncthreads();
    const R s = s_v;
    if (!(s >= TLim<R>::min_pos())) {  // factor.rs:339-347 (s is never NaN: NaN entries are never chosen)
      if (leader)
        for (int t = k; t < size; ++t) {
          w.hist[t] = t;
          w.hist[size + t] = t;
        }
      break;
    }
    const i64 r = s_i % m, c = s_i / m;

    // ---- S: swap rows k / r and columns k / c (factor.rs:349-358), copy the pivot column and row ----
    for (i64 i = gt; i < m; i += T) {  // column swap over the rows other than k and r
      if (i == k || i == r) continue;
      Sc<R> v;
      if (c != k) {
        const Sc<R> a = fld<R, CX>(at(i, k)), b = fld<R, CX>(at(i, c));
        fst<R, CX>(at(i, k), b);
        fst<R, CX>(at(i, c), a);
        v = b;
      } else {
        if (i <= k) continue;
        v = fld<R, CX>(at(i, k));
      }
      if (i > k) fst<R, CX>(w.col + W * i, v);
    }
    for (i64 j = gt; j < n; j += T) {  // row swap over the columns other than k and c
      if (j == k || j == c) continue;
      Sc<R> v;
      if (r != k) {
        const Sc<R> a = fld<R, CX>(at(k, j)), b = fld<R, CX>(at(r, j));
        fst<R, CX>(at(k, j), b);
        fst<R, CX>(at(r, j), a);
        v = b;
      } else {
        if (j <= k) continue;
        v = fld<R, CX>(at(k, j));
      }
      if (j > k) fst<R, CX>(w.row + W * j, v);
    }
    if (leader) {
      // the corner rows {k, r} x columns {k, c}: new(i, j) = old(swap_r(i), swap_c(j))
      const Sc<R> o_kk = fld<R, CX>(at(k, k)), o_kc = fld<R, CX>(at(k, c)), o_rk = fld<R, CX>(at(r, k)), o_rc = fld<R, CX>(at(r, c));
      fst<R, CX>(at(k, k), o_rc);
      fst<R, CX>(w.col + W * k, o_rc);  // the pivot
      if (c != k) {
        fst<R, CX>(at(k, c), o_rk);
        fst<R, CX>(w.row + W * c, o_rk);
      }
      if (r != k) {
        fst<R, CX>(at(r, k), o_kc);
        fst<R, CX>(w.col + W * r, o_kc);
      }
      if (r != k && c != k) fst<R, CX>(at(r, c), o_kk);
      w.hist[k] = (int)r;
      w.hist[size + k] = (int)c;
    }
    barrier();

    // ---- U: scaled side (factor.rs:359-368), then the rank-one update fused with the next search (369-430) ----
    const Sc<R> inv = recip_rn<R, CX>(fld<R, CX>(w.col + W * k));
    if (!tr) {
      for (i64 i = k + 1 + gt; i < m; i += T) fst<R, CX>(at(i, k), cmul_rn<R, CX>(fld<R, CX>(w.col + W * i), inv));
    } else {
      for (i64 j = k + 1 + gt; j < n; j += T) fst<R, CX>(at(k, j), cmul_rn<R, CX>(fld<R, CX>(w.row + W * j), inv));
    }
    if (k + 1 == size) break;
    pass(k + 1, true, inv);
    barrier();
  }
}

// In-place full-pivoting LU (views in element units of the scalar kind; complex: COMPLEX units on an R* base). transpose: factor
// A^T (the reference's branch for |row_stride| >= |col_stride|). row_t / col_t (host, min(m, n) entries) receive A's row and
// column transpositions. Returns the transposition count.
template <class R, bool CX>
i64 full_piv_lu_in_place_t(cudaStream_t st, View<R> A, bool transpose, std::vector<long long>& row_t, std::vector<long long>& col_t) {
  constexpr int W = CX ? 2 : 1;
  const View<R> V = transpose ? A.t() : A;
  const i64 m = V.nrows, n = V.ncols, size = std::min(m, n);
  FB_ASSERT(m < (i64)INT_MAX && n < (i64)INT_MAX, "full-pivoting LU: dimension too large");
  row_t.assign((size_t)size, 0);
  col_t.assign((size_t)size, 0);
  if (size == 0) return 0;

  // the kernel works on a column-major, 16-byte aligned matrix; other views go through a compact copy
  const bool compact = V.rs == 1 && V.cs >= m && ((uintptr_t)V.ptr % 16 == 0 || !(CX && sizeof(R) == 8));
  R* work = V.ptr;
  i64 ld = V.cs;
  if (!compact) {
    work = (R*)ws_alloc((size_t)m * (size_t)n * W * sizeof(R));
    ld = m;
    piv_copy_t<R, CX>(st, View<R>{work, m, n, 1, m}, cview(V));
  }

  const int sms = stream_sms(st);
  int occ = 0;
  FB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, full_piv_lu_kernel<R, CX>, FPL_THREADS, 0));
  FB_ASSERT(occ > 0, "full-pivoting LU kernel cannot be resident");
  const int G = sms * std::min(occ, 2);  // 16 warps per SM keep the trailing pass fed; more CTAs only lengthen the barriers

  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t b_rec = (size_t)G * sizeof(FplRec<R>), b_col = (size_t)W * m * sizeof(R), b_row = (size_t)W * n * sizeof(R);
  const size_t b_hist = (size_t)2 * size * sizeof(int);
  char* buf = (char*)ws_alloc(up(b_rec) + up(b_col) + up(b_row) + up(b_hist) + 256);
  FplWs<R> w;
  char* p = buf;
  w.rec = (FplRec<R>*)p; p += up(b_rec);
  w.col = (R*)p; p += up(b_col);
  w.row = (R*)p; p += up(b_row);
  w.hist = (int*)p; p += up(b_hist);
  w.bar = (unsigned long long*)p;
  FB_CUDA_CHECK(cudaMemsetAsync(w.bar, 0, sizeof(unsigned long long), st));
  {
    int mi = (int)m, ni = (int)n, tri = transpose ? 1 : 0;
    void* args[] = {&work, &ld, &mi, &ni, &tri, &w};
    FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)full_piv_lu_kernel<R, CX>, dim3(G), dim3(FPL_THREADS), args, 0, st));
    note_launch();
  }
  if (!compact) {
    piv_copy_t<R, CX>(st, V, View<const R>{work, m, n, 1, m});
  }
  std::vector<int> hist((size_t)(2 * size));
  FB_CUDA_CHECK(cudaMemcpyAsync(hist.data(), w.hist, b_hist, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(buf);
  if (!compact) ws_free(work);
  i64 count = 0;
  for (i64 k = 0; k < size; ++k) {
    const long long hr = hist[(size_t)k], hc = hist[(size_t)(size + k)];
    count += (hr != k) + (hc != k);
    (transpose ? col_t : row_t)[(size_t)k] = hr;
    (transpose ? row_t : col_t)[(size_t)k] = hc;
  }
  return count;
}

// rhs <- A^-1 rhs (solve.rs:21-56) or A^-T rhs (solve.rs:58-93), conj(A) with `conj`. Permutations: host int64[n].
template <class R, bool CX>
void full_piv_lu_solve_t(cudaStream_t st, View<const R> L, View<const R> U, const long long* row_fwd, const long long* row_bwd,
                         const long long* col_fwd, const long long* col_bwd, bool conj, bool transpose, View<R> rhs) {
  const i64 n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "full-pivoting LU solve shape mismatch");
  if (n == 0 || rhs.ncols == 0) return;
  if (!transpose) {
    permute_rows_t<R, CX>(st, rhs, row_fwd);
    solve_lower_t<R, CX>(st, L, true, conj, rhs);
    solve_upper_t<R, CX>(st, U, false, conj, rhs);
    permute_rows_t<R, CX>(st, rhs, col_bwd);
  } else {
    permute_rows_t<R, CX>(st, rhs, col_fwd);
    solve_lower_t<R, CX>(st, U.t(), false, conj, rhs);
    solve_upper_t<R, CX>(st, L.t(), true, conj, rhs);
    permute_rows_t<R, CX>(st, rhs, row_bwd);
  }
}

// out (m x n) <- P^-1 L U Q^-1: tmp = L U by structured products, out[i, j] = tmp[row_bwd[i], col_bwd[j]] (reconstruct.rs:13-82)
template <class R, bool CX>
void full_piv_lu_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L, View<const R> U, const long long* row_bwd,
                               const long long* col_bwd) {
  constexpr int W = CX ? 2 : 1;
  const i64 m = L.nrows, n = U.ncols, size = std::min(m, n);
  FB_ASSERT(out.nrows == m && out.ncols == n && L.ncols >= size && U.nrows >= size, "full-pivoting LU reconstruct shape mismatch");
  if (m == 0 || n == 0) return;
  R* buf = (R*)ws_alloc((size_t)m * (size_t)n * W * sizeof(R));
  const View<R> tmp{buf, m, n, 1, m};
  const View<const R> Ls = sub_t<R, CX>(L, 0, 0, size, size), Us = sub_t<R, CX>(U, 0, 0, size, size);
  gemm_t<R, CX>(st, sub_t<R, CX>(tmp, 0, 0, size, size), RECT, 0, Ls, UNIT_LOWER, false, Us, TRI_UPPER, false, R(1));
  if (m > n)
    gemm_t<R, CX>(st, sub_t<R, CX>(tmp, size, 0, m - size, size), RECT, 0, sub_t<R, CX>(L, size, 0, m - size, size), RECT, false, Us,
                  TRI_UPPER, false, R(1));
  if (m < n)
    gemm_t<R, CX>(st, sub_t<R, CX>(tmp, 0, size, size, n - size), RECT, 0, Ls, UNIT_LOWER, false, sub_t<R, CX>(U, 0, size, size, n - size),
                  RECT, false, R(1));
  gather_2d_t<R, CX>(st, out, View<const R>{buf, m, n, 1, m}, row_bwd, col_bwd);
  ws_free(buf);
}

// out <- A^-1 = Q U^-1 L^-1 P: both triangular inverses in out, tmp = U^-1 L^-1, out[i, j] = tmp[col_bwd[i], row_bwd[j]]
// (inverse.rs:12-63)
template <class R, bool CX>
void full_piv_lu_inverse_t(cudaStream_t st, View<R> out, View<const R> L, View<const R> U, const long long* row_bwd,
                           const long long* col_bwd) {
  constexpr int W = CX ? 2 : 1;
  const i64 n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && out.nrows == n && out.ncols == n, "full-pivoting LU inverse shape mismatch");
  if (n == 0) return;
  inverse_triangular_t<R, CX>(st, out, L, true, true);
  inverse_triangular_t<R, CX>(st, out, U, false, false);
  R* buf = (R*)ws_alloc((size_t)n * (size_t)n * W * sizeof(R));
  const View<const R> o{out.ptr, n, n, out.rs, out.cs};
  gemm_t<R, CX>(st, View<R>{buf, n, n, 1, n}, RECT, 0, o, TRI_UPPER, false, o, UNIT_LOWER, false, R(1));
  gather_2d_t<R, CX>(st, out, View<const R>{buf, n, n, 1, n}, col_bwd, row_bwd);
  ws_free(buf);
}

}  // namespace

}  // namespace fb

// ---- C ABI (faer-ffi/src/lib.rs:2125-2325; declarations in include/faer_b200_full_piv_lu.h) ----
using namespace fb;

namespace {

template <class R, bool CX>
FaerV0_24_FullPivLuStatus full_piv_lu_factor_entry(FaerV0_24_MatMut A, FaerV0_24_SliceMut row_fwd, FaerV0_24_SliceMut row_bwd,
                                                   FaerV0_24_SliceMut col_fwd, FaerV0_24_SliceMut col_bwd, int idx_bytes) {
  FB_ENTRY();
  const size_t m = A.nrows, n = A.ncols;
  FB_ASSERT(m == 0 || (row_fwd.ptr != nullptr && row_bwd.ptr != nullptr), "null row permutation slice");
  FB_ASSERT(n == 0 || (col_fwd.ptr != nullptr && col_bwd.ptr != nullptr), "null column permutation slice");
  cudaStream_t st = current_stream();
  std::vector<long long> rt, ct;
  i64 count = 0;
  if (m > 0 && n > 0) {
    // the branch reads the CALLER's strides (factor.rs:492): the staged mirror may be laid out differently
    const bool transpose = !(std::llabs((long long)A.row_stride) < std::llabs((long long)A.col_stride));
    StagedMat a = stage<R, CX>(A, true, st);
    count = full_piv_lu_in_place_t<R, CX>(st, a.view<R>(), transpose, rt, ct);
    finish_all(st, {&a});
  }
  // factor.rs:511-528: the transpositions applied in order to the identity, and the inverses
  std::vector<long long> rf, rb, cf, cb;
  perm_from_transpositions(m, rt, rf, rb);
  perm_from_transpositions(n, ct, cf, cb);
  write_perm(row_fwd.ptr, rf, idx_bytes);
  write_perm(row_bwd.ptr, rb, idx_bytes);
  write_perm(col_fwd.ptr, cf, idx_bytes);
  write_perm(col_bwd.ptr, cb, idx_bytes);
  FaerV0_24_FullPivLuStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_FullPivLuStatus_Ok;
  out.ok.transposition_count = (size_t)count;
  return out;
}

template <class R, bool CX>
void full_piv_lu_solve_entry(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj conj, FaerV0_24_SliceRef row_fwd,
                             FaerV0_24_SliceRef row_bwd, FaerV0_24_SliceRef col_fwd, FaerV0_24_SliceRef col_bwd, FaerV0_24_MatMut rhs,
                             int idx_bytes, bool transpose) {
  FB_ENTRY();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && U.nrows == n && U.ncols == n && rhs.nrows == n, "full-pivoting LU solve shape mismatch");
  cudaStream_t st = current_stream();
  const std::vector<long long> rf = read_perm_checked(row_fwd, n, idx_bytes), rb = read_perm_checked(row_bwd, n, idx_bytes);
  const std::vector<long long> cf = read_perm_checked(col_fwd, n, idx_bytes), cb = read_perm_checked(col_bwd, n, idx_bytes);
  StagedMat l = stage<R, CX>(L, st);
  StagedMat u = stage<R, CX>(U, st);
  StagedMat r = stage<R, CX>(rhs, true, st);
  full_piv_lu_solve_t<R, CX>(st, l.view<const R>(), u.view<const R>(), rf.data(), rb.data(), cf.data(), cb.data(),
                             conj == FaerV0_24_Conj_Yes, transpose, r.view<R>());
  finish_all(st, {&l, &u, &r});
}

template <class R, bool CX>
void full_piv_lu_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_SliceRef row_bwd,
                             FaerV0_24_SliceRef col_bwd, int idx_bytes, bool inverse) {
  FB_ENTRY();
  const size_t m = L.nrows, n = U.ncols;
  if (inverse)
    FB_ASSERT(L.ncols == m && U.nrows == m && n == m && A.nrows == m && A.ncols == m, "full-pivoting LU inverse shape mismatch");
  else
    FB_ASSERT(A.nrows == m && A.ncols == n && L.ncols >= (m < n ? m : n) && U.nrows >= (m < n ? m : n),
              "full-pivoting LU reconstruct shape mismatch");
  cudaStream_t st = current_stream();
  const std::vector<long long> rb = read_perm_checked(row_bwd, m, idx_bytes), cb = read_perm_checked(col_bwd, n, idx_bytes);
  StagedMat a = stage<R, CX>(A, false, st);
  StagedMat l = stage<R, CX>(L, st);
  StagedMat u = stage<R, CX>(U, st);
  if (inverse) full_piv_lu_inverse_t<R, CX>(st, a.view<R>(), l.view<const R>(), u.view<const R>(), rb.data(), cb.data());
  else full_piv_lu_reconstruct_t<R, CX>(st, a.view<R>(), l.view<const R>(), u.view<const R>(), rb.data(), cb.data());
  finish_all(st, {&a, &l, &u});
}

}  // namespace

extern "C" {

// Scratch layouts are the reference's (factor.rs:450-461, solve.rs:4-19, reconstruct.rs:4-11, inverse.rs:4-10); the GPU paths keep
// their workspace in the device pool and ignore `mem`.
#define FB_FPL_FFI(SUF, R, CX, IT, BYTES)                                                                                             \
  FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_##IT##_##SUF(size_t dim, size_t block_size, FaerV0_24_Par par,    \
                                                                                  FaerV0_24_FullPivLuParams params) {                 \
    (void)par; (void)params;                                                                                                          \
    /* faer-ffi forwards (dim, block_size) as (nrows, ncols): StackReq::new::<usize>(min(nrows, ncols)).array(2) */                  \
    const size_t size = dim < block_size ? dim : block_size;                                                                          \
    return FaerV0_24_Layout{2 * size * sizeof(size_t), alignof(size_t)};                                                              \
  }                                                                                                                                   \
  FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_##IT##_##SUF(                                                   \
      FaerV0_24_MatMut A, FaerV0_24_SliceMut row_perm_fwd, FaerV0_24_SliceMut row_perm_bwd, FaerV0_24_SliceMut col_perm_fwd,          \
      FaerV0_24_SliceMut col_perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem, FaerV0_24_FullPivLuParams params) {                  \
    (void)par; (void)mem; (void)params;                                                                                               \
    return full_piv_lu_factor_entry<R, CX>(A, row_perm_fwd, row_perm_bwd, col_perm_fwd, col_perm_bwd, BYTES);                        \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {   \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{dim * rhs_ncols * (CX ? 2 : 1) * sizeof(R), 64}; /* permute_rows_in_place_scratch::<I, T>(dim, k) */       \
  }                                                                                                                                   \
  void libfaer_v0_23_full_piv_lu_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj,           \
                                                             FaerV0_24_SliceRef row_perm_fwd, FaerV0_24_SliceRef row_perm_bwd,         \
                                                             FaerV0_24_SliceRef col_perm_fwd, FaerV0_24_SliceRef col_perm_bwd,         \
                                                             FaerV0_24_MatMut rhs, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {        \
    (void)par; (void)mem;                                                                                                             \
    full_piv_lu_solve_entry<R, CX>(L, U, A_conj, row_perm_fwd, row_perm_bwd, col_perm_fwd, col_perm_bwd, rhs, BYTES, false);          \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols,              \
                                                                                           FaerV0_24_Par par) {                       \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{dim * rhs_ncols * (CX ? 2 : 1) * sizeof(R), 64};                                                          \
  }                                                                                                                                   \
  void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_##IT##_##SUF(                                                               \
      FaerV0_24_MatRef L, FaerV0_24_MatRef U, FaerV0_24_Conj A_conj, FaerV0_24_SliceRef row_perm_fwd, FaerV0_24_SliceRef row_perm_bwd, \
      FaerV0_24_SliceRef col_perm_fwd, FaerV0_24_SliceRef col_perm_bwd, FaerV0_24_MatMut rhs, FaerV0_24_Par par,                      \
      FaerV0_24_MemAlloc mem) {                                                                                                       \
    (void)par; (void)mem;                                                                                                             \
    full_piv_lu_solve_entry<R, CX>(L, U, A_conj, row_perm_fwd, row_perm_bwd, col_perm_fwd, col_perm_bwd, rhs, BYTES, true);           \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_##IT##_##SUF(size_t nrows, size_t ncols, FaerV0_24_Par par) {         \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{nrows * ncols * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(nrows, ncols) */                  \
  }                                                                                                                                   \
  void libfaer_v0_23_full_piv_lu_reconstruct_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,                 \
                                                          FaerV0_24_SliceRef row_perm_fwd, FaerV0_24_SliceRef row_perm_bwd,            \
                                                          FaerV0_24_SliceRef col_perm_fwd, FaerV0_24_SliceRef col_perm_bwd,            \
                                                          FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                 \
    (void)row_perm_fwd; (void)col_perm_fwd; (void)par; (void)mem;                                                                     \
    full_piv_lu_recon_entry<R, CX>(A, L, U, row_perm_bwd, col_perm_bwd, BYTES, false);                                                \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                             \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{dim * dim * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, dim) */                          \
  }                                                                                                                                   \
  void libfaer_v0_23_full_piv_lu_inverse_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_MatRef U,                     \
                                                      FaerV0_24_SliceRef row_perm_fwd, FaerV0_24_SliceRef row_perm_bwd,                \
                                                      FaerV0_24_SliceRef col_perm_fwd, FaerV0_24_SliceRef col_perm_bwd,                \
                                                      FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                     \
    (void)row_perm_fwd; (void)col_perm_fwd; (void)par; (void)mem;                                                                     \
    full_piv_lu_recon_entry<R, CX>(A, L, U, row_perm_bwd, col_perm_bwd, BYTES, true);                                                 \
  }
#define FB_FPL_DTYPE(SUF, R, CX)                                                                                                 \
  FaerV0_24_FullPivLuParams libfaer_v0_23_FullPivLuParams_##SUF(void) { return FaerV0_24_FullPivLuParams{256 * 512}; } /* factor.rs:441-449 */ \
  FB_FPL_FFI(SUF, R, CX, u32, 4)                                                                                                 \
  FB_FPL_FFI(SUF, R, CX, u64, 8)
FB_FPL_DTYPE(f64, double, false)
FB_FPL_DTYPE(f32, float, false)
FB_FPL_DTYPE(c64, double, true)
FB_FPL_DTYPE(c32, float, true)
#undef FB_FPL_DTYPE
#undef FB_FPL_FFI

}  // extern "C"
