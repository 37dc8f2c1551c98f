// Bunch-Kaufman LBL^H (faer's `cholesky::lblt`, the reference's `bunch_kaufman` module) for f64 / f32 / c64 / c32: factor, solve,
// reconstruct, inverse, and their C ABI (include/faer_b200_lblt.h, included by include/faer_b200.h: `libfaer_v0_23_lblt_*`).
//
// Reference: faer/src/linalg/cholesky/bunch_kaufman/factor.rs (cholesky_in_place 1161-1234, lblt_blocked 700-782,
// lblt_blocked_step 491-699, lblt_unblocked 784-902, lblt_full_piv 264-429, rank1/rank2_update 913-1125), solve.rs:35-104,
// reconstruct.rs:12-87, inverse.rs:11-42. The factorization follows the reference's operation sequence:
//   * Full -> lblt_full_piv; the other strategies -> lblt_blocked with (rook, diagonal) = Partial (F, F), PartialDiag (F, T),
//     Rook (T, F), RookDiag (T, T); bs = block_size, 0 when bs < 2 or n <= bs (no clamp: bs decides where the unblocked tail starts);
//   * blocked: while more than bs columns remain, a left-looking step of at most bs - 1 columns (bs after a closing 2 x 2 pivot),
//     then ONE product A22(strict lower) -= W Al^H, the diagonal made real, and the step's row interchanges applied to the
//     columns left of the block; the last <= bs columns (or all of them when bs is 0) are factored right-looking;
//   * the pivot rules: abs1 first maxima with strict `>` from 0, the diagonal excluded from the column search; 1 x 1 when
//     |Re a_i0i0| >= alpha gamma_i; otherwise (non-rook) |Re a_i0i0| >= alpha gamma_r (gamma_r / gamma_i), then
//     |Re a_i1i1| >= alpha gamma_r, else 2 x 2; rook: abs1 of the diagonal, ending on s == i0 (blocked step only) or
//     gamma_i == gamma_r. gamma_i == 0 or the last column: no scaling, no update, subdiag[k] NOT written;
//   * Full: the whole matrix (strict upper triangle included) scaled by 1 / norm_max and never restored; abs2 comparisons of
//     the largest diagonal entry with alpha^2 max_offdiag; the next off-diagonal maximum is taken during the rank-1 / rank-2
//     update in column-major order (the Seq rule: see DESIGN.md §3 for the Rayon split's ties); after max_offdiag == 0 only
//     diagonal interchanges; diag and subdiag multiplied back by norm_max at the end.
//
// GPU mapping (one stream; the only host synchronisation inside the factorization reads the column count of each blocked step):
//   lblt_panel_kernel   one cooperative launch per blocked step over the trailing rows. Thread t owns rows t, t + T, ... of the
//                       step (T = grid threads) in every phase, so a phase that only touches owned rows needs no barrier. Per
//                       column: [scale L of the previous pivot and update the owned diagonal entries (+ the diagonal argmax for
//                       the Diag strategies)] -> barrier -> [W column of the candidate: row / column of the trailing matrix minus
//                       Al conj(Wl[i0, :]), its abs1 argmax] -> barrier -> [the same record reduction and decision in every CTA,
//                       the symmetric interchange spread over the grid] -> barrier. That is 3 grid barriers per column when a
//                       1 x 1 pivot passes the first test (2 for Partial / Rook, whose first phase needs no reduction). Each
//                       further candidate column (the second test, the rook walk) adds one barrier, a 2 x 2 pivot two, and a
//                       1 x 1 pivot on the candidate one (its W column is copied before the interchange reads it).
//   trailing update     gemm_f64 / f32 / c64 / c32 with a STRICT_LOWER destination, lhs W, rhs Al^H, alpha = -1; then the diagonal
//                       made real (complex kinds). At the default block size the f64 product has k = 63 and, for a trailing
//                       matrix of at least 3 waves of 128 x 128 tiles, takes the wide TMA-fed configuration (gemm_f64.cu's
//                       triangular-destination rule for k <= 1024).
//   left interchanges   piv_laswp_t (piv_common.cuh), the pivot list with TOP_BIT stripped.
//   lblt_rl_kernel      one persistent cooperative kernel for the right-looking loops: lblt_unblocked and lblt_full_piv. Per
//                       pivot: [the pending rank-1 / rank-2 update of the trailing lower triangle fused with the next search
//                       (column argmax, diagonal argmax, or Full's off-diagonal maximum)] -> barrier -> [decision, interchange]
//                       -> barrier, plus one barrier per extra candidate column. The scaled L columns of a pivot are written one
//                       pivot later (the update reads them unscaled; row interchanges commute with the per-row scaling), which
//                       keeps the writers and the readers of a pivot column in different phases. The trailing pass is tiled:
//                       a warp owns 128 consecutive rows of one column. Records and their publish are pivot_record.cuh's.
// Pivots and 2 x 2 flags stay on the device and are read back once, after the factorization.
// Record sets: A (diagonal argmax), B (the first candidate column) and C. Further candidate columns of one decision (the second
// test, the rook walk) alternate C, B, C, ... (lb_cand): every CTA reads a set after a barrier, and a CTA that leaves the barrier
// early may publish the next candidate before the slowest CTA has read the last one, so a set is never rewritten before the
// barrier of the publication in between. This costs no barrier.
// ptxas -v: no spills. The two cooperative kernels are declared __launch_bounds__(256, 1): with the block size alone, ptxas
// allocated fewer registers than lblt_panel_kernel<double, false> (140 registers now), <float, false> and
// lblt_rl_kernel<double, true, true> need and spilled up to 140 bytes. Their grids are sized from the occupancy they get.
// Solve / reconstruct / inverse use the unit-triangular solves and structured products of each kind, the shared row gathers,
// and two small kernels (the 1 x 1 / 2 x 2 block solve, the L B column pass).
#include <algorithm>
#include <climits>
#include <cstring>
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

constexpr int LB_THREADS = 256;
constexpr int LB_WARPS = LB_THREADS / 32;
constexpr int LB_TR = 128;  // rows of a trailing tile of the right-looking kernel: 4 per lane

// a pivot block whose scaling / update is pending: kind 0 none (also "nothing to do"), 1 a 1 x 1 pivot at column p, 2 a 2 x 2 pivot
// at columns p, p + 1 (factor.rs:620-670 / 867-891 / 337-393)
template <class R>
struct LbPiv {
  int kind, p;
  R dg, dinv;          // 1 x 1: Re a_pp, recip
  R d, d00, d11;       // 2 x 2
  Sc<R> d10;
};
template <class R, bool CX>
__device__ __forceinline__ LbPiv<R> lb_one(int p, R dg) {
  LbPiv<R> q{};
  q.kind = 1;
  q.p = p;
  q.dg = dg;
  q.dinv = R(1) / dg;
  return q;
}
template <class R, bool CX>
__device__ __forceinline__ LbPiv<R> lb_two(int p, R a00, R a11, Sc<R> a10) {
  LbPiv<R> q{};
  q.kind = 2;
  q.p = p;
  const R d10 = cabs<R, CX>(a10);
  const R d10_inv = R(1) / d10;
  q.d00 = a00 * d10_inv;
  q.d11 = a11 * d10_inv;
  const R t = R(1) / (q.d00 * q.d11 - R(1));
  q.d10 = cscale(a10, d10_inv);
  q.d = t * d10_inv;
  return q;
}
// w0 = (x0 d11 - x1 d10) d, w1 = (x1 d00 - x0 conj(d10)) d
template <class R, bool CX>
__device__ __forceinline__ void lb_w(const LbPiv<R>& q, Sc<R> x0, Sc<R> x1, Sc<R>& w0, Sc<R>& w1) {
  w0 = cscale(csub(cscale(x0, q.d11), cmul<R, CX>(x1, q.d10)), q.d);
  w1 = cscale(csub(cscale(x1, q.d00), cmul<R, CX>(x0, cconj(q.d10))), q.d);
}

template <class R>
struct LbWs {
  FplRec<R>* rec;           // [3 * grid]: record sets A (diagonal), B (column / off-diagonal) and C; see lb_cand
  unsigned long long* bar;  // grid barrier counter (zeroed before each launch)
  long long* piv;           // [n] pivot row of column j (global, TOP_BIT stripped)
  int* two;                 // [n] 1 where column j belongs to a 2 x 2 block
  int* kstep;               // columns factored by the last panel launch
};

// this CTA's first maximum into rec[blockIdx.x] (every thread of the CTA calls it)
template <class R>
__device__ void lb_publish(FplRec<R>* rec, R v, long long i, R* s_v, long long* s_i) {
  cta_publish<LB_WARPS>(rec, v, i, s_v, s_i);
  __syncthreads();
}
// the same reduction of the grid's records in every CTA (after a grid barrier)
template <class R>
__device__ void lb_collect(const FplRec<R>* rec, R& v, long long& i, R* s_v, long long* s_i) {
  if (threadIdx.x < 32) {
    R bv = R(0);
    long long bi = LLONG_MAX;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += 32) {
      const R v2 = __ldcg(&rec[b].score);
      const long long i2 = __ldcg(&rec[b].idx);
      if (better(v2, i2, bv, bi)) {
        bv = v2;
        bi = i2;
      }
    }
    fpl_warp_argmax(bv, bi);
    if (threadIdx.x == 0) {
      s_v[0] = bv;
      s_i[0] = bi;
    }
  }
  __syncthreads();
  v = s_v[0];
  i = s_i[0];
  __syncthreads();
}

// The record set of the k-th further candidate column of a pivot decision (k = 0, 1, ...): C, B, C, ... Every CTA reads a set
// after a grid barrier and may publish the next candidate's records before the slowest CTA has finished reading, so
// consecutive publications alternate between two sets; a set is rewritten only after the barrier of the publication in between.
template <class R>
__device__ __forceinline__ FplRec<R>* lb_cand(FplRec<R>* rec, int k) {
  return rec + (k & 1 ? 1 : 2) * gridDim.x;
}

// swap_self_adjoint(A, i, j), i < j (factor.rs:37-53), on a matrix whose first `c` columns are the factored ones: rows i / j over
// columns 0..i (the factored part and the trailing part `..i` together), columns i / j below j, the middle segment
// (A[t, i], A[j, t]) = (conj A[j, t], conj A[t, i]), A[j, i] conjugated, the diagonal exchanged as real parts; with Wb, rows i / j
// of W's columns 0..nw as well. Element pairs are spread over the grid; the single entries go to the leader.
template <class R, bool CX, class At, class Wa>
__device__ void lb_swap(At at, Wa wa, bool with_w, int m, int i, int j, int nw, i64 gt, i64 T, bool leader) {
  const i64 na = (i64)m - 1 - j, nb = i, nc = (i64)j - i - 1, nd = with_w ? nw : 0;
  for (i64 e = gt; e < na + nb + nc + nd; e += T) {
    if (e < na) {
      const i64 r = j + 1 + e;
      const Sc<R> x = sc_ld<R, CX>(at(r, i)), y = sc_ld<R, CX>(at(r, j));
      sc_st<R, CX>(at(r, i), y);
      sc_st<R, CX>(at(r, j), x);
    } else if (e < na + nb) {
      const i64 col = e - na;
      const Sc<R> x = sc_ld<R, CX>(at(i, col)), y = sc_ld<R, CX>(at(j, col));
      sc_st<R, CX>(at(i, col), y);
      sc_st<R, CX>(at(j, col), x);
    } else if (e < na + nb + nc) {
      const i64 t = i + 1 + (e - na - nb);
      const Sc<R> x = sc_ld<R, CX>(at(t, i)), y = sc_ld<R, CX>(at(j, t));
      sc_st<R, CX>(at(t, i), cconj(y));
      sc_st<R, CX>(at(j, t), cconj(x));
    } else {
      const i64 col = e - na - nb - nc;
      const Sc<R> x = sc_ld<R, CX>(wa(i, col)), y = sc_ld<R, CX>(wa(j, col));
      sc_st<R, CX>(wa(i, col), y);
      sc_st<R, CX>(wa(j, col), x);
    }
  }
  if (leader) {
    const R aii = __ldcg(at(i, i)), ajj = __ldcg(at(j, j));
    sc_st<R, CX>(at(i, i), Sc<R>{ajj, R(0)});
    sc_st<R, CX>(at(j, j), Sc<R>{aii, R(0)});
    if (CX) {
      R* o = at(j, i);
      o[1] = -__ldcg(o + 1);
    }
  }
}

// One left-looking step (lblt_blocked_step) on the trailing matrix A (m x m, A[k0, k0] of the caller's matrix) with W (m x bs,
// leading dimension ldw). sub: subdiag[k0..]. See the file comment for the per-column schedule.
template <class R, bool CX>
__global__ void __launch_bounds__(LB_THREADS, 1) lblt_panel_kernel(R* __restrict__ A, i64 rs, i64 cs, int m, int k0, int bs,
                                                                R* __restrict__ Wb, i64 ldw, R* __restrict__ sub, i64 sds,
                                                                int rook, int diagonal, LbWs<R> w) {
  constexpr int W = CX ? 2 : 1;
  __shared__ R s_v[LB_WARPS];
  __shared__ long long s_i[LB_WARPS];
  const int G = gridDim.x;
  const i64 T = (i64)G * LB_THREADS, gt = (i64)blockIdx.x * LB_THREADS + threadIdx.x;
  const bool leader = blockIdx.x == 0 && threadIdx.x == 0;
  auto at = [&](i64 i, i64 j) { return A + W * (i * rs + j * cs); };
  auto wa = [&](i64 i, i64 j) { return Wb + W * (i + j * ldw); };
  auto sd = [&](i64 i) { return sub + W * i * sds; };
  FplRec<R>* recA = w.rec;
  FplRec<R>* recB = w.rec + G;
  unsigned long long target = 0;
  auto barrier = [&]() {
    target += G;
    grid_barrier(w.bar, target);
  };
  const R alpha = (R(1) + sqrt(R(17))) * R(0.125);

  // owned rows >= c: L of the pending pivot q and the diagonal update (factor.rs:620-637 / 638-670); the diagonal argmax (abs1)
  auto apply = [&](const LbPiv<R>& q, int c, bool want) {
    R bv = R(0);
    long long bi = LLONG_MAX;
    for (i64 r = gt; r < m; r += T) {
      if (r < c) continue;
      if (q.kind == 1) {
        const Sc<R> l = cscale(sc_ld<R, CX>(wa(r, q.p)), q.dinv);
        sc_st<R, CX>(at(r, q.p), l);
        sc_st<R, CX>(at(r, r), Sc<R>{__ldcg(at(r, r)) - q.dg * cabs2(l), R(0)});
      } else if (q.kind == 2) {
        const Sc<R> x0 = sc_ld<R, CX>(wa(r, q.p)), x1 = sc_ld<R, CX>(wa(r, q.p + 1));
        Sc<R> w0, w1;
        lb_w<R, CX>(q, x0, x1, w0, w1);
        const Sc<R> a = csub(csub(sc_ld<R, CX>(at(r, r)), cmul<R, CX>(x0, cconj(w0))), cmul<R, CX>(x1, cconj(w1)));
        sc_st<R, CX>(at(r, r), Sc<R>{a.re, R(0)});
        sc_st<R, CX>(at(r, q.p), w0);
        sc_st<R, CX>(at(r, q.p + 1), w1);
      }
      if (want) {
        const R s = cabs1(sc_ld<R, CX>(at(r, r)));
        if (s > bv) {
          bv = s;
          bi = r;
        }
      }
    }
    if (leader && q.kind == 2) sc_st<R, CX>(at(q.p + 1, q.p), Sc<R>{R(0), R(0)});
    if (want) lb_publish(recA, bv, bi, s_v, s_i);
  };
  // W[:, wc] <- column x of the updated trailing matrix, rows c.. (update_and_offdiag_argmax, factor.rs:461-489), and the
  // abs1 first maximum off x
  auto build = [&](int c, int x, int wc, FplRec<R>* set) {
    R bv = R(0);
    long long bi = LLONG_MAX;
    for (i64 r = gt; r < m; r += T) {
      if (r < c) continue;
      if (r == x) {
        sc_st<R, CX>(wa(r, wc), Sc<R>{__ldcg(at(r, r)), R(0)});
        continue;
      }
      Sc<R> v = r < x ? cconj(sc_ld<R, CX>(at(x, r))) : sc_ld<R, CX>(at(r, x));
      Sc<R> acc{R(0), R(0)};
      for (int t = 0; t < c; ++t) {
        const Sc<R> a = sc_ld<R, CX>(at(r, t)), b = sc_ld<R, CX>(wa(x, t));
        acc = cfms_conj<R, CX>(acc, a, b);  // acc -= Al[r, t] conj(Wl[x, t])
      }
      v = Sc<R>{v.re + acc.re, v.im + acc.im};
      sc_st<R, CX>(wa(r, wc), v);
      const R s = cabs1(v);
      if (s > bv) {
        bv = s;
        bi = r;
      }
    }
    lb_publish(set, bv, bi, s_v, s_i);
  };
  auto copy_col = [&](int c, int from, int to) {
    for (i64 r = gt; r < m; r += T)
      if (r >= c) sc_st<R, CX>(wa(r, to), sc_ld<R, CX>(wa(r, from)));
  };

  LbPiv<R> q{};
  int c = 0;
  const int kmax = min(bs - 1, m);
  while (c < kmax) {
    int i0 = c;
    if (diagonal) {
      apply(q, c, true);
      barrier();
      R v;
      long long ix;
      lb_collect(recA, v, ix, s_v, s_i);
      if (ix != LLONG_MAX) i0 = (int)ix;
      build(c, i0, c, recB);
    } else {
      apply(q, c, false);
      build(c, i0, c, recB);
    }
    barrier();
    R gi;
    long long r;
    lb_collect(recB, gi, r, s_v, s_i);
    int npiv = 1, i1 = -1;
    bool nothing = false, moved = false;
    if (c + 1 == m || gi == R(0)) {
      nothing = true;
    } else if (fabs(__ldcg(at(i0, i0))) >= alpha * gi) {
      npiv = 1;
    } else {
      i1 = (int)r;
      if (rook) {
        for (int cand = 0;; ++cand) {
          FplRec<R>* set = lb_cand(w.rec, cand);
          build(c, i1, c + 1, set);
          barrier();
          R gr;
          long long s;
          lb_collect(set, gr, s, s_v, s_i);
          if (s == LLONG_MAX) s = c;
          if (cabs1(sc_ld<R, CX>(at(i1, i1))) >= alpha * gr) {
            npiv = 1;
            i0 = i1;
            i1 = -1;
            copy_col(c, c + 1, c);
            moved = true;
            break;
          } else if (s == i0 || gi == gr) {
            npiv = 2;
            break;
          } else {
            i0 = i1;
            i1 = (int)s;
            gi = gr;
            copy_col(c, c + 1, c);
          }
        }
      } else {
        FplRec<R>* set = lb_cand(w.rec, 0);
        build(c, i1, c + 1, set);
        barrier();
        R gr;
        long long s;
        lb_collect(set, gr, s, s_v, s_i);
        if (fabs(__ldcg(at(i0, i0))) >= (alpha * gr) * (gr / gi)) {
          npiv = 1;
        } else if (fabs(__ldcg(at(i1, i1))) >= alpha * gr) {
          npiv = 1;
          i0 = i1;
          i1 = -1;
          copy_col(c, c + 1, c);
          moved = true;
        } else {
          npiv = 2;
        }
      }
    }
    if (npiv == 2) {
      if (i0 > i1) {
        for (i64 rr = gt; rr < m; rr += T) {
          if (rr < c) continue;
          const Sc<R> x = sc_ld<R, CX>(wa(rr, c)), y = sc_ld<R, CX>(wa(rr, c + 1));
          sc_st<R, CX>(wa(rr, c), y);
          sc_st<R, CX>(wa(rr, c + 1), x);
        }
        const int t = i0;
        i0 = i1;
        i1 = t;
      }
      moved = true;
    }
    if (moved) barrier();  // the interchanges read W rows owned by other threads
    if (i0 != c) lb_swap<R, CX>(at, wa, true, m, c, i0, c + npiv, gt, T, leader);
    if (npiv == 2) {
      barrier();
      if (i1 != c + 1) lb_swap<R, CX>(at, wa, true, m, c + 1, i1, c + 2, gt, T, leader);
    }
    if (leader) {
      w.piv[k0 + c] = k0 + i0;
      w.two[k0 + c] = npiv == 2;
      if (npiv == 2) {
        w.piv[k0 + c + 1] = k0 + i1;
        w.two[k0 + c + 1] = 1;
      }
    }
    barrier();
    if (nothing) {
      q.kind = 0;
    } else if (npiv == 1) {
      q = lb_one<R, CX>(c, __ldcg(wa(c, c)));
      if (leader) sc_st<R, CX>(sd(c), Sc<R>{R(0), R(0)});
    } else {
      const Sc<R> a10 = sc_ld<R, CX>(wa(c + 1, c));
      q = lb_two<R, CX>(c, __ldcg(wa(c, c)), __ldcg(wa(c + 1, c + 1)), a10);
      if (leader) {
        sc_st<R, CX>(sd(c), a10);
        sc_st<R, CX>(sd(c + 1), Sc<R>{R(0), R(0)});
      }
    }
    c += npiv;
  }
  apply(q, c, false);
  if (leader) *w.kstep = c;
}

// The right-looking loops on the m x m matrix A (A[k0, k0] of the caller's; the factored columns of this launch are its columns
// 0..c): lblt_unblocked (FULL = false) and lblt_full_piv (FULL = true, k0 = 0). piv / two / sub: entries k0.. .
template <class R, bool CX, bool FULL>
__global__ void __launch_bounds__(LB_THREADS, 1) lblt_rl_kernel(R* __restrict__ A, i64 rs, i64 cs, int m, int k0, R* __restrict__ sub,
                                                             i64 sds, int rook, int diagonal, LbWs<R> w) {
  constexpr int W = CX ? 2 : 1;
  __shared__ R s_v[LB_WARPS];
  __shared__ long long s_i[LB_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x;
  const i64 warps = (i64)G * LB_WARPS, gw = (i64)blockIdx.x * LB_WARPS + warp;
  const i64 T = (i64)G * LB_THREADS, gt = (i64)blockIdx.x * LB_THREADS + tid;
  const bool leader = blockIdx.x == 0 && tid == 0;
  auto at = [&](i64 i, i64 j) { return A + W * (i * rs + j * cs); };
  auto sd = [&](i64 i) { return sub + W * i * sds; };
  auto nowa = [&](i64, i64) { return (R*)nullptr; };
  FplRec<R>* recA = w.rec;
  FplRec<R>* recB = w.rec + G;
  unsigned long long target = 0;
  auto barrier = [&]() {
    target += G;
    grid_barrier(w.bar, target);
  };
  const R alpha = (R(1) + sqrt(R(17))) * R(0.125);

  // the deferred L columns of pivot s (rows below the block; the update read them unscaled)
  auto scale_cols = [&](const LbPiv<R>& s) {
    if (s.kind == 0) return;
    for (i64 r = s.p + s.kind + gt; r < m; r += T) {
      if (s.kind == 1) {
        sc_st<R, CX>(at(r, s.p), cscale(sc_ld<R, CX>(at(r, s.p)), s.dinv));
      } else {
        Sc<R> w0, w1;
        lb_w<R, CX>(s, sc_ld<R, CX>(at(r, s.p)), sc_ld<R, CX>(at(r, s.p + 1)), w0, w1);
        sc_st<R, CX>(at(r, s.p), w0);
        sc_st<R, CX>(at(r, s.p + 1), w1);
      }
    }
    if (leader && s.kind == 2) sc_st<R, CX>(at(s.p + 1, s.p), Sc<R>{R(0), R(0)});
  };
  // The trailing lower triangle from column c: the update of pivot q (rank1_update / rank2_update, or Full's
  // rank_*_update_and_argmax with its diagonal update), the deferred columns of s, and the records: A = diagonal (abs1, Full:
  // abs2), B = column c below the diagonal (abs1, non-Diag strategies) or Full's strict lower triangle (abs2, column-major).
  auto pass = [&](const LbPiv<R>& q, const LbPiv<R>& s, int c) {
    scale_cols(s);
    R va = R(0), vb = R(0);
    long long ia = LLONG_MAX, ib = LLONG_MAX;
    const i64 nr = (i64)m - c;
    const i64 tr = (nr + LB_TR - 1) / LB_TR;
    const bool full_pass = FULL || q.kind != 0;
    for (i64 t = gw; t < tr * nr; t += warps) {
      const i64 rb = t % tr, j = c + t / tr;
      const i64 i0 = c + rb * LB_TR;
      if (i0 + LB_TR <= j) continue;  // above the diagonal
      if (!full_pass && !(diagonal ? (j >= i0) : (j == c))) continue;
      Sc<R> w0{R(0), R(0)}, w1{R(0), R(0)};
      if (q.kind == 1) {
        w0 = cscale(sc_ld<R, CX>(at(j, q.p)), q.dinv);  // unblocked: w0 = L[j] d; Full: L[j] scaled
      } else if (q.kind == 2) {
        lb_w<R, CX>(q, sc_ld<R, CX>(at(j, q.p)), sc_ld<R, CX>(at(j, q.p + 1)), w0, w1);
      }
#pragma unroll
      for (int u = 0; u < LB_TR / 32; ++u) {
        const i64 i = i0 + lane + 32 * u;
        if (i < j || i >= m) continue;
        R* p = at(i, j);
        Sc<R> a = sc_ld<R, CX>(p);
        if (q.kind == 1) {
          const Sc<R> li = sc_ld<R, CX>(at(i, q.p));
          if (!FULL) {
            a = cfms_conj<R, CX>(a, li, w0);
            if (i == j) a.im = R(0);
          } else if (i > j) {
            const Sc<R> lsi = cscale(li, q.dinv);
            a = csub(a, cscale(cmul<R, CX>(lsi, cconj(w0)), q.dg));
          } else {
            a = Sc<R>{a.re - q.dg * cabs2(w0), R(0)};
          }
          sc_st<R, CX>(p, a);
        } else if (q.kind == 2) {
          const Sc<R> l0 = sc_ld<R, CX>(at(i, q.p)), l1 = sc_ld<R, CX>(at(i, q.p + 1));
          if (!FULL) {
            a = cfms_conj<R, CX>(cfms_conj<R, CX>(a, l0, w0), l1, w1);
          } else {
            a = csub(csub(a, cmul<R, CX>(l0, cconj(w0))), cmul<R, CX>(l1, cconj(w1)));
          }
          if (i == j) a.im = R(0);
          sc_st<R, CX>(p, a);
        }
        if (i == j) {
          const R sc = FULL ? cabs2(a) : cabs1(a);
          if ((FULL || diagonal) && better(sc, (long long)i, va, ia)) {
            va = sc;
            ia = i;
          }
        } else if (FULL) {
          const R sc = cabs2(a);
          const long long ix = i + j * (long long)m;
          if (better(sc, ix, vb, ib)) {
            vb = sc;
            ib = ix;
          }
        } else if (!diagonal && j == c) {
          const R sc = cabs1(a);
          if (better(sc, (long long)i, vb, ib)) {
            vb = sc;
            ib = i;
          }
        }
      }
    }
    // rows ascend within a lane's tile but not across tiles: ties go to the smaller index in the record order
    lb_publish(recA, va, ia, s_v, s_i);
    lb_publish(recB, vb, ib, s_v, s_i);
  };
  // offdiag_argmax (factor.rs:448-460) of column x of the trailing matrix from c: row part A[x, c..x), column part A(x.., x)
  auto oa = [&](int c, int x, FplRec<R>* set) {
    R bv = R(0);
    long long bi = LLONG_MAX;
    for (i64 t = c + gt; t < m; t += T) {
      if (t == x) continue;
      const R v = cabs1(t < x ? sc_ld<R, CX>(at(x, t)) : sc_ld<R, CX>(at(t, x)));
      if (v > bv) {
        bv = v;
        bi = t;
      }
    }
    lb_publish(set, bv, bi, s_v, s_i);
  };
  auto record = [&](int c, int i0, int i1, int npiv) {
    if (leader) {
      w.piv[k0 + c] = k0 + i0;
      w.two[k0 + c] = npiv == 2;
      if (npiv == 2) {
        w.piv[k0 + c + 1] = k0 + i1;
        w.two[k0 + c + 1] = 1;
      }
    }
  };
  // the new pending block after the interchanges; subdiag as the reference writes it
  auto take = [&](int c, int npiv) {
    if (npiv == 1) {
      if (leader) sc_st<R, CX>(sd(c), Sc<R>{R(0), R(0)});
      return lb_one<R, CX>(c, __ldcg(at(c, c)));
    }
    const Sc<R> a10 = sc_ld<R, CX>(at(c + 1, c));
    if (leader) {
      sc_st<R, CX>(sd(c), a10);
      sc_st<R, CX>(sd(c + 1), Sc<R>{R(0), R(0)});
    }
    return lb_two<R, CX>(c, __ldcg(at(c, c)), __ldcg(at(c + 1, c + 1)), a10);
  };

  LbPiv<R> q{}, s{};
  int c = 0;
  R scale_fwd = R(1);
  if (FULL) {
    // norm_max, then the whole matrix scaled by its recip, the first searches fused with the scaling
    R mx = R(0);
    for (i64 e = gt; e < (i64)m * m; e += T) {
      const Sc<R> a = sc_ld<R, CX>(at(e % m, e / m));
      const R v = fmax(fabs(a.re), fabs(a.im));  // norm_max: the largest |re| or |im| (faer-traits simd_abs_max)
      if (v > mx) mx = v;
    }
    lb_publish(recA, mx, 0, s_v, s_i);
    barrier();
    long long ix;
    lb_collect(recA, scale_fwd, ix, s_v, s_i);
    const R scale_bwd = R(1) / scale_fwd;
    barrier();  // recA is reused below
    R va = R(0), vb = R(0);
    long long ia = LLONG_MAX, ib = LLONG_MAX;
    for (i64 e = gt; e < (i64)m * m; e += T) {
      const i64 i = e % m, j = e / m;
      const Sc<R> a = cscale(sc_ld<R, CX>(at(i, j)), scale_bwd);
      sc_st<R, CX>(at(i, j), a);
      const R sc = cabs2(a);
      if (i == j) {
        if (better(sc, (long long)i, va, ia)) {
          va = sc;
          ia = i;
        }
      } else if (i > j && better(sc, (long long)e, vb, ib)) {
        vb = sc;
        ib = e;
      }
    }
    lb_publish(recA, va, ia, s_v, s_i);
    lb_publish(recB, vb, ib, s_v, s_i);
    barrier();
    const R alpha2 = alpha * alpha;
    bool offdiag = true;
    while (c < m) {
      R md, mo;
      long long is, io;
      lb_collect(recA, md, is, s_v, s_i);
      if (is == LLONG_MAX) is = c;
      if (offdiag) {
        lb_collect(recB, mo, io, s_v, s_i);
        if (mo == R(0)) offdiag = false;
      }
      if (!offdiag) {  // factor.rs:402-425: diagonal interchanges only
        const int sdx = (int)is;
        if (sdx != c) {
          for (i64 col = gt; col < c; col += T) {
            const Sc<R> x = sc_ld<R, CX>(at(c, col)), y = sc_ld<R, CX>(at(sdx, col));
            sc_st<R, CX>(at(c, col), y);
            sc_st<R, CX>(at(sdx, col), x);
          }
          if (leader) {
            const Sc<R> x = sc_ld<R, CX>(at(c, c)), y = sc_ld<R, CX>(at(sdx, sdx));
            sc_st<R, CX>(at(c, c), y);
            sc_st<R, CX>(at(sdx, sdx), x);
          }
        }
        if (leader) sc_st<R, CX>(sd(c), Sc<R>{R(0), R(0)});
        record(c, sdx, -1, 1);
        c += 1;
        barrier();
        if (c < m) {
          R bv = R(0);
          long long bi = LLONG_MAX;
          for (i64 t = c + gt; t < m; t += T) {
            const R v = cabs2(sc_ld<R, CX>(at(t, t)));
            if (v > bv) {
              bv = v;
              bi = t;
            }
          }
          lb_publish(recA, bv, bi, s_v, s_i);
          barrier();
        }
        continue;
      }
      int npiv, i0, i1 = -1;
      if (md >= alpha2 * mo) {
        npiv = 1;
        i0 = (int)is;
      } else {
        npiv = 2;
        i0 = (int)(io / m);
        i1 = (int)(io % m);
      }
      if (i0 != c) lb_swap<R, CX>(at, nowa, false, m, c, i0, 0, gt, T, leader);
      if (npiv == 2) {
        barrier();
        if (i1 != c + 1) lb_swap<R, CX>(at, nowa, false, m, c + 1, i1, 0, gt, T, leader);
      }
      record(c, i0, i1, npiv);
      barrier();
      q = take(c, npiv);
      c += npiv;
      if (c < m) {
        pass(q, s, c);
        s = q;
        q.kind = 0;
        barrier();
      }
    }
  } else {
    while (c < m) {
      pass(q, s, c);
      s = q;
      q.kind = 0;
      barrier();
      int i0 = c;
      R gi;
      long long r;
      if (diagonal) {
        R v;
        long long ix;
        lb_collect(recA, v, ix, s_v, s_i);
        if (ix != LLONG_MAX) i0 = (int)ix;
        oa(c, i0, recB);
        barrier();
      }
      lb_collect(recB, gi, r, s_v, s_i);
      int npiv = 1, i1 = -1;
      bool nothing = false;
      if (c + 1 == m || gi == R(0)) {
        nothing = true;
      } else if (fabs(__ldcg(at(i0, i0))) >= alpha * gi) {
        npiv = 1;
      } else {
        i1 = (int)r;
        if (rook) {
          for (int cand = 0;; ++cand) {
            FplRec<R>* set = lb_cand(w.rec, cand);
            oa(c, i1, set);
            barrier();
            R gr;
            long long sx;
            lb_collect(set, gr, sx, s_v, s_i);
            if (sx == LLONG_MAX) sx = c;
            if (cabs1(sc_ld<R, CX>(at(i1, i1))) >= alpha * gr) {
              npiv = 1;
              i0 = i1;
              i1 = -1;
              break;
            } else if (gi == gr) {
              npiv = 2;
              break;
            } else {
              i0 = i1;
              i1 = (int)sx;
              gi = gr;
            }
          }
        } else {
          FplRec<R>* set = lb_cand(w.rec, 0);
          oa(c, i1, set);
          barrier();
          R gr;
          long long sx;
          lb_collect(set, gr, sx, s_v, s_i);
          if (fabs(__ldcg(at(i0, i0))) >= (alpha * gr) * (gr / gi)) {
            npiv = 1;
          } else if (fabs(__ldcg(at(i1, i1))) >= alpha * gr) {
            npiv = 1;
            i0 = i1;
            i1 = -1;
          } else {
            npiv = 2;
          }
        }
      }
      if (npiv == 2 && i0 > i1) {
        const int t = i0;
        i0 = i1;
        i1 = t;
      }
      if (i0 != c) lb_swap<R, CX>(at, nowa, false, m, c, i0, 0, gt, T, leader);
      if (npiv == 2) {
        barrier();
        if (i1 != c + 1) lb_swap<R, CX>(at, nowa, false, m, c + 1, i1, 0, gt, T, leader);
      }
      record(c, i0, i1, npiv);
      barrier();
      if (!nothing) q = take(c, npiv);
      c += npiv;
    }
  }
  // the last deferred columns (two blocks at most, disjoint columns)
  scale_cols(s);
  scale_cols(q);
  if (FULL) {
    barrier();
    for (i64 t = gt; t < m; t += T) {
      sc_st<R, CX>(at(t, t), cscale(sc_ld<R, CX>(at(t, t)), scale_fwd));
      sc_st<R, CX>(sd(t), cscale(sc_ld<R, CX>(sd(t)), scale_fwd));
    }
  }
}

// the imaginary part of the diagonal of an n x n block set to zero (as_real)
template <class R>
__global__ void lblt_real_diag_kernel(R* __restrict__ A, i64 rs, i64 cs, i64 n) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) A[2 * (i * rs + i * cs) + 1] = R(0);
}

// out <- identity (L == null) or the unit-lower L with zeros above (reconstruct.rs:35-37)
template <class R, bool CX>
__global__ void lblt_init_kernel(R* __restrict__ out, i64 ors, i64 ocs, const R* __restrict__ L, i64 lrs, i64 lcs, i64 n) {
  constexpr int W = CX ? 2 : 1;
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * n) return;
  const i64 i = e % n, j = e / n;
  R* o = out + W * (i * ors + j * ocs);
  if (i > j && L != nullptr) {
    const R* l = L + W * (i * lrs + j * lcs);
    o[0] = l[0];
    if (CX) o[1] = l[1];
  } else {
    o[0] = i == j ? R(1) : R(0);
    if (CX) o[1] = R(0);
  }
}

// the 1 x 1 / 2 x 2 block solve of solve.rs:63-96 on column-major X (n x k); dg / sd: compact diag / subdiag; kind: 0 a 1 x 1
// block, 1 the first column of a 2 x 2 block, 2 its second
template <class R, bool CX>
__global__ void lblt_block_solve_kernel(R* __restrict__ X, i64 n, i64 k, const R* __restrict__ dg, const R* __restrict__ sdg,
                                        const int* __restrict__ kind, int conj) {
  constexpr int W = CX ? 2 : 1;
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * k) return;
  const i64 i = e % n, j = e / n;
  const int kd = kind[i];
  if (kd == 2) return;
  R* x0 = X + W * (i + j * n);
  if (kd == 0) {
    const R dinv = R(1) / dg[W * i];
    x0[0] *= dinv;
    if (CX) x0[1] *= dinv;
    return;
  }
  R* x1 = X + W * (i + 1 + j * n);
  Sc<R> s{sdg[W * i], CX ? sdg[W * i + 1] : R(0)};
  if (conj) s = cconj(s);
  Sc<R> rk;  // recip(s)
  if (!CX) {
    rk = Sc<R>{R(1) / s.re, R(0)};
  } else {
    const R den = s.re * s.re + s.im * s.im;
    rk = Sc<R>{s.re / den, -s.im / den};
  }
  const Sc<R> ak = cscale(cconj(rk), dg[W * i]);
  const Sc<R> akp1 = cscale(rk, dg[W * (i + 1)]);
  const R denom = R(1) / (cmul<R, CX>(ak, akp1).re - R(1));
  const Sc<R> xk = cmul<R, CX>(Sc<R>{x0[0], CX ? x0[1] : R(0)}, cconj(rk));
  const Sc<R> xkp1 = cmul<R, CX>(Sc<R>{x1[0], CX ? x1[1] : R(0)}, rk);
  const Sc<R> y0 = cscale(csub(cmul<R, CX>(akp1, xk), xkp1), denom);
  const Sc<R> y1 = cscale(csub(cmul<R, CX>(ak, xkp1), xk), denom);
  x0[0] = y0.re;
  x1[0] = y1.re;
  if (CX) {
    x0[1] = y0.im;
    x1[1] = y1.im;
  }
}

// out <- out B, column blocks by `kind` (reconstruct.rs:38-60): the diagonal of B is Re L[j, j], the off-diagonal entry subdiag[j]
template <class R, bool CX>
__global__ void lblt_lb_kernel(R* __restrict__ out, i64 ors, i64 ocs, const R* __restrict__ L, i64 lrs, i64 lcs, i64 n,
                               const R* __restrict__ sdg, const int* __restrict__ kind) {
  constexpr int W = CX ? 2 : 1;
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * n) return;
  const i64 i = e % n, j = e / n;
  const int kd = kind[j];
  if (kd == 2) return;
  R* o0 = out + W * (i * ors + j * ocs);
  const R ak = L[W * (j * lrs + j * lcs)];
  if (kd == 0) {
    o0[0] *= ak;
    if (CX) o0[1] *= ak;
    return;
  }
  R* o1 = out + W * (i * ors + (j + 1) * ocs);
  const R akp1 = L[W * ((j + 1) * lrs + (j + 1) * lcs)];
  const Sc<R> s{sdg[W * j], CX ? sdg[W * j + 1] : R(0)};
  const Sc<R> xk{o0[0], CX ? o0[1] : R(0)}, xkp1{o1[0], CX ? o1[1] : R(0)};
  const Sc<R> y0 = cscale(xk, ak), y0b = cmul<R, CX>(xkp1, s);
  const Sc<R> y1 = cscale(xkp1, akp1), y1b = cmul<R, CX>(xk, cconj(s));
  o0[0] = y0.re + y0b.re;
  o1[0] = y1.re + y1b.re;
  if (CX) {
    o0[1] = y0.im + y0b.im;
    o1[1] = y1.im + y1b.im;
  }
}

template <class K>
int lb_grid(K kernel, cudaStream_t st) {
  int occ = 0;
  FB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, LB_THREADS, 0));
  FB_ASSERT(occ > 0, "LBLT kernel cannot be resident");
  return stream_sms(st) * std::min(occ, 2);
}

}  // namespace

// Pivoting strategies, faer-ffi's PivotingStrategy discriminants
enum LbStrategy : int { LB_PARTIAL = 0, LB_PARTIAL_DIAG = 1, LB_ROOK = 2, LB_ROOK_DIAG = 3, LB_FULL = 4 };

// In-place LBL^H of A (lower triangle; Full also scales the strict upper triangle). sub: n x 1 view of subdiag (device).
// pivots (host, n entries): the pivot row of each column, TOP_BIT set for the columns of 2 x 2 blocks.
template <class R, bool CX>
void lblt_in_place_t(cudaStream_t st, View<R> A, View<R> sub, int strategy, i64 block_size, std::vector<unsigned long long>& pivots) {
  constexpr int Wd = CX ? 2 : 1;
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n && sub.nrows == n, "LBLT shape mismatch");
  FB_ASSERT(n < (i64)INT_MAX / 2, "LBLT: dimension too large");
  pivots.assign((size_t)n, 0);
  if (n == 0) return;
  const bool rook = strategy == LB_ROOK || strategy == LB_ROOK_DIAG;
  const bool diagonal = strategy == LB_PARTIAL_DIAG || strategy == LB_ROOK_DIAG;
  i64 bs = block_size;
  if (bs < 2 || n <= bs) bs = 0;

  const int g_rl = std::min(lb_grid(lblt_rl_kernel<R, CX, false>, st), lb_grid(lblt_rl_kernel<R, CX, true>, st));
  const int g_pn = lb_grid(lblt_panel_kernel<R, CX>, st);
  const int gmax = std::max(g_rl, g_pn);
  const size_t rec_bytes = 3 * (size_t)gmax * sizeof(FplRec<R>);
  const size_t bytes = rec_bytes + (size_t)n * 8 + (size_t)n * 4 + 64;
  char* buf = (char*)ws_alloc(bytes);
  LbWs<R> w;
  w.rec = (FplRec<R>*)buf;
  w.piv = (long long*)(buf + rec_bytes);
  w.two = (int*)(w.piv + n);
  w.bar = (unsigned long long*)(((uintptr_t)(w.two + n) + 7) & ~(uintptr_t)7);
  w.kstep = (int*)(w.bar + 1);
  R* Wb = bs > 0 ? (R*)ws_alloc((size_t)n * (size_t)bs * Wd * sizeof(R)) : nullptr;
  const int rk = rook, dg = diagonal;

  auto launch_rl = [&](i64 k, bool full) {
    const int m = (int)(n - k);
    const int G = (int)std::min<i64>(g_rl, std::max<i64>(1, (i64)m * m / (64 * 1024) + 1));
    FB_CUDA_CHECK(cudaMemsetAsync(w.bar, 0, sizeof(unsigned long long), st));
    R* Ap = A.ptr + Wd * (k * A.rs + k * A.cs);
    R* sp = sub.ptr + Wd * k * sub.rs;
    i64 rs = A.rs, cs = A.cs, sds = sub.rs;
    int mi = m, ki = (int)k, r_ = rk, d_ = dg;
    void* args[] = {&Ap, &rs, &cs, &mi, &ki, &sp, &sds, &r_, &d_, &w};
    void* fn = full ? (void*)lblt_rl_kernel<R, CX, true> : (void*)lblt_rl_kernel<R, CX, false>;
    FB_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(G), dim3(LB_THREADS), args, 0, st));
    note_launch();
  };

  if (strategy == LB_FULL) {
    launch_rl(0, true);
  } else {
    i64 k = 0;
    while (k < n) {
      i64 next;
      if (bs < 2 || n - k <= bs) {
        launch_rl(k, false);
        next = n;
      } else {
        const i64 m = n - k;
        const int G = (int)std::min<i64>(g_pn, (m + LB_THREADS - 1) / LB_THREADS);
        FB_CUDA_CHECK(cudaMemsetAsync(w.bar, 0, sizeof(unsigned long long), st));
        {
          R* Ap = A.ptr + Wd * (k * A.rs + k * A.cs);
          R* sp = sub.ptr + Wd * k * sub.rs;
          i64 rs = A.rs, cs = A.cs, ldw = m, sds = sub.rs;
          int mi = (int)m, ki = (int)k, bi = (int)bs, r_ = rk, d_ = dg;
          void* args[] = {&Ap, &rs, &cs, &mi, &ki, &bi, &Wb, &ldw, &sp, &sds, &r_, &d_, &w};
          FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)lblt_panel_kernel<R, CX>, dim3(G), dim3(LB_THREADS), args, 0, st));
          note_launch();
        }
        int ks = 0;
        FB_CUDA_CHECK(cudaMemcpyAsync(&ks, w.kstep, sizeof(int), cudaMemcpyDeviceToHost, st));
        FB_CUDA_CHECK(cudaStreamSynchronize(st));
        const i64 mm = m - ks;
        if (mm > 0) {
          View<R> dst = sub_t<R, CX>(A, k + ks, k + ks, mm, mm);
          View<const R> Wv{Wb + Wd * (i64)ks, mm, ks, 1, m};
          const View<const R> Al = cview(sub_t<R, CX>(A, k + ks, k, mm, ks));
          gemm_t<R, CX>(st, dst, STRICT_LOWER, 1, Wv, RECT, false, Al.t(), RECT, true, R(-1));  // dst(strict lower) -= W Al^H
          if (CX) {
            lblt_real_diag_kernel<R><<<grid_1d(mm), 256, 0, st>>>(dst.ptr, dst.rs, dst.cs, mm);
            FB_CUDA_CHECK(cudaGetLastError());
            note_launch();
          }
        }
        next = k + ks;
      }
      piv_laswp_t<R, CX>(st, A, k, next - k, w.piv);
      k = next;
    }
  }
  std::vector<long long> piv((size_t)n);
  std::vector<int> two((size_t)n);
  FB_CUDA_CHECK(cudaMemcpyAsync(piv.data(), w.piv, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(two.data(), w.two, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (Wb) ws_free(Wb);
  ws_free(buf);
  for (i64 i = 0; i < n; ++i)
    pivots[(size_t)i] = (unsigned long long)piv[(size_t)i] | (two[(size_t)i] ? (1ull << 63) : 0ull);
}

// block kinds of solve.rs:63-96 / reconstruct.rs:38-60 from the subdiagonal (host, compact): 0 a 1 x 1 block, 1 / 2 the columns
// of a 2 x 2 block (subdiag[i] != 0 opens one)
template <class R, bool CX>
std::vector<int> lb_kinds(const std::vector<unsigned char>& sd, i64 n) {
  std::vector<int> kind((size_t)n, 0);
  const R* s = (const R*)sd.data();
  for (i64 i = 0; i < n;) {
    const bool zero = s[(CX ? 2 : 1) * i] == R(0) && (!CX || s[2 * i + 1] == R(0));
    if (zero) {
      i += 1;
    } else {
      FB_ASSERT(i + 1 < n, "LBLT: a 2 x 2 block starts at the last row (subdiag[n - 1] != 0)");
      kind[(size_t)i] = 1;
      kind[(size_t)i + 1] = 2;
      i += 2;
    }
  }
  return kind;
}

// rhs <- A^-1 rhs (conj(A)^-1 rhs) from the factors (solve.rs:35-104). dg / sd: host compact diag / subdiag; pf / pb: host perms.
template <class R, bool CX>
void lblt_solve_t(cudaStream_t st, View<const R> L, const std::vector<unsigned char>& dgv, const std::vector<unsigned char>& sdv,
                  const long long* pf, const long long* pb, bool conj, View<R> rhs) {
  constexpr int Wd = CX ? 2 : 1;
  const i64 n = L.nrows, k = rhs.ncols;
  if (n == 0 || k == 0) return;
  const std::vector<int> kind = lb_kinds<R, CX>(sdv, n);
  const size_t vb = (size_t)n * Wd * sizeof(R);
  char* aux = (char*)ws_alloc(16 * (size_t)n + 2 * vb + 4 * (size_t)n + 64);
  long long* d_p = (long long*)aux;
  R* d_dg = (R*)(aux + 16 * (size_t)n);
  R* d_sd = (R*)((char*)d_dg + vb);
  int* d_kind = (int*)((char*)d_sd + vb);
  R* tmp = (R*)ws_alloc((size_t)n * (size_t)k * Wd * sizeof(R));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p, pf, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p + n, pb, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_dg, dgv.data(), vb, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_sd, sdv.data(), vb, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_kind, kind.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  View<R> X{tmp, n, k, 1, n};
  piv_gather_rows_t<R, CX>(st, X, cview(rhs), d_p);
  solve_lower_t<R, CX>(st, L, true, conj, X);
  lblt_block_solve_kernel<R, CX><<<grid_1d(n * k), 256, 0, st>>>(tmp, n, k, d_dg, d_sd, d_kind, conj ? 1 : 0);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  solve_upper_t<R, CX>(st, L.t(), true, !conj, X);
  piv_gather_rows_t<R, CX>(st, rhs, cview(X), d_p + n);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(tmp);
  ws_free(aux);
}

// out <- P^T (L B L^H) P in the lower triangle, L B in the strict upper triangle (reconstruct.rs:12-87). pb: host perm_bwd.
template <class R, bool CX>
void lblt_reconstruct_t(cudaStream_t st, View<R> out, View<const R> L, const std::vector<unsigned char>& sdv, const long long* pb) {
  constexpr int Wd = CX ? 2 : 1;
  const i64 n = L.nrows;
  if (n == 0) return;
  const std::vector<int> kind = lb_kinds<R, CX>(sdv, n);
  const size_t vb = (size_t)n * Wd * sizeof(R);
  char* aux = (char*)ws_alloc(8 * (size_t)n + vb + 4 * (size_t)n + 64);
  long long* d_p = (long long*)aux;
  R* d_sd = (R*)(aux + 8 * (size_t)n);
  int* d_kind = (int*)((char*)d_sd + vb);
  R* tmp = (R*)ws_alloc((size_t)n * (size_t)n * Wd * sizeof(R));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_p, pb, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_sd, sdv.data(), vb, cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(d_kind, kind.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  lblt_init_kernel<R, CX><<<grid_1d(n * n), 256, 0, st>>>(out.ptr, out.rs, out.cs, L.ptr, L.rs, L.cs, n);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  lblt_lb_kernel<R, CX><<<grid_1d(n * n), 256, 0, st>>>(out.ptr, out.rs, out.cs, L.ptr, L.rs, L.cs, n, d_sd, d_kind);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  View<R> Tm{tmp, n, n, 1, n};
  gemm_t<R, CX>(st, Tm, TRI_LOWER, 0, L, UNIT_LOWER, false, cview(out).t(), RECT, true, R(1));  // tmp(lower) = L(unit lower) X^H
  piv_sym_gather_t<R, CX>(st, out, tmp, n, d_p);
  if (CX) {
    lblt_real_diag_kernel<R><<<grid_1d(n), 256, 0, st>>>(out.ptr, out.rs, out.cs, n);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(tmp);
  ws_free(aux);
}

// out <- identity, then the solve (inverse.rs:11-42)
template <class R, bool CX>
void lblt_inverse_t(cudaStream_t st, View<R> out, View<const R> L, const std::vector<unsigned char>& dgv,
                    const std::vector<unsigned char>& sdv, const long long* pf, const long long* pb) {
  const i64 n = L.nrows;
  if (n == 0) return;
  lblt_init_kernel<R, CX><<<grid_1d(n * n), 256, 0, st>>>(out.ptr, out.rs, out.cs, nullptr, 0, 0, n);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  lblt_solve_t<R, CX>(st, L, dgv, sdv, pf, pb, false, out);
}

}  // namespace fb

// ---- C ABI (faer-ffi/src/lib.rs:1288-1420; declarations in include/faer_b200_lblt.h) ----
using namespace fb;

namespace {

// a VecRef / VecMut of either residency and any positive stride, as compact host bytes
std::vector<unsigned char> lb_read_vec(const void* p, size_t n, ptrdiff_t stride, size_t es) {
  std::vector<unsigned char> out(n * es);
  if (n == 0) return out;
  FB_ASSERT(p != nullptr, "null vector");
  FB_ASSERT(stride >= 1 || n == 1, "LBLT vectors need a positive stride");
  const size_t pitch = (size_t)(n == 1 ? 1 : stride) * es;
  if (is_device_pointer(p)) FB_CUDA_CHECK(cudaMemcpy2D(out.data(), es, p, pitch, es, n, cudaMemcpyDeviceToHost));
  else
    for (size_t i = 0; i < n; ++i) memcpy(out.data() + i * es, (const char*)p + i * pitch, es);
  return out;
}

template <class R, bool CX>
FaerV0_24_LbltStatus lblt_factor_entry(FaerV0_24_MatMut A, FaerV0_24_VecMut subdiag, FaerV0_24_SliceMut perm_fwd,
                                       FaerV0_24_SliceMut perm_bwd, FaerV0_24_LbltParams params, int idx_bytes) {
  FB_ENTRY();
  FB_ASSERT((int)params.pivoting >= 0 && (int)params.pivoting <= 4, "LbltParams.pivoting is not a PivotingStrategy");
  const size_t n = A.nrows;
  FB_ASSERT(A.ncols == n && subdiag.len == n && perm_fwd.len == n && perm_bwd.len == n, "LBLT shape mismatch");
  FaerV0_24_LbltStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_LbltStatus_Ok;
  if (n == 0) return out;
  FB_ASSERT(perm_fwd.ptr != nullptr && perm_bwd.ptr != nullptr, "null permutation slice");
  FB_ASSERT(subdiag.ptr != nullptr && (subdiag.stride >= 1 || n == 1), "LBLT subdiag needs a positive stride");
  cudaStream_t st = current_stream();
  const size_t es = (CX ? 2 : 1) * sizeof(R);
  StagedMat a = stage<R, CX>(A, true, st);
  const i64 sstride = n == 1 ? 1 : (i64)subdiag.stride;
  StagedMat s(subdiag.ptr, (i64)n, 1, sstride, (i64)n * sstride, es, true, true, st);
  std::vector<unsigned long long> piv;
  lblt_in_place_t<R, CX>(st, a.view<R>(), s.view<R>(), (int)params.pivoting, (i64)params.block_size, piv);
  finish_all(st, {&a, &s});
  // perm_fwd / perm_bwd / transposition_count from the pivots (factor.rs:1214-1227)
  std::vector<long long> trans(n), fwd, bwd;
  size_t count = 0;
  for (size_t i = 0; i < n; ++i) {
    trans[i] = (long long)(piv[i] & ~(1ull << 63));
    count += (size_t)trans[i] != i;
  }
  perm_from_transpositions(n, trans, fwd, bwd);
  write_perm(perm_fwd.ptr, fwd, idx_bytes);
  write_perm(perm_bwd.ptr, bwd, idx_bytes);
  out.ok.transposition_count = count;
  return out;
}

template <class R, bool CX>
void lblt_solve_entry(FaerV0_24_MatRef L, FaerV0_24_VecRef diag, FaerV0_24_VecRef subdiag, FaerV0_24_Conj A_conj,
                      FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd, FaerV0_24_MatMut rhs, int idx_bytes) {
  FB_ENTRY();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && rhs.nrows == n && diag.len == n && subdiag.len == n, "LBLT solve shape mismatch");
  FB_ASSERT(std::min(perm_fwd.len, perm_bwd.len) == n, "LBLT solve: permutation length mismatch");
  if (n == 0 || rhs.ncols == 0) return;
  cudaStream_t st = current_stream();
  const size_t es = (CX ? 2 : 1) * sizeof(R);
  const std::vector<long long> pf = read_perm_checked(perm_fwd, n, idx_bytes), pb = read_perm_checked(perm_bwd, n, idx_bytes);
  const std::vector<unsigned char> dg = lb_read_vec(diag.ptr, n, diag.stride, es), sd = lb_read_vec(subdiag.ptr, n, subdiag.stride, es);
  StagedMat l = stage<R, CX>(L, st);
  StagedMat r = stage<R, CX>(rhs, true, st);
  lblt_solve_t<R, CX>(st, l.view<const R>(), dg, sd, pf.data(), pb.data(), A_conj == FaerV0_24_Conj_Yes, r.view<R>());
  finish_all(st, {&l, &r});
}

template <class R, bool CX>
void lblt_recon_entry(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_VecRef diag, FaerV0_24_VecRef subdiag,
                      FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd, int idx_bytes, bool inverse) {
  FB_ENTRY();
  const size_t n = L.nrows;
  FB_ASSERT(L.ncols == n && A.nrows == n && A.ncols == n && diag.len == n && subdiag.len == n,
            "LBLT reconstruct / inverse shape mismatch");
  FB_ASSERT(std::min(perm_fwd.len, perm_bwd.len) == n, "LBLT reconstruct / inverse: permutation length mismatch");
  if (n == 0) return;
  cudaStream_t st = current_stream();
  const size_t es = (CX ? 2 : 1) * sizeof(R);
  const std::vector<long long> pf = read_perm_checked(perm_fwd, n, idx_bytes), pb = read_perm_checked(perm_bwd, n, idx_bytes);
  const std::vector<unsigned char> sd = lb_read_vec(subdiag.ptr, n, subdiag.stride, es);
  // every entry of the output is written
  StagedMat a = stage<R, CX>(A, false, st);
  StagedMat l = stage<R, CX>(L, st);
  if (inverse) {
    const std::vector<unsigned char> dg = lb_read_vec(diag.ptr, n, diag.stride, es);
    lblt_inverse_t<R, CX>(st, a.view<R>(), l.view<const R>(), dg, sd, pf.data(), pb.data());
  } else {
    lblt_reconstruct_t<R, CX>(st, a.view<R>(), l.view<const R>(), sd, pb.data());
  }
  finish_all(st, {&a, &l});
}

}  // namespace

extern "C" {

// Scratch layouts are the reference's (factor.rs:1128-1140, solve.rs:11-18, reconstruct.rs:4-10, inverse.rs:3-9); the GPU paths
// keep their workspace in the device pool and ignore `mem`.
#define FB_LBLT_FFI(SUF, R, CX, IT, BYTES)                                                                                            \
  FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par, FaerV0_24_LbltParams params) { \
    (void)par;                                                                                                                        \
    size_t bs = params.block_size;                                                                                                    \
    if (bs < 2 || dim <= bs) bs = 0;                                                                                                  \
    /* StackReq::new::<usize>(dim).and(temp_mat_scratch::<T>(dim, bs)) */                                                             \
    return layout_and(FaerV0_24_Layout{dim * sizeof(size_t), alignof(size_t)}, dim * bs * (CX ? 2 : 1) * sizeof(R));                  \
  }                                                                                                                                   \
  FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_VecMut subdiag,                   \
                                                                       FaerV0_24_SliceMut perm_fwd, FaerV0_24_SliceMut perm_bwd,     \
                                                                       FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                    \
                                                                       FaerV0_24_LbltParams params) {                                \
    (void)par; (void)mem;                                                                                                             \
    return lblt_factor_entry<R, CX>(A, subdiag, perm_fwd, perm_bwd, params, BYTES);                                                   \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_##IT##_##SUF(size_t dim, size_t rhs_ncols, FaerV0_24_Par par) {          \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{dim * rhs_ncols * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, rhs_ncols) */               \
  }                                                                                                                                   \
  void libfaer_v0_23_lblt_solve_in_place_##IT##_##SUF(FaerV0_24_MatRef L, FaerV0_24_VecRef diag, FaerV0_24_VecRef subdiag,             \
                                                      FaerV0_24_Conj A_conj, FaerV0_24_SliceRef perm_fwd,                             \
                                                      FaerV0_24_SliceRef perm_bwd, FaerV0_24_MatMut rhs, FaerV0_24_Par par,           \
                                                      FaerV0_24_MemAlloc mem) {                                                       \
    (void)par; (void)mem;                                                                                                             \
    lblt_solve_entry<R, CX>(L, diag, subdiag, A_conj, perm_fwd, perm_bwd, rhs, BYTES);                                                \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                              \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{dim * dim * (CX ? 2 : 1) * sizeof(R), 64}; /* temp_mat_scratch::<T>(dim, dim) */                           \
  }                                                                                                                                   \
  void libfaer_v0_23_lblt_reconstruct_##IT##_##SUF(FaerV0_24_MatMut A, FaerV0_24_MatRef L, FaerV0_24_VecRef diag,                     \
                                                   FaerV0_24_VecRef subdiag, FaerV0_24_SliceRef perm_fwd,                             \
                                                   FaerV0_24_SliceRef perm_bwd, FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {          \
    (void)par; (void)mem;                                                                                                             \
    lblt_recon_entry<R, CX>(A, L, diag, subdiag, perm_fwd, perm_bwd, BYTES, false);                                                   \
  }                                                                                                                                   \
  FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_##IT##_##SUF(size_t dim, FaerV0_24_Par par) {                                  \
    (void)par;                                                                                                                        \
    return FaerV0_24_Layout{dim * dim * (CX ? 2 : 1) * sizeof(R), 64}; /* solve_in_place_scratch(dim, dim) */                          \
  }                                                                                                                                   \
  void libfaer_v0_23_lblt_inverse_##IT##_##SUF(FaerV0_24_MatMut A_inv, FaerV0_24_MatRef L, FaerV0_24_VecRef diag,                     \
                                               FaerV0_24_VecRef subdiag, FaerV0_24_SliceRef perm_fwd, FaerV0_24_SliceRef perm_bwd,    \
                                               FaerV0_24_Par par, FaerV0_24_MemAlloc mem) {                                           \
    (void)par; (void)mem;                                                                                                             \
    lblt_recon_entry<R, CX>(A_inv, L, diag, subdiag, perm_fwd, perm_bwd, BYTES, true);                                                \
  }
#define FB_LBLT_DTYPE(SUF, R, CX)                                                                                                 \
  FaerV0_24_LbltParams libfaer_v0_23_LbltParams_##SUF(void) { /* factor.rs:903-910 */                                             \
    return FaerV0_24_LbltParams{FaerV0_24_PivotingStrategy_PartialDiag, 128 * 128, 64};                                           \
  }                                                                                                                               \
  FB_LBLT_FFI(SUF, R, CX, u32, 4)                                                                                                 \
  FB_LBLT_FFI(SUF, R, CX, u64, 8)
FB_LBLT_DTYPE(f64, double, false)
FB_LBLT_DTYPE(f32, float, false)
FB_LBLT_DTYPE(c64, double, true)
FB_LBLT_DTYPE(c32, float, true)
#undef FB_LBLT_DTYPE
#undef FB_LBLT_FFI

}  // extern "C"
