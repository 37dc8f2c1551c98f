// Double-double (fx128 / cx128) Householder QR and block-Householder sequences: the shared blocked driver of qr_blocked.cuh on the
// dd GEMM and triangular solves, with a cooperative dd panel kernel as its unblocked leaf.
//
// The leaf is qr_in_place_unblocked (qr/no_pivoting/factor.rs:11-86) with its column-skipping rank logic (reflectors written out
// of place into column `row`, the zero fill of factor.rs:33-38), applied to sub-panels of at most QD_PW columns; when a leaf spans
// more columns (block size 1, or a matrix under the blocking threshold), each sub-panel's reflectors reach the columns to its
// right as one block reflector, as in qr.cu's general driver. In dd arithmetic (dd.cuh):
//   householder.rs:59-107        tau = 1/2 (1 + (tail_norm |1 / (head + signed_norm)|)^2), +inf when the tail vanishes, and the
//                                head flushed to zero below min_positive; |.| and hypot are faer's abs_impl
//   reductions/norm_l2.rs        three scaled accumulators with fx128's sqrt_min_positive / sqrt_max_positive
//   factor.rs:41-83              the rank test with fx128's eps
// The rows of the panel are sliced over at most one CTA per SM (fewer when few rows remain, down to one CTA); the slices stay in
// global memory (L2). Each column has one grid-wide exchange: every CTA publishes its partial norm accumulators (above and below
// the pivot row) and its partial dots with the panel's remaining columns, and the CTA owning the pivot row publishes that row.
// After the barrier every CTA reduces the partials in the same fixed order, so all of them compute identical scalars and take the
// same skip / advance decision, and two identical calls give identical bits.
#include <algorithm>

#include "panel_common.cuh"  // before dd.cuh: its fb::__ldcg(const dd*) would hide the builtin overloads t_ldcg calls
#include "dd.cuh"
#include "qr_blocked.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

constexpr int QD_PW = 16;                 // panel columns per launch
constexpr int QD_THREADS = 256;           // 16 row groups x 16 column lanes
constexpr int QD_NWARP = QD_THREADS / 32;
constexpr int QD_NR = 2 * QD_PW + 6;      // per-CTA record: dots (re, im) of 16 columns, tail s / m / b, above s / m / b
constexpr int QD_MIN_ROWS = 128;          // the grid shrinks so that every CTA keeps at least this many rows

template <bool CX>
__device__ __forceinline__ cdd qd_ld(const dd* p, i64 off) {
  return CX ? cdd{p[2 * off], p[2 * off + 1]} : cdd{p[off], dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ void qd_st(dd* p, i64 off, cdd v) {
  if (CX) {
    p[2 * off] = v.re;
    p[2 * off + 1] = v.im;
  } else {
    p[off] = v.re;
  }
}
template <bool CX>
__device__ __forceinline__ cdd qd_mul(cdd a, cdd b) {
  return CX ? a * b : cdd{a.re * b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd qd_add(cdd a, cdd b) {
  return CX ? a + b : cdd{a.re + b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd qd_conj(cdd a) {
  return CX ? cdd_conj(a) : a;
}
template <bool CX>
__device__ __forceinline__ dd qd_abs(cdd a) {
  return CX ? cdd_abs(a) : fabs(a.re);
}
template <bool CX>
__device__ __forceinline__ cdd qd_recip(cdd a) {
  return CX ? cdd_recip_scaled(a) : cdd{dd_recip(a.re), dd(0.0)};
}
__device__ __forceinline__ dd qd_shfl_xor(dd v, int off) {
  return dd(__shfl_xor_sync(0xffffffffu, v.hi, off), __shfl_xor_sync(0xffffffffu, v.lo, off));
}
// dd addition is commutative, so the xor butterfly leaves the same bits in every lane
__device__ __forceinline__ dd qd_warp_sum(dd v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = v + qd_shfl_xor(v, off);
  return v;
}
// norm_l2.rs:161-172
__device__ __forceinline__ dd qd_norm_select(dd s, dd m, dd b, dd sml, dd big) {
  if (s >= dd(1.0)) return sqrt(s) * big;
  if (m >= dd(1.0)) return sqrt(m);
  return sqrt(b) * sml;
}
// (x sml)^2, x^2, (x big)^2 of the modulus of x, added to the three accumulators
template <bool CX>
__device__ __forceinline__ void qd_norm_add(dd* acc, cdd x, dd sml, dd big) {
  const dd rs = x.re * sml, rm = x.re, rb = x.re * big;
  acc[0] = dd_mul_add(rs, rs, acc[0]);
  acc[1] = dd_mul_add(rm, rm, acc[1]);
  acc[2] = dd_mul_add(rb, rb, acc[2]);
  if (CX) {
    const dd is = x.im * sml, im = x.im, ib = x.im * big;
    acc[0] = dd_mul_add(is, is, acc[0]);
    acc[1] = dd_mul_add(im, im, acc[1]);
    acc[2] = dd_mul_add(ib, ib, acc[2]);
  }
}

struct QdScratch {
  dd* part;                 // [2][G][QD_NR], by column parity
  dd* rowv;                 // [2][QD_PW] complex entries (2 dd each), by column parity
  unsigned long long* bar;  // grid barrier counter, zeroed before each launch
  int* out_row;
};

// Columns [c0, c0 + w) of A (m rows) from pivot row `row0`; the reflector taus go to H[row * h_stride] (rows < row_end).
// CTA b owns the rows [row0 + b * rpc, row0 + (b + 1) * rpc) of the panel; the rows above row0 only enter the column norms.
template <bool CX>
__global__ void __launch_bounds__(QD_THREADS) qr_panel_dd_kernel(dd* __restrict__ A, i64 rs, i64 cs, int m, int c0, int w, int row0,
                                                                 int row_end, dd* __restrict__ H, i64 h_stride, int rpc, QdScratch sc) {
  __shared__ dd s_norm[QD_NWARP][6];
  __shared__ cdd s_dot[QD_NWARP][QD_PW];
  __shared__ dd tot[QD_NR];
  __shared__ cdd s_row[QD_PW];
  __shared__ cdd s_k[QD_PW];
  __shared__ cdd s_inv, s_head;
  __shared__ dd s_tau_inv;
  __shared__ int s_action, s_scale;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tl = tid & 15, rg = tid >> 4;
  const int G = gridDim.x, bid = blockIdx.x;
  const int r_lo = row0 + bid * rpc, r_hi = min(m, r_lo + rpc);
  const dd sml = dd_sqrt_min_positive(), big = dd_sqrt_max_positive(), min_pos = dd_min_positive();
  const dd zero(0.0);
  const cdd czero{zero, zero};
  const int cend = c0 + w;

  unsigned long long nbar = 0;
  int row = row0;
  for (int col = c0; col < cend && row < row_end; ++col) {
    const int par = col & 1;
    // ---- phase A: partial norms and dots over this CTA's rows ----
    dd acc[6] = {zero, zero, zero, zero, zero, zero};  // tail s / m / b, above s / m / b
    cdd dacc = czero;
    const int c = col + 1 + tl;
    for (int i = r_lo + rg; i < r_hi; i += QD_THREADS / QD_PW) {
      const cdd x = qd_ld<CX>(A, (i64)i * rs + (i64)col * cs);
      if (i > row) {
        if (c < cend) dacc = qd_add<CX>(qd_mul<CX>(qd_conj<CX>(x), qd_ld<CX>(A, (i64)i * rs + (i64)c * cs)), dacc);
        if (tl == 0) qd_norm_add<CX>(acc, x, sml, big);
      } else if (i < row && tl == 0) {
        qd_norm_add<CX>(acc + 3, x, sml, big);
      }
    }
    for (int i = bid * QD_THREADS + tid; i < row0; i += G * QD_THREADS)
      qd_norm_add<CX>(acc + 3, qd_ld<CX>(A, (i64)i * rs + (i64)col * cs), sml, big);
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      const dd s = qd_warp_sum(acc[q]);
      if (lane == 0) s_norm[warp][q] = s;
    }
    {  // the two row groups of a warp hold the same column
      const cdd o{qd_shfl_xor(dacc.re, 16), qd_shfl_xor(dacc.im, 16)};
      if (lane < 16) s_dot[warp][tl] = cdd{dacc.re + o.re, dacc.im + o.im};
    }
    __syncthreads();
    dd* part = sc.part + ((i64)par * G + bid) * QD_NR;
    if (tid < QD_NR) {
      dd s = zero;
      if (tid < 2 * QD_PW) {
        for (int q = 0; q < QD_NWARP; ++q) s = s + (tid & 1 ? s_dot[q][tid >> 1].im : s_dot[q][tid >> 1].re);
      } else {
        for (int q = 0; q < QD_NWARP; ++q) s = s + s_norm[q][tid - 2 * QD_PW];
      }
      part[tid] = s;
    }
    if (row >= r_lo && row < r_hi && tid < w) {
      const cdd v = qd_ld<CX>(A, (i64)row * rs + (i64)(c0 + tid) * cs);
      sc.rowv[(par * QD_PW + tid) * 2] = v.re;
      sc.rowv[(par * QD_PW + tid) * 2 + 1] = v.im;
    }
    ++nbar;
    grid_barrier(sc.bar, nbar * (unsigned long long)G);

    // ---- phase B: the same fixed-order reduction in every CTA ----
    for (int v = warp; v < QD_NR; v += QD_NWARP) {
      dd s = zero;
      for (int b = lane; b < G; b += 32) s = s + __ldcg(&sc.part[((i64)par * G + b) * QD_NR + v]);
      s = qd_warp_sum(s);
      if (lane == 0) tot[v] = s;
    }
    if (tid < w) s_row[tid] = cdd{__ldcg(&sc.rowv[(par * QD_PW + tid) * 2]), __ldcg(&sc.rowv[(par * QD_PW + tid) * 2 + 1])};
    __syncthreads();
    if (tid == 0) {
      // make_householder_imp (householder.rs:59-107)
      const dd tail_norm = qd_norm_select(tot[2 * QD_PW], tot[2 * QD_PW + 1], tot[2 * QD_PW + 2], sml, big);
      const dd norm_above = qd_norm_select(tot[2 * QD_PW + 3], tot[2 * QD_PW + 4], tot[2 * QD_PW + 5], sml, big);
      cdd head = s_row[col - c0];
      dd head_norm = qd_abs<CX>(head);
      if (head_norm < min_pos) {
        head = czero;
        head_norm = zero;
      }
      dd tau, info_norm;
      cdd inv = czero;
      int scale = 0;
      if (tail_norm < min_pos) {
        tau = dd_infinity();
        info_norm = head_norm;
      } else {
        const dd norm = dd_hypot(head_norm, tail_norm);
        cdd sign{dd(1.0), zero};
        if (head_norm != zero) {
          const dd hi = dd_recip(head_norm);
          sign = cdd{head.re * hi, CX ? head.im * hi : zero};
        }
        const cdd signed_norm{sign.re * norm, CX ? sign.im * norm : zero};
        inv = qd_recip<CX>(qd_add<CX>(head, signed_norm));
        head = -signed_norm;
        const dd t = tail_norm * qd_abs<CX>(inv);
        tau = dd(0.5) * (dd(1.0) + t * t);
        info_norm = norm;
        scale = 1;
      }
      // rank test (factor.rs:41-53)
      const dd nrm = dd_hypot(info_norm, norm_above);
      const dd threshold = dd_eps() * dd((double)(m - row) * 16.0) * nrm;
      const dd tau_inv = dd_recip(tau);
      if (bid == 0) qd_st<CX>(H, (i64)row * h_stride, cdd{tau, zero});
      int action = 0;
      if (tau_inv < min_pos) {
        if (info_norm > zero) action = 1;
      } else if (info_norm > threshold) {
        action = 2;
      }
      s_inv = inv;
      s_head = head;
      s_scale = scale;
      s_action = action;
      s_tau_inv = tau_inv;
    }
    __syncthreads();
    const int action = s_action, scale = s_scale;
    const cdd inv = s_inv;
    // k_c = -(head_c + v^H a_c) / tau with v^H a_c = conj(inv) sum conj(x_i) a_ic
    if (tid < w) {
      const int cc = c0 + tid;
      cdd k = czero;
      if (action == 2 && cc > col) {
        const dd tau_inv = s_tau_inv;
        const cdd dot = qd_add<CX>(s_row[tid], qd_mul<CX>(qd_conj<CX>(inv), cdd{tot[2 * (cc - col - 1)], tot[2 * (cc - col - 1) + 1]}));
        k = cdd{-(dot.re * tau_inv), CX ? -(dot.im * tau_inv) : zero};
      }
      s_k[tid] = k;
    }
    __syncthreads();

    // ---- phase C: head, reflector, zero fill, update of the remaining panel columns ----
    const int z = col - row;  // rows row + 1 .. row + z of column col are cleared when row != col (factor.rs:33-38)
    if (row >= r_lo && row < r_hi && tid < w) {
      const int cc = c0 + tid;
      if (cc == col) qd_st<CX>(A, (i64)row * rs + (i64)col * cs, s_head);
      else if (action == 2 && cc > col) qd_st<CX>(A, (i64)row * rs + (i64)cc * cs, qd_add<CX>(s_row[tid], s_k[tid]));
    }
    for (int i = max(r_lo, row + 1) + tid; i < r_hi; i += QD_THREADS) {
      const i64 r_ = (i64)i * rs;
      if (scale) qd_st<CX>(A, r_ + (i64)row * cs, qd_mul<CX>(qd_ld<CX>(A, r_ + (i64)col * cs), inv));
      if (row != col && i <= row + z) qd_st<CX>(A, r_ + (i64)col * cs, czero);
    }
    __syncthreads();
    if (action == 2 && c < cend) {
      const cdd k = s_k[c - c0];
      for (int i = max(r_lo, row + 1) + rg; i < r_hi; i += QD_THREADS / QD_PW) {
        const i64 r_ = (i64)i * rs;
        qd_st<CX>(A, r_ + (i64)c * cs, qd_add<CX>(qd_mul<CX>(k, qd_ld<CX>(A, r_ + (i64)row * cs)), qd_ld<CX>(A, r_ + (i64)c * cs)));
      }
    }
    if (action != 0) ++row;
    __syncthreads();
  }
  if (bid == 0 && tid == 0) sc.out_row[0] = row;
}

// T's diagonal: Ts[l, l] = tau of reflector row0 + l, zero elsewhere
template <bool CX>
__global__ void qd_tdiag_kernel(dd* __restrict__ Ts, int nl, const dd* __restrict__ H, i64 h_stride, int row0) {
  for (int e = threadIdx.x; e < nl * nl; e += blockDim.x) {
    const int i = e % nl, j = e / nl;
    qd_st<CX>(Ts, (i64)j * nl + i, i == j ? qd_ld<CX>(H, (i64)(row0 + i) * h_stride) : cdd{dd(0.0), dd(0.0)});
  }
}

// CTAs of one panel launch on the current device: one per SM (the kernel needs at least one resident CTA per SM for the
// cooperative launch); queried per call, so devices of different sizes each get their own grid
template <bool CX>
int qd_grid_max() {
  int dev = 0, sms = 0, per_sm = 0;
  FB_CUDA_CHECK(cudaGetDevice(&dev));
  FB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  FB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, qr_panel_dd_kernel<CX>, QD_THREADS, 0));
  FB_ASSERT(per_sm >= 1, "the dd QR panel kernel cannot be resident");
  return sms;
}

template <bool CX>
i64 qr_unblocked_dd(const QrCtx<dd>& cx, View<dd> A, View<dd> Hrow, i64 row_start, i64 col_start) {
  const i64 m = A.nrows, n = A.ncols, row_end = std::min(Hrow.ncols, m);
  if (!(row_start < row_end && col_start < n)) return row_start;
  const int Gmax = qd_grid_max<CX>();
  const size_t ES = (CX ? 2 : 1) * sizeof(dd);
  char* buf = (char*)ws_alloc((size_t)2 * Gmax * QD_NR * sizeof(dd) + (size_t)4 * QD_PW * sizeof(dd) + 64);
  QdScratch sc{(dd*)buf, (dd*)(buf + (size_t)2 * Gmax * QD_NR * sizeof(dd)), nullptr, cx.d_row};
  sc.bar = (unsigned long long*)(buf + (size_t)2 * Gmax * QD_NR * sizeof(dd) + (size_t)4 * QD_PW * sizeof(dd));
  dd *Ts = nullptr, *tmp = nullptr;
  i64 row = row_start, col = col_start;
  while (row < row_end && col < n) {
    const i64 w = std::min<i64>(QD_PW, n - col), mp = m - row;
    int G = (int)std::min<i64>(Gmax, (mp + QD_MIN_ROWS - 1) / QD_MIN_ROWS);
    if (G < 1) G = 1;
    int rpc = (int)((mp + G - 1) / G);
    FB_CUDA_CHECK(cudaMemsetAsync(sc.bar, 0, 8, cx.st));
    dd* Ap = A.ptr;
    dd* Hp = Hrow.ptr;
    i64 rs = A.rs, cs = A.cs, hs = Hrow.cs;
    int mi = (int)m, c0 = (int)col, wi = (int)w, r0 = (int)row, re = (int)row_end;
    void* args[] = {&Ap, &rs, &cs, &mi, &c0, &wi, &r0, &re, &Hp, &hs, &rpc, &sc};
    {
      LaunchTag tag(LAUNCH_PANEL);
      FB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)qr_panel_dd_kernel<CX>, dim3(G), dim3(QD_THREADS), args, 0, cx.st));
      note_launch();
    }
    int new_row = 0;
    FB_CUDA_CHECK(cudaMemcpyAsync(&new_row, cx.d_row, sizeof(int), cudaMemcpyDeviceToHost, cx.st));
    FB_CUDA_CHECK(cudaStreamSynchronize(cx.st));
    const i64 local = new_row - row, rest = n - (col + w);
    FB_ASSERT(local >= 0 && local <= w, "dd QR panel returned an impossible reflector count");
    if (local > 0 && rest > 0) {
      // the sub-panel's reflectors reach the rest of the leaf's columns as one block reflector: T = striu(V^H V) + diag(tau)
      if (!Ts) {
        Ts = (dd*)ws_alloc((size_t)QD_PW * QD_PW * ES);
        tmp = (dd*)ws_alloc((size_t)QD_PW * (size_t)rest * ES);
      }
      {
        LaunchTag tag(LAUNCH_TBUILD);
        qd_tdiag_kernel<CX><<<1, 256, 0, cx.st>>>(Ts, (int)local, Hrow.ptr, Hrow.cs, (int)row);
        FB_CUDA_CHECK(cudaGetLastError());
        note_launch();
      }
      const View<dd> Tv{Ts, local, local, 1, local};
      const View<const dd> V = cview(sub_t<dd, CX>(A, row, row, m - row, local));
      upgrade_householder_factor_t<dd, CX>(cx.st, Tv, V, local, 1);
      apply_block_householder_left_t<dd, CX>(cx.st, V, cview(Tv), false, sub_t<dd, CX>(A, row, col + w, m - row, rest), true, tmp);
    }
    row = new_row;
    col += w;
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(cx.st));
  if (Ts) {
    ws_free(tmp);
    ws_free(Ts);
  }
  ws_free(buf);
  return row;
}

}  // namespace

template <>
i64 qr_unblocked_t<dd, false>(const QrCtx<dd>& cx, View<dd> A, View<dd> Hrow, i64 row_start, i64 col_start) {
  return qr_unblocked_dd<false>(cx, A, Hrow, row_start, col_start);
}
template <>
i64 qr_unblocked_t<dd, true>(const QrCtx<dd>& cx, View<dd> A, View<dd> Hrow, i64 row_start, i64 col_start) {
  return qr_unblocked_dd<true>(cx, A, Hrow, row_start, col_start);
}

template <bool CX>
i64 qr_dd(cudaStream_t st, View<dd> A, View<dd> Q_coeff, i64 blocking_threshold) {
  return qr_in_place_t<dd, CX>(st, A, Q_coeff, blocking_threshold);
}
template <bool CX>
void householder_sequence_dd(cudaStream_t st, View<const dd> basis, View<const dd> factor, bool conj, View<dd> rhs, bool transpose) {
  apply_householder_sequence_left_t<dd, CX>(st, basis, factor, conj, rhs, transpose);
}
template i64 qr_dd<false>(cudaStream_t, View<dd>, View<dd>, i64);
template i64 qr_dd<true>(cudaStream_t, View<dd>, View<dd>, i64);
template void householder_sequence_dd<false>(cudaStream_t, View<const dd>, View<const dd>, bool, View<dd>, bool);
template void householder_sequence_dd<true>(cudaStream_t, View<const dd>, View<const dd>, bool, View<dd>, bool);

}  // namespace fb
