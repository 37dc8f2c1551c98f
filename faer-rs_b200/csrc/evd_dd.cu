// Double-double (fx128 / cx128) self-adjoint eigendecomposition A = U diag(S) U^H on the GPU, every step in faer's fx128 arithmetic
// (dd.cuh). Reference: faer/src/linalg/evd/mod.rs:270-418 (`self_adjoint_evd`): copy_from_triangular_lower, tridiag_in_place
// (evd/tridiag.rs:274-529), for complex input the diagonal unitary that makes the tridiagonal real, the real tridiagonal problem
// (divide and conquer with vectors, values only otherwise), and the back-transform U = Q D Z.
//
// Arrangement (DESIGN.md §7 item 15):
//   reduction   one Householder reflector per column, H = I - v v^H / tau with faer's make_householder (householder.rs:59-107, as
//               qr_dd.cu computes it). The copy of A is kept full (both triangles), so that p = A22 v is a coalesced
//               column-chunked product; per column: reflector (one CTA), p (row blocks x 64-column chunks, partial sums), the
//               reduction of the chunks and w = p - (v^H p / 2 tau) v (one CTA), and the rank-2 update A22 -= v w^H + w v^H of the
//               whole trailing square. Every sum is in a fixed order, so repeated calls give identical bits. The stage is
//               bandwidth-bound: about 3 x 16 (32) bytes per trailing element per column.
//   real form   cx128: d_i = re a_ii, e_i = |a_{i+1,i}|, and the phases delta_0 = 1, delta_{i+1} = delta_i a_{i+1,i} / |a_{i+1,i}|
//               (D^H T D is real, mod.rs:300-330); the eigenvector rows are scaled by delta before the back-transform.
//   values      Sturm bisection (tridiag_ev.cuh) with fx128's eps, one thread per value, as evd.cu does for f64.
//   vectors     tridiag_dc.cu's divide and conquer (same tree, tear, deflation, secular solver, Gu-Eisenstat vectors and Givens
//               folding, all from tridiag_dc_core.cuh) in dd, with the merges through gemm_dd. Two departures from f64:
//                 * the differences d_i - d_j and d_i - lambda_j are formed with dd_sub_accurate (dc_sub), because dd's own
//                   subtraction (faer's add(a, -b)) loses relative accuracy as |a| / |a - b|, and non-deflated gaps reach 2^-98
//                   relative;
//                 * the leaf (32 rows) runs its implicit QL in ONE thread over d, e and the 32 x 32 eigenvector block in shared
//                   memory (per-lane dd[32] / ee[32] would need 256 registers); the scaling is by a power of two.
//   back-transform  Q = H_0 ... H_{n-2} as a block-Householder sequence (qr_blocked.cuh): T blocks of 64 reflectors, applied
//               with gemm_dd.
#include <algorithm>
#include <vector>

#include "panel_common.cuh"  // before dd.cuh: its fb::__ldcg(const dd*) would hide the builtin overloads t_ldcg calls
#include "dd.cuh"
#include "qr_blocked.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"
#include "tridiag_dd.cuh"

namespace fb {

namespace {

constexpr int ED_LEAF = 32;   // divide-and-conquer leaf rows (tridiag_dc.cu's DC_LEAF)
constexpr int ED_CHUNK = 64;  // columns per partial sum of p = A22 v
constexpr int ED_BS = 64;     // reflectors per block of the back-transform

template <bool CX>
__device__ __forceinline__ cdd ed_ld(const dd* p, i64 off) {
  return CX ? cdd{p[2 * off], p[2 * off + 1]} : cdd{p[off], dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ void ed_st(dd* p, i64 off, cdd v) {
  if (CX) {
    p[2 * off] = v.re;
    p[2 * off + 1] = v.im;
  } else {
    p[off] = v.re;
  }
}
template <bool CX>
__device__ __forceinline__ cdd ed_mul(cdd a, cdd b) {
  return CX ? a * b : cdd{a.re * b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd ed_add(cdd a, cdd b) {
  return CX ? a + b : cdd{a.re + b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd ed_conj(cdd a) {
  return CX ? cdd_conj(a) : a;
}
__device__ __forceinline__ dd ed_shfl_xor(dd v, int off) {
  return dd(__shfl_xor_sync(0xffffffffu, v.hi, off), __shfl_xor_sync(0xffffffffu, v.lo, off));
}
// dd addition is commutative, so the xor butterfly leaves the same bits in every lane
__device__ __forceinline__ dd ed_warp_sum(dd v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = v + ed_shfl_xor(v, off);
  return v;
}
// sum over the CTA in a fixed order (warp butterflies, then the warps in order); every thread gets the result
template <int NT>
__device__ __forceinline__ dd ed_block_sum(dd v, dd* red) {
  v = ed_warp_sum(v);
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  dd s(0.0);
  for (int q = 0; q < NT / 32; ++q) s = s + red[q];
  return s;
}
// norm_l2.rs:161-172, three scaled accumulators
__device__ __forceinline__ dd ed_norm_select(dd s, dd m, dd b, dd sml, dd big) {
  if (s >= dd(1.0)) return sqrt(s) * big;
  if (m >= dd(1.0)) return sqrt(m);
  return sqrt(b) * sml;
}

// dst (n x n, ld n) <- the self-adjoint matrix whose lower triangle is src; the diagonal's imaginary part is dropped
template <bool CX>
__global__ void ed_copy_kernel(dd* __restrict__ dst, i64 n, const dd* __restrict__ src, i64 rs, i64 cs) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n) return;
  cdd v = i >= j ? ed_ld<CX>(src, i * rs + j * cs) : ed_conj<CX>(ed_ld<CX>(src, j * rs + i * cs));
  if (i == j) v.im = dd(0.0);
  ed_st<CX>(dst, j * n + i, v);
}

// reflector of column k (rows k+1 ..): tau[k], tau_inv (scal[0]), beta into W(k+1, k), v (v_0 = 1) into vbuf and below beta
template <bool CX>
__global__ void __launch_bounds__(512) ed_house_kernel(dd* W, int n, int k, dd* tau, dd* scal, cdd* vbuf) {
  __shared__ dd red[16];
  __shared__ cdd s_inv;
  const int L = n - k - 1;
  dd* col = W + (CX ? 2 : 1) * (i64)k * n;
  const dd sml = dd_sqrt_min_positive(), big = dd_sqrt_max_positive(), min_pos = dd_min_positive(), zero(0.0);
  dd acc[3] = {zero, zero, zero};
  for (int i = 1 + threadIdx.x; i < L; i += 512) {
    const cdd x = ed_ld<CX>(col, k + 1 + i);
    const dd rs = x.re * sml, rb = x.re * big;
    acc[0] = dd_mul_add(rs, rs, acc[0]);
    acc[1] = dd_mul_add(x.re, x.re, acc[1]);
    acc[2] = dd_mul_add(rb, rb, acc[2]);
    if (CX) {
      const dd is = x.im * sml, ib = x.im * big;
      acc[0] = dd_mul_add(is, is, acc[0]);
      acc[1] = dd_mul_add(x.im, x.im, acc[1]);
      acc[2] = dd_mul_add(ib, ib, acc[2]);
    }
  }
  const dd s0 = ed_block_sum<512>(acc[0], red), s1 = ed_block_sum<512>(acc[1], red), s2 = ed_block_sum<512>(acc[2], red);
  if (threadIdx.x == 0) {
    // make_householder_imp (householder.rs:59-107)
    const dd tail_norm = ed_norm_select(s0, s1, s2, sml, big);
    cdd head = ed_ld<CX>(col, k + 1);
    dd head_norm = CX ? cdd_abs(head) : fabs(head.re);
    if (head_norm < min_pos) {
      head = cdd{zero, zero};
      head_norm = zero;
    }
    dd t_au;
    cdd inv{dd(1.0), zero};
    if (tail_norm < min_pos) {
      t_au = dd_infinity();
    } else {
      const dd norm = dd_hypot(head_norm, tail_norm);
      cdd sign{dd(1.0), zero};
      if (head_norm != zero) {
        const dd hi = dd_recip(head_norm);
        sign = cdd{head.re * hi, CX ? head.im * hi : zero};
      }
      const cdd signed_norm{sign.re * norm, CX ? sign.im * norm : zero};
      const cdd hs = ed_add<CX>(head, signed_norm);
      inv = CX ? cdd_recip_scaled(hs) : cdd{dd_recip(hs.re), zero};
      head = -signed_norm;
      const dd t = tail_norm * (CX ? cdd_abs(inv) : fabs(inv.re));
      t_au = dd(0.5) * (dd(1.0) + t * t);
    }
    tau[k] = t_au;
    scal[0] = dd_recip(t_au);
    ed_st<CX>(col, k + 1, head);
    vbuf[0] = cdd{dd(1.0), zero};
    s_inv = inv;
  }
  __syncthreads();
  const cdd inv = s_inv;
  for (int i = 1 + threadIdx.x; i < L; i += 512) {
    const cdd x = ed_mul<CX>(ed_ld<CX>(col, k + 1 + i), inv);
    ed_st<CX>(col, k + 1 + i, x);
    vbuf[i] = x;
  }
}

// part[c][i] = sum_{j in chunk c} A22(i, j) v_j
template <bool CX>
__global__ void __launch_bounds__(128) ed_symv_kernel(const dd* __restrict__ W, int n, int k, const cdd* __restrict__ vbuf,
                                                      cdd* __restrict__ part) {
  __shared__ cdd vs[ED_CHUNK];
  const int L = n - k - 1, c = blockIdx.y, j0 = c * ED_CHUNK, j1 = min(L, j0 + ED_CHUNK);
  if (threadIdx.x < j1 - j0) vs[threadIdx.x] = vbuf[j0 + threadIdx.x];
  __syncthreads();
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= L) return;
  const dd* base = W + (CX ? 2 : 1) * ((i64)(k + 1) * n + k + 1);
  cdd acc{dd(0.0), dd(0.0)};
  for (int j = j0; j < j1; ++j) acc = ed_add<CX>(acc, ed_mul<CX>(ed_ld<CX>(base, (i64)j * n + i), vs[j - j0]));
  part[(i64)c * n + i] = acc;
}

// p = (sum of the chunks) / tau, then w = p - (v^H p / (2 tau)) v  (tridiag.rs:462-491 in the unblocked form)
template <bool CX>
__global__ void __launch_bounds__(1024) ed_w_kernel(int n, int k, const cdd* __restrict__ part, int nchunk, const cdd* __restrict__ vbuf,
                                                    cdd* __restrict__ wbuf, const dd* scal) {
  __shared__ dd red[32];
  const int L = n - k - 1;
  const dd tau_inv = scal[0];
  dd dot(0.0);
  for (int i = threadIdx.x; i < L; i += 1024) {
    cdd s = part[i];
    for (int c = 1; c < nchunk; ++c) s = ed_add<CX>(s, part[(i64)c * n + i]);
    const cdd p{s.re * tau_inv, CX ? s.im * tau_inv : dd(0.0)};
    wbuf[i] = p;
    const cdd v = vbuf[i];
    dot = dot + (CX ? v.re * p.re + v.im * p.im : v.re * p.re);  // re(conj(v) p); the imaginary part vanishes
  }
  const dd K = ed_block_sum<1024>(dot, red) * tau_inv * dd(0.5);
  for (int i = threadIdx.x; i < L; i += 1024) {
    const cdd v = vbuf[i], p = wbuf[i];
    wbuf[i] = cdd{p.re - K * v.re, CX ? p.im - K * v.im : dd(0.0)};
  }
}

// A22 -= v w^H + w v^H, 4 columns per thread
template <bool CX>
__global__ void __launch_bounds__(128) ed_rank2_kernel(dd* W, int n, int k, const cdd* __restrict__ vbuf, const cdd* __restrict__ wbuf) {
  const int L = n - k - 1;
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= L) return;
  dd* base = W + (CX ? 2 : 1) * ((i64)(k + 1) * n + k + 1);
  const cdd vi = vbuf[i], wi = wbuf[i];
  for (int j = blockIdx.y * 4; j < min(L, (int)blockIdx.y * 4 + 4); ++j) {
    const i64 off = (i64)j * n + i;
    const cdd a = ed_ld<CX>(base, off);
    const cdd t = ed_add<CX>(ed_mul<CX>(vi, ed_conj<CX>(wbuf[j])), ed_mul<CX>(wi, ed_conj<CX>(vbuf[j])));
    ed_st<CX>(base, off, cdd{a.re - t.re, CX ? a.im - t.im : dd(0.0)});
  }
}

// the real tridiagonal (d, e) and, for cx128, the phases; flag[0] = 1 on a non-finite entry
template <bool CX>
__global__ void ed_extract_kernel(const dd* __restrict__ W, int n, dd* __restrict__ d, dd* __restrict__ e, cdd* __restrict__ ph,
                                  int* flag) {
  int bad = 0;
  cdd delta{dd(1.0), dd(0.0)};
  for (int i = 0; i < n; ++i) {
    d[i] = ed_ld<CX>(W, (i64)i * n + i).re;
    if (!dd_is_finite(d[i])) bad = 1;
    if (CX) ph[i] = delta;
    if (i + 1 < n) {
      const cdd b = ed_ld<CX>(W, (i64)i * n + i + 1);
      if (!dd_is_finite(b.re) || !dd_is_finite(b.im)) bad = 1;
      if (CX) {
        const dd a = cdd_abs(b);
        e[i] = a;
        if (a != dd(0.0) && dd_is_finite(a)) {
          const dd ai = dd_recip(a);
          delta = delta * cdd{b.re * ai, b.im * ai};
        }
      } else {
        e[i] = b.re;
      }
    }
  }
  flag[0] = bad;
}

// ---- values only: Gershgorin interval and bisection ----
__global__ void ed_bounds_kernel(const dd* __restrict__ d, const dd* __restrict__ e, int n, dd* __restrict__ bb) {
  dd lo = d[0], hi = d[0], e2(0.0);
  for (int i = 0; i < n; ++i) {
    const dd r = (i > 0 ? fabs(e[i - 1]) : dd(0.0)) + (i + 1 < n ? fabs(e[i]) : dd(0.0));
    lo = fmin(lo, d[i] - r);
    hi = fmax(hi, d[i] + r);
    if (i + 1 < n) e2 = fmax(e2, e[i] * e[i]);
  }
  const dd span = fmax(fabs(lo), fabs(hi));
  const dd pad = dd(4.0) * dd_eps() * span * dd((double)n) + dd_min_positive();
  bb[0] = lo - pad;
  bb[1] = hi + pad;
  bb[2] = e2;
}

__global__ void __launch_bounds__(64) ed_values_kernel(const dd* __restrict__ d, const dd* __restrict__ e, int n,
                                                        const dd* __restrict__ bb, dd* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = tev::st_kth_smallest<dd>(d, e, n, k, bb[0], bb[1], bb[2]);
}

// ---- divide and conquer (tridiag_dc.cu's kernels in dd) ----
struct EdMerge {
  int lo, mid, hi;
};

struct EdBuf {
  dd *d, *e, *dsort, *zsort, *dl, *w, *dd_, *rc, *rs, *lam, *zh, *dnew, *rho, *sgn;
  int *colsort, *cnd, *cdf, *ra, *rb, *outcol, *kcnt, *nrot;
  dd* scale;  // [1]: the power of two the problem was divided by
};

// d, e /= 2^k with 2^k > max |d_i|, |e_i| (exact), e[n-1] = 0
__global__ void ed_scale_kernel(dd* d, dd* e, int n, dd* scale) {
  double mx = 0.0;
  for (int i = 0; i < n; ++i) mx = fmax(mx, fmax(fabs(d[i].hi), i + 1 < n ? fabs(e[i].hi) : 0.0));
  int ex = 0;
  if (mx > 0.0) frexp(mx, &ex);
  const dd s(ldexp(1.0, ex)), si(ldexp(1.0, -ex));
  scale[0] = s;
  for (int i = 0; i < n; ++i) {
    d[i] = d[i] * si;
    e[i] = i + 1 < n ? e[i] * si : dd(0.0);
  }
}

__global__ void ed_tear_kernel(dd* d, const dd* e, const EdMerge* merges, int nmerge, dd* rho, dd* sgn) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= nmerge) return;
  const int mid = merges[m].mid;
  const dd beta = e[mid - 1];
  rho[m] = fabs(beta);
  sgn[m] = beta < dd(0.0) ? dd(-1.0) : dd(1.0);
  d[mid - 1] = d[mid - 1] - fabs(beta);
  d[mid] = d[mid] - fabs(beta);
}

// one thread runs the implicit QL of a leaf over shared d, e and eigenvector block; the warp loads and stores
__global__ void __launch_bounds__(32) ed_leaf_kernel(dd* d, const dd* e, dd* Q, i64 ldq, int n, int nlev, int* fail) {
  __shared__ dd Z[ED_LEAF][ED_LEAF + 1];
  __shared__ dd sd[ED_LEAF], se[ED_LEAF];
  const int leaf = blockIdx.x, lane = threadIdx.x;
  const int lo = (int)(((long long)leaf * n) >> nlev), hi = (int)(((long long)(leaf + 1) * n) >> nlev);
  const int s = hi - lo;
  sd[lane] = lane < s ? d[lo + lane] : dd(0.0);
  se[lane] = lane + 1 < s ? e[lo + lane] : dd(0.0);
  for (int j = 0; j < ED_LEAF; ++j) Z[lane][j] = dd(lane == j ? 1.0 : 0.0);
  __syncwarp();
  if (lane == 0) {
    const bool ok = dc::ql_implicit(sd, se, s, [&](int i, dd c, dd sn) {
      for (int r = 0; r < s; ++r) {
        const dd f = Z[r][i + 1];
        Z[r][i + 1] = sn * Z[r][i] + c * f;
        Z[r][i] = c * Z[r][i] - sn * f;
      }
    });
    if (!ok) *fail = 1;
    for (int i = 0; i < s; ++i) {
      int kmin = i;
      for (int j = i + 1; j < s; ++j)
        if (sd[j] < sd[kmin]) kmin = j;
      if (kmin != i) {
        const dd t = sd[i];
        sd[i] = sd[kmin];
        sd[kmin] = t;
        for (int r = 0; r < s; ++r) {
          const dd u = Z[r][i];
          Z[r][i] = Z[r][kmin];
          Z[r][kmin] = u;
        }
      }
    }
  }
  __syncwarp();
  if (lane < s) d[lo + lane] = sd[lane];
  for (int c = 0; c < s; ++c)
    if (lane < s) Q[(i64)(lo + c) * ldq + lo + lane] = Z[lane][c];
}

__device__ __forceinline__ int ed_count_less(const dd* a, int n, dd x, bool or_equal) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const bool lt = or_equal ? (a[mid] <= x) : (a[mid] < x);
    if (lt) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(256) ed_prepare_kernel(EdBuf b, const dd* Q, i64 ldq, const EdMerge* merges, int mbase) {
  const int m = mbase + blockIdx.x;
  const int lo = merges[m].lo, mid = merges[m].mid, hi = merges[m].hi, s = hi - lo;
  const dd sg = b.sgn[m], r2 = sqrt(dd(0.5));
  for (int i = lo + threadIdx.x; i < hi; i += 256) {
    const dd zi = (i < mid ? Q[(i64)i * ldq + (mid - 1)] : sg * Q[(i64)i * ldq + mid]) * r2;
    const dd di = b.d[i];
    int pos;
    if (i < mid) pos = (i - lo) + ed_count_less(b.d + mid, hi - mid, di, false);
    else pos = (i - mid) + ed_count_less(b.d + lo, mid - lo, di, true);
    b.dsort[lo + pos] = di;
    b.zsort[lo + pos] = zi;
    b.colsort[lo + pos] = i - lo;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int nrot = 0;
    const int k = dc::deflate_scan<dd>(b.dsort + lo, b.zsort + lo, b.colsort + lo, s, dd(2.0) * b.rho[m], b.dl + lo, b.w + lo,
                                       b.cnd + lo, b.dd_ + lo, b.cdf + lo, b.ra + lo, b.rb + lo, b.rc + lo, b.rs + lo, &nrot);
    b.kcnt[m] = k;
    b.nrot[m] = nrot;
  }
}

// one warp per root; every lane holds the same sums (ed_warp_sum), so all take the same bisection steps
__global__ void __launch_bounds__(256) ed_secular_kernel(EdBuf b, dd* DEL, i64 ldw, const EdMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo;
  const int k = b.kcnt[m];
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= k) return;
  const dd rho = dd(2.0) * b.rho[m], rhoinv = dd_recip(rho);
  const dd* dl = b.dl + lo;
  const dd* w = b.w + lo;
  dd zz(0.0);
  for (int i = lane; i < k; i += 32) zz = zz + w[i] * w[i];
  zz = ed_warp_sum(zz);
  int org = 0;
  dd tau;
  if (k == 1) {
    tau = rho * zz;
  } else {
    tau = dc::secular_root<dd>(dl, k, j, rho, zz,
                               [&](int o, dd t) {
                                 const dd dorg = dl[o];
                                 dd f(0.0);
                                 for (int i = lane; i < k; i += 32) {
                                   const dd del = dc::dc_sub(dc::dc_sub(dl[i], dorg), t);
                                   f = f + w[i] * (w[i] / del);
                                 }
                                 return rhoinv + ed_warp_sum(f);
                               },
                               &org);
  }
  const dd dorg = dl[org];
  if (lane == 0) b.lam[lo + j] = dorg + tau;
  dd* col = DEL + (i64)(lo + j) * ldw + lo;
  for (int i = lane; i < k; i += 32) col[i] = dc::dc_sub(dc::dc_sub(dl[i], dorg), tau);
}

__global__ void __launch_bounds__(256) ed_zhat_kernel(EdBuf b, const dd* DEL, i64 ldw, const EdMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo;
  const int k = b.kcnt[m];
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= k) return;
  const dd* dl = b.dl + lo;
  const dd di = dl[i];
  dd prod = DEL[(i64)(lo + i) * ldw + lo + i];
  for (int j = 0; j < k; ++j)
    if (j != i) prod = prod * (DEL[(i64)(lo + j) * ldw + lo + i] / dc::dc_sub(di, dl[j]));
  const dd r = sqrt(fabs(prod));
  b.zh[lo + i] = b.w[lo + i] < dd(0.0) ? -r : r;
}

__global__ void __launch_bounds__(256) ed_order_kernel(EdBuf b, const EdMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo, s = merges[m].hi - lo;
  const int k = b.kcnt[m], nd = s - k;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= s) return;
  const dd* lam = b.lam + lo;
  const dd* dd0 = b.dd_ + lo;
  int c;
  dd val;
  if (t < k) {
    val = lam[t];
    c = t;
    for (int u = 0; u < nd; ++u) c += dd0[u] < val;
  } else {
    const int td = t - k;
    val = dd0[td];
    c = ed_count_less(lam, k, val, true);
    for (int u = 0; u < nd; ++u) c += (dd0[u] < val) || (dd0[u] == val && u < td);
  }
  b.outcol[lo + t] = c;
  b.dnew[lo + c] = val;
}

__global__ void __launch_bounds__(128) ed_vectors_kernel(EdBuf b, const dd* DEL, dd* W, i64 ldw, const EdMerge* merges, int mbase) {
  __shared__ dd red[4];
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo, s = merges[m].hi - lo;
  const int k = b.kcnt[m];
  const int t = blockIdx.x;
  if (t >= s) return;
  const int oc = b.outcol[lo + t];
  dd* wcol = W + (i64)(lo + oc) * ldw + lo;
  if (t >= k) {
    if (threadIdx.x == 0) wcol[b.cdf[lo + t - k]] = dd(1.0);
    return;
  }
  const dd* dcol = DEL + (i64)(lo + t) * ldw + lo;
  dd acc(0.0);
  for (int i = threadIdx.x; i < k; i += 128) {
    const dd v = b.zh[lo + i] / dcol[i];
    acc = dd_mul_add(v, v, acc);
  }
  const dd inv = dd_recip(sqrt(ed_block_sum<128>(acc, red)));
  for (int i = threadIdx.x; i < k; i += 128) wcol[b.cnd[lo + i]] = (b.zh[lo + i] / dcol[i]) * inv;
}

__global__ void __launch_bounds__(256) ed_rotate_kernel(EdBuf b, dd* W, i64 ldw, const EdMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo, s = merges[m].hi - lo;
  const int nrot = b.nrot[m];
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= s || nrot == 0) return;
  dd* wcol = W + (i64)(lo + c) * ldw + lo;
  for (int r = nrot - 1; r >= 0; --r) {
    const int a = b.ra[lo + r], bb = b.rb[lo + r];
    const dd cs = b.rc[lo + r], sn = b.rs[lo + r];
    const dd x = wcol[a], y = wcol[bb];
    wcol[a] = cs * x - sn * y;
    wcol[bb] = sn * x + cs * y;
  }
}

__global__ void ed_finish_kernel(const dd* d, dd* lam, int n, const dd* scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lam[i] = d[i] * scale[0];
}

int ed_num_levels(i64 n) {
  int lv = 0;
  while (((n + (1ll << lv) - 1) >> lv) > ED_LEAF) ++lv;
  return lv;
}

}  // namespace

// (d, e) real tridiagonal on the device -> lam ascending, Z (n x n, ld n) its eigenvectors; false if a leaf failed
bool tridiag_dc_dd(cudaStream_t st, const dd* d_in, const dd* e_in, i64 n, dd* lam, dd* Z) {
  LaunchTag tag(LAUNCH_SOLVE);  // the merges' GEMMs included
  const int nlev = ed_num_levels(n);
  std::vector<EdMerge> merges;
  std::vector<int> first((size_t)nlev + 1, 0);
  for (int l = 0; l < nlev; ++l) {
    first[(size_t)l] = (int)merges.size();
    for (long long i = 0; i < (1ll << l); ++i)
      merges.push_back(EdMerge{(int)((i * n) >> l), (int)(((2 * i + 1) * n) >> (l + 1)), (int)(((i + 1) * n) >> l)});
  }
  first[(size_t)nlev] = (int)merges.size();
  const int nm = std::max<int>(1, (int)merges.size());
  const size_t nd = (size_t)n;
  const size_t bytes = 12 * nd * sizeof(dd) + (2 * (size_t)nm + 1) * sizeof(dd) + (6 * nd + 2 * (size_t)nm + 2) * sizeof(int) +
                       (size_t)nm * sizeof(EdMerge) + 256;
  char* pool = (char*)ws_alloc(bytes);
  EdBuf b;
  dd* pd = (dd*)pool;
  dd** dptrs[] = {&b.d, &b.e, &b.dsort, &b.zsort, &b.dl, &b.w, &b.dd_, &b.rc, &b.rs, &b.lam, &b.zh, &b.dnew};
  for (dd** p : dptrs) {
    *p = pd;
    pd += nd;
  }
  b.rho = pd; pd += nm; b.sgn = pd; pd += nm; b.scale = pd; pd += 1;
  int* pi = (int*)pd;
  int** iptrs[] = {&b.colsort, &b.cnd, &b.cdf, &b.ra, &b.rb, &b.outcol};
  for (int** p : iptrs) {
    *p = pi;
    pi += nd;
  }
  b.kcnt = pi; pi += nm; b.nrot = pi; pi += nm;
  int* d_fail = pi; pi += 2;
  EdMerge* d_merges = (EdMerge*)(((uintptr_t)pi + 15) & ~(uintptr_t)15);
  FB_ASSERT((char*)(d_merges + nm) <= pool + bytes, "workspace layout");
  if (!merges.empty())
    FB_CUDA_CHECK(cudaMemcpyAsync(d_merges, merges.data(), merges.size() * sizeof(EdMerge), cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemsetAsync(d_fail, 0, 8, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(b.d, d_in, nd * sizeof(dd), cudaMemcpyDeviceToDevice, st));
  FB_CUDA_CHECK(cudaMemsetAsync(b.e, 0, nd * sizeof(dd), st));
  if (n > 1) FB_CUDA_CHECK(cudaMemcpyAsync(b.e, e_in, (nd - 1) * sizeof(dd), cudaMemcpyDeviceToDevice, st));
  ed_scale_kernel<<<1, 1, 0, st>>>(b.d, b.e, (int)n, b.scale);
  note_launch();
  if (!merges.empty()) {
    ed_tear_kernel<<<(unsigned)((merges.size() + 127) / 128), 128, 0, st>>>(b.d, b.e, d_merges, (int)merges.size(), b.rho, b.sgn);
    note_launch();
  }
  dd* Qs = nlev > 0 ? (dd*)ws_alloc(nd * nd * sizeof(dd)) : nullptr;
  dd* Wm = nlev > 0 ? (dd*)ws_alloc(nd * nd * sizeof(dd)) : nullptr;
  dd* DEL = nlev > 0 ? (dd*)ws_alloc(nd * nd * sizeof(dd)) : nullptr;
  dd* cur = (nlev % 2 == 0) ? Z : Qs;
  FB_CUDA_CHECK(cudaMemsetAsync(cur, 0, nd * nd * sizeof(dd), st));
  ed_leaf_kernel<<<(unsigned)(1u << nlev), 32, 0, st>>>(b.d, b.e, cur, n, (int)n, nlev, d_fail);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  for (int l = nlev - 1; l >= 0; --l) {
    const int mb = first[(size_t)l], cnt = first[(size_t)l + 1] - mb;
    int smax = 0;
    for (int i = 0; i < cnt; ++i) smax = std::max(smax, merges[(size_t)(mb + i)].hi - merges[(size_t)(mb + i)].lo);
    dd* nxt = (cur == Z) ? Qs : Z;
    FB_CUDA_CHECK(cudaMemsetAsync(Wm, 0, nd * nd * sizeof(dd), st));
    ed_prepare_kernel<<<(unsigned)cnt, 256, 0, st>>>(b, cur, n, d_merges, mb);
    ed_secular_kernel<<<dim3((unsigned)((smax + 7) / 8), (unsigned)cnt), 256, 0, st>>>(b, DEL, n, d_merges, mb);
    ed_zhat_kernel<<<dim3((unsigned)((smax + 255) / 256), (unsigned)cnt), 256, 0, st>>>(b, DEL, n, d_merges, mb);
    ed_order_kernel<<<dim3((unsigned)((smax + 255) / 256), (unsigned)cnt), 256, 0, st>>>(b, d_merges, mb);
    ed_vectors_kernel<<<dim3((unsigned)smax, (unsigned)cnt), 128, 0, st>>>(b, DEL, Wm, n, d_merges, mb);
    ed_rotate_kernel<<<dim3((unsigned)((smax + 255) / 256), (unsigned)cnt), 256, 0, st>>>(b, Wm, n, d_merges, mb);
    FB_CUDA_CHECK(cudaGetLastError());
    for (int q = 0; q < 6; ++q) note_launch();
    for (int i = 0; i < cnt; ++i) {
      const EdMerge& mg = merges[(size_t)(mb + i)];
      const i64 lo = mg.lo, mid = mg.mid, hi = mg.hi, s = hi - lo, s1 = mid - lo, s2 = hi - mid;
      View<const dd> Q1{cur + lo * n + lo, s1, s1, 1, n}, Q2{cur + mid * n + mid, s2, s2, 1, n};
      View<const dd> W1{Wm + lo * n + lo, s1, s, 1, n}, W2{Wm + lo * n + mid, s2, s, 1, n};
      gemm_dd(st, View<dd>{nxt + lo * n + lo, s1, s, 1, n}, RECT, 0, Q1, RECT, false, W1, RECT, false, false, dd(1.0), dd(0.0));
      gemm_dd(st, View<dd>{nxt + lo * n + mid, s2, s, 1, n}, RECT, 0, Q2, RECT, false, W2, RECT, false, false, dd(1.0), dd(0.0));
    }
    FB_CUDA_CHECK(cudaMemcpyAsync(b.d, b.dnew, nd * sizeof(dd), cudaMemcpyDeviceToDevice, st));
    cur = nxt;
  }
  FB_ASSERT(cur == Z, "eigenvector ping-pong ended in the scratch buffer");
  ed_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(b.d, lam, (int)n, b.scale);
  note_launch();
  int h_fail = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(&h_fail, d_fail, 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (DEL) ws_free(DEL);
  if (Wm) ws_free(Wm);
  if (Qs) ws_free(Qs);
  ws_free(pool);
  return h_fail == 0;
}

namespace {

// ---- back-transform helpers ----
// Uc (n x n, ld n) = D Z: Z's rows scaled by the phases (cx128) or copied (fx128)
template <bool CX>
__global__ void ed_lift_kernel(dd* __restrict__ Uc, const dd* __restrict__ Z, const cdd* __restrict__ ph, i64 n) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= n) return;
  const dd z = Z[j * n + i];
  if (CX) ed_st<CX>(Uc, j * n + i, cdd{ph[i].re * z, ph[i].im * z});
  else Uc[j * n + i] = z;
}
// T blocks' diagonals: Tf(j % bs, j) = tau_j
template <bool CX>
__global__ void ed_tdiag_kernel(dd* Tf, const dd* tau, int bs, int n1) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n1) ed_st<CX>(Tf, (i64)j * bs + j % bs, cdd{tau[j], dd(0.0)});
}
template <bool CX>
__global__ void ed_store_kernel(View<dd> U, const dd* __restrict__ Uc) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i < U.nrows) ed_st<CX>(U.ptr, i * U.rs + j * U.cs, ed_ld<CX>(Uc, j * U.nrows + i));
}
// S (compact, element units) <- the real values (cx128: (value, 0))
template <bool CX>
__global__ void ed_values_out_kernel(dd* S, const dd* lam, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ed_st<CX>(S, i, cdd{lam[i], dd(0.0)});
}

}  // namespace

// A: the lower triangle of a self-adjoint n x n matrix (device view, element units); U: n x n device view, or no columns for the
// eigenvalues only; S: n device entries in element units. Returns false for non-finite input (or a leaf QL that did not converge).
template <bool CX>
bool self_adjoint_evd_dd(cudaStream_t st, View<const dd> A, View<dd> U, dd* S) {
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n, "self_adjoint_evd: square matrix required");
  if (n == 0) return true;
  FB_ASSERT(n < 65536, "self_adjoint_evd: dimension too large for the copy launch");
  const size_t esz = (CX ? 2 : 1) * sizeof(dd), nd = (size_t)n;
  dd* W = (dd*)ws_alloc(nd * nd * esz);
  ed_copy_kernel<CX><<<dim3((unsigned)((n + 255) / 256), (unsigned)n), 256, 0, st>>>(W, n, A.ptr, A.rs, A.cs);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  const int nchunk = (int)std::max<i64>(1, (n + ED_CHUNK - 1) / ED_CHUNK);
  dd* tau = (dd*)ws_alloc((nd + 1) * sizeof(dd));
  dd* scal = (dd*)ws_alloc(4 * sizeof(dd));
  cdd* vbuf = (cdd*)ws_alloc(nd * sizeof(cdd));
  cdd* wbuf = (cdd*)ws_alloc(nd * sizeof(cdd));
  cdd* part = (cdd*)ws_alloc((size_t)nchunk * nd * sizeof(cdd));
  {
    LaunchTag tag(LAUNCH_PANEL);
    for (int k = 0; k + 2 < n; ++k) {  // the last column (k = n-2) has a one-entry tail: H = I (tau = +inf)
      const int L = (int)n - k - 1, nc = (L + ED_CHUNK - 1) / ED_CHUNK;
      ed_house_kernel<CX><<<1, 512, 0, st>>>(W, (int)n, k, tau, scal, vbuf);
      ed_symv_kernel<CX><<<dim3((unsigned)((L + 127) / 128), (unsigned)nc), 128, 0, st>>>(W, (int)n, k, vbuf, part);
      ed_w_kernel<CX><<<1, 1024, 0, st>>>((int)n, k, part, nc, vbuf, wbuf, scal);
      ed_rank2_kernel<CX><<<dim3((unsigned)((L + 127) / 128), (unsigned)((L + 3) / 4)), 128, 0, st>>>(W, (int)n, k, vbuf, wbuf);
      FB_CUDA_CHECK(cudaGetLastError());
      for (int q = 0; q < 4; ++q) note_launch();
    }
    if (n >= 2) {  // tridiag.rs: the last reflector has no tail; +inf makes it the identity in the block sequence
      const dd inf = dd_infinity();
      FB_CUDA_CHECK(cudaMemcpyAsync(tau + (n - 2), &inf, sizeof(dd), cudaMemcpyHostToDevice, st));
    }
  }
  dd* de = (dd*)ws_alloc((3 * nd + 4) * sizeof(dd));
  dd *d = de, *e = de + n, *bb = de + 2 * n + 1;
  cdd* ph = CX ? (cdd*)ws_alloc(nd * sizeof(cdd)) : nullptr;
  int* flag = (int*)ws_alloc(16);
  ed_extract_kernel<CX><<<1, 1, 0, st>>>(W, (int)n, d, e, ph, flag);
  note_launch();
  int h_flag = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, flag, 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  bool ok = h_flag == 0;
  if (ok && U.ncols == 0) {
    dd* lam = (dd*)ws_alloc(nd * sizeof(dd));
    LaunchTag tag(LAUNCH_SOLVE);
    ed_bounds_kernel<<<1, 1, 0, st>>>(d, e, (int)n, bb);
    ed_values_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(d, e, (int)n, bb, lam);
    ed_values_out_kernel<CX><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, lam, (int)n);
    FB_CUDA_CHECK(cudaGetLastError());
    for (int q = 0; q < 3; ++q) note_launch();
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    ws_free(lam);
  } else if (ok) {
    FB_ASSERT(U.nrows == n && U.ncols == n, "self_adjoint_evd: U must be n x n");
    dd* lam = (dd*)ws_alloc(nd * sizeof(dd));
    dd* Z = (dd*)ws_alloc(nd * nd * sizeof(dd));
    ok = tridiag_dc_dd(st, d, e, n, lam, Z);
    if (ok) {
      ed_values_out_kernel<CX><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, lam, (int)n);
      note_launch();
      dd* Uc = (dd*)ws_alloc(nd * nd * esz);
      const cdd* phc = ph;
      ed_lift_kernel<CX><<<dim3((unsigned)((n + 255) / 256), (unsigned)n), 256, 0, st>>>(Uc, Z, phc, n);
      FB_CUDA_CHECK(cudaGetLastError());
      note_launch();
      const i64 n1 = n - 1;
      if (n1 > 0) {
        const i64 bs = std::min<i64>(ED_BS, n1);
        dd* Tf = (dd*)ws_alloc((size_t)bs * (size_t)n1 * esz);
        FB_CUDA_CHECK(cudaMemsetAsync(Tf, 0, (size_t)bs * (size_t)n1 * esz, st));
        ed_tdiag_kernel<CX><<<(unsigned)((n1 + 255) / 256), 256, 0, st>>>(Tf, tau, (int)bs, (int)n1);
        note_launch();
        const View<dd> Tv{Tf, bs, n1, 1, bs};
        const View<const dd> basis{W + (CX ? 2 : 1) * 1, n1, n1, 1, n};  // A[1.., 0..n-1]: unit lower, beta on the diagonal unread
        for (i64 j = 0; j < n1; j += bs) {
          const i64 b = std::min(bs, n1 - j);
          upgrade_householder_factor_t<dd, CX>(st, sub_t<dd, CX>(Tv, 0, j, b, b), sub_t<dd, CX>(basis, j, j, n1 - j, b), b, 1);
        }
        const View<dd> Uv{Uc, n, n, 1, n};
        apply_householder_sequence_left_t<dd, CX>(st, basis, cview(Tv), false, sub_t<dd, CX>(Uv, 1, 0, n1, n), false);
        ws_free(Tf);
      }
      ed_store_kernel<CX><<<dim3((unsigned)((n + 255) / 256), (unsigned)n), 256, 0, st>>>(U, Uc);
      FB_CUDA_CHECK(cudaGetLastError());
      note_launch();
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(Uc);
    }
    ws_free(Z);
    ws_free(lam);
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(flag);
  if (ph) ws_free(ph);
  ws_free(de);
  ws_free(part);
  ws_free(wbuf);
  ws_free(vbuf);
  ws_free(scal);
  ws_free(tau);
  ws_free(W);
  return ok;
}

template bool self_adjoint_evd_dd<false>(cudaStream_t, View<const dd>, View<dd>, dd*);
template bool self_adjoint_evd_dd<true>(cudaStream_t, View<const dd>, View<dd>, dd*);

}  // namespace fb
