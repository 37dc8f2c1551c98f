// Double-double (fx128 / cx128) singular value decomposition A = U diag(S) V^H on the GPU, every step in faer's fx128 arithmetic
// (dd.cuh). Reference: faer/src/linalg/svd/mod.rs:530-672 (`svd`: wide inputs through the transpose with the outputs conjugated,
// QR first above qr_ratio_threshold) and 326-431 (`svd_imp`: bidiagonalize, the real bidiagonal problem, back-transforms 403-429).
//
// Arrangement (DESIGN.md §7 item 16):
//   reduction   bidiag_in_place (svd/bidiag.rs:47-256) in its unblocked form, faer's make_householder (householder.rs:59-107, as
//               qr_dd.cu / evd_dd.cu compute it) on the left and on the right; left reflector k below the diagonal of column k,
//               right reflector k right of the superdiagonal in row k. Per column, six launches with every sum in a fixed order:
//                 1. the left reflector (one CTA);
//                 2. y = v^H A22 / tau_l, one CTA per column;
//                 3. row k -= y, then the right reflector of row k (one CTA);
//                 4. A22 -= v y over row blocks x 64-column chunks, with the partial sums of z = A22 conj(u) of each chunk;
//                 5. z = (sum of the chunks) / tau_r;
//                 6. A22 -= z u^T.
//               No state lives in shared memory across columns, so the row count is not limited (bidiag.cu's persistent f64 kernel
//               keeps 8192-row vectors there and is real only).
//   real form   cx128: B = D_l B_real D_r^H with r_0 = 1, l_k = phase(d_k r_k), r_{k+1} = conj(phase(conj(l_k) f_k))
//               (cplx_condensed_core.cuh's BidiagPhases).
//   values      Golub-Kahan bisection (bidiag_sv.cuh) with fx128's eps, one thread per value, as svd.cu does for f64.
//   vectors     svd_vectors.cu's stabilised scheme in dd: the Golub-Kahan tridiagonal of order 2n through evd_dd.cu's divide and
//               conquer, the v parts of its n largest eigenvectors, Q_v from their dd QR, W = B Q_v, U_B from the dd QR of W, the
//               signs of diag R into U_B, a stable descending sort. U_B and Q_v are orthogonal by construction whatever the rank.
//   back-transform  U = H_left [D_l U_B 0; 0 I] and V = diag(1, conj H_right) D_r V_B through qr_blocked.cuh's block-Householder
//               sequences with T blocks of 64 reflectors; tall inputs lift U through the first QR's sequence.
// The dd glue kernels of the vectors path are written here rather than by templating svd_vectors.cu, so that the f64 object
// keeps its code and no dd code is compiled into it.
#include <algorithm>

#include "panel_common.cuh"  // before dd.cuh: its fb::__ldcg(const dd*) would hide the builtin overloads t_ldcg calls
#include "dd.cuh"
#include "qr_blocked.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"
#include "tridiag_dd.cuh"

namespace fb {

namespace {

constexpr int SD_CHUNK = 64;  // columns per partial sum of z = A22 conj(u)
constexpr int SD_BS = 64;     // reflectors per T block of the back-transforms
constexpr i64 SD_QR_BLOCKING = 48 * 48;  // QrParams::blocking_threshold default (qr/no_pivoting/factor.rs)

template <bool CX>
__device__ __forceinline__ cdd sd_ld(const dd* p, i64 off) {
  return CX ? cdd{p[2 * off], p[2 * off + 1]} : cdd{p[off], dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ void sd_st(dd* p, i64 off, cdd v) {
  if (CX) {
    p[2 * off] = v.re;
    p[2 * off + 1] = v.im;
  } else {
    p[off] = v.re;
  }
}
template <bool CX>
__device__ __forceinline__ cdd sd_mul(cdd a, cdd b) {
  return CX ? a * b : cdd{a.re * b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd sd_add(cdd a, cdd b) {
  return CX ? a + b : cdd{a.re + b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd sd_sub(cdd a, cdd b) {
  return CX ? cdd{a.re - b.re, a.im - b.im} : cdd{a.re - b.re, dd(0.0)};
}
template <bool CX>
__device__ __forceinline__ cdd sd_conj(cdd a) {
  return CX ? cdd_conj(a) : a;
}
__device__ __forceinline__ dd sd_shfl_xor(dd v, int off) {
  return dd(__shfl_xor_sync(0xffffffffu, v.hi, off), __shfl_xor_sync(0xffffffffu, v.lo, off));
}
// dd addition is commutative, so the xor butterfly leaves the same bits in every lane
__device__ __forceinline__ dd sd_warp_sum(dd v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = v + sd_shfl_xor(v, off);
  return v;
}
// sum over the CTA in a fixed order (warp butterflies, then the warps in order); every thread gets the result
template <int NT>
__device__ __forceinline__ dd sd_block_sum(dd v, dd* red) {
  v = sd_warp_sum(v);
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  dd s(0.0);
  for (int q = 0; q < NT / 32; ++q) s = s + red[q];
  return s;
}
// norm_l2.rs:161-172, three scaled accumulators
__device__ __forceinline__ dd sd_norm_select(dd s, dd m, dd b, dd sml, dd big) {
  if (s >= dd(1.0)) return sqrt(s) * big;
  if (m >= dd(1.0)) return sqrt(m);
  return sqrt(b) * sml;
}
// z / |z|, 1 for z = 0 or a non-finite z (svd/mod.rs:214-222 `normalized`: scaled by the larger part first)
__device__ __forceinline__ cdd sd_phase(cdd z) {
  const dd mx = fmax(fabs(z.re), fabs(z.im));
  if (mx == dd(0.0) || !dd_is_finite(mx)) return cdd{dd(1.0), dd(0.0)};
  const dd s = dd_recip(mx);
  const cdd y{z.re * s, z.im * s};
  const dd a = dd_recip(cdd_abs(y));
  return cdd{y.re * a, y.im * a};
}

// faer's make_householder on x[0], x[stride], ..., x[(len - 1) stride] (head x[0]) by one CTA of NT threads: beta into x[0], the
// essential part (tail / (head + signed_norm)) into the tail, tau into *tau, 1 / tau into *tau_inv (0 when tau = +inf, i.e. the
// tail vanishes and H = I); u = [1, essential] into ubuf when given
template <bool CX, int NT>
__device__ void sd_householder(dd* x, i64 stride, int len, dd* tau, dd* tau_inv, cdd* ubuf, dd* red, cdd* s_inv) {
  const dd sml = dd_sqrt_min_positive(), big = dd_sqrt_max_positive(), min_pos = dd_min_positive(), zero(0.0);
  dd acc[3] = {zero, zero, zero};
  for (int i = 1 + threadIdx.x; i < len; i += NT) {
    const cdd v = sd_ld<CX>(x, (i64)i * stride);
    const dd rs = v.re * sml, rb = v.re * big;
    acc[0] = dd_mul_add(rs, rs, acc[0]);
    acc[1] = dd_mul_add(v.re, v.re, acc[1]);
    acc[2] = dd_mul_add(rb, rb, acc[2]);
    if (CX) {
      const dd is = v.im * sml, ib = v.im * big;
      acc[0] = dd_mul_add(is, is, acc[0]);
      acc[1] = dd_mul_add(v.im, v.im, acc[1]);
      acc[2] = dd_mul_add(ib, ib, acc[2]);
    }
  }
  const dd s0 = sd_block_sum<NT>(acc[0], red), s1 = sd_block_sum<NT>(acc[1], red), s2 = sd_block_sum<NT>(acc[2], red);
  if (threadIdx.x == 0) {
    // make_householder_imp (householder.rs:59-107)
    const dd tail_norm = sd_norm_select(s0, s1, s2, sml, big);
    cdd head = sd_ld<CX>(x, 0);
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
      const cdd hs = sd_add<CX>(head, signed_norm);
      inv = CX ? cdd_recip_scaled(hs) : cdd{dd_recip(hs.re), zero};
      head = -signed_norm;
      const dd t = tail_norm * (CX ? cdd_abs(inv) : fabs(inv.re));
      t_au = dd(0.5) * (dd(1.0) + t * t);
    }
    *tau = t_au;
    *tau_inv = dd_recip(t_au);
    sd_st<CX>(x, 0, head);
    if (ubuf) ubuf[0] = cdd{dd(1.0), zero};
    *s_inv = inv;
  }
  __syncthreads();
  const cdd inv = *s_inv;
  for (int i = 1 + threadIdx.x; i < len; i += NT) {
    const cdd e = sd_mul<CX>(sd_ld<CX>(x, (i64)i * stride), inv);
    sd_st<CX>(x, (i64)i * stride, e);
    if (ubuf) ubuf[i] = e;
  }
}

// W (m x n, ld m) <- the source view, columns [c0, c0 + gridDim.y)
template <bool CX>
__global__ void sd_copy_kernel(dd* __restrict__ W, i64 m, const dd* __restrict__ src, i64 rs, i64 cs, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < m) sd_st<CX>(W, j * m + i, sd_ld<CX>(src, i * rs + j * cs));
}
// flag[0] <- 1 if any of the cnt dd values is not finite
__global__ void sd_finite_kernel(const dd* __restrict__ x, i64 cnt, int* flag) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt && !dd_is_finite(x[i])) *flag = 1;
}
// R (n x n, ld n) <- the upper triangle of the leading n x n block of QR (ld ldq), zero below
template <bool CX>
__global__ void sd_copy_upper_kernel(dd* __restrict__ R, i64 n, const dd* __restrict__ QR, i64 ldq, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < n) sd_st<CX>(R, j * n + i, i <= j ? sd_ld<CX>(QR, j * ldq + i) : cdd{dd(0.0), dd(0.0)});
}

// ---- bidiagonalization, column k of W (m x n, ld m); tl / tr: the left / right taus; sc[0] = 1 / tau_l, sc[1] = 1 / tau_r ----
// 1. the left reflector of column k (rows k ..)
template <bool CX>
__global__ void __launch_bounds__(512) sd_left_house_kernel(dd* W, int m, int k, dd* tl, dd* sc) {
  __shared__ dd red[16];
  __shared__ cdd s_inv;
  sd_householder<CX, 512>(W + (CX ? 2 : 1) * ((i64)k * m + k), 1, m - k, tl + k, sc, nullptr, red, &s_inv);
}
// 2. y_j = (1 / tau_l) sum_i conj(v_i) W(k + i, k + 1 + j), v_0 = 1; one CTA per column
template <bool CX>
__global__ void __launch_bounds__(256) sd_vhm_kernel(const dd* __restrict__ W, int m, int k, const dd* __restrict__ sc,
                                                     cdd* __restrict__ y) {
  __shared__ dd red[8];
  const int rows = m - k, j = blockIdx.x;
  const dd* v = W + (CX ? 2 : 1) * ((i64)k * m + k);
  const dd* a = W + (CX ? 2 : 1) * ((i64)(k + 1 + j) * m + k);
  cdd acc{dd(0.0), dd(0.0)};
  for (int i = threadIdx.x; i < rows; i += 256) {
    const cdd vi = i == 0 ? cdd{dd(1.0), dd(0.0)} : sd_ld<CX>(v, i);
    acc = sd_add<CX>(acc, sd_mul<CX>(sd_conj<CX>(vi), sd_ld<CX>(a, i)));
  }
  const dd re = sd_block_sum<256>(acc.re, red);
  const dd im = CX ? sd_block_sum<256>(acc.im, red) : dd(0.0);
  if (threadIdx.x == 0) y[j] = cdd{re * sc[0], CX ? im * sc[0] : dd(0.0)};
}
// 3. row k (columns k + 1 ..) -= y, then the right reflector of that row; u = [1, essential] into ubuf
template <bool CX>
__global__ void __launch_bounds__(512) sd_right_house_kernel(dd* W, int m, int n, int k, const cdd* __restrict__ y, dd* tr, dd* sc,
                                                             cdd* ubuf) {
  __shared__ dd red[16];
  __shared__ cdd s_inv;
  const int cols = n - k - 1;
  dd* row = W + (CX ? 2 : 1) * ((i64)(k + 1) * m + k);
  for (int j = threadIdx.x; j < cols; j += 512) sd_st<CX>(row, (i64)j * m, sd_sub<CX>(sd_ld<CX>(row, (i64)j * m), y[j]));
  __syncthreads();
  sd_householder<CX, 512>(row, m, cols, tr + k, sc + 1, ubuf, red, &s_inv);
}
// 4. A22 = W[k+1.., k+1..] -= v y (v: column k below the diagonal), and part[c][i] = sum_{j in chunk c} A22(i, j) conj(u_j)
template <bool CX>
__global__ void __launch_bounds__(128) sd_left_update_kernel(dd* W, int m, int n, int k, const cdd* __restrict__ y,
                                                             const cdd* __restrict__ ubuf, cdd* __restrict__ part) {
  __shared__ cdd ys[SD_CHUNK], us[SD_CHUNK];
  const int rows = m - k - 1, cols = n - k - 1, c = blockIdx.y, j0 = c * SD_CHUNK, j1 = min(cols, j0 + SD_CHUNK);
  if (threadIdx.x < j1 - j0) {
    ys[threadIdx.x] = y[j0 + threadIdx.x];
    us[threadIdx.x] = sd_conj<CX>(ubuf[j0 + threadIdx.x]);
  }
  __syncthreads();
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= rows) return;
  const cdd vi = sd_ld<CX>(W, (i64)k * m + k + 1 + i);
  dd* base = W + (CX ? 2 : 1) * ((i64)(k + 1) * m + k + 1);
  cdd acc{dd(0.0), dd(0.0)};
  for (int j = j0; j < j1; ++j) {
    const i64 off = (i64)j * m + i;
    const cdd a = sd_sub<CX>(sd_ld<CX>(base, off), sd_mul<CX>(vi, ys[j - j0]));
    sd_st<CX>(base, off, a);
    acc = sd_add<CX>(acc, sd_mul<CX>(a, us[j - j0]));
  }
  part[(i64)c * m + i] = acc;
}
// 5. z_i = (1 / tau_r) sum_c part[c][i], the chunks in order
template <bool CX>
__global__ void __launch_bounds__(256) sd_z_kernel(int m, int k, const cdd* __restrict__ part, int nchunk, const dd* __restrict__ sc,
                                                   cdd* __restrict__ z) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= m - k - 1) return;
  cdd s = part[i];
  for (int c = 1; c < nchunk; ++c) s = sd_add<CX>(s, part[(i64)c * m + i]);
  z[i] = cdd{s.re * sc[1], CX ? s.im * sc[1] : dd(0.0)};
}
// 6. A22 -= z u^T, 16 columns per thread
template <bool CX>
__global__ void __launch_bounds__(128) sd_right_update_kernel(dd* W, int m, int n, int k, const cdd* __restrict__ z,
                                                              const cdd* __restrict__ ubuf) {
  const int rows = m - k - 1, cols = n - k - 1;
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i >= rows) return;
  dd* base = W + (CX ? 2 : 1) * ((i64)(k + 1) * m + k + 1);
  const cdd zi = z[i];
  for (int j = blockIdx.y * 16; j < min(cols, (int)blockIdx.y * 16 + 16); ++j) {
    const i64 off = (i64)j * m + i;
    sd_st<CX>(base, off, sd_sub<CX>(sd_ld<CX>(base, off), sd_mul<CX>(zi, ubuf[j])));
  }
}

// the real bidiagonal (d, f) and, for cx128, the phases l, r (B = D_l B_real D_r^H); flag[0] = 1 on a non-finite entry. One thread.
template <bool CX>
__global__ void sd_extract_kernel(const dd* __restrict__ W, int m, int n, dd* __restrict__ d, dd* __restrict__ f, cdd* __restrict__ l,
                                  cdd* __restrict__ r, int* flag) {
  int bad = 0;
  cdd rk{dd(1.0), dd(0.0)};
  for (int k = 0; k < n; ++k) {
    const cdd dk = sd_ld<CX>(W, (i64)k * m + k);
    if (!dd_is_finite(dk.re) || !dd_is_finite(dk.im)) bad = 1;
    if (CX) {
      r[k] = rk;
      const cdd lk = sd_phase(dk * rk);
      l[k] = lk;
      d[k] = cdd_abs(dk);
      if (k + 1 < n) {
        const cdd fk = sd_ld<CX>(W, (i64)(k + 1) * m + k);
        if (!dd_is_finite(fk.re) || !dd_is_finite(fk.im)) bad = 1;
        f[k] = cdd_abs(fk);
        rk = cdd_conj(sd_phase(cdd_conj(lk) * fk));
      }
    } else {
      d[k] = dk.re;
      if (k + 1 < n) {
        f[k] = sd_ld<CX>(W, (i64)(k + 1) * m + k).re;
        if (!dd_is_finite(f[k])) bad = 1;
      }
    }
  }
  if (n > 0) f[n - 1] = dd(0.0);
  flag[0] |= bad;
}

// ---- values only: Gershgorin bound of the Golub-Kahan form and one bisection thread per value ----
// bb[0] >= sigma_max, bb[1] = max b_j^2 (svd.cu's gk_bound_kernel in one thread)
__global__ void sd_gk_bound_kernel(const dd* __restrict__ d, const dd* __restrict__ f, int n, dd* __restrict__ bb) {
  dd bound(0.0), b2(0.0);
  for (int i = 0; i < n; ++i) {
    const dd a = fabs(d[i]), b = i + 1 < n ? fabs(f[i]) : dd(0.0), c = i > 0 ? fabs(f[i - 1]) : dd(0.0);
    bound = fmax(bound, fmax(a + b, a + c));
    b2 = fmax(b2, fmax(a * a, b * b));
  }
  bb[0] = bound * (dd(1.0) + dd(4.0) * bsv::Lim<dd>::eps()) + bsv::Lim<dd>::safmin();
  bb[1] = b2;
}
__global__ void __launch_bounds__(64) sd_gk_values_kernel(const dd* __restrict__ d, const dd* __restrict__ f, int n,
                                                           const dd* __restrict__ bb, dd* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = bsv::gk_kth_largest<dd>(d, f, n, 1, 1, k, bb[0], bb[1]);
}

// ---- with vectors: svd_vectors.cu's glue kernels in dd ----
// Golub-Kahan off-diagonals (d_0, f_0, d_1, ..., d_{n-1}); diag <- 0
__global__ void sd_tgk_kernel(const dd* __restrict__ d, const dd* __restrict__ f, int n, dd* __restrict__ diag, dd* __restrict__ off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    off[2 * i] = d[i];
    if (i + 1 < n) off[2 * i + 1] = f[i];
    diag[2 * i] = dd(0.0);
    diag[2 * i + 1] = dd(0.0);
  }
}
// Vh(i, j) = QT(2 i, 2n - 1 - j): the v parts of the eigenvectors of the n largest eigenvalues, largest first
__global__ void sd_vparts_kernel(dd* __restrict__ Vh, i64 n, const dd* __restrict__ QT, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < n) Vh[j * n + i] = QT[(2 * n - 1 - j) * (2 * n) + 2 * i];
}
// W = B X, B upper bidiagonal (d, f): W(i, :) = d_i X(i, :) + f_i X(i + 1, :)
__global__ void sd_bidiag_times_kernel(dd* __restrict__ W, const dd* __restrict__ X, i64 n, const dd* __restrict__ d,
                                       const dd* __restrict__ f, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < n) W[j * n + i] = d[i] * X[j * n + i] + (i + 1 < n ? f[i] * X[j * n + i + 1] : dd(0.0));
}
// s_j = |R_jj|, sg_j = sign(R_jj) (1 for 0)
__global__ void sd_diag_sign_kernel(const dd* __restrict__ R, i64 ld, int n, dd* __restrict__ s, dd* __restrict__ sg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const dd r = R[(i64)i + (i64)i * ld];
    s[i] = fabs(r);
    sg[i] = r < dd(0.0) ? dd(-1.0) : dd(1.0);
  }
}
// pos[j] = position of s_j in non-increasing order (stable); sorted[pos[j]] = s_j
__global__ void sd_rank_desc_kernel(const dd* __restrict__ s, int n, int* __restrict__ pos, dd* __restrict__ sorted) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const dd v = s[j];
  int c = 0;
  for (int u = 0; u < n; ++u) c += (s[u] > v) || (s[u] == v && u < j);
  pos[j] = c;
  sorted[c] = v;
}
// dst(:, pos[j]) = scale[j] * src(:, j) (scale == nullptr: 1), n x n, ld n
__global__ void sd_scatter_kernel(dd* __restrict__ dst, const dd* __restrict__ src, i64 n, const int* __restrict__ pos,
                                  const dd* __restrict__ scale, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < n) dst[(i64)pos[j] * n + i] = scale ? scale[j] * src[j * n + i] : src[j * n + i];
}
// M (rows x cols, ld rows) <- identity
__global__ void sd_identity_kernel(dd* __restrict__ M, i64 rows, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < rows) M[j * rows + i] = dd(i == j ? 1.0 : 0.0);
}

// ---- back-transforms ----
// out (rows x cols, ld rows) <- [diag(ph) Q 0; 0 I] with Q real (k x k, ld k); ph == nullptr: no phases (fx128)
template <bool CX>
__global__ void sd_embed_kernel(dd* __restrict__ out, i64 rows, const dd* __restrict__ Q, i64 k, const cdd* __restrict__ ph, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i >= rows) return;
  cdd v{dd(i == j ? 1.0 : 0.0), dd(0.0)};
  if (i < k && j < k) {
    const dd q = Q[j * k + i];
    v = CX ? cdd{ph[i].re * q, ph[i].im * q} : cdd{q, dd(0.0)};
  }
  sd_st<CX>(out, j * rows + i, v);
}
// T blocks' diagonals: Tf(j % bs, j) = tau_j
template <bool CX>
__global__ void sd_tdiag_kernel(dd* Tf, const dd* tau, int bs, int cnt) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < cnt) sd_st<CX>(Tf, (i64)j * bs + j % bs, cdd{tau[j], dd(0.0)});
}
// T (n - 1 x n - 1, ld n - 1) <- the rows of W right of the diagonal as columns: T(i, j) = W(j, i + 1) (svd/mod.rs:413-419)
template <bool CX>
__global__ void sd_transpose_rows_kernel(dd* __restrict__ T, const dd* __restrict__ W, i64 ldw, i64 n1, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i < n1) sd_st<CX>(T, j * n1 + i, sd_ld<CX>(W, (i + 1) * ldw + j));
}
// out view <- src (rows x cols, ld rows), conjugated when asked (the swapped outputs of a wide cx128 input)
template <bool CX>
__global__ void sd_store_kernel(View<dd> out, const dd* __restrict__ src, bool conj, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x, j = c0 + blockIdx.y;
  if (i >= out.nrows) return;
  const cdd v = sd_ld<CX>(src, j * out.nrows + i);
  sd_st<CX>(out.ptr, i * out.rs + j * out.cs, conj ? sd_conj<CX>(v) : v);
}
// S (compact, element units) <- the real values (cx128: (value, 0))
template <bool CX>
__global__ void sd_values_out_kernel(dd* S, const dd* s, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sd_st<CX>(S, i, cdd{s[i], dd(0.0)});
}

// launches over (rows in blocks of 256) x (columns in chunks of <= 65535)
template <class F>
void sd_cols(i64 rows, i64 cols, F&& f) {
  for (i64 c0 = 0; c0 < cols; c0 += 65535) {
    f(dim3((unsigned)((rows + 255) / 256), (unsigned)std::min<i64>(65535, cols - c0)), c0);
    note_launch();
  }
  FB_CUDA_CHECK(cudaGetLastError());
}

// Q factor (n x n, ld n) of the dd QR stored in QR (n x n) with its block factor H (bs x n)
void sd_form_q(cudaStream_t st, const dd* QR, i64 n, const dd* H, i64 bs, dd* Q) {
  sd_cols(n, n, [&](dim3 g, i64 c0) { sd_identity_kernel<<<g, 256, 0, st>>>(Q, n, c0); });
  apply_householder_sequence_left_t<dd, false>(st, View<const dd>{QR, n, n, 1, n}, View<const dd>{H, bs, n, 1, bs}, false,
                                               View<dd>{Q, n, n, 1, n}, false);
}

// SVD of the real upper-bidiagonal (d, f) of order n: S_sorted non-increasing, UB and VB (n x n, ld n) with B = UB diag(S) VB^T, the
// columns in the sorted order. False if a leaf of the divide and conquer did not converge.
bool sd_bidiag_svd_vectors(cudaStream_t st, const dd* d, const dd* f, i64 n, dd* S_sorted, dd* UB, dd* VB) {
  const i64 n2 = 2 * n;
  dd* tg = (dd*)ws_alloc((size_t)(3 * n2 + 8) * sizeof(dd));
  dd *tdiag = tg, *toff = tg + n2, *tlam = tg + 2 * n2;
  dd* QT = (dd*)ws_alloc((size_t)n2 * (size_t)n2 * sizeof(dd));
  bool ok;
  {
    LaunchTag tag(LAUNCH_SOLVE);
    sd_tgk_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d, f, (int)n, tdiag, toff);
    note_launch();
    ok = tridiag_dc_dd(st, tdiag, toff, n2, tlam, QT);
  }
  dd* Vh = (dd*)ws_alloc((size_t)n * (size_t)n * sizeof(dd));
  sd_cols(n, n, [&](dim3 g, i64 c0) { sd_vparts_kernel<<<g, 256, 0, st>>>(Vh, n, QT, c0); });
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(QT);
  const i64 bs = qr_recommended_block_size(n, n);
  dd* H = (dd*)ws_alloc((size_t)bs * (size_t)n * sizeof(dd));
  // Q_v
  qr_dd<false>(st, View<dd>{Vh, n, n, 1, n}, View<dd>{H, bs, n, 1, bs}, SD_QR_BLOCKING);
  dd* Qv = (dd*)ws_alloc((size_t)n * (size_t)n * sizeof(dd));
  sd_form_q(st, Vh, n, H, bs, Qv);
  // W = B Q_v, its QR, U_B
  dd* Wm = Vh;
  sd_cols(n, n, [&](dim3 g, i64 c0) { sd_bidiag_times_kernel<<<g, 256, 0, st>>>(Wm, Qv, n, d, f, c0); });
  qr_dd<false>(st, View<dd>{Wm, n, n, 1, n}, View<dd>{H, bs, n, 1, bs}, SD_QR_BLOCKING);
  dd* sv = (dd*)ws_alloc((size_t)(2 * n + 2) * sizeof(dd) + (size_t)n * 4 + 16);
  dd *s_raw = sv, *sg = sv + n;
  int* pos = (int*)(sv + 2 * n + 2);
  sd_diag_sign_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(Wm, n, (int)n, s_raw, sg);
  sd_rank_desc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s_raw, (int)n, pos, S_sorted);
  note_launch();
  note_launch();
  dd* Ub = (dd*)ws_alloc((size_t)n * (size_t)n * sizeof(dd));
  sd_form_q(st, Wm, n, H, bs, Ub);
  sd_cols(n, n, [&](dim3 g, i64 c0) { sd_scatter_kernel<<<g, 256, 0, st>>>(UB, Ub, n, pos, sg, c0); });
  sd_cols(n, n, [&](dim3 g, i64 c0) { sd_scatter_kernel<<<g, 256, 0, st>>>(VB, Qv, n, pos, nullptr, c0); });
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(Ub);
  ws_free(sv);
  ws_free(Qv);
  ws_free(H);
  ws_free(Vh);
  ws_free(tg);
  return ok;
}

// Tf (bs x cnt, ld bs) <- the T blocks of the cnt reflectors in the columns of basis (upgrade_householder_factor per block)
template <bool CX>
dd* sd_tblocks(cudaStream_t st, View<const dd> basis, const dd* tau, i64 cnt, i64 bs) {
  const size_t esz = (CX ? 2 : 1) * sizeof(dd);
  dd* Tf = (dd*)ws_alloc((size_t)bs * (size_t)cnt * esz);
  FB_CUDA_CHECK(cudaMemsetAsync(Tf, 0, (size_t)bs * (size_t)cnt * esz, st));
  sd_tdiag_kernel<CX><<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(Tf, tau, (int)bs, (int)cnt);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  const View<dd> Tv{Tf, bs, cnt, 1, bs};
  for (i64 j = 0; j < cnt; j += bs) {
    const i64 b = std::min(bs, cnt - j);
    upgrade_householder_factor_t<dd, CX>(st, sub_t<dd, CX>(Tv, 0, j, b, b), sub_t<dd, CX>(basis, j, j, basis.nrows - j, b), b, 1);
  }
  return Tf;
}

}  // namespace

// A: device view (element units; complex units for cx128); U, V: device views, or ptr == nullptr / ncols == 0 for "not computed";
// U is nrows x {size, nrows}, V is ncols x {size, ncols}; S: min(m, n) device entries in element units, non-increasing. Returns
// false for non-finite input (SvdError::NoConvergence) or a divide-and-conquer leaf that did not converge.
template <bool CX>
bool svd_dd(cudaStream_t st, View<const dd> A, View<dd> U, dd* S, View<dd> V, double qr_ratio_threshold) {
  // svd/mod.rs:560-575: a wide input is transposed (not conjugated), U and V swap, and the outputs are conjugated at the end
  const bool transpose = A.ncols > A.nrows;
  const View<const dd> M = transpose ? A.t() : A;
  const View<dd> Um = transpose ? V : U, Vm = transpose ? U : V;
  const bool conj_out = CX && transpose;
  const i64 m = M.nrows, n = M.ncols;
  const bool want_u = Um.ptr != nullptr && Um.ncols > 0, want_v = Vm.ptr != nullptr && Vm.ncols > 0;
  const size_t esz = (CX ? 2 : 1) * sizeof(dd);
  if (want_u) FB_ASSERT(Um.nrows == m && (Um.ncols == n || Um.ncols == m), "svd: the left factor must be nrows x {size, nrows}");
  if (want_v) FB_ASSERT(Vm.nrows == n && Vm.ncols == n, "svd: the right factor must be ncols x {size, ncols}");
  if (n == 0) {
    if (want_u) {  // no singular values: the full left factor is the identity
      dd* I = (dd*)ws_alloc((size_t)std::max<i64>(1, m * Um.ncols) * esz);
      sd_cols(m, Um.ncols, [&](dim3 g, i64 c0) { sd_embed_kernel<CX><<<g, 256, 0, st>>>(I, m, nullptr, 0, nullptr, c0); });
      sd_cols(m, Um.ncols, [&](dim3 g, i64 c0) { sd_store_kernel<CX><<<g, 256, 0, st>>>(Um, I, false, c0); });
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(I);
    }
    return true;
  }
  FB_ASSERT(m < (1ll << 31), "svd: dimension too large");
  dd* Wk = (dd*)ws_alloc((size_t)m * (size_t)n * esz);
  sd_cols(m, n, [&](dim3 g, i64 c0) { sd_copy_kernel<CX><<<g, 256, 0, st>>>(Wk, m, M.ptr, M.rs, M.cs, c0); });
  int* flag = (int*)ws_alloc(16);
  FB_CUDA_CHECK(cudaMemsetAsync(flag, 0, 4, st));
  {
    const i64 cnt = (i64)m * n * (CX ? 2 : 1);
    sd_finite_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(Wk, cnt, flag);
    note_launch();
  }
  // ---- QR first for tall inputs (svd/mod.rs:594-633) ----
  const bool qr_first = (double)m / (double)n > qr_ratio_threshold && n > 1;
  dd *Hq = nullptr, *R = nullptr;
  i64 bsq = 0, mb = m;
  if (qr_first) {
    bsq = qr_recommended_block_size(m, n);
    Hq = (dd*)ws_alloc((size_t)bsq * (size_t)n * esz);
    qr_dd<CX>(st, View<dd>{Wk, m, n, 1, m}, View<dd>{Hq, bsq, n, 1, bsq}, SD_QR_BLOCKING);
    R = (dd*)ws_alloc((size_t)n * (size_t)n * esz);
    sd_cols(n, n, [&](dim3 g, i64 c0) { sd_copy_upper_kernel<CX><<<g, 256, 0, st>>>(R, n, Wk, m, c0); });
    mb = n;
  }
  dd* Bm = R ? R : Wk;
  // ---- bidiagonalization (svd/bidiag.rs:47-256) ----
  dd* taus = (dd*)ws_alloc((size_t)(2 * n + 4) * sizeof(dd));
  dd *tl = taus, *tr = taus + n, *sc = taus + 2 * n;
  const int nchunk = (int)std::max<i64>(1, (n + SD_CHUNK - 1) / SD_CHUNK);
  cdd* y = (cdd*)ws_alloc((size_t)n * sizeof(cdd));
  cdd* ubuf = (cdd*)ws_alloc((size_t)n * sizeof(cdd));
  cdd* z = (cdd*)ws_alloc((size_t)mb * sizeof(cdd));
  cdd* part = (cdd*)ws_alloc((size_t)nchunk * (size_t)mb * sizeof(cdd));
  {
    LaunchTag tag(LAUNCH_PANEL);
    const int mi = (int)mb, ni = (int)n;
    for (int k = 0; k < ni; ++k) {
      const int rows = mi - k - 1, cols = ni - k - 1;
      sd_left_house_kernel<CX><<<1, 512, 0, st>>>(Bm, mi, k, tl, sc);
      note_launch();
      if (cols == 0) break;
      sd_vhm_kernel<CX><<<(unsigned)cols, 256, 0, st>>>(Bm, mi, k, sc, y);
      sd_right_house_kernel<CX><<<1, 512, 0, st>>>(Bm, mi, ni, k, y, tr, sc, ubuf);
      for (int q = 0; q < 2; ++q) note_launch();
      if (rows > 0) {
        const int nc = (cols + SD_CHUNK - 1) / SD_CHUNK;
        sd_left_update_kernel<CX><<<dim3((unsigned)((rows + 127) / 128), (unsigned)nc), 128, 0, st>>>(Bm, mi, ni, k, y, ubuf, part);
        note_launch();
        if (cols > 1) {  // a one-entry row has tau_r = +inf: z = 0
          sd_z_kernel<CX><<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(mi, k, part, nc, sc, z);
          sd_right_update_kernel<CX><<<dim3((unsigned)((rows + 127) / 128), (unsigned)((cols + 15) / 16)), 128, 0, st>>>(Bm, mi, ni, k, z,
                                                                                                                       ubuf);
          for (int q = 0; q < 2; ++q) note_launch();
        }
      }
      FB_CUDA_CHECK(cudaGetLastError());
    }
  }
  dd* de = (dd*)ws_alloc((size_t)(4 * n + 4) * sizeof(dd));
  dd *d = de, *f = de + n, *s_sorted = de + 2 * n, *bb = de + 3 * n;
  cdd* ph = CX ? (cdd*)ws_alloc((size_t)(2 * n) * sizeof(cdd)) : nullptr;
  cdd *pl = ph, *pr = CX ? ph + n : nullptr;
  sd_extract_kernel<CX><<<1, 1, 0, st>>>(Bm, (int)mb, (int)n, d, f, pl, pr, flag);
  note_launch();
  int h_flag = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, flag, 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  bool ok = h_flag == 0;
  if (ok && !want_u && !want_v) {
    LaunchTag tag(LAUNCH_SOLVE);
    sd_gk_bound_kernel<<<1, 1, 0, st>>>(d, f, (int)n, bb);
    sd_gk_values_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(d, f, (int)n, bb, s_sorted);
    FB_CUDA_CHECK(cudaGetLastError());
    for (int q = 0; q < 2; ++q) note_launch();
  } else if (ok) {
    dd* UB = (dd*)ws_alloc((size_t)n * (size_t)n * sizeof(dd));
    dd* VB = (dd*)ws_alloc((size_t)n * (size_t)n * sizeof(dd));
    ok = sd_bidiag_svd_vectors(st, d, f, n, s_sorted, UB, VB);
    const i64 bs = std::min<i64>(SD_BS, n);
    if (ok && want_u) {
      // U = H_left [D_l U_B 0; 0 I] (svd/mod.rs:403-412, Conj::No); tall inputs: the bidiagonal's sequence on the leading n x n
      // block, then the QR's sequence on all of U (svd/mod.rs:634-658)
      const i64 ku = Um.ncols;
      dd* Uw = (dd*)ws_alloc((size_t)m * (size_t)ku * esz);
      sd_cols(m, ku, [&](dim3 g, i64 c0) { sd_embed_kernel<CX><<<g, 256, 0, st>>>(Uw, m, UB, n, pl, c0); });
      const View<dd> Uv{Uw, m, ku, 1, m};
      const View<const dd> basis{Bm, mb, n, 1, mb};
      dd* Tl = sd_tblocks<CX>(st, basis, tl, n, bs);
      apply_householder_sequence_left_t<dd, CX>(st, basis, View<const dd>{Tl, bs, n, 1, bs}, false,
                                                qr_first ? sub_t<dd, CX>(Uv, 0, 0, n, n) : Uv, false);
      if (qr_first)
        apply_householder_sequence_left_t<dd, CX>(st, View<const dd>{Wk, m, n, 1, m}, View<const dd>{Hq, bsq, n, 1, bsq}, false, Uv, false);
      sd_cols(m, ku, [&](dim3 g, i64 c0) { sd_store_kernel<CX><<<g, 256, 0, st>>>(Um, Uw, conj_out, c0); });
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(Tl);
      ws_free(Uw);
    }
    if (ok && want_v) {
      // V = diag(1, H_right) D_r V_B: the right reflectors are the rows right of the superdiagonal, applied as columns with
      // Conj::Yes (svd/mod.rs:413-429)
      dd* Vw = (dd*)ws_alloc((size_t)n * (size_t)n * esz);
      sd_cols(n, n, [&](dim3 g, i64 c0) { sd_embed_kernel<CX><<<g, 256, 0, st>>>(Vw, n, VB, n, pr, c0); });
      if (n > 1) {
        const i64 n1 = n - 1, bsr = std::min<i64>(SD_BS, n1);
        dd* Tb = (dd*)ws_alloc((size_t)n1 * (size_t)n1 * esz);
        sd_cols(n1, n1, [&](dim3 g, i64 c0) { sd_transpose_rows_kernel<CX><<<g, 256, 0, st>>>(Tb, Bm, mb, n1, c0); });
        const View<const dd> basis{Tb, n1, n1, 1, n1};
        dd* Tr = sd_tblocks<CX>(st, basis, tr, n1, bsr);
        apply_householder_sequence_left_t<dd, CX>(st, basis, View<const dd>{Tr, bsr, n1, 1, bsr}, true,
                                                  sub_t<dd, CX>(View<dd>{Vw, n, n, 1, n}, 1, 0, n1, n), false);
        FB_CUDA_CHECK(cudaStreamSynchronize(st));
        ws_free(Tr);
        ws_free(Tb);
      }
      sd_cols(n, n, [&](dim3 g, i64 c0) { sd_store_kernel<CX><<<g, 256, 0, st>>>(Vm, Vw, conj_out, c0); });
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(Vw);
    }
    ws_free(VB);
    ws_free(UB);
  }
  if (ok) {
    sd_values_out_kernel<CX><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, s_sorted, (int)n);
    note_launch();
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (ph) ws_free(ph);
  ws_free(de);
  ws_free(part);
  ws_free(z);
  ws_free(ubuf);
  ws_free(y);
  ws_free(taus);
  if (R) ws_free(R);
  if (Hq) ws_free(Hq);
  ws_free(flag);
  ws_free(Wk);
  return ok;
}

template bool svd_dd<false>(cudaStream_t, View<const dd>, View<dd>, dd*, View<dd>, double);
template bool svd_dd<true>(cudaStream_t, View<const dd>, View<dd>, dd*, View<dd>, double);

}  // namespace fb
