// Divide-and-conquer eigensolver for symmetric tridiagonal matrices on the GPU (f64), all eigenvectors.
//
// Replaces `evd::tridiag_evd::divide_and_conquer` + `qr_algorithm` (reference faer/src/linalg/evd/tridiag_evd.rs:270-665,
// 8-268) and, through the Golub-Kahan form, the vector part of `svd::bidiag_svd` (svd/bidiag_svd.rs:1005-...; svd.cu explains
// how). The scalar numerics live in tridiag_dc_core.cuh (shared with the CPU harness tools/emul/tridiag_dc_host.cpp, which
// runs the same steps in the same order); this file is their parallel arrangement:
//
//   * balanced tree: L levels, 2^L leaves of 16..32 rows; block j of level l is [ (j n) >> l, ((j+1) n) >> l ). Every
//     tear (Cuppen) is applied up front: |beta| comes off the two diagonal entries next to each cut;
//   * leaves: one warp per leaf runs implicit QL redundantly in every lane (private d, e), lane r owning row r of the leaf's
//     eigenvector block in shared memory;
//   * one pass per level, every merge of the level in the same launches (grid.y = merge), no host synchronisation:
//       prepare   z from the adjacent rows of the two eigenvector blocks, merged order by ranks (binary searches), then ONE
//                 thread runs the dlaed2-style deflation scan (inherently sequential, O(s))
//       secular   one warp per root: safeguarded bisection on the shifted secular function, the sum shared by the lanes;
//                 writes lambda_j and column j of DELTA = (d_i - lambda_j), formed without cancellation
//       zhat      Gu-Eisenstat: z-hat_i from products over DELTA's rows (thread per i, coalesced along i)
//       order     output position of every new eigenvalue by counting (roots and deflated values interleave)
//       vectors   one CTA per root: v = z-hat / DELTA[:, j], normalised, scattered into the merge matrix W (s x s) at the
//                 rows of the non-deflated columns; deflated columns get a unit entry
//       rotate    the deflation's Givens rotations folded into W's rows (last first), so the old eigenvector blocks stay
//                 block diagonal and
//       Q_new[lo:mid, lo:hi] = Q1 * W[0:s1, :],  Q_new[mid:hi, lo:hi] = Q2 * W[s1:, :]   — two DMMA GEMMs per merge
//     (4/3 n^3 flop over all levels; deflation is not exploited to shrink them).
// Eigenvalues come out ascending, eigenvectors orthogonal to working precision whatever the clustering (tests:
// tests/test_tridiag_dc_cpu.py on the CPU harness, tests/test_gpu_zz11_evd_svd_vectors.py and
// tests/test_gpu_zz24_spectral_exact.py on the device).
#include <algorithm>
#include <vector>

#include "panel_common.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"
#include "tridiag_dc_core.cuh"

namespace fb {

namespace {

constexpr int DC_LEAF = 32;

struct DcMerge {
  int lo, mid, hi;
};

struct DcBuf {
  double *d, *e;          // [n] working diagonal (sorted per block) / off-diagonal
  double *dsort, *zsort;  // [n]
  double *dl, *w, *dd;    // [n] non-deflated d / z, deflated d
  double *rc, *rs;        // [n] rotations
  double *lam, *zh, *dnew;
  double *rho, *sgn;      // [nmerge_total]
  int *colsort, *cnd, *cdf, *ra, *rb, *outcol;
  int *kcnt, *nrot;       // [nmerge_total]
  double* scale;          // [2]: scale, nonfinite flag
};

__global__ void dc_scale_kernel(double* d, double* e, int n, double* scale) {
  __shared__ double red[256];
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  double mx = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const double a = fabs(d[i]), b = i + 1 < n ? fabs(e[i]) : 0.0;
    if (!(a < TLim<double>::inf()) || !(b < TLim<double>::inf())) bad = 1;
    mx = fmax(mx, fmax(a, b));
  }
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if ((int)threadIdx.x < off) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + off]);
    __syncthreads();
  }
  const double s = (red[0] > 0.0 && !bad) ? red[0] : 1.0;
  if (threadIdx.x == 0) {
    scale[0] = s;
    scale[1] = bad ? 1.0 : 0.0;
  }
  for (int i = threadIdx.x; i < n; i += 256) {
    d[i] /= s;
    if (i + 1 < n) e[i] /= s;
    else e[i] = 0.0;
  }
}

// every cut of every level: rho, sign, and the two diagonal entries next to it
__global__ void dc_tear_kernel(double* d, const double* e, const DcMerge* merges, int nmerge, double* rho, double* sgn) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= nmerge) return;
  const int mid = merges[m].mid;
  const double beta = e[mid - 1];
  rho[m] = fabs(beta);
  sgn[m] = beta < 0.0 ? -1.0 : 1.0;
  // cuts are at least 16 rows apart: no two threads touch the same entry
  d[mid - 1] -= fabs(beta);
  d[mid] -= fabs(beta);
}

__global__ void __launch_bounds__(32) dc_leaf_kernel(double* d, const double* e, double* Q, i64 ldq, int n, int nlev, int* fail) {
  __shared__ double Z[DC_LEAF][DC_LEAF + 1];
  const int leaf = blockIdx.x, lane = threadIdx.x;
  const int lo = (int)(((long long)leaf * n) >> nlev), hi = (int)(((long long)(leaf + 1) * n) >> nlev);
  const int s = hi - lo;
  double dd[DC_LEAF], ee[DC_LEAF];
#pragma unroll
  for (int i = 0; i < DC_LEAF; ++i) {
    dd[i] = i < s ? d[lo + i] : 0.0;
    ee[i] = (i + 1 < s) ? e[lo + i] : 0.0;
  }
  for (int j = 0; j < DC_LEAF; ++j) Z[lane][j] = lane == j ? 1.0 : 0.0;
  __syncwarp();
  const bool ok = dc::ql_implicit(dd, ee, s, [&](int i, double c, double sn) {
    if (lane < s) {
      const double f = Z[lane][i + 1];
      Z[lane][i + 1] = sn * Z[lane][i] + c * f;
      Z[lane][i] = c * Z[lane][i] - sn * f;
    }
  });
  if (!ok && lane == 0) *fail = 1;
  // ascending order (selection sort, the same in every lane) with column swaps of this lane's row
  for (int i = 0; i < s; ++i) {
    int kmin = i;
    for (int j = i + 1; j < s; ++j)
      if (dd[j] < dd[kmin]) kmin = j;
    if (kmin != i) {
      const double t = dd[i];
      dd[i] = dd[kmin];
      dd[kmin] = t;
      if (lane < s) {
        const double u = Z[lane][i];
        Z[lane][i] = Z[lane][kmin];
        Z[lane][kmin] = u;
      }
    }
  }
  __syncwarp();
  if (lane < s) d[lo + lane] = dd[lane];
  // Q block (column-major): element (row r, column c) at Q[(lo + c) * ldq + lo + r]; lane = row -> coalesced
  for (int c = 0; c < s; ++c)
    if (lane < s) Q[(i64)(lo + c) * ldq + lo + lane] = Z[lane][c];
}

// number of elements of the ascending array a[0..n) that are < x (strict) or <= x
__device__ __forceinline__ int count_less(const double* a, int n, double x, bool or_equal) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const bool lt = or_equal ? (a[mid] <= x) : (a[mid] < x);
    if (lt) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(256) dc_prepare_kernel(DcBuf b, const double* Q, i64 ldq, const DcMerge* merges, int mbase) {
  const int m = mbase + blockIdx.x;
  const int lo = merges[m].lo, mid = merges[m].mid, hi = merges[m].hi, s = hi - lo;
  const double sg = b.sgn[m];
  for (int i = lo + threadIdx.x; i < hi; i += 256) {
    const double zi = (i < mid ? Q[(i64)i * ldq + (mid - 1)] : sg * Q[(i64)i * ldq + mid]) * 0.70710678118654752440;
    const double di = b.d[i];
    int pos;
    if (i < mid) pos = (i - lo) + count_less(b.d + mid, hi - mid, di, false);
    else pos = (i - mid) + count_less(b.d + lo, mid - lo, di, true);
    b.dsort[lo + pos] = di;
    b.zsort[lo + pos] = zi;
    b.colsort[lo + pos] = i - lo;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int nrot = 0;
    const int k = dc::deflate_scan<double>(b.dsort + lo, b.zsort + lo, b.colsort + lo, s, 2.0 * b.rho[m], b.dl + lo, b.w + lo,
                                           b.cnd + lo, b.dd + lo, b.cdf + lo, b.ra + lo, b.rb + lo, b.rc + lo, b.rs + lo, &nrot);
    b.kcnt[m] = k;
    b.nrot[m] = nrot;
  }
}

// one warp per root
__global__ void __launch_bounds__(256) dc_secular_kernel(DcBuf b, double* DEL, i64 ldw, const DcMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo;
  const int k = b.kcnt[m];
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= k) return;
  const double rho = 2.0 * b.rho[m], rhoinv = 1.0 / rho;
  const double* dl = b.dl + lo;
  const double* w = b.w + lo;
  double zz = 0.0;
  for (int i = lane; i < k; i += 32) zz += w[i] * w[i];
  zz = warp_sum(zz);
  int org = 0;
  double tau;
  if (k == 1) {
    tau = rho * zz;
  } else {
    tau = dc::secular_root<double>(dl, k, j, rho, zz,
                                   [&](int o, double t) {
                                     const double dorg = dl[o];
                                     double f = 0.0;
                                     for (int i = lane; i < k; i += 32) {
                                       const double del = (dl[i] - dorg) - t;
                                       f += w[i] * (w[i] / del);
                                     }
                                     return rhoinv + warp_sum(f);
                                   },
                                   &org);
  }
  const double dorg = dl[org];
  if (lane == 0) b.lam[lo + j] = dorg + tau;
  double* col = DEL + (i64)(lo + j) * ldw + lo;
  for (int i = lane; i < k; i += 32) col[i] = (dl[i] - dorg) - tau;
}

__global__ void __launch_bounds__(256) dc_zhat_kernel(DcBuf b, const double* DEL, i64 ldw, const DcMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo;
  const int k = b.kcnt[m];
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= k) return;
  const double* dl = b.dl + lo;
  const double di = dl[i];
  double prod = DEL[(i64)(lo + i) * ldw + lo + i];
  for (int j = 0; j < k; ++j)
    if (j != i) prod *= DEL[(i64)(lo + j) * ldw + lo + i] / (di - dl[j]);
  b.zh[lo + i] = copysign(sqrt(fabs(prod)), b.w[lo + i]);
}

// output column of every new eigenvalue: roots before deflated values on ties, deflated ties by index
__global__ void __launch_bounds__(256) dc_order_kernel(DcBuf b, const DcMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo, s = merges[m].hi - lo;
  const int k = b.kcnt[m], nd = s - k;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= s) return;
  const double* lam = b.lam + lo;
  const double* dd = b.dd + lo;
  int c;
  double val;
  if (t < k) {
    val = lam[t];
    c = t;
    for (int u = 0; u < nd; ++u) c += dd[u] < val;
  } else {
    const int td = t - k;
    val = dd[td];
    c = count_less(lam, k, val, true);  // roots are ascending
    for (int u = 0; u < nd; ++u) c += (dd[u] < val) || (dd[u] == val && u < td);
  }
  b.outcol[lo + t] = c;
  b.dnew[lo + c] = val;
}

// one CTA per new column: roots j < k get the normalised secular vector, deflated values a unit entry
__global__ void __launch_bounds__(128) dc_vectors_kernel(DcBuf b, const double* DEL, double* W, i64 ldw, const DcMerge* merges,
                                                         int mbase) {
  __shared__ double red[128];
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo, s = merges[m].hi - lo;
  const int k = b.kcnt[m];
  const int t = blockIdx.x;
  if (t >= s) return;
  const int oc = b.outcol[lo + t];
  double* wcol = W + (i64)(lo + oc) * ldw + lo;
  if (t >= k) {
    if (threadIdx.x == 0) wcol[b.cdf[lo + t - k]] = 1.0;
    return;
  }
  const double* dcol = DEL + (i64)(lo + t) * ldw + lo;
  double acc = 0.0;
  for (int i = threadIdx.x; i < k; i += 128) {
    const double v = b.zh[lo + i] / dcol[i];
    acc = fma(v, v, acc);
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int off = 64; off > 0; off >>= 1) {
    if ((int)threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  const double inv = 1.0 / sqrt(red[0]);
  for (int i = threadIdx.x; i < k; i += 128) wcol[b.cnd[lo + i]] = (b.zh[lo + i] / dcol[i]) * inv;
}

// rows a, b of W <- G rows a, b, rotations in reverse order; thread per column of W
__global__ void __launch_bounds__(256) dc_rotate_kernel(DcBuf b, double* W, i64 ldw, const DcMerge* merges, int mbase) {
  const int m = mbase + blockIdx.y;
  const int lo = merges[m].lo, s = merges[m].hi - lo;
  const int nrot = b.nrot[m];
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= s || nrot == 0) return;
  double* wcol = W + (i64)(lo + c) * ldw + lo;
  for (int r = nrot - 1; r >= 0; --r) {
    const int a = b.ra[lo + r], bb = b.rb[lo + r];
    const double cs = b.rc[lo + r], sn = b.rs[lo + r];
    const double x = wcol[a], y = wcol[bb];
    wcol[a] = cs * x - sn * y;
    wcol[bb] = sn * x + cs * y;
  }
}

__global__ void dc_finish_kernel(const double* d, double* lam, int n, const double* scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lam[i] = d[i] * scale[0];
}

int dc_num_levels(i64 n) {
  int lv = 0;
  while (((n + (1ll << lv) - 1) >> lv) > DC_LEAF) ++lv;
  return lv;
}

}  // namespace

// d[n], e[n-1] (device, read only) -> lam[n] ascending (device), Q (device, column-major n x n, ld = ldq >= n) = eigenvectors.
// Returns false for non-finite input (nothing meaningful is written then).
bool tridiag_dc_f64(cudaStream_t st, const double* d_in, const double* e_in, i64 n, double* lam, double* Q, i64 ldq) {
  if (n == 0) return true;
  FB_ASSERT(n < (1ll << 30), "dimension too large");
  const int nlev = dc_num_levels(n);
  // merges of all levels, level l at [first[l], first[l + 1])
  std::vector<DcMerge> merges;
  std::vector<int> first((size_t)nlev + 1, 0);
  for (int l = 0; l < nlev; ++l) {
    first[(size_t)l] = (int)merges.size();
    for (long long i = 0; i < (1ll << l); ++i)
      merges.push_back(DcMerge{(int)((i * n) >> l), (int)(((2 * i + 1) * n) >> (l + 1)), (int)(((i + 1) * n) >> l)});
  }
  first[(size_t)nlev] = (int)merges.size();
  const int nm = std::max<int>(1, (int)merges.size());

  const size_t nd = (size_t)n;
  const size_t dbl_n = 13, int_n = 6;
  char* pool = (char*)ws_alloc(dbl_n * nd * 8 + int_n * nd * 4 + (size_t)nm * (2 * 8 + 2 * 4 + sizeof(DcMerge)) + 256);
  DcBuf b;
  double* pd = (double*)pool;
  b.d = pd; pd += nd; b.e = pd; pd += nd; b.dsort = pd; pd += nd; b.zsort = pd; pd += nd; b.dl = pd; pd += nd; b.w = pd; pd += nd;
  b.dd = pd; pd += nd; b.rc = pd; pd += nd; b.rs = pd; pd += nd; b.lam = pd; pd += nd; b.zh = pd; pd += nd; b.dnew = pd; pd += nd;
  b.rho = pd; pd += nm; b.sgn = pd; pd += nm; b.scale = pd; pd += 4;
  (void)dbl_n;
  int* pi = (int*)pd;
  b.colsort = pi; pi += nd; b.cnd = pi; pi += nd; b.cdf = pi; pi += nd; b.ra = pi; pi += nd; b.rb = pi; pi += nd; b.outcol = pi; pi += nd;
  b.kcnt = pi; pi += nm; b.nrot = pi; pi += nm;
  int* d_fail = pi; pi += 2;
  DcMerge* d_merges = (DcMerge*)(((uintptr_t)pi + 15) & ~(uintptr_t)15);
  FB_ASSERT((char*)(d_merges + nm) <= pool + dbl_n * nd * 8 + int_n * nd * 4 + (size_t)nm * (2 * 8 + 2 * 4 + sizeof(DcMerge)) + 256,
            "workspace layout");
  if (!merges.empty())
    FB_CUDA_CHECK(cudaMemcpyAsync(d_merges, merges.data(), merges.size() * sizeof(DcMerge), cudaMemcpyHostToDevice, st));
  FB_CUDA_CHECK(cudaMemsetAsync(d_fail, 0, 8, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(b.d, d_in, nd * 8, cudaMemcpyDeviceToDevice, st));
  FB_CUDA_CHECK(cudaMemsetAsync(b.e, 0, nd * 8, st));
  if (n > 1) FB_CUDA_CHECK(cudaMemcpyAsync(b.e, e_in, (nd - 1) * 8, cudaMemcpyDeviceToDevice, st));
  dc_scale_kernel<<<1, 256, 0, st>>>(b.d, b.e, (int)n, b.scale);
  note_launch();
  {
    // non-finite input: stop here (the reference returns NoConvergence, svd/mod.rs:282-286); NaNs in the deflation /
    // sorting stages would otherwise turn into wild indices
    double h_sc[2] = {1.0, 0.0};
    FB_CUDA_CHECK(cudaMemcpyAsync(h_sc, b.scale, 16, cudaMemcpyDeviceToHost, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (h_sc[1] != 0.0) {
      ws_free(pool);
      return false;
    }
  }
  if (!merges.empty()) {
    dc_tear_kernel<<<(unsigned)((merges.size() + 127) / 128), 128, 0, st>>>(b.d, b.e, d_merges, (int)merges.size(), b.rho, b.sgn);
    note_launch();
  }
  // eigenvector blocks ping-pong between Q (the output) and a scratch matrix so that the LAST level lands in Q
  double* Qs = nlev > 0 ? (double*)ws_alloc(nd * nd * 8) : nullptr;
  double* Wm = nlev > 0 ? (double*)ws_alloc(nd * nd * 8) : nullptr;
  double* DEL = nlev > 0 ? (double*)ws_alloc(nd * nd * 8) : nullptr;
  double* cur = (nlev % 2 == 0) ? Q : Qs;
  i64 ldc = (nlev % 2 == 0) ? ldq : n;
  FB_CUDA_CHECK(cudaMemset2DAsync(cur, (size_t)ldc * 8, 0, nd * 8, nd, st));
  dc_leaf_kernel<<<(unsigned)(1u << nlev), 32, 0, st>>>(b.d, b.e, cur, ldc, (int)n, nlev, d_fail);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  for (int l = nlev - 1; l >= 0; --l) {
    const int mb = first[(size_t)l], cnt = first[(size_t)l + 1] - mb;
    int smax = 0;
    for (int i = 0; i < cnt; ++i) smax = std::max(smax, merges[(size_t)(mb + i)].hi - merges[(size_t)(mb + i)].lo);
    double* nxt = (cur == Q) ? Qs : Q;
    const i64 ldn = (cur == Q) ? n : ldq;
    FB_CUDA_CHECK(cudaMemsetAsync(Wm, 0, nd * nd * 8, st));
    dc_prepare_kernel<<<(unsigned)cnt, 256, 0, st>>>(b, cur, ldc, d_merges, mb);
    dc_secular_kernel<<<dim3((unsigned)((smax + 7) / 8), (unsigned)cnt), 256, 0, st>>>(b, DEL, n, d_merges, mb);
    dc_zhat_kernel<<<dim3((unsigned)((smax + 255) / 256), (unsigned)cnt), 256, 0, st>>>(b, DEL, n, d_merges, mb);
    dc_order_kernel<<<dim3((unsigned)((smax + 255) / 256), (unsigned)cnt), 256, 0, st>>>(b, d_merges, mb);
    dc_vectors_kernel<<<dim3((unsigned)smax, (unsigned)cnt), 128, 0, st>>>(b, DEL, Wm, n, d_merges, mb);
    dc_rotate_kernel<<<dim3((unsigned)((smax + 255) / 256), (unsigned)cnt), 256, 0, st>>>(b, Wm, n, d_merges, mb);
    FB_CUDA_CHECK(cudaGetLastError());
    for (int q = 0; q < 6; ++q) note_launch();
    for (int i = 0; i < cnt; ++i) {
      const DcMerge& mg = merges[(size_t)(mb + i)];
      const i64 lo = mg.lo, mid = mg.mid, hi = mg.hi, s = hi - lo, s1 = mid - lo, s2 = hi - mid;
      VCD Q1{cur + lo * ldc + lo, s1, s1, 1, ldc}, Q2{cur + mid * ldc + mid, s2, s2, 1, ldc};
      VCD W1{Wm + lo * n + lo, s1, s, 1, n}, W2{Wm + lo * n + mid, s2, s, 1, n};
      gemm_f64(st, VD{nxt + lo * ldn + lo, s1, s, 1, ldn}, 0, Q1, W1, 1.0);
      gemm_f64(st, VD{nxt + lo * ldn + mid, s2, s, 1, ldn}, 0, Q2, W2, 1.0);
    }
    // the level's sorted eigenvalues become the blocks' diagonals
    FB_CUDA_CHECK(cudaMemcpyAsync(b.d, b.dnew, nd * 8, cudaMemcpyDeviceToDevice, st));
    cur = nxt;
    ldc = ldn;
  }
  FB_ASSERT(cur == Q, "eigenvector ping-pong ended in the scratch buffer");
  dc_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(b.d, lam, (int)n, b.scale);
  note_launch();
  double h_scale[2] = {1.0, 0.0};
  int h_fail = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(h_scale, b.scale, 16, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaMemcpyAsync(&h_fail, d_fail, 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (DEL) ws_free(DEL);
  if (Wm) ws_free(Wm);
  if (Qs) ws_free(Qs);
  ws_free(pool);
  return h_scale[1] == 0.0 && h_fail == 0;
}

}  // namespace fb
