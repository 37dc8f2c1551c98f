// SVD and self-adjoint EVD WITH vectors (f64 arithmetic; f32 entry points go through an f64 copy).
//
// Reference:
//   svd::svd               faer/src/linalg/svd/mod.rs:530-672   (transpose wide inputs, QR first above qr_ratio_threshold,
//                                                                 conjugation of the swapped outputs)
//   svd_imp                svd/mod.rs:326-431                    (bidiagonalize, SVD of the bidiagonal, back-transforms 403-429)
//   bidiag_svd             svd/bidiag_svd.rs:1005-...            (divide and conquer on the bidiagonal, merges as matmuls)
//   self_adjoint_evd       evd/mod.rs:270-418                    (tridiagonalize, tridiag_evd, back-transform 411-418)
//
// GPU arrangement. The reductions to condensed form are the HBM-bound persistent kernels of bidiag.cu / tridiag.cu, the
// back-transforms the block-Householder GEMM compositions of householder.cu. The condensed problems go through ONE
// divide-and-conquer code, the symmetric tridiagonal eigensolver of tridiag_dc.cu (all work in DMMA GEMMs + parallel
// secular solves):
//   * EVD: directly.
//   * SVD of the bidiagonal B (n x n, upper): its Golub-Kahan form T_GK = P [0 B^T; B 0] P^T (order 2n, zero diagonal,
//     off-diagonals d_1, e_1, d_2, ..., d_n) has the eigenpairs (+-sigma_i, (v_i, u_i) / sqrt 2 interleaved). The n largest
//     eigenpairs give sigma_i and the directions v_i. The eigensolver is backward stable for T_GK, which pins sigma_i to
//     eps |B| and v_i to its direction, but not the SPLIT of an eigenvector into u and v parts when sigma_i is small
//     (|u_i| - |v_i| = O(eps |B| / sigma_i)). So only the v parts are used, and the rest is made exact by construction:
//         V^ = v parts  ->  Householder QR, Q_v its orthogonal factor (orthonormal whatever V^'s rank: for sigma = 0
//         the completion IS a basis of the null space)
//         W = B Q_v (O(n^2): B is bidiagonal)  ->  Householder QR, W = U_B R
//     Then B = U_B R Q_v^T holds to rounding for ANY orthogonal Q_v, U_B is orthogonal by construction, and R is diagonal
//     up to eps |B| because the columns of Q_v are right singular directions in decreasing order of sigma: the part of
//     column j along an earlier left singular vector u_i is (error of v_j towards v_i) * sigma_i <= eps |B|. S = |diag R|,
//     the signs go into U_B, and a final stable ordering makes S non-increasing as the reference promises.
//   Cost at n = 8192: eigensolver on 2n (4/3 (2n)^3 flop of GEMM), two QRs and two applications of their Q to the
//   identity: ~16 n^3 flop on the DMMA path, a fraction of the 1 s the HBM-bound bidiagonalization takes.
// STATUS: validated on hardware (tests/test_gpu_zz11_evd_svd_vectors.py; exact spectra, rank-deficient and repeated singular
// values, and sizes past 8192 rows in tests/test_gpu_zz24_spectral_exact.py).
#include <algorithm>

#include "bidiag_sv.cuh"
#include "panel_common.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

bool tridiag_dc_f64(cudaStream_t st, const double* d_in, const double* e_in, i64 n, double* lam, double* Q, i64 ldq);

namespace {

// launches over (rows in blocks of 256) x (columns in chunks of <= 65535)
template <class F>
void for_each_col_chunk(i64 ncols, F&& f) {
  for (i64 c0 = 0; c0 < ncols; c0 += 65535) f(c0, std::min<i64>(65535, ncols - c0));
}

template <class TD, class TS>
__global__ void copy_cast_kernel(TD* __restrict__ dst, i64 drs, i64 dcs, const TS* __restrict__ src, i64 srs, i64 scs, i64 m, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < m) dst[i * drs + j * dcs] = (TD)src[i * srs + j * scs];
}
template <class TD, class TS>
void copy_cast(cudaStream_t st, TD* dst, i64 drs, i64 dcs, const TS* src, i64 srs, i64 scs, i64 m, i64 n) {
  if (m == 0 || n == 0) return;
  for_each_col_chunk(n, [&](i64 c0, i64 nc) {
    copy_cast_kernel<TD, TS><<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(dst, drs, dcs, src, srs, scs, m, c0);
    note_launch();
  });
  FB_CUDA_CHECK(cudaGetLastError());
}

// dst (column-major, ld) <- lower triangle of src, zero above
__global__ void copy_lower_f64_kernel(double* __restrict__ dst, i64 ld, const double* __restrict__ src, i64 rs, i64 cs, i64 n, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < n) dst[j * ld + i] = i >= j ? src[i * rs + j * cs] : 0.0;
}
// dst (n x n column-major) <- upper triangle of the leading n x n block of src (ld lds), zero below
__global__ void copy_upper_f64_kernel(double* __restrict__ dst, i64 n, const double* __restrict__ src, i64 lds, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < n) dst[j * n + i] = i <= j ? src[j * lds + i] : 0.0;
}
// M (column-major, ld) <- [X 0; 0 I]: X = top-left k x k block of src (ld lds) — rows / columns beyond k get the identity
__global__ void embed_kernel(double* __restrict__ M, i64 ld, i64 rows, const double* __restrict__ src, i64 lds, i64 k, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i >= rows) return;
  M[j * ld + i] = (i < k && j < k) ? src[j * lds + i] : (i == j ? 1.0 : 0.0);
}
__global__ void identity_kernel(double* __restrict__ M, i64 ld, i64 rows, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < rows) M[j * ld + i] = i == j ? 1.0 : 0.0;
}
void set_identity(cudaStream_t st, double* M, i64 ld, i64 rows, i64 cols) {
  for_each_col_chunk(cols, [&](i64 c0, i64 nc) {
    identity_kernel<<<dim3((unsigned)((rows + 255) / 256), (unsigned)nc), 256, 0, st>>>(M, ld, rows, c0);
    note_launch();
  });
}

// diagonal / superdiagonal (super = true) or subdiagonal of a column-major matrix
__global__ void extract_diags_kernel(const double* __restrict__ A, i64 ld, int n, bool super, double* __restrict__ d, double* __restrict__ e) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    d[i] = A[(i64)i + (i64)i * ld];
    if (i + 1 < n) e[i] = super ? A[(i64)i + (i64)(i + 1) * ld] : A[(i64)(i + 1) + (i64)i * ld];
  }
}
// flag[0] <- 1 if any of the n values is not finite
__global__ void finite_check_kernel(const double* __restrict__ x, i64 n, int* __restrict__ flag) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(fabs(x[i]) < TLim<double>::inf())) *flag = 1;
}
// Golub-Kahan off-diagonals (d_0, e_0, d_1, ..., d_{n-1}); diag <- 0
__global__ void tgk_kernel(const double* __restrict__ d, const double* __restrict__ e, int n, double* __restrict__ diag, double* __restrict__ off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    off[2 * i] = d[i];
    if (i + 1 < n) off[2 * i + 1] = e[i];
    diag[2 * i] = 0.0;
    diag[2 * i + 1] = 0.0;
  }
}
// V^(i, j) = QT(2 i, 2n - 1 - j): the v parts of the eigenvectors of the n largest eigenvalues, largest first
__global__ void vparts_kernel(double* __restrict__ Vh, i64 n, const double* __restrict__ QT, i64 ldq, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < n) Vh[j * n + i] = QT[(2 * n - 1 - j) * ldq + 2 * i];
}
// W = B X, B upper bidiagonal (d, e): W(i, :) = d_i X(i, :) + e_i X(i + 1, :)
__global__ void bidiag_times_kernel(double* __restrict__ W, const double* __restrict__ X, i64 n, const double* __restrict__ d,
                                    const double* __restrict__ e, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < n) W[j * n + i] = d[i] * X[j * n + i] + (i + 1 < n ? e[i] * X[j * n + i + 1] : 0.0);
}
// s_j = |R_jj|, sg_j = sign(R_jj) (1 for 0)
__global__ void diag_sign_kernel(const double* __restrict__ R, i64 ld, int n, double* __restrict__ s, double* __restrict__ sg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double r = R[(i64)i + (i64)i * ld];
    s[i] = fabs(r);
    sg[i] = r < 0.0 ? -1.0 : 1.0;
  }
}
// pos[j] = position of s_j in non-increasing order (stable); sorted[pos[j]] = s_j
__global__ void rank_desc_kernel(const double* __restrict__ s, int n, int* __restrict__ pos, double* __restrict__ sorted) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double v = s[j];
  int c = 0;
  for (int u = 0; u < n; ++u) c += (s[u] > v) || (s[u] == v && u < j);
  pos[j] = c;
  sorted[c] = v;
}
// dst(:, pos[j]) = scale[j] * src(:, j) for j < k (pos == nullptr: identity); columns j >= k are copied in place
template <class TD>
__global__ void scatter_cols_kernel(TD* __restrict__ dst, i64 drs, i64 dcs, const double* __restrict__ src, i64 lds, i64 rows, i64 k,
                                    const int* __restrict__ pos, const double* __restrict__ scale, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i >= rows) return;
  const i64 jd = (j < k && pos) ? pos[j] : j;
  const double sc = (j < k && scale) ? scale[j] : 1.0;
  dst[i * drs + jd * dcs] = (TD)(sc * src[j * lds + i]);
}
template <class TD>
void scatter_cols(cudaStream_t st, View<TD> dst, const double* src, i64 lds, i64 k, const int* pos, const double* scale) {
  if (dst.nrows == 0 || dst.ncols == 0) return;
  for_each_col_chunk(dst.ncols, [&](i64 c0, i64 nc) {
    scatter_cols_kernel<TD><<<dim3((unsigned)((dst.nrows + 255) / 256), (unsigned)nc), 256, 0, st>>>(dst.ptr, dst.rs, dst.cs, src, lds,
                                                                                                   dst.nrows, k, pos, scale, c0);
    note_launch();
  });
  FB_CUDA_CHECK(cudaGetLastError());
}
template <class TD>
__global__ void copy_vec_kernel(TD* __restrict__ dst, i64 stride, const double* __restrict__ src, i64 n) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i * stride] = (TD)src[i];
}

// Q factor of a Householder QR (packed factors in QR, T blocks in H), written to Qout (n x n, column-major, ld n)
void form_q(cudaStream_t st, const double* QR, i64 n, const double* H, i64 bs, double* Qout) {
  set_identity(st, Qout, n, n, n);
  apply_block_householder_sequence_on_the_left<double>(st, VCD{QR, n, n, 1, n}, VCD{H, bs, n, 1, bs}, VD{Qout, n, n, 1, n});
}

// SVD of the upper-bidiagonal (d, e) of order n: S_sorted (non-increasing), UB and VB (n x n, column-major, ld n) with columns
// already in the sorted order. Returns false if the eigensolver reports non-finite input.
bool bidiag_svd_vectors(cudaStream_t st, const double* d, const double* e, i64 n, double* S_sorted, double* UB, double* VB) {
  const i64 n2 = 2 * n;
  double* tg = (double*)ws_alloc((size_t)(3 * n2 + 8) * 8);
  double *tdiag = tg, *toff = tg + n2, *tlam = tg + 2 * n2;
  tgk_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d, e, (int)n, tdiag, toff);
  note_launch();
  double* QT = (double*)ws_alloc((size_t)n2 * (size_t)n2 * 8);
  const bool ok = tridiag_dc_f64(st, tdiag, toff, n2, tlam, QT, n2);
  double* Vh = (double*)ws_alloc((size_t)n * (size_t)n * 8);
  for_each_col_chunk(n, [&](i64 c0, i64 nc) {
    vparts_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)nc), 256, 0, st>>>(Vh, n, QT, n2, c0);
    note_launch();
  });
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(QT);
  const i64 bs = qr_recommended_block_size(n, n);
  double* H = (double*)ws_alloc((size_t)bs * (size_t)n * 8);
  // Q_v
  qr_in_place<double>(st, VD{Vh, n, n, 1, n}, VD{H, bs, n, 1, bs});
  double* Qv = (double*)ws_alloc((size_t)n * (size_t)n * 8);
  form_q(st, Vh, n, H, bs, Qv);
  // W = B Q_v, its QR, U_B
  double* Wm = Vh;  // reuse
  for_each_col_chunk(n, [&](i64 c0, i64 nc) {
    bidiag_times_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)nc), 256, 0, st>>>(Wm, Qv, n, d, e, c0);
    note_launch();
  });
  qr_in_place<double>(st, VD{Wm, n, n, 1, n}, VD{H, bs, n, 1, bs});
  double* sv = (double*)ws_alloc((size_t)(2 * n + 2) * 8 + (size_t)n * 4 + 16);
  double *s_raw = sv, *sg = sv + n;
  int* pos = (int*)(sv + 2 * n + 2);
  diag_sign_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(Wm, n, (int)n, s_raw, sg);
  rank_desc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s_raw, (int)n, pos, S_sorted);
  note_launch();
  note_launch();
  double* Ub = (double*)ws_alloc((size_t)n * (size_t)n * 8);
  form_q(st, Wm, n, H, bs, Ub);
  scatter_cols<double>(st, VD{UB, n, n, 1, n}, Ub, n, n, pos, sg);
  scatter_cols<double>(st, VD{VB, n, n, 1, n}, Qv, n, n, pos, nullptr);
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(Ub);
  ws_free(sv);
  ws_free(Qv);
  ws_free(H);
  ws_free(Vh);
  ws_free(tg);
  return ok;
}

}  // namespace

// the real bidiagonal solver for the complex driver (cplx_condensed.cu)
bool bidiag_svd_vectors_f64(cudaStream_t st, const double* d, const double* e, i64 n, double* S_sorted, double* UB, double* VB) {
  return bidiag_svd_vectors(st, d, e, n, S_sorted, UB, VB);
}

// Full driver. A: device view (any strides) of element type TA (float / double); U, V: device views or ncols == 0 / ptr == null
// ("do not compute"); U is nrows x {size, nrows}, V is ncols x {size, ncols}; S: device, `sstride` elements apart.
// Returns false on non-finite input (SvdError::NoConvergence, svd/mod.rs:282-286).
template <class TA>
bool svd_with_vectors(cudaStream_t st, View<const TA> A, View<TA> U, TA* S, i64 sstride, View<TA> V, double qr_ratio_threshold) {
  const bool transpose = A.ncols > A.nrows;
  View<const TA> M = transpose ? A.t() : A;
  View<TA> Um = transpose ? V : U, Vm = transpose ? U : V;  // real types: no conjugation needed (svd/mod.rs:661-669)
  const i64 m = M.nrows, n = M.ncols;
  const bool want_u = Um.ptr != nullptr && Um.ncols > 0, want_v = Vm.ptr != nullptr && Vm.ncols > 0;
  if (n == 0) {
    if (want_u) {
      double* I = (double*)ws_alloc((size_t)std::max<i64>(1, m * Um.ncols) * 8);
      set_identity(st, I, m, m, Um.ncols);
      scatter_cols<TA>(st, Um, I, m, 0, nullptr, nullptr);
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(I);
    }
    return true;
  }
  double* Wk = (double*)ws_alloc((size_t)m * (size_t)n * 8);
  copy_cast<double, TA>(st, Wk, 1, m, M.ptr, M.rs, M.cs, m, n);
  int* d_flag = (int*)ws_alloc(16);
  FB_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, 4, st));
  // ---- QR first for tall inputs (svd/mod.rs:594-633) ----
  const bool qr_first = (double)m / (double)n > qr_ratio_threshold && n > 1;
  double *Hq = nullptr, *R = nullptr;
  i64 bsq = 0, mb = m;
  if (qr_first) {
    bsq = qr_recommended_block_size(m, n);
    Hq = (double*)ws_alloc((size_t)bsq * (size_t)n * 8);
    qr_in_place<double>(st, VD{Wk, m, n, 1, m}, VD{Hq, bsq, n, 1, bsq});
    R = (double*)ws_alloc((size_t)n * (size_t)n * 8);
    for_each_col_chunk(n, [&](i64 c0, i64 nc) {
      copy_upper_f64_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)nc), 256, 0, st>>>(R, n, Wk, m, c0);
      note_launch();
    });
    mb = n;
  }
  double* Bm = R ? R : Wk;
  // ---- bidiagonalization (svd/mod.rs:346-363) ----
  const i64 bs = (want_u || want_v) ? qr_recommended_block_size(mb, n) : 1;
  double* Hl = (double*)ws_alloc((size_t)bs * (size_t)n * 8);
  double* Hr = (double*)ws_alloc((size_t)bs * (size_t)std::max<i64>(1, n - 1) * 8);
  bidiag_in_place<double>(st, VD{Bm, mb, n, 1, mb}, VD{Hl, bs, n, 1, bs}, VD{Hr, bs, n - 1, 1, bs});
  double* de = (double*)ws_alloc((size_t)(3 * n + 8) * 8);
  double *d = de, *e = de + n, *s_sorted = de + 2 * n;
  FB_CUDA_CHECK(cudaMemsetAsync(e, 0, (size_t)n * 8, st));
  extract_diags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(Bm, mb, (int)n, true, d, e);
  finite_check_kernel<<<(unsigned)((2 * n + 255) / 256), 256, 0, st>>>(de, 2 * n, d_flag);
  note_launch();
  note_launch();
  int h_flag = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, d_flag, 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  bool ok = h_flag == 0;
  FB_ASSERT(want_u || want_v, "svd_with_vectors: the values-only path is singular_values (svd.cu)");
  if (ok) {
    double* UB = (double*)ws_alloc((size_t)n * (size_t)n * 8);
    double* VB = (double*)ws_alloc((size_t)n * (size_t)n * 8);
    ok = bidiag_svd_vectors(st, d, e, n, s_sorted, UB, VB);
    if (ok && want_u) {
      const i64 ku = Um.ncols;  // size or m
      double* Uw = (double*)ws_alloc((size_t)m * (size_t)ku * 8);
      if (!qr_first) {
        // U = H_left-sequence * [U_B 0; 0 I]  (svd/mod.rs:403-412)
        for_each_col_chunk(ku, [&](i64 c0, i64 nc) {
          embed_kernel<<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(Uw, m, m, UB, n, n, c0);
          note_launch();
        });
        apply_block_householder_sequence_on_the_left<double>(st, VCD{Bm, m, n, 1, m}, VCD{Hl, bs, n, 1, bs}, VD{Uw, m, ku, 1, m});
      } else {
        // U_R = H_left-sequence * U_B (n x n), then U = Q_qr * [U_R 0; 0 I]  (svd/mod.rs:621-658)
        apply_block_householder_sequence_on_the_left<double>(st, VCD{Bm, n, n, 1, n}, VCD{Hl, bs, n, 1, bs}, VD{UB, n, n, 1, n});
        for_each_col_chunk(ku, [&](i64 c0, i64 nc) {
          embed_kernel<<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(Uw, m, m, UB, n, n, c0);
          note_launch();
        });
        apply_block_householder_sequence_on_the_left<double>(st, VCD{Wk, m, n, 1, m}, VCD{Hq, bsq, n, 1, bsq}, VD{Uw, m, ku, 1, m});
      }
      scatter_cols<TA>(st, Um, Uw, m, 0, nullptr, nullptr);
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(Uw);
    }
    if (ok && want_v) {
      // V = diag(1, H_right-sequence) * V_B; the right reflectors are the ROWS of the bidiagonalised matrix to the right of
      // the superdiagonal: basis = transposed view (svd/mod.rs:413-428)
      if (n > 1)
        apply_block_householder_sequence_on_the_left<double>(st, VCD{Bm + mb, n - 1, n - 1, mb, 1}, VCD{Hr, bs, n - 1, 1, bs},
                                                             VD{VB + 1, n - 1, n, 1, n});
      scatter_cols<TA>(st, Vm, VB, n, 0, nullptr, nullptr);
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    ws_free(VB);
    ws_free(UB);
  }
  if (ok) {
    copy_vec_kernel<TA><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, sstride, s_sorted, n);
    note_launch();
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(de);
  ws_free(Hr);
  ws_free(Hl);
  if (R) ws_free(R);
  if (Hq) ws_free(Hq);
  ws_free(d_flag);
  ws_free(Wk);
  return ok;
}

// Self-adjoint EVD with eigenvectors: A's LOWER triangle (device view, any strides); S nondecreasing; U n x n (device view).
// Returns false on non-finite input.
template <class TA>
bool self_adjoint_evd_with_vectors(cudaStream_t st, View<const TA> A, View<TA> U, TA* S, i64 sstride) {
  const i64 n = A.nrows;
  if (n == 0) return true;
  double* W = (double*)ws_alloc((size_t)n * (size_t)n * 8);
  // lower triangle in f64, column-major
  {
    double* tmp = W;
    if (sizeof(TA) == 8) {
      for_each_col_chunk(n, [&](i64 c0, i64 nc) {
        copy_lower_f64_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)nc), 256, 0, st>>>(tmp, n, (const double*)A.ptr, A.rs, A.cs, n, c0);
        note_launch();
      });
    } else {
      copy_cast<double, TA>(st, tmp, 1, n, A.ptr, A.rs, A.cs, n, n);  // the upper triangle is never read by tridiag_in_place
    }
  }
  const i64 bs = qr_recommended_block_size(n, n);
  double* H = (double*)ws_alloc((size_t)bs * (size_t)std::max<i64>(1, n - 1) * 8);
  tridiag_in_place<double>(st, VD{W, n, n, 1, n}, VD{H, bs, n - 1, 1, bs});
  double* de = (double*)ws_alloc((size_t)(3 * n + 8) * 8);
  double *d = de, *e = de + n, *lam = de + 2 * n;
  FB_CUDA_CHECK(cudaMemsetAsync(e, 0, (size_t)n * 8, st));
  extract_diags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, n, (int)n, false, d, e);
  note_launch();
  double* Q = (double*)ws_alloc((size_t)n * (size_t)n * 8);
  const bool ok = tridiag_dc_f64(st, d, e, n, lam, Q, n);
  if (ok) {
    if (n > 1)
      apply_block_householder_sequence_on_the_left<double>(st, VCD{W + 1, n - 1, n - 1, 1, n}, VCD{H, bs, n - 1, 1, bs},
                                                           VD{Q + 1, n - 1, n, 1, n});
    scatter_cols<TA>(st, U, Q, n, 0, nullptr, nullptr);
    copy_vec_kernel<TA><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, sstride, lam, n);
    note_launch();
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(Q);
  ws_free(de);
  ws_free(H);
  ws_free(W);
  return ok;
}

template <class T>
__global__ void finite_check_t_kernel(const T* __restrict__ x, i64 n, int* __restrict__ flag) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(fabs((double)x[i]) < TLim<double>::inf())) *flag = 1;
}
// true iff all n device values are finite (one small launch + read-back)
template <class T>
bool device_all_finite(cudaStream_t st, const T* x, i64 n) {
  if (n == 0) return true;
  int* d_flag = (int*)ws_alloc(16);
  FB_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, 4, st));
  finite_check_t_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, n, d_flag);
  note_launch();
  int h = 0;
  FB_CUDA_CHECK(cudaMemcpyAsync(&h, d_flag, 4, cudaMemcpyDeviceToHost, st));
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(d_flag);
  return h == 0;
}
template bool device_all_finite<double>(cudaStream_t, const double*, i64);
template bool device_all_finite<float>(cudaStream_t, const float*, i64);

template bool svd_with_vectors<double>(cudaStream_t, View<const double>, View<double>, double*, i64, View<double>, double);
template bool svd_with_vectors<float>(cudaStream_t, View<const float>, View<float>, float*, i64, View<float>, double);
template bool self_adjoint_evd_with_vectors<double>(cudaStream_t, View<const double>, View<double>, double*, i64);
template bool self_adjoint_evd_with_vectors<float>(cudaStream_t, View<const float>, View<float>, float*, i64);

}  // namespace fb
