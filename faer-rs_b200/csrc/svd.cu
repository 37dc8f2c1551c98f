// Singular values on the GPU (BASELINE.json configs[4], "SVD via bidiagonalization"; SURVEY.md §8f rank 4, values only):
// A (or A^T for wide inputs, svd/mod.rs:560-575) is copied, reduced to bidiagonal form by the HBM-bound persistent kernel
// of bidiag.cu, and the singular values of the bidiagonal come from one bisection thread per value (bidiag_sv.cuh).
// Reference: faer/src/linalg/svd/mod.rs:530-648 (`svd` with u = v = None, as `MatRef::singular_values`, solvers.rs:457-487).
// Like the reference, a QR factorization comes first when nrows / ncols exceeds params.qr_ratio_threshold (11/6) and R is
// bidiagonalised instead. Differences, both documented in DESIGN.md: (1) the reference reaches the values of the bidiagonal
// through bidiag_svd (QR iteration / divide and conquer); here they are located by Sturm counts — same values to
// n * eps * sigma_max, the small ones to high relative accuracy; (2) this file is the VALUES-ONLY path (U and V passed with no
// columns); with vectors the entry point goes to svd_vectors.cu (divide and conquer + back-transforms).
// STATUS: validated on hardware (tests/test_gpu_zz7_singular_values.py and the fixture files of tests/test_gpu_zz11_evd_svd_vectors.py,
// exact spectra in tests/test_gpu_zz24_spectral_exact.py);
// bidiag_sv.cuh is also checked on the CPU (the same header compiled for the host, tests/test_bidiag_sv_cpu.py).
#include "bidiag_sv.cuh"
#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

template <class T>
__global__ void copy_to_colmajor_kernel(T* __restrict__ dst, i64 ld, const T* __restrict__ src, i64 rs, i64 cs, i64 m, i64 n) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = blockIdx.y;
  if (i < m && j < n) dst[j * ld + i] = src[i * rs + j * cs];
}

// R (n x n, column-major, ld = n) <- the upper triangle of the leading n x n block of QR (ld = ldq), zero below the diagonal
template <class T>
__global__ void copy_upper_kernel(T* __restrict__ R, i64 n, const T* __restrict__ QR, i64 ldq) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = blockIdx.y;
  if (i < n && j < n) R[j * n + i] = i <= j ? QR[j * ldq + i] : T(0);
}

template <class T>
__global__ void extract_bidiag_kernel(const T* __restrict__ A, i64 cs, int n, T* __restrict__ d, T* __restrict__ e) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    d[i] = A[(i64)i + (i64)i * cs];
    if (i + 1 < n) e[i] = A[(i64)i + (i64)(i + 1) * cs];
  }
}

// bb[0] = Gershgorin bound of T_GK (>= sigma_max), bb[1] = max b_j^2
template <class T>
__global__ void __launch_bounds__(256) gk_bound_kernel(const T* __restrict__ d, const T* __restrict__ e, int n,
                                                        T* __restrict__ bb) {
  __shared__ T s_bound[256], s_b2[256];
  T bound = 0, b2 = 0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const T a = fabs(d[i]), b = i + 1 < n ? fabs(e[i]) : T(0), c = i > 0 ? fabs(e[i - 1]) : T(0);
    bound = fmax(bound, fmax(a + b, a + c));
    b2 = fmax(b2, fmax(a * a, b * b));
  }
  s_bound[threadIdx.x] = bound;
  s_b2[threadIdx.x] = b2;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_bound[threadIdx.x] = fmax(s_bound[threadIdx.x], s_bound[threadIdx.x + s]);
      s_b2[threadIdx.x] = fmax(s_b2[threadIdx.x], s_b2[threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    bb[0] = s_bound[0] * (T(1) + T(4) * bsv::Lim<T>::eps()) + bsv::Lim<T>::safmin();
    bb[1] = s_b2[0];
  }
}

template <class T>
__global__ void __launch_bounds__(64) gk_values_kernel(const T* __restrict__ d, const T* __restrict__ e, int n,
                                                        const T* __restrict__ bb, T* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = bsv::gk_kth_largest<T>(d, e, n, 1, 1, k, bb[0], bb[1]);
}

}  // namespace

// S (device, compact, min(m, n) entries) <- singular values of A in non-increasing order. A: device view, any strides.
template <class T>
bool singular_values(cudaStream_t st, View<const T> A, T* S, double qr_ratio_threshold) {
  View<const T> M = A.ncols > A.nrows ? A.t() : A;
  const i64 m = M.nrows, n = M.ncols;
  if (n == 0) return true;
  FB_ASSERT(n < 65536 && m < (1ll << 31), "singular_values: dimension too large for the copy launch");
  T* W = (T*)ws_alloc((size_t)m * (size_t)n * sizeof(T));
  auto copy_in = [&]() {
    dim3 grid((unsigned)((m + 255) / 256), (unsigned)n);
    copy_to_colmajor_kernel<T><<<grid, 256, 0, st>>>(W, m, M.ptr, M.rs, M.cs, m, n);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  };
  copy_in();
  // Tall inputs: the singular values of A are those of R (svd/mod.rs:594-633): one QR (GEMM-rich) and then an n x n
  // bidiagonalization instead of an m x n one (every column step of which streams the whole trailing matrix).
  // A rank-deficient input is reported by the QR driver; then the copy is restored and bidiagonalised directly.
  i64 mb = m;  // rows of the matrix that is bidiagonalised
  T* R = nullptr;
  if ((double)m / (double)n > qr_ratio_threshold && n > 1) {
    const i64 bs = qr_recommended_block_size(m, n);
    T* Hq = (T*)ws_alloc((size_t)bs * (size_t)n * sizeof(T));
    const i64 rank = qr_in_place<T>(st, View<T>{W, m, n, 1, m}, View<T>{Hq, bs, n, 1, bs});
    ws_free(Hq);
    if (rank == n) {
      R = (T*)ws_alloc((size_t)n * (size_t)n * sizeof(T));
      dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
      copy_upper_kernel<T><<<grid, 256, 0, st>>>(R, n, W, m);
      FB_CUDA_CHECK(cudaGetLastError());
      note_launch();
      mb = n;
    } else {
      copy_in();
    }
  }
  T* Bm = R ? R : W;
  // one-row Householder factors: only the taus are produced, no T blocks (bidiag.cu skips them for a single row)
  T* h = (T*)ws_alloc((size_t)(2 * n + 2) * sizeof(T));
  View<T> Hl{h, 1, n, 1, 1}, Hr{h + n, 1, n - 1, 1, 1};
  bidiag_in_place<T>(st, View<T>{Bm, mb, n, 1, mb}, Hl, Hr);
  T* de = (T*)ws_alloc((size_t)(2 * n + 2) * sizeof(T));
  T *d = de, *e = de + n, *bb = de + 2 * n;
  extract_bidiag_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(Bm, mb, (int)n, d, e);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  // a non-finite bidiagonal has no singular values: the reference returns SvdError::NoConvergence (svd/mod.rs:282-286);
  // fmax / fmin in the bounds kernel would silently drop the NaNs otherwise
  const bool finite = device_all_finite<T>(st, d, n) && (n < 2 || device_all_finite<T>(st, e, n - 1));
  gk_bound_kernel<T><<<1, 256, 0, st>>>(d, e, (int)n, bb);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  gk_values_kernel<T><<<(unsigned)((n + 63) / 64), 64, 0, st>>>(d, e, (int)n, bb, S);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(de);
  ws_free(h);
  if (R) ws_free(R);
  ws_free(W);
  return finite;
}

template bool singular_values<double>(cudaStream_t, View<const double>, double*, double);

namespace {
template <class TD, class TS>
__global__ void cast_copy_kernel(TD* __restrict__ dst, i64 ld, const TS* __restrict__ src, i64 rs, i64 cs, i64 m, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < m) dst[j * ld + i] = (TD)src[i * rs + j * cs];
}
}  // namespace

// f32: the condensed form is computed in f64 on a copy (as the f32 decompositions with vectors do, svd_vectors.cu): the
// values come out to f32 accuracy relative to sigma_max at least, and an exactly rank-deficient f32 input cannot push
// subnormal intermediates through the f32 bidiagonalization kernel
template <>
bool singular_values<float>(cudaStream_t st, View<const float> A, float* S, double qr_ratio_threshold) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n);
  if (size == 0) return true;
  double* W = (double*)ws_alloc((size_t)m * (size_t)n * 8);
  for (i64 c0 = 0; c0 < n; c0 += 65535) {
    const i64 nc = std::min<i64>(65535, n - c0);
    cast_copy_kernel<double, float><<<dim3((unsigned)((m + 255) / 256), (unsigned)nc), 256, 0, st>>>(W, m, A.ptr, A.rs, A.cs, m, c0);
    note_launch();
  }
  double* S64 = (double*)ws_alloc((size_t)size * 8);
  const bool ok = singular_values<double>(st, View<const double>{W, m, n, 1, m}, S64, qr_ratio_threshold);
  cast_copy_kernel<float, double><<<dim3((unsigned)((size + 255) / 256), 1), 256, 0, st>>>(S, size, S64, 1, size, size, 0);
  note_launch();
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(S64);
  ws_free(W);
  return ok;
}

}  // namespace fb
