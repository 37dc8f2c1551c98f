// Eigenvalues of a self-adjoint matrix on the GPU (SURVEY.md §8f rank 4, values only): the lower triangle of A is copied,
// reduced to tridiagonal form by the HBM-bound persistent kernel of tridiag.cu, and the eigenvalues of the tridiagonal
// come from one bisection thread per value (tridiag_ev.cuh).
// Reference: faer/src/linalg/evd/mod.rs:270-353 (`self_adjoint_evd` with u = None: copy_from_triangular_lower, tridiag_in_place,
// tridiag_evd::qr_algorithm on (diag, offdiag); nondecreasing order), as `MatRef::self_adjoint_eigenvalues` (solvers.rs:417-456).
// This file is the VALUES-ONLY path (U passed with no columns); with eigenvectors the entry point goes to svd_vectors.cu
// (divide and conquer of the tridiagonal, tridiag_dc.cu, + the Householder back-transform). Any n (tridiag.cu keeps its
// per-CTA vectors in global memory above n = 8192).
// STATUS: validated on hardware (tests/test_gpu_zz8_self_adjoint_eigenvalues.py, tests/test_gpu_zz11_evd_svd_vectors.py,
// tests/test_gpu_zz24_spectral_exact.py); tridiag_ev.cuh is also
// checked on the CPU (the same header compiled for the host, tests/test_tridiag_ev_cpu.py).
#include "runtime.cuh"
#include "tensor_ops.cuh"
#include "tridiag_ev.cuh"

namespace fb {

namespace {

// dst (column-major, ld = n) lower triangle <- src lower triangle; the strict upper part of dst is zero-filled (never read)
template <class T>
__global__ void copy_lower_kernel(T* __restrict__ dst, i64 n, const T* __restrict__ src, i64 rs, i64 cs) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = blockIdx.y;
  if (i < n && j < n) dst[j * n + i] = i >= j ? src[i * rs + j * cs] : T(0);
}

template <class T>
__global__ void extract_tridiag_kernel(const T* __restrict__ A, i64 cs, int n, T* __restrict__ d, T* __restrict__ e) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    d[i] = A[(i64)i + (i64)i * cs];
    if (i + 1 < n) e[i] = A[(i64)(i + 1) + (i64)i * cs];
  }
}

// bb[0], bb[1] = padded Gershgorin interval, bb[2] = max e_i^2
template <class T>
__global__ void __launch_bounds__(256) st_bounds_kernel(const T* __restrict__ d, const T* __restrict__ e, int n,
                                                         T* __restrict__ bb) {
  __shared__ T s_lo[256], s_hi[256], s_e2[256];
  T lo = d[0], hi = d[0], e2 = 0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const T r = (i > 0 ? fabs(e[i - 1]) : T(0)) + (i + 1 < n ? fabs(e[i]) : T(0));
    lo = fmin(lo, d[i] - r);
    hi = fmax(hi, d[i] + r);
    if (i + 1 < n) e2 = fmax(e2, e[i] * e[i]);
  }
  s_lo[threadIdx.x] = lo;
  s_hi[threadIdx.x] = hi;
  s_e2[threadIdx.x] = e2;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_lo[threadIdx.x] = fmin(s_lo[threadIdx.x], s_lo[threadIdx.x + s]);
      s_hi[threadIdx.x] = fmax(s_hi[threadIdx.x], s_hi[threadIdx.x + s]);
      s_e2[threadIdx.x] = fmax(s_e2[threadIdx.x], s_e2[threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const T span = fmax(fabs(s_lo[0]), fabs(s_hi[0]));
    const T pad = T(4) * tev::Lim<T>::eps() * span * T(n) + tev::Lim<T>::safmin();
    bb[0] = s_lo[0] - pad;
    bb[1] = s_hi[0] + pad;
    bb[2] = s_e2[0];
  }
}

template <class T>
__global__ void __launch_bounds__(64) st_values_kernel(const T* __restrict__ d, const T* __restrict__ e, int n,
                                                        const T* __restrict__ bb, T* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = tev::st_kth_smallest<T>(d, e, n, k, bb[0], bb[1], bb[2]);
}

}  // namespace

// S (device, compact, n entries) <- eigenvalues of the self-adjoint matrix whose LOWER triangle is in A, nondecreasing.
template <class T>
bool self_adjoint_eigenvalues(cudaStream_t st, View<const T> A, T* S) {
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n, "self_adjoint_eigenvalues: square matrix required");
  if (n == 0) return true;
  FB_ASSERT(n < 65536, "self_adjoint_eigenvalues: dimension too large for the copy launch");
  T* W = (T*)ws_alloc((size_t)n * (size_t)n * sizeof(T));
  {
    dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
    copy_lower_kernel<T><<<grid, 256, 0, st>>>(W, n, A.ptr, A.rs, A.cs);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
  T* h = (T*)ws_alloc((size_t)(n + 1) * sizeof(T));
  tridiag_in_place<T>(st, View<T>{W, n, n, 1, n}, View<T>{h, 1, n - 1, 1, 1});  // one-row factor: taus only, no T blocks
  T* de = (T*)ws_alloc((size_t)(2 * n + 4) * sizeof(T));
  T *d = de, *e = de + n, *bb = de + 2 * n;
  extract_tridiag_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, n, (int)n, d, e);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  const bool finite = device_all_finite<T>(st, d, n) && (n < 2 || device_all_finite<T>(st, e, n - 1));
  st_bounds_kernel<T><<<1, 256, 0, st>>>(d, e, (int)n, bb);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  st_values_kernel<T><<<(unsigned)((n + 63) / 64), 64, 0, st>>>(d, e, (int)n, bb, S);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(de);
  ws_free(h);
  ws_free(W);
  return finite;
}

template bool self_adjoint_eigenvalues<double>(cudaStream_t, View<const double>, double*);

namespace {
template <class TD, class TS>
__global__ void evd_cast_copy_kernel(TD* __restrict__ dst, i64 ld, const TS* __restrict__ src, i64 rs, i64 cs, i64 m, i64 c0) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  const i64 j = c0 + blockIdx.y;
  if (i < m) dst[j * ld + i] = (TD)src[i * rs + j * cs];
}
}  // namespace

// f32 through an f64 copy (see svd.cu: same reasons)
template <>
bool self_adjoint_eigenvalues<float>(cudaStream_t st, View<const float> A, float* S) {
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n, "self_adjoint_eigenvalues: square matrix required");
  if (n == 0) return true;
  double* W = (double*)ws_alloc((size_t)n * (size_t)n * 8);
  for (i64 c0 = 0; c0 < n; c0 += 65535) {
    const i64 nc = std::min<i64>(65535, n - c0);
    evd_cast_copy_kernel<double, float><<<dim3((unsigned)((n + 255) / 256), (unsigned)nc), 256, 0, st>>>(W, n, A.ptr, A.rs, A.cs, n, c0);
    note_launch();
  }
  double* S64 = (double*)ws_alloc((size_t)n * 8);
  const bool ok = self_adjoint_eigenvalues<double>(st, View<const double>{W, n, n, 1, n}, S64);
  evd_cast_copy_kernel<float, double><<<dim3((unsigned)((n + 255) / 256), 1), 256, 0, st>>>(S, n, S64, 1, n, n, 0);
  note_launch();
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(S64);
  ws_free(W);
  return ok;
}

}  // namespace fb
