// General (non-symmetric) eigendecomposition on the GPU: faer::linalg::evd::evd_real / evd_cplx (evd/mod.rs:1007-1246).
//   stage A  H <- A, Hessenberg reduction and Z = Q (cplx_condensed.cu, householder.cu / cplx.cu: existing code)
//   stage B  Hessenberg -> Schur form T with Z accumulated: the sweep driver of schur_core.cuh. Every reflector is generated and
//            applied inside a diagonal window held by ONE CTA (schur_window_qr_kernel: lahqr on a whole window;
//            schur_window_chase_kernel: a stretch of a small-bulge multishift sweep), which also yields the window's unitary U;
//            the rows above, the columns to the right and Z are updated with U on the f64 / c64 tensor GEMMs. One 16-byte
//            read-back per sweep (schur_scan_kernel's next active block); shapes of every launch are known on the host.
//   stage C  eigenvectors of T by back substitution (evd_from_schur_kernel, one CTA per eigenvalue or conjugate pair), then
//            UR = Z X (X upper triangular) and UL = Z X' (X' lower triangular) on the structured GEMM.
// f32 / c32 compute in f64 / c64 like `svd` and `self_adjoint_evd`. What the reference has and this does not (aggressive early
// deflation above all) is listed in DESIGN.md §7.
// STATUS: validated on hardware (tests/test_gpu_zz20_evd.py); the core also runs on the CPU (tests/test_schur_core_cpu.py).
#include <algorithm>
#include <memory>

#include "ffi_common.cuh"
#include "runtime.cuh"
#include "schur_core.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {
using sch::Cx;
using sch::Lim;
using sch::Num;

constexpr int WIN_THREADS = 256;
// status word read back once per sweep
enum { ST_ILO = 0, ST_IHI = 1, ST_FAILED = 2, ST_COUNT = 4 };

template <bool CX>
constexpr int win_ld() { return Lim<CX>::W + 1; }  // odd leading dimension: column walks do not hit one shared-memory bank
template <bool CX>
constexpr size_t win_smem() {
  return (size_t)2 * win_ld<CX>() * Lim<CX>::W * sizeof(typename Num<CX>::T) +
         Lim<CX>::NB * (sizeof(sch::Refl<typename Num<CX>::T>) + sizeof(typename Num<CX>::T));
}

template <class S>
__device__ void window_load(S* Hs, S* Us, int lds, const S* H, i64 ld, int lo, int wn, bool with_u) {
  for (int idx = threadIdx.x; idx < wn * wn; idx += blockDim.x) {
    const int i = idx % wn, j = idx / wn;
    Hs[i + j * lds] = H[(lo + i) + (i64)(lo + j) * ld];
    if (with_u) sch::set_real(Us[i + j * lds], i == j ? 1.0 : 0.0);
  }
}
template <class S>
__device__ void window_store(const S* Hs, const S* Us, int lds, S* H, i64 ld, int lo, int wn, S* Uout, int ldu) {
  for (int idx = threadIdx.x; idx < wn * wn; idx += blockDim.x) {
    const int i = idx % wn, j = idx / wn;
    H[(lo + i) + (i64)(lo + j) * ld] = Hs[i + j * lds];
    Uout[i + j * ldu] = Us[i + j * lds];
  }
}

// lahqr on the window H[lo : lo + wn, lo : lo + wn]. shifts_out == null: the window is replaced by its Schur form and Uout (leading
// dimension W) receives the transformation. Otherwise the window is only read, and its eigenvalues become the next sweep's shifts
// (or the exceptional shifts, from the subdiagonal, when `exceptional`).
template <bool CX>
__global__ void __launch_bounds__(WIN_THREADS, 1)
    schur_window_qr_kernel(typename Num<CX>::T* H, i64 ld, int lo, int wn, typename Num<CX>::T* Uout,
                           typename Num<CX>::T* shifts_out, int exceptional, int* status) {
  typedef typename Num<CX>::T S;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int LDS = Lim<CX>::W + 1;
  S* Hs = (S*)smem_raw;
  S* Us = Hs + LDS * Lim<CX>::W;
  if (shifts_out && exceptional) {
    if (threadIdx.x == 0) sch::exceptional_shifts(H, ld, lo + wn, wn, shifts_out);
    return;
  }
  window_load(Hs, Us, LDS, H, ld, lo, wn, shifts_out == nullptr);
  const int left = sch::window_qr<CX>(Hs, shifts_out ? (S*)nullptr : Us, LDS, wn, threadIdx.x, blockDim.x);
  __syncthreads();
  if (shifts_out) {
    if (threadIdx.x == 0) sch::pair_shifts(Hs, LDS, wn, shifts_out);
    return;
  }
  if (left != 0 && threadIdx.x == 0) status[ST_FAILED] = 1;
  window_store(Hs, Us, LDS, H, ld, lo, wn, Uout, Lim<CX>::W);
}

// one stretch of a multishift sweep on its window (schur_core.cuh: window_chase)
template <bool CX>
__global__ void __launch_bounds__(WIN_THREADS, 1)
    schur_window_chase_kernel(typename Num<CX>::T* H, i64 ld, sch::Stretch s, const typename Num<CX>::T* shifts,
                              typename Num<CX>::T* Uout) {
  typedef typename Num<CX>::T S;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int LDS = Lim<CX>::W + 1;
  S* Hs = (S*)smem_raw;
  S* Us = Hs + LDS * Lim<CX>::W;
  sch::Refl<S>* refl = (sch::Refl<S>*)(Us + LDS * Lim<CX>::W);
  S* beta = (S*)(refl + Lim<CX>::NB);
  __shared__ S sh[4 * Lim<CX>::NB];
  for (int i = threadIdx.x; i < (CX ? 1 : 4) * s.nb; i += blockDim.x) sh[i] = shifts[i];
  window_load(Hs, Us, LDS, H, ld, s.w0, s.wn, true);
  sch::window_chase<CX>(Hs, Us, LDS, s, sh, refl, beta, threadIdx.x, blockDim.x);
  window_store(Hs, Us, LDS, H, ld, s.w0, s.wn, Uout, Lim<CX>::W);
}

// One warp: clear negligible subdiagonals upwards from row ihi - 1 and skip deflated 1 x 1 blocks; status <- the bottom unreduced
// block [ilo, ihi) (ihi = 0: the matrix is reduced).
template <bool CX>
__global__ void __launch_bounds__(32) schur_scan_kernel(typename Num<CX>::T* H, i64 ld, int ihi, int* status) {
  const int lane = threadIdx.x;
  int ilo = 0;
  while (ihi > 0) {
    int found = 0;
    for (int base = ihi - 1; base > 0 && found == 0; base -= 32) {
      const int k = base - lane;
      const bool neg = k > 0 && sch::negligible(H, ld, k, 0, ihi);
      const unsigned m = __ballot_sync(0xffffffffu, neg);
      if (m) found = base - (__ffs(m) - 1);
    }
    if (found > 0 && lane == 0) sch::set_real(H[found + (i64)(found - 1) * ld], 0.0);
    __syncwarp();
    if (found < ihi - 1) {
      ilo = found;
      break;
    }
    ihi = found;
  }
  if (lane == 0) {
    status[ST_ILO] = ilo;
    status[ST_IHI] = ihi;
  }
}

// eigenvalues from the diagonal blocks of T (2 x 2 blocks are in standard form: a conjugate pair a +- i sqrt|b| sqrt|c|)
__global__ void schur_eigenvalues_kernel(const double* T, i64 ld, int n, double* s_re, double* s_im) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  double im = 0.0;
  if (k + 1 < n && T[(k + 1) + (i64)k * ld] != 0.0) im = sqrt(fabs(T[(k + 1) + (i64)k * ld])) * sqrt(fabs(T[k + (i64)(k + 1) * ld]));
  else if (k > 0 && T[k + (i64)(k - 1) * ld] != 0.0) im = -sqrt(fabs(T[k + (i64)(k - 1) * ld])) * sqrt(fabs(T[(k - 1) + (i64)k * ld]));
  s_re[k] = T[k + (i64)k * ld];
  s_im[k] = im;
}
__global__ void schur_eigenvalues_kernel(const Cx* T, i64 ld, int n, Cx* s, Cx*) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) s[k] = T[k + (i64)k * ld];
}

// norm <- sum of |T(i, j)| over the (quasi-)triangle, the scale of the eigenvector solves' perturbation (mod.rs:567-572, 632-637)
template <bool CX>
__global__ void __launch_bounds__(256) schur_norm_kernel(const typename Num<CX>::T* T, i64 ld, int n, double* norm) {
  __shared__ double part[256];
  double acc = 0.0;
  for (int j = blockIdx.x; j < n; j += gridDim.x) {
    const int rows = min(j + (CX ? 1 : 2), n);
    for (int i = threadIdx.x; i < rows; i += 256) acc += sch::abs1(T[i + (i64)j * ld]);
  }
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) part[threadIdx.x] += part[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *norm = part[0];
}

// CTA k: the eigenvector of T's k-th eigenvalue (a real conjugate pair: the CTA of its first column does both columns)
template <bool CX>
__global__ void __launch_bounds__(256)
    evd_from_schur_kernel(sch::MatV<const typename Num<CX>::T> T, sch::MatV<typename Num<CX>::T> X, int n, int conj,
                          const double* norm) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int k = blockIdx.x;
  if constexpr (CX) {
    sch::eigvec_cplx(T, conj != 0, X, k, *norm, (Cx*)smem_raw, threadIdx.x, blockDim.x);
  } else {
    if (k > 0 && T(k, k - 1) != 0.0) return;
    double* b = (double*)smem_raw;
    sch::eigvec_real(T, X, n, k, *norm, b, b + n + 2, threadIdx.x, blockDim.x);
  }
}

// compact column-major f64 / c64 working copies of strided f32 / f64 / c32 / c64 views (nc scalars per element)
template <class TS>
__global__ void widen_in_kernel(double* dst, i64 ld, const TS* src, i64 rs, i64 cs, i64 n, int nc) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  for (i64 j = blockIdx.y; i < n && j < n; j += gridDim.y)
    for (int c = 0; c < nc; ++c) dst[(j * ld + i) * nc + c] = (double)src[(i * rs + j * cs) * nc + c];
}
template <class TD>
__global__ void narrow_out_kernel(TD* dst, i64 rs, i64 cs, const double* src, i64 ld, i64 m, i64 n, int nc) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  for (i64 j = blockIdx.y; i < m && j < n; j += gridDim.y)
    for (int c = 0; c < nc; ++c) dst[(i * rs + j * cs) * nc + c] = (TD)src[(j * ld + i) * nc + c];
}
// H <- upper Hessenberg part (the reflectors below the subdiagonal are dropped); Z <- identity
template <class S>
__global__ void hessenberg_part_kernel(S* H, S* Z, i64 n) {
  const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  for (i64 j = blockIdx.y; i < n && j < n; j += gridDim.y) {
    if (H && i > j + 1) sch::set_real(H[i + j * n], 0.0);
    if (Z) sch::set_real(Z[i + j * n], i == j ? 1.0 : 0.0);
  }
}
inline dim3 grid2d(i64 n) { return dim3((unsigned)((n + 255) / 256), (unsigned)std::min<i64>(n, 65535)); }

template <bool CX>
void product(cudaStream_t st, VD dst, VCD lhs, bool conj_lhs, VCD rhs, int rhs_struct) {
  if (CX) gemm_c64(st, dst, RECT, 0, lhs, RECT, conj_lhs, rhs, rhs_struct, false, 1.0, 0.0);
  else gemm_f64(st, dst, RECT, 0, lhs, RECT, rhs, rhs_struct, 1.0);
}

// the device side of schur_core.cuh's sweep driver
template <bool CX>
struct DevOps {
  typedef typename Num<CX>::T S;
  static constexpr int W = Lim<CX>::W;
  cudaStream_t st;
  i64 n;
  S *H, *Z, *Ubuf, *tmp, *shifts;
  int* status;
  long long sweeps = 0, windows = 0;

  VD view(S* p, i64 m, i64 k, i64 ld) const { return VD{(double*)p, m, k, 1, ld}; }
  void copy_back(S* dst, i64 ld_dst, const S* src, i64 ld_src, i64 rows, i64 cols) const {
    FB_CUDA_CHECK(cudaMemcpy2DAsync(dst, (size_t)ld_dst * sizeof(S), src, (size_t)ld_src * sizeof(S), (size_t)rows * sizeof(S),
                                    (size_t)cols, cudaMemcpyDeviceToDevice, st));
  }
  // H[:lo, win] U, Z[:, win] U and U^H H[win, hi:] for the window [lo, lo + wn) whose U a window kernel has just written
  void apply_u(int lo, int wn) {
    const i64 hi = lo + wn;
    const VCD U = cv(view(Ubuf, wn, wn, W));
    if (lo > 0) {
      product<CX>(st, view(tmp, lo, wn, n), cv(view(H + (i64)lo * n, lo, wn, n)), false, U, RECT);
      copy_back(H + (i64)lo * n, n, tmp, n, lo, wn);
    }
    if (Z) {
      product<CX>(st, view(tmp, n, wn, n), cv(view(Z + (i64)lo * n, n, wn, n)), false, U, RECT);
      copy_back(Z + (i64)lo * n, n, tmp, n, n, wn);
    }
    if (hi < n) {
      product<CX>(st, view(tmp, wn, n - hi, W), U.t(), true, cv(view(H + lo + hi * n, wn, n - hi, n)), RECT);
      copy_back(H + lo + hi * n, n, tmp, W, wn, n - hi);
    }
  }
  bool scan(int ihi, int* ilo, int* ihi_out) {
    schur_scan_kernel<CX><<<1, 32, 0, st>>>(H, n, ihi, status);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    int h[ST_COUNT];
    FB_CUDA_CHECK(cudaMemcpyAsync(h, status, sizeof(h), cudaMemcpyDeviceToHost, st));
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    *ilo = h[ST_ILO];
    *ihi_out = h[ST_IHI];
    return h[ST_FAILED] == 0;
  }
  void finish_block(int lo, int hi) {
    schur_window_qr_kernel<CX><<<1, WIN_THREADS, win_smem<CX>(), st>>>(H, n, lo, hi - lo, Ubuf, nullptr, 0, status);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    apply_u(lo, hi - lo);
  }
  void make_shifts(int ilo, int ihi, int ns, bool exceptional) {
    (void)ilo;
    ++sweeps;
    schur_window_qr_kernel<CX><<<1, WIN_THREADS, win_smem<CX>(), st>>>(H, n, ihi - ns, ns, nullptr, shifts, exceptional ? 1 : 0, status);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
  void chase(const sch::Stretch& s) {
    ++windows;
    schur_window_chase_kernel<CX><<<1, WIN_THREADS, win_smem<CX>(), st>>>(H, n, s, shifts, Ubuf);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
    apply_u(s.w0, s.wn);
  }
};

template <bool CX>
void configure_kernels() {
  static bool done = false;
  if (done) return;
  FB_CUDA_CHECK(cudaFuncSetAttribute(schur_window_qr_kernel<CX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)win_smem<CX>()));
  FB_CUDA_CHECK(cudaFuncSetAttribute(schur_window_chase_kernel<CX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)win_smem<CX>()));
  FB_CUDA_CHECK(cudaFuncSetAttribute(evd_from_schur_kernel<CX>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  done = true;
}

}  // namespace

long long g_evd_last_sweeps = 0, g_evd_last_windows = 0;

// A: n x n (TO = double / float, complex views in complex units). UL / UR: n x n or ptr == null (not wanted). S, S_im: device,
// compact, n entries of TO's kind (S_im unused for complex). ns_limit: upper bound on the shifts of a sweep. False: a non-finite
// entry in A (nothing written) or the iteration cap.
template <class TO, bool CX>
bool evd_general(cudaStream_t st, View<const TO> A, View<TO> UL, View<TO> UR, TO* S_out, TO* S_im_out, size_t ns_limit) {
  typedef typename Num<CX>::T S;
  constexpr int NC = CX ? 2 : 1;
  const i64 n = A.nrows;
  FB_ASSERT(A.ncols == n, "evd: square matrix required");
  if (n == 0) return true;
  const size_t vec_smem = (size_t)(CX ? (n + 1) * sizeof(Cx) : 2 * (n + 2) * sizeof(double));
  FB_ASSERT(vec_smem <= 200 * 1024 && n < (1 << 24), "evd: dimension too large for the eigenvector kernel's shared memory");
  configure_kernels<CX>();
  const bool want_l = UL.ptr != nullptr, want_r = UR.ptr != nullptr, want_z = want_l || want_r;
  const size_t mat = (size_t)n * (size_t)n * sizeof(S);
  S* H = (S*)ws_alloc(mat);
  widen_in_kernel<TO><<<grid2d(n), 256, 0, st>>>((double*)H, n, A.ptr, A.rs, A.cs, n, NC);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  if (!device_all_finite<double>(st, (const double*)H, n * n * NC)) {  // evd/mod.rs:1021-1027
    ws_free(H);
    return false;
  }
  S* Z = want_z ? (S*)ws_alloc(mat) : nullptr;
  S* tmp = (S*)ws_alloc((size_t)n * Lim<CX>::W * sizeof(S));
  S* small = (S*)ws_alloc((size_t)(Lim<CX>::W * Lim<CX>::W + 4 * Lim<CX>::NB) * sizeof(S) + 64);
  S *Ubuf = small, *shifts = small + Lim<CX>::W * Lim<CX>::W;
  int* status = (int*)(shifts + 4 * Lim<CX>::NB);
  double* norm = (double*)(status + ST_COUNT);
  FB_CUDA_CHECK(cudaMemsetAsync(status, 0, 64, st));
  // stage A
  if (n > 1) {
    const i64 bs = std::min<i64>(32, n - 1);
    S* Hf = (S*)ws_alloc((size_t)bs * (size_t)(n - 1) * sizeof(S));
    hessenberg_in_place_t<double, CX>(st, View<double>{(double*)H, n, n, 1, n}, View<double>{(double*)Hf, bs, n - 1, 1, bs});
    if (want_z) {
      hessenberg_part_kernel<S><<<grid2d(n), 256, 0, st>>>(nullptr, Z, n);
      note_launch();
      const VCD basis{(const double*)(H + 1), n - 1, n - 1, 1, n}, factor{(const double*)Hf, bs, n - 1, 1, bs};
      const VD z11{(double*)(Z + 1 + n), n - 1, n - 1, 1, n};
      householder_sequence_t<double, CX>(st, basis, factor, false, z11, false);
    }
    hessenberg_part_kernel<S><<<grid2d(n), 256, 0, st>>>(H, nullptr, n);
    note_launch();
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    ws_free(Hf);
  } else if (want_z) {
    hessenberg_part_kernel<S><<<grid2d(n), 256, 0, st>>>(nullptr, Z, n);
    note_launch();
  }
  // stage B
  DevOps<CX> ops{st, n, H, Z, Ubuf, tmp, shifts, status};
  const bool ok = sch::schur_drive<CX>(ops, (int)n, (int)std::min<size_t>(ns_limit, 1 << 20));
  g_evd_last_sweeps = ops.sweeps;
  g_evd_last_windows = ops.windows;
  if (ok) {
    S* sv = (S*)ws_alloc((size_t)2 * n * sizeof(S));
    schur_eigenvalues_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const S*)H, n, (int)n, sv, sv + n);
    note_launch();
    narrow_out_kernel<TO><<<dim3((unsigned)((n + 255) / 256), 1), 256, 0, st>>>(S_out, 1, n, (const double*)sv, n, n, 1, NC);
    if (!CX) narrow_out_kernel<TO><<<dim3((unsigned)((n + 255) / 256), 1), 256, 0, st>>>(S_im_out, 1, n, (const double*)(sv + n), n, n, 1, NC);
    note_launch();
    // stage C
    if (want_z) {
      S* X = (S*)ws_alloc(mat);
      S* P = (S*)ws_alloc(mat);
      schur_norm_kernel<CX><<<1, 256, 0, st>>>(H, n, (int)n, norm);  // one CTA: the same sum order in every call
      note_launch();
      const i64 last = (n - 1) + (n - 1) * n;
      for (int side = 0; side < 2; ++side) {
        if (!(side == 0 ? want_r : want_l)) continue;
        // right: T and X as they are; left: T^T (conjugated) and X reversed in rows and columns, which puts the lower
        // triangular X' of evd/mod.rs:1140-1171 in place
        const sch::MatV<const S> Tv = side == 0 ? sch::MatV<const S>{H, 1, n} : sch::MatV<const S>{H + last, -n, -1};
        const sch::MatV<S> Xv = side == 0 ? sch::MatV<S>{X, 1, n} : sch::MatV<S>{X + last, -1, -n};
        evd_from_schur_kernel<CX><<<(unsigned)n, 256, vec_smem, st>>>(Tv, Xv, (int)n, side, norm);
        FB_CUDA_CHECK(cudaGetLastError());
        note_launch();
        product<CX>(st, VD{(double*)P, n, n, 1, n}, VCD{(const double*)Z, n, n, 1, n}, false, VCD{(const double*)X, n, n, 1, n},
                    side == 0 ? TRI_UPPER : TRI_LOWER);
        const View<TO> out = side == 0 ? UR : UL;
        narrow_out_kernel<TO><<<grid2d(n), 256, 0, st>>>(out.ptr, out.rs, out.cs, (const double*)P, n, n, n, NC);
        note_launch();
      }
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
      ws_free(P);
      ws_free(X);
    }
    FB_CUDA_CHECK(cudaStreamSynchronize(st));
    ws_free(sv);
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(small);
  ws_free(tmp);
  if (Z) ws_free(Z);
  ws_free(H);
  return ok;
}

template bool evd_general<double, false>(cudaStream_t, View<const double>, View<double>, View<double>, double*, double*, size_t);
template bool evd_general<float, false>(cudaStream_t, View<const float>, View<float>, View<float>, float*, float*, size_t);
template bool evd_general<double, true>(cudaStream_t, View<const double>, View<double>, View<double>, double*, double*, size_t);
template bool evd_general<float, true>(cudaStream_t, View<const float>, View<float>, View<float>, float*, float*, size_t);

}  // namespace fb

// ---- C ABI (faer-ffi/src/lib.rs:2402-2457; declarations in include/faer_b200_evd.h) ----
using namespace fb;

namespace {

// the reference's tables (evd/schur/mod.rs:59-107)
extern "C" size_t default_recommended_shift_count(size_t n, size_t) {
  return n < 30 ? 2 : n < 60 ? 4 : n < 150 ? 12 : n < 590 ? 32 : n < 3000 ? 64 : n < 6000 ? 128 : 256;
}
extern "C" size_t default_recommended_deflation_window(size_t n, size_t) {
  return n < 30 ? 2 : n < 60 ? 4 : n < 150 ? 10 : n < 590 ? (size_t)((double)n / log2((double)n)) : n < 3000 ? 96 : n < 6000 ? 192 : 384;
}
FaerV0_24_SchurParams schur_params_default() {
  return FaerV0_24_SchurParams{default_recommended_shift_count, default_recommended_deflation_window, 75, 50};
}
FaerV0_24_EvdParams evd_params_default() {
  return FaerV0_24_EvdParams{FaerV0_24_HessenbergParams{192 * 256, 256 * 256}, schur_params_default(), FaerV0_24_EvdFromSchurParams{64}};
}

template <class R, bool CX>
FaerV0_24_EvdStatus evd_entry(FaerV0_24_MatRef A, FaerV0_24_MatMut UL, FaerV0_24_MatMut UR, FaerV0_24_VecMut S, FaerV0_24_VecMut S_im,
                              FaerV0_24_EvdParams params) {
  FB_ENTRY();
  cudaStream_t st = current_stream();
  const size_t n = A.nrows, es = (CX ? 2 : 1) * sizeof(R);
  FB_ASSERT(A.ncols == n && S.len == n && (n == 0 || S.stride >= 1), "evd: square A, S of length n, positive stride");
  if (!CX) FB_ASSERT(S_im.len == n && (n == 0 || S_im.stride >= 1), "evd: S_im of length n, positive stride");
  const bool want_l = UL.ncols != 0, want_r = UR.ncols != 0;
  if (want_l) FB_ASSERT(UL.nrows == n && UL.ncols == n, "evd: UL must be n x n (or have no columns)");
  if (want_r) FB_ASSERT(UR.nrows == n && UR.ncols == n, "evd: UR must be n x n (or have no columns)");
  if (n == 0) return evd_status(true);
  size_t ns_limit = ~(size_t)0;
  if (params.schur.recommended_shift_count) ns_limit = params.schur.recommended_shift_count(n, n);
  StagedMat a = stage<R, CX>(A, st);
  std::unique_ptr<StagedMat> ul, ur;
  if (want_l) ul.reset(new StagedMat(UL.ptr, (i64)n, (i64)n, (i64)UL.row_stride, (i64)UL.col_stride, es, true, true, st));
  if (want_r) ur.reset(new StagedMat(UR.ptr, (i64)n, (i64)n, (i64)UR.row_stride, (i64)UR.col_stride, es, true, true, st));
  R* s_dev = (R*)ws_alloc(2 * n * es);
  const View<R> none{nullptr, 0, 0, 1, 1};
  const bool ok = evd_general<R, CX>(st, a.view<const R>(), want_l ? ul->view<R>() : none, want_r ? ur->view<R>() : none, s_dev,
                                     s_dev + n * (CX ? 2 : 1), ns_limit);
  if (ok) {
    FB_CUDA_CHECK(cudaMemcpy2DAsync(S.ptr, (size_t)S.stride * es, s_dev, es, es, n, cudaMemcpyDefault, st));
    if (!CX) FB_CUDA_CHECK(cudaMemcpy2DAsync(S_im.ptr, (size_t)S_im.stride * es, s_dev + n, es, es, n, cudaMemcpyDefault, st));
  }
  // the eigenvector mirrors were filled from the caller's memory, so a failed call copies back what was there
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  a.finish();
  if (ul) ul->finish();
  if (ur) ur->finish();
  ws_free(s_dev);
  return evd_status(ok);
}

}  // namespace

extern "C" {

#define FB_EVD_GENERAL_FFI(SUF, R, CX)                                                                                         \
  FaerV0_24_EvdFromSchurParams libfaer_v0_23_EvdFromSchurParams_##SUF(void) { return FaerV0_24_EvdFromSchurParams{64}; }       \
  FaerV0_24_SchurParams libfaer_v0_23_SchurParams_##SUF(void) { return schur_params_default(); }                               \
  FaerV0_24_EvdParams libfaer_v0_23_EvdParams_##SUF(void) { return evd_params_default(); }                                     \
  FaerV0_24_Layout libfaer_v0_23_evd_scratch_##SUF(size_t dim, FaerV0_24_ComputeEigenvectors compute_left,                     \
                                                   FaerV0_24_ComputeEigenvectors compute_right, FaerV0_24_Par par,             \
                                                   FaerV0_24_EvdParams params) {                                               \
    (void)compute_left; (void)compute_right; (void)par; (void)params;                                                          \
    return FaerV0_24_Layout{dim * dim * (CX ? 2 : 1) * sizeof(R), 64};                                                         \
  }                                                                                                                            \
  FaerV0_24_EvdStatus libfaer_v0_23_evd_##SUF(FaerV0_24_MatRef A, FaerV0_24_MatMut UL, FaerV0_24_MatMut UR, FaerV0_24_VecMut S, \
                                              FaerV0_24_VecMut S_im, FaerV0_24_Par par, FaerV0_24_MemAlloc mem,                \
                                              FaerV0_24_EvdParams params) {                                                    \
    (void)par; (void)mem;                                                                                                      \
    return evd_entry<R, CX>(A, UL, UR, S, S_im, params);                                                                       \
  }
FB_EVD_GENERAL_FFI(f64, double, false)
FB_EVD_GENERAL_FFI(f32, float, false)
FB_EVD_GENERAL_FFI(c64, double, true)
FB_EVD_GENERAL_FFI(c32, float, true)
#undef FB_EVD_GENERAL_FFI

void faer_b200_evd_last_sweep_counts(long long* out) {
  out[0] = g_evd_last_sweeps;
  out[1] = g_evd_last_windows;
}

}  // extern "C"
