// Host run of the general eigensolver's middle and last stages from faer-rs_b200/csrc/schur_core.cuh: the sweep driver, the two
// window routines (one "thread"), the deflation scan, the shift selection and the eigenvector back substitution are the header's;
// what the GPU does with kernels and GEMMs around them (window load / store, the off-window products with U) is written here as
// plain loops. Test infrastructure for tests/test_schur_core_cpu.py, not product code.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../faer-rs_b200/csrc/schur_core.cuh"

namespace {
using namespace fb::sch;

template <bool CX>
struct HostOps {
  typedef typename Num<CX>::T S;
  static constexpr int W = Lim<CX>::W;
  int n;
  S* H;  // n x n, column-major
  S* Z;  // n x n or null
  std::vector<S> win, U, shifts, E, tmp;
  bool failed = false;
  long long sweeps = 0, stretches = 0;

  HostOps(int n_, S* H_, S* Z_) : n(n_), H(H_), Z(Z_), win(W * W), U(W * W), shifts(4 * Lim<CX>::NB), E(W * W), tmp((size_t)n_ * W) {}

  bool scan(int ihi, int* ilo, int* ihi_out) {
    while (ihi > 0) {
      int k = ihi - 1;
      while (k > 0 && !negligible(H, (long long)n, k, 0, ihi)) --k;
      if (k > 0) set_real(H[k + (size_t)(k - 1) * n], 0.0);
      if (k < ihi - 1) {
        *ilo = k;
        *ihi_out = ihi;
        return !failed;
      }
      ihi = k;
    }
    *ilo = 0;
    *ihi_out = 0;
    return !failed;
  }
  void load(int lo, int wn) {
    for (int j = 0; j < wn; ++j)
      for (int i = 0; i < wn; ++i) {
        win[i + j * W] = H[(lo + i) + (size_t)(lo + j) * n];
        set_real(U[i + j * W], i == j ? 1.0 : 0.0);
      }
  }
  // window back, then H[:lo, win] U, U^H H[win, hi:], Z[:, win] U
  void apply_u(int lo, int wn) {
    const int hi = lo + wn;
    for (int j = 0; j < wn; ++j)
      for (int i = 0; i < wn; ++i) H[(lo + i) + (size_t)(lo + j) * n] = win[i + j * W];
    auto right = [&](S* M, int rows) {
      for (int j = 0; j < wn; ++j)
        for (int i = 0; i < rows; ++i) {
          S acc;
          set_real(acc, 0.0);
          for (int k = 0; k < wn; ++k) acc = acc + M[i + (size_t)(lo + k) * n] * U[k + j * W];
          tmp[i + (size_t)j * n] = acc;
        }
      for (int j = 0; j < wn; ++j)
        for (int i = 0; i < rows; ++i) M[i + (size_t)(lo + j) * n] = tmp[i + (size_t)j * n];
    };
    right(H, lo);
    if (Z) right(Z, n);
    for (int j = hi; j < n; ++j) {
      for (int i = 0; i < wn; ++i) {
        S acc;
        set_real(acc, 0.0);
        for (int k = 0; k < wn; ++k) acc = acc + conj_(U[k + i * W]) * H[(lo + k) + (size_t)j * n];
        tmp[i] = acc;
      }
      for (int i = 0; i < wn; ++i) H[(lo + i) + (size_t)j * n] = tmp[i];
    }
  }
  void finish_block(int lo, int hi) {
    load(lo, hi - lo);
    if (window_qr<CX>(win.data(), U.data(), W, hi - lo, 0, 1) != 0) failed = true;
    apply_u(lo, hi - lo);
  }
  void make_shifts(int ilo, int ihi, int ns, bool exceptional) {
    (void)ilo;
    ++sweeps;
    if (exceptional) {
      exceptional_shifts(H, (long long)n, ihi, ns, shifts.data());
      return;
    }
    for (int j = 0; j < ns; ++j)
      for (int i = 0; i < ns; ++i) E[i + j * W] = H[(ihi - ns + i) + (size_t)(ihi - ns + j) * n];
    window_qr<CX>(E.data(), (S*)nullptr, W, ns, 0, 1);
    pair_shifts(E.data(), W, ns, shifts.data());
  }
  void chase(const Stretch& s) {
    ++stretches;
    load(s.w0, s.wn);
    Refl<S> refl[Lim<CX>::NB];
    S beta[Lim<CX>::NB];
    window_chase<CX>(win.data(), U.data(), W, s, shifts.data(), refl, beta, 0, 1);
    apply_u(s.w0, s.wn);
  }
};

template <bool CX>
double schur_norm(const typename Num<CX>::T* T, int n) {
  double norm = 0.0;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < std::min(j + (CX ? 1 : 2), n); ++i) norm += abs1(T[i + (size_t)j * n]);
  return norm;
}
}  // namespace

// H (n x n Hessenberg, column-major) <- T, Z <- Z U; s_re / s_im <- eigenvalues; XR / XL (n x n, zero on entry) <- the upper / lower
// triangular eigenvector matrices of T. info[0] = sweeps, info[1] = windows chased. Returns 0, or 1 when the iteration cap was hit.
extern "C" int schur_host_f64(int n, double* H, double* Z, double* s_re, double* s_im, double* XR, double* XL, int ns_limit,
                              long long* info) {
  HostOps<false> ops(n, H, Z);
  const bool ok = schur_drive<false>(ops, n, ns_limit);
  info[0] = ops.sweeps;
  info[1] = ops.stretches;
  if (!ok) return 1;
  for (int k = 0; k < n; ++k) {
    s_re[k] = H[k + (size_t)k * n];
    s_im[k] = 0.0;
    if (k + 1 < n && H[(k + 1) + (size_t)k * n] != 0.0) {
      const double im = sqrt(fabs(H[(k + 1) + (size_t)k * n])) * sqrt(fabs(H[k + (size_t)(k + 1) * n]));
      s_re[k + 1] = H[(k + 1) + (size_t)(k + 1) * n];
      s_im[k] = im;
      s_im[k + 1] = -im;
      ++k;
    }
  }
  const double norm = schur_norm<false>(H, n);
  std::vector<double> b(2 * (size_t)n + 4);
  const size_t last = (size_t)(n - 1) + (size_t)(n - 1) * n;
  for (int side = 0; side < 2; ++side) {
    // right: T and X as they are; left: T^T and X, both reversed in rows and columns (evd/mod.rs:1140-1171)
    MatV<const double> Tv = side == 0 ? MatV<const double>{H, 1, n} : MatV<const double>{H + last, -(long long)n, -1};
    MatV<double> Xv = side == 0 ? MatV<double>{XR, 1, n} : MatV<double>{XL + last, -1, -(long long)n};
    for (int k = 0; k < n; ++k) {
      if (k > 0 && Tv(k, k - 1) != 0.0) continue;  // second column of a pair
      eigvec_real(Tv, Xv, n, k, norm, b.data(), b.data() + n + 2, 0, 1);
    }
  }
  return 0;
}

// the same for interleaved complex matrices; s holds n complex eigenvalues
extern "C" int schur_host_c64(int n, double* H_, double* Z_, double* s_, double* XR_, double* XL_, int ns_limit, long long* info) {
  Cx *H = (Cx*)H_, *Z = (Cx*)Z_, *s = (Cx*)s_, *XR = (Cx*)XR_, *XL = (Cx*)XL_;
  HostOps<true> ops(n, H, Z);
  const bool ok = schur_drive<true>(ops, n, ns_limit);
  info[0] = ops.sweeps;
  info[1] = ops.stretches;
  if (!ok) return 1;
  for (int k = 0; k < n; ++k) s[k] = H[k + (size_t)k * n];
  const double norm = schur_norm<true>(H, n);
  std::vector<Cx> b((size_t)n + 1);
  const size_t last = (size_t)(n - 1) + (size_t)(n - 1) * n;
  for (int k = 0; k < n; ++k) {
    eigvec_cplx(MatV<const Cx>{H, 1, n}, false, MatV<Cx>{XR, 1, n}, k, norm, b.data(), 0, 1);
    eigvec_cplx(MatV<const Cx>{H + last, -(long long)n, -1}, true, MatV<Cx>{XL + last, -1, -(long long)n}, k, norm, b.data(), 0, 1);
  }
  return 0;
}
