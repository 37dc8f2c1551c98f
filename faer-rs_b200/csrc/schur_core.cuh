// Hessenberg -> Schur form and eigenvectors of the Schur form: the scalar routines, the two diagonal-window routines and the sweep
// driver, shared by the CUDA build (schur.cu) and a host build (tools/emul/schur_host.cpp, tests/test_schur_core_cpu.py).
//
// Reference: faer/src/linalg/evd/schur/{real,complex}_schur.rs (lahqr, the small-bulge multishift sweep) and evd/mod.rs:557-958
// (eigenvectors of the Schur form); the formulas of lahqr / lanv2 / laqr1 are LAPACK's, which the reference follows.
//
// One principle: every reflector is generated and applied inside a diagonal window of at most W rows that one CTA holds in shared
// memory together with the accumulated unitary U of the window; the driver updates what lies outside the window with U by GEMM.
// The window routines are written over (tid, nt): each phase partitions its rows / columns over the nt threads and SCH_SYNC()
// separates the phases, so a host build with nt = 1 runs the same statements in the same order.
//
// Reflectors are P = I - tau w w^H with w = (1, v1, v2) and tau real, so P is Hermitian and unitary for real and complex scalars
// alike: P x = beta e1 with beta = -phase(x0) |x|. The complex Schur form therefore has complex subdiagonals while it iterates.
//
// Not built (DESIGN.md §7): aggressive early deflation, the search for two consecutive small subdiagonals inside lahqr, vigilant
// deflation and re-introduction of collapsed bulges inside a sweep (a collapsed bulge is an identity reflector here).
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define SCH_HD __host__ __device__
#else
#define SCH_HD
#endif
#if defined(__CUDA_ARCH__)
#define SCH_SYNC() __syncthreads()
#else
#define SCH_SYNC() ((void)0)
#endif

namespace fb {
namespace sch {

constexpr double EPS = 2.220446049250313e-16;      // the reference's eps::<f64>()
constexpr double SMALL_NUM = 2.2250738585072014e-308 / EPS;

struct Cx {
  double re, im;
};
SCH_HD inline Cx operator+(Cx a, Cx b) { return Cx{a.re + b.re, a.im + b.im}; }
SCH_HD inline Cx operator-(Cx a, Cx b) { return Cx{a.re - b.re, a.im - b.im}; }
SCH_HD inline Cx operator-(Cx a) { return Cx{-a.re, -a.im}; }
SCH_HD inline Cx operator*(Cx a, Cx b) { return Cx{a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }
SCH_HD inline Cx operator*(Cx a, double s) { return Cx{a.re * s, a.im * s}; }
SCH_HD inline Cx operator*(double s, Cx a) { return Cx{a.re * s, a.im * s}; }
SCH_HD inline Cx conj_(Cx a) { return Cx{a.re, -a.im}; }
SCH_HD inline double conj_(double a) { return a; }
SCH_HD inline double abs1(Cx a) { return fabs(a.re) + fabs(a.im); }
SCH_HD inline double abs1(double a) { return fabs(a); }
SCH_HD inline double abs2(Cx a) { return a.re * a.re + a.im * a.im; }
SCH_HD inline double abs2(double a) { return a * a; }
SCH_HD inline double absv(Cx a) { return hypot(a.re, a.im); }
SCH_HD inline double absv(double a) { return fabs(a); }
SCH_HD inline bool is_zero(Cx a) { return a.re == 0.0 && a.im == 0.0; }
SCH_HD inline bool is_zero(double a) { return a == 0.0; }
SCH_HD inline void set_real(Cx& a, double r) { a = Cx{r, 0.0}; }
SCH_HD inline void set_real(double& a, double r) { a = r; }
// a / b, scaled so that |b|^2 cannot overflow or underflow
SCH_HD inline Cx div_(Cx a, Cx b) {
  const double m = fmax(fabs(b.re), fabs(b.im));
  const double br = b.re / m, bi = b.im / m, d = br * br + bi * bi;
  return Cx{(a.re * br + a.im * bi) / d / m, (a.im * br - a.re * bi) / d / m};
}
SCH_HD inline double div_(double a, double b) { return a / b; }
SCH_HD inline Cx sqrt_(Cx a) {
  const double r = absv(a);
  if (r == 0.0) return Cx{0.0, 0.0};
  const double s = sqrt(0.5 * (r + fabs(a.re)));
  const double t = 0.5 * a.im / s;
  return a.re >= 0.0 ? Cx{s, t} : Cx{fabs(t), a.im >= 0.0 ? s : -s};
}

template <bool CX>
struct Num {
  typedef double T;
};
template <>
struct Num<true> {
  typedef Cx T;
};

// window and shift-count limits: H and U of a window (2 W^2 scalars) fit the 227 KB of shared memory a CTA can have
template <bool CX>
struct Lim {
  static constexpr int W = CX ? 64 : 96;      // rows of a diagonal window
  static constexpr int NR = CX ? 2 : 3;       // rows of a bulge's reflector (single / double shift)
  static constexpr int NB = 16;               // bulges of a chain
  static constexpr int NS = CX ? NB : 2 * NB;  // shifts of a sweep
};

// ---- reflectors ----------------------------------------------------------------------------------------------------------------
template <class S>
struct Refl {
  S v1, v2;
  double tau;
};
// P (x0, x1, x2) = (beta, 0, 0); nr = 2 ignores x2. A zero tail gives the identity (tau = 0, beta = x0).
template <class S>
SCH_HD inline Refl<S> make_reflector(int nr, S x0, S x1, S x2, S* beta) {
  Refl<S> r;
  set_real(r.v1, 0.0);
  set_real(r.v2, 0.0);
  r.tau = 0.0;
  *beta = x0;
  if (nr < 3) set_real(x2, 0.0);
  const double tail = fmax(abs1(x1), abs1(x2));
  if (!(tail > 0.0)) return r;
  const double m = fmax(tail, abs1(x0));
  const S y0 = x0 * (1.0 / m), y1 = x1 * (1.0 / m), y2 = x2 * (1.0 / m);
  const double nrm = sqrt(abs2(y0) + abs2(y1) + abs2(y2));
  const double a0 = absv(y0);
  S ph;
  set_real(ph, 1.0);
  if (a0 > 0.0) ph = y0 * (1.0 / a0);
  const S b = ph * (-nrm);
  const S u0 = y0 - b;
  r.v1 = div_(y1, u0);
  r.v2 = div_(y2, u0);
  r.tau = 2.0 / (1.0 + abs2(r.v1) + abs2(r.v2));
  *beta = b * m;
  return r;
}
// rows (a0, a1, a2) of one column <- P (a0, a1, a2)
template <class S>
SCH_HD inline void refl_left(const Refl<S>& r, int nr, S& a0, S& a1, S& a2) {
  S s = a0 + conj_(r.v1) * a1;
  if (nr == 3) s = s + conj_(r.v2) * a2;
  s = s * r.tau;
  a0 = a0 - s;
  a1 = a1 - r.v1 * s;
  if (nr == 3) a2 = a2 - r.v2 * s;
}
// columns (a0, a1, a2) of one row <- (a0, a1, a2) P
template <class S>
SCH_HD inline void refl_right(const Refl<S>& r, int nr, S& a0, S& a1, S& a2) {
  S s = a0 + a1 * r.v1;
  if (nr == 3) s = s + a2 * r.v2;
  s = s * r.tau;
  a0 = a0 - s;
  a1 = a1 - s * conj_(r.v1);
  if (nr == 3) a2 = a2 - s * conj_(r.v2);
}

// ---- 2 x 2 blocks --------------------------------------------------------------------------------------------------------------
SCH_HD inline double sign_(double a, double b) { return b >= 0.0 ? fabs(a) : -fabs(a); }
// Standard form of a real 2 x 2 block (LAPACK dlanv2; the reference's lahqr_schur22): [a b; c d] <- R^T [a b; c d] R with
// R = [cs -sn; sn cs], so that either c = 0 or a = d and b c < 0. (rt1r, rt1i), (rt2r, rt2i) are the eigenvalues.
SCH_HD inline void standardize22(double& a, double& b, double& c, double& d, double& rt1r, double& rt1i, double& rt2r, double& rt2i,
                                 double& cs, double& sn) {
  const double multpl = 4.0;
  if (c == 0.0) {
    cs = 1.0;
    sn = 0.0;
  } else if (b == 0.0) {
    cs = 0.0;
    sn = 1.0;
    const double t = d;
    d = a;
    a = t;
    b = -c;
    c = 0.0;
  } else if (a - d == 0.0 && sign_(1.0, b) != sign_(1.0, c)) {
    cs = 1.0;
    sn = 0.0;
  } else {
    double temp = a - d;
    double p = 0.5 * temp;
    const double bcmax = fmax(fabs(b), fabs(c));
    const double bcmis = fmin(fabs(b), fabs(c)) * sign_(1.0, b) * sign_(1.0, c);
    const double scale = fmax(fabs(p), bcmax);
    double z = (p / scale) * p + (bcmax / scale) * bcmis;
    if (z >= multpl * EPS) {
      z = p + sign_(sqrt(scale) * sqrt(z), p);
      a = d + z;
      d = d - (bcmax / z) * bcmis;
      const double tau = hypot(c, z);
      cs = z / tau;
      sn = c / tau;
      b = b - c;
      c = 0.0;
    } else {
      const double sigma = b + c;
      const double tau = hypot(sigma, temp);
      cs = sqrt(0.5 * (1.0 + fabs(sigma) / tau));
      sn = -(p / (tau * cs)) * sign_(1.0, sigma);
      const double aa = a * cs + b * sn, bb = -a * sn + b * cs, cc = c * cs + d * sn, dd = -c * sn + d * cs;
      a = aa * cs + cc * sn;
      b = bb * cs + dd * sn;
      c = -aa * sn + cc * cs;
      d = -bb * sn + dd * cs;
      temp = 0.5 * (a + d);
      a = temp;
      d = temp;
      if (c != 0.0) {
        if (b != 0.0) {
          if (sign_(1.0, b) == sign_(1.0, c)) {
            const double sab = sqrt(fabs(b)), sac = sqrt(fabs(c));
            p = sign_(sab * sac, c);
            const double tau2 = 1.0 / sqrt(fabs(b + c));
            a = temp + p;
            d = temp - p;
            b = b - c;
            c = 0.0;
            const double cs1 = sab * tau2, sn1 = sac * tau2;
            temp = cs * cs1 - sn * sn1;
            sn = cs * sn1 + sn * cs1;
            cs = temp;
          }
        } else {
          b = -c;
          c = 0.0;
          temp = cs;
          cs = -sn;
          sn = temp;
        }
      }
    }
  }
  rt1r = a;
  rt2r = d;
  if (c == 0.0) {
    rt1i = rt2i = 0.0;
  } else {
    rt1i = sqrt(fabs(b)) * sqrt(fabs(c));
    rt2i = -rt1i;
  }
}

// eigenvalues of a real 2 x 2 block as lahqr takes its two shifts: a conjugate pair, or the real eigenvalue nearer h22 twice
SCH_HD inline void shifts22(double h11, double h12, double h21, double h22, double& r1, double& i1, double& r2, double& i2) {
  const double s = fabs(h11) + fabs(h12) + fabs(h21) + fabs(h22);
  if (s == 0.0) {
    r1 = i1 = r2 = i2 = 0.0;
    return;
  }
  h11 /= s;
  h12 /= s;
  h21 /= s;
  h22 /= s;
  const double tr = 0.5 * (h11 + h22);
  const double det = (h11 - tr) * (h22 - tr) - h12 * h21;
  const double rtdisc = sqrt(fabs(det));
  if (det >= 0.0) {
    r1 = r2 = tr * s;
    i1 = rtdisc * s;
    i2 = -i1;
  } else {
    const double a = tr + rtdisc, b = tr - rtdisc;
    r1 = r2 = (fabs(a - h22) <= fabs(b - h22) ? a : b) * s;
    i1 = i2 = 0.0;
  }
}
// Wilkinson shift of a complex 2 x 2 block: the eigenvalue nearer h22 (zlahqr)
SCH_HD inline Cx wilkinson(Cx h11, Cx h12, Cx h21, Cx h22) {
  Cx t = h22;
  const Cx u = sqrt_(h12) * sqrt_(h21);
  double s = abs1(u);
  if (s != 0.0) {
    const Cx x = (h11 - t) * 0.5;
    const double sx = abs1(x);
    s = fmax(s, sx);
    const Cx xs = x * (1.0 / s), us = u * (1.0 / s);
    Cx y = sqrt_(xs * xs + us * us) * s;
    if (sx > 0.0) {
      const Cx xn = x * (1.0 / sx);
      if (xn.re * y.re + xn.im * y.im < 0.0) y = -y;
    }
    t = t - u * div_(u, x + y);
  }
  return t;
}

// First column of (H - s1)(H - s2) for the leading 3 x 3 of H (LAPACK dlaqr1; the reference's lahqr_shiftcolumn). h points at
// H(l, l), column-major with leading dimension ld. The shifts are a conjugate pair or two reals.
SCH_HD inline void shift_column(const double* h, int ld, const double* sh, double& x0, double& x1, double& x2) {
  const double sr1 = sh[0], si1 = sh[1], sr2 = sh[2], si2 = sh[3];
  const double h11 = h[0], h21 = h[1], h12 = h[ld], h22 = h[ld + 1], h32 = h[ld + 2];
  const double s = fabs(h11 - sr2) + fabs(si2) + fabs(h21);
  if (s == 0.0) {
    x0 = x1 = x2 = 0.0;
    return;
  }
  const double h21s = h21 / s;
  x0 = h21s * h12 + (h11 - sr1) * ((h11 - sr2) / s) - si1 * (si2 / s);
  x1 = h21s * (h11 + h22 - sr1 - sr2);
  x2 = h21s * h32;
}
// first column of H - s for the leading 2 x 2 (single shift)
SCH_HD inline void shift_column(const Cx* h, int ld, const Cx* sh, Cx& x0, Cx& x1, Cx& x2) {
  (void)ld;
  x0 = h[0] - sh[0];
  x1 = h[1];
  x2 = Cx{0.0, 0.0};
}

// The reference's deflation test of the subdiagonal H(k, k - 1) inside the block [lo, hi) (lahqr: the classic criterion, then
// Ahues and Tisseur's)
template <class S>
SCH_HD inline bool negligible(const S* H, long long ld, int k, int lo, int hi) {
  const double sub = abs1(H[k + (k - 1) * ld]);
  if (sub <= SMALL_NUM) return true;
  const S hkk = H[k + k * ld], hmm = H[(k - 1) + (k - 1) * ld];
  double tst = abs1(hmm) + abs1(hkk);
  if (tst == 0.0) {
    if (k - 2 >= lo) tst += abs1(H[(k - 1) + (k - 2) * ld]);
    if (k + 1 < hi) tst += abs1(H[(k + 1) + k * ld]);
  }
  if (sub > EPS * tst) return false;
  const double sup = abs1(H[(k - 1) + k * ld]);
  const double ab = fmax(sub, sup), ba = fmin(sub, sup);
  const double dd = abs1(hmm - hkk);
  const double aa = fmax(abs1(hkk), dd), bb = fmin(abs1(hkk), dd);
  const double s = aa + ab;
  return ba * (ab / s) <= fmax(SMALL_NUM, EPS * (bb * (aa / s)));
}

// ---- window routine 1: lahqr on a whole window ------------------------------------------------------------------------------------
// One reflector of a QR step on the n x n window: rows k .. k + nr - 1. x is the generating vector; when from_column, column k - 1
// receives (beta, 0, 0).
template <class S>
SCH_HD inline void window_reflect(S* H, S* U, int ld, int n, int k, int nr, int last, S x0, S x1, S x2, bool from_column, int tid,
                                  int nt) {
  S beta;
  const Refl<S> r = make_reflector(nr, x0, x1, x2, &beta);
  SCH_SYNC();  // every thread has read x
  for (int j = k + tid; j < n; j += nt) {
    S z;
    set_real(z, 0.0);
    S* c = H + k + j * ld;
    refl_left(r, nr, c[0], c[1], nr == 3 ? c[2] : z);
  }
  if (from_column && tid == 0) {
    S* c = H + k + (k - 1) * ld;
    c[0] = beta;
    set_real(c[1], 0.0);
    if (nr == 3) set_real(c[2], 0.0);
  }
  SCH_SYNC();
  const int rmax = k + nr < last ? k + nr : last;  // the reflector's columns are nonzero down to row min(k + nr, last)
  for (int i = tid; i <= rmax; i += nt) {
    S z;
    set_real(z, 0.0);
    S* p = H + i + k * ld;
    refl_right(r, nr, p[0], p[ld], nr == 3 ? p[2 * ld] : z);
  }
  if (U)
    for (int i = tid; i < n; i += nt) {
      S z;
      set_real(z, 0.0);
      S* p = U + i + k * ld;
      refl_right(r, nr, p[0], p[ld], nr == 3 ? p[2 * ld] : z);
    }
  SCH_SYNC();
}

// Standardise the real 2 x 2 block at (i - 1, i - 1) of the window and apply its rotation to the rest of the window and to U
SCH_HD inline void window_schur22(double* H, double* U, int ld, int n, int i, int tid, int nt) {
  double a = H[(i - 1) + (i - 1) * ld], b = H[(i - 1) + i * ld], c = H[i + (i - 1) * ld], d = H[i + i * ld];
  double r1, i1, r2, i2, cs, sn;
  standardize22(a, b, c, d, r1, i1, r2, i2, cs, sn);
  SCH_SYNC();
  if (tid == 0) {
    H[(i - 1) + (i - 1) * ld] = a;
    H[(i - 1) + i * ld] = b;
    H[i + (i - 1) * ld] = c;
    H[i + i * ld] = d;
  }
  for (int j = i + 1 + tid; j < n; j += nt) {
    const double x = H[(i - 1) + j * ld], y = H[i + j * ld];
    H[(i - 1) + j * ld] = cs * x + sn * y;
    H[i + j * ld] = cs * y - sn * x;
  }
  for (int r = tid; r < i - 1; r += nt) {
    const double x = H[r + (i - 1) * ld], y = H[r + i * ld];
    H[r + (i - 1) * ld] = cs * x + sn * y;
    H[r + i * ld] = cs * y - sn * x;
  }
  if (U)
    for (int r = tid; r < n; r += nt) {
      const double x = U[r + (i - 1) * ld], y = U[r + i * ld];
      U[r + (i - 1) * ld] = cs * x + sn * y;
      U[r + i * ld] = cs * y - sn * x;
    }
  SCH_SYNC();
}
SCH_HD inline void window_schur22(Cx*, Cx*, int, int, int, int, int) {}

// the shifts of one lahqr iteration on the active block [l, i] (exceptional at iterations 10 and 20, as the reference)
SCH_HD inline void lahqr_shifts(const double* H, int ld, int l, int i, int its, double* sh) {
  double h11, h12, h21, h22;
  if (its == 10) {
    const double s = fabs(H[(l + 1) + l * ld]) + fabs(H[(l + 2) + (l + 1) * ld]);
    h11 = 0.75 * s + H[l + l * ld];
    h12 = -0.4375 * s;
    h21 = s;
    h22 = h11;
  } else if (its == 20) {
    const double s = fabs(H[i + (i - 1) * ld]) + fabs(H[(i - 1) + (i - 2) * ld]);
    h11 = 0.75 * s + H[i + i * ld];
    h12 = -0.4375 * s;
    h21 = s;
    h22 = h11;
  } else {
    h11 = H[(i - 1) + (i - 1) * ld];
    h21 = H[i + (i - 1) * ld];
    h12 = H[(i - 1) + i * ld];
    h22 = H[i + i * ld];
  }
  shifts22(h11, h12, h21, h22, sh[0], sh[1], sh[2], sh[3]);
}
SCH_HD inline void lahqr_shifts(const Cx* H, int ld, int l, int i, int its, Cx* sh) {
  if (its == 10)
    sh[0] = H[l + l * ld] + Cx{0.75 * absv(H[(l + 1) + l * ld]), 0.0};
  else if (its == 20)
    sh[0] = H[i + i * ld] + Cx{0.75 * absv(H[i + (i - 1) * ld]), 0.0};
  else
    sh[0] = wilkinson(H[(i - 1) + (i - 1) * ld], H[(i - 1) + i * ld], H[i + (i - 1) * ld], H[i + i * ld]);
}

// The n x n Hessenberg window H (leading dimension ld) <- its Schur form U^H H U, real 2 x 2 blocks in standard form; U (identity
// on entry, or null) accumulates the transformations. Every thread runs the same control flow on the same shared data. Returns the
// number of rows that did not deflate within the reference's iteration cap (0 = converged).
template <bool CX>
SCH_HD inline int window_qr(typename Num<CX>::T* H, typename Num<CX>::T* U, int ld, int n, int tid, int nt) {
  typedef typename Num<CX>::T S;
  constexpr int NR = Lim<CX>::NR;
  const int itmax = 30 * (n > 10 ? n : 10);
  int i = n - 1, its = 0, total = 0;
  SCH_SYNC();
  while (i >= 0) {
    int l = i;
    while (l > 0 && !negligible(H, ld, l, 0, n)) --l;
    SCH_SYNC();  // every thread has finished the scan before the subdiagonal is cleared
    if (l > 0 && tid == 0) set_real(H[l + (l - 1) * ld], 0.0);
    SCH_SYNC();
    if (l == i) {
      i = l - 1;
      its = 0;
      continue;
    }
    if (!CX && l == i - 1) {
      window_schur22(H, U, ld, n, i, tid, nt);
      i = l - 1;
      its = 0;
      continue;
    }
    if (total >= itmax) return i + 1;
    S sh[4];
    lahqr_shifts(H, ld, l, i, its, sh);
    ++its;
    ++total;
    for (int k = l; k < i; ++k) {
      const int nr = (i - k + 1 < NR) ? i - k + 1 : NR;
      S x0, x1, x2;
      set_real(x2, 0.0);
      if (k == l) {
        shift_column(H + l + l * ld, ld, sh, x0, x1, x2);
      } else {
        const S* c = H + k + (k - 1) * ld;
        x0 = c[0];
        x1 = c[1];
        if (nr == 3) x2 = c[2];
      }
      window_reflect(H, U, ld, n, k, nr, i, x0, x1, x2, k > l, tid, nt);
    }
  }
  return 0;
}

// ---- window routine 2: one stretch of a small-bulge multishift sweep -----------------------------------------------------------------
// A sweep over the active block [ilo, ihi) moves a chain of nb bulges, NR columns apart, from the top to the bottom in steps. At
// step t bulge j sits at column p = ilo - 1 + t - NR j: p = ilo - 1 introduces it from its shift pair, ilo <= p <= ihi - 3 moves it
// one row down by the reflector that clears column p below the subdiagonal, later steps have nothing left to do. The reflectors
// of one step act on disjoint rows and columns, so a step is: generate all, apply all from the left, apply all from the right.
struct Stretch {
  int ilo, ihi;  // the active block
  int w0, wn;    // the window [w0, w0 + wn) holds every row and column the steps touch
  int t0, t1;    // steps [t0, t1)
  int nb;        // bulges in the chain
};
template <bool CX>
SCH_HD inline int sweep_steps(int nh, int nb) { return nh - 1 + Lim<CX>::NR * (nb - 1); }
// the stretch that starts at step t0: as many steps as the window allows
template <bool CX>
SCH_HD inline Stretch plan_stretch(int ilo, int ihi, int nb, int t0) {
  constexpr int NR = Lim<CX>::NR, W = Lim<CX>::W;
  Stretch s;
  s.ilo = ilo;
  s.ihi = ihi;
  s.nb = nb;
  s.t0 = t0;
  const int last = ilo - 1 + t0 - NR * (nb - 1);  // column of the last bulge at t0
  s.w0 = last > ilo ? last : ilo;
  const int total = sweep_steps<CX>(ihi - ilo, nb);
  int t1 = s.w0 + W - ilo - NR;  // the lead bulge's fill row p + NR + 1 at step t1 - 1 stays inside the window
  if (s.w0 + W >= ihi || t1 > total) t1 = total;
  s.t1 = t1;
  const int hi = ilo + t1 + NR < ihi ? ilo + t1 + NR : ihi;
  s.wn = hi - s.w0;
  return s;
}

// H, U: the wn x wn window and its accumulated transformation (identity on entry); shifts: NS scalars per chain as shift_column
// takes them (4 doubles per real bulge, one complex per complex bulge); refl: scratch for nb reflectors.
template <bool CX>
SCH_HD inline void window_chase(typename Num<CX>::T* H, typename Num<CX>::T* U, int ld, const Stretch& s,
                                const typename Num<CX>::T* shifts, Refl<typename Num<CX>::T>* refl,
                                typename Num<CX>::T* beta, int tid, int nt) {
  typedef typename Num<CX>::T S;
  constexpr int NR = Lim<CX>::NR;
  const int wn = s.wn;
  SCH_SYNC();
  for (int t = s.t0; t < s.t1; ++t) {
    for (int j = tid; j < s.nb; j += nt) {
      const int p = s.ilo - 1 + t - NR * j;
      refl[j].tau = -1.0;  // not active at this step
      if (p < s.ilo - 1 || p > s.ihi - 3) continue;
      const int nr = (s.ihi - 1 - p < NR) ? s.ihi - 1 - p : NR;
      S x0, x1, x2;
      set_real(x2, 0.0);
      if (p == s.ilo - 1) {
        const int o = s.ilo - s.w0;
        shift_column(H + o + o * ld, ld, shifts + (CX ? 1 : 4) * j, x0, x1, x2);
      } else {
        const S* c = H + (p + 1 - s.w0) + (p - s.w0) * ld;
        x0 = c[0];
        x1 = c[1];
        if (nr == 3) x2 = c[2];
      }
      refl[j] = make_reflector(nr, x0, x1, x2, &beta[j]);
    }
    SCH_SYNC();
    for (int idx = tid; idx < wn * s.nb; idx += nt) {
      const int j = idx / wn, c = idx - j * wn;
      if (refl[j].tau < 0.0) continue;
      const int p = s.ilo - 1 + t - NR * j, col = s.w0 + c;
      const int nr = (s.ihi - 1 - p < NR) ? s.ihi - 1 - p : NR;
      S* a = H + (p + 1 - s.w0) + c * ld;
      S z;
      set_real(z, 0.0);
      if (col == p) {
        a[0] = beta[j];
        set_real(a[1], 0.0);
        if (nr == 3) set_real(a[2], 0.0);
      } else if (col > p) {
        refl_left(refl[j], nr, a[0], a[1], nr == 3 ? a[2] : z);
      }
    }
    SCH_SYNC();
    for (int idx = tid; idx < 2 * wn * s.nb; idx += nt) {
      const int j = idx / (2 * wn), q = idx - j * 2 * wn;
      if (refl[j].tau < 0.0) continue;
      const int p = s.ilo - 1 + t - NR * j;
      const int nr = (s.ihi - 1 - p < NR) ? s.ihi - 1 - p : NR;
      S z;
      set_real(z, 0.0);
      if (q < wn) {  // a row of H: nonzero down to the fill row p + nr + 1
        const int row = s.w0 + q;
        if (row > p + nr + 1 || row >= s.ihi) continue;
        S* a = H + q + (p + 1 - s.w0) * ld;
        refl_right(refl[j], nr, a[0], a[ld], nr == 3 ? a[2 * ld] : z);
      } else {
        S* a = U + (q - wn) + (p + 1 - s.w0) * ld;
        refl_right(refl[j], nr, a[0], a[ld], nr == 3 ? a[2 * ld] : z);
      }
    }
    SCH_SYNC();
  }
}

// ---- shifts of a sweep ---------------------------------------------------------------------------------------------------------
// E: the ns x ns trailing block of the active block after window_qr (eigenvalues on its diagonal blocks); out: the chain's shifts.
// Real shifts are paired two by two in diagonal order; one left over (only when window_qr stopped early) is used twice. Returns
// the number of bulges, always ns / 2 (ns for complex).
SCH_HD inline int pair_shifts(const double* E, int ld, int ns, double* out) {
  int nb = 0;
  double odd = 0.0;
  bool have_odd = false;
  for (int k = 0; k < ns; ++k) {
    if (k + 1 < ns && E[(k + 1) + k * ld] != 0.0) {
      const double re = E[k + k * ld], im = sqrt(fabs(E[k + (k + 1) * ld])) * sqrt(fabs(E[(k + 1) + k * ld]));
      double* o = out + 4 * nb++;
      o[0] = re;
      o[1] = im;
      o[2] = re;
      o[3] = -im;
      ++k;
    } else if (have_odd) {
      double* o = out + 4 * nb++;
      o[0] = odd;
      o[1] = 0.0;
      o[2] = E[k + k * ld];
      o[3] = 0.0;
      have_odd = false;
    } else {
      odd = E[k + k * ld];
      have_odd = true;
    }
  }
  if (have_odd && 2 * nb + 2 <= ns) {
    double* o = out + 4 * nb++;
    o[0] = o[2] = odd;
    o[1] = o[3] = 0.0;
  }
  return nb;
}
SCH_HD inline int pair_shifts(const Cx* E, int ld, int ns, Cx* out) {
  for (int k = 0; k < ns; ++k) out[k] = E[k + k * ld];
  return ns;
}
// Exceptional shifts of a sweep that follows 5 sweeps without a deflation (LAPACK dlaqr0 / zlaqr0): from the subdiagonal of the
// trailing block of H (the global matrix, leading dimension ld), active block ending at ihi.
SCH_HD inline int exceptional_shifts(const double* H, long long ld, int ihi, int ns, double* out) {
  int nb = 0;
  for (int i = ihi - 1; i >= ihi - ns + 1; i -= 2) {
    const double ss = fabs(H[i + (i - 1) * ld]) + fabs(H[(i - 1) + (i - 2) * ld]);
    const double aa = 0.75 * ss + H[i + i * ld];
    double* o = out + 4 * nb++;
    shifts22(aa, ss, -0.4375 * ss, aa, o[0], o[1], o[2], o[3]);
  }
  return nb;
}
SCH_HD inline int exceptional_shifts(const Cx* H, long long ld, int ihi, int ns, Cx* out) {
  for (int k = 0; k < ns; ++k) {
    const int i = ihi - 1 - k;
    out[k] = H[i + i * ld] + Cx{0.75 * abs1(H[i + (i - 1) * ld]), 0.0};
  }
  return ns;
}

// ---- the sweep driver ------------------------------------------------------------------------------------------------------------
// Ops supplies the steps on its side of the host / device boundary; shapes are host-known, and the only value that comes back
// per sweep is the next active block:
//   bool scan(int ihi, int* ilo, int* ihi_out)   clear negligible subdiagonals upwards from row ihi - 1, skip deflated 1 x 1 blocks;
//                                                 the bottom unreduced block [ilo, ihi_out) (ihi_out = 0: done); false: window_qr failed
//   void finish_block(int lo, int hi)             window_qr on H[lo:hi, lo:hi], then apply_u
//   void make_shifts(int ilo, int ihi, int ns, bool exceptional)   the chain's shifts from the trailing ns x ns block
//   void chase(const Stretch&)                    window_chase on the stretch's window, then apply_u
// Returns false when the reference's cap of 30 max(10, n) sweeps is reached.
template <bool CX, class Ops>
inline bool schur_drive(Ops& ops, int n, int ns_limit) {
  constexpr int W = Lim<CX>::W, NS = Lim<CX>::NS, PER = CX ? 1 : 2;
  int ns = ns_limit < NS ? ns_limit : NS;
  ns -= ns % PER;
  if (ns < PER) ns = PER;
  const long long itmax = 30ll * (n > 10 ? n : 10);
  int ihi = n, stall = 0, last_ihi = -1, last_ilo = -1;
  for (long long it = 0; it < itmax; ++it) {
    int ilo;
    if (!ops.scan(ihi, &ilo, &ihi)) return false;
    if (ihi == 0) return true;
    if (ihi - ilo <= W) {
      ops.finish_block(ilo, ihi);
      ihi = ilo;
      stall = 0;
      continue;
    }
    stall = (ihi == last_ihi && ilo == last_ilo) ? stall + 1 : 0;
    last_ihi = ihi;
    last_ilo = ilo;
    ops.make_shifts(ilo, ihi, ns, stall > 0 && stall % 6 == 5);
    const int nb = ns / PER;
    const int total = sweep_steps<CX>(ihi - ilo, nb);
    for (int t = 0; t < total;) {
      const Stretch s = plan_stretch<CX>(ilo, ihi, nb, t);
      ops.chase(s);
      t = s.t1;
    }
  }
  return false;
}

// ---- eigenvectors of the Schur form (evd/mod.rs:557-958) ---------------------------------------------------------------------------
// A strided view of T (or of its transpose reversed in both directions, for left eigenvectors) and of the matrix X of eigenvectors
template <class S>
struct MatV {
  S* p;
  long long rs, cs;
  SCH_HD S& operator()(long long i, long long j) const { return p[i * rs + j * cs]; }
};

// Real T, columns k0 (and k0 + 1 when T(k0 + 1, k0) != 0: a conjugate pair p +- i q) of X. The pair is one complex system
// (T00 - (p + i q)) (x_re + i x_im) = rhs solved by back substitution, x_re in column k0 and x_im in column k0 + 1
// (solve_cplx_shifted_upper_quasi_triangular_system, mod.rs:759-846); a real eigenvalue is the same with q = 0 and no
// imaginary column (mod.rs:670-725; the `x != 0` guard of 704 is kept). A shifted diagonal (block) smaller than eps * norm is
// replaced by eps * norm (mod.rs:701-703, 794-798, 828-832). b_re / b_im: 2 * (k0 + 2) scratch scalars.
SCH_HD inline void eigvec_real(MatV<const double> T, MatV<double> X, int n, int k0, double norm, double* b_re, double* b_im, int tid,
                               int nt) {
  const bool pair = k0 + 1 < n && T(k0 + 1, k0) != 0.0;
  const double p = T(k0, k0);
  double q = 0.0, d0 = 1.0, d1 = 0.0;
  int m = k0;  // rows of the system
  if (pair) {
    const double up = T(k0, k0 + 1), lo = T(k0 + 1, k0);
    q = sqrt(fabs(lo)) * sqrt(fabs(up));
    if (fabs(up) >= fabs(lo)) {
      d0 = 1.0;
      d1 = q / up;
    } else {
      d0 = -q / lo;
      d1 = 1.0;
    }
  }
  for (int i = tid; i < m; i += nt) {
    b_re[i] = -d0 * T(i, k0);
    b_im[i] = pair ? -d1 * T(i, k0 + 1) : 0.0;
  }
  if (tid == 0) {
    X(k0, k0) = d0;
    if (pair) {
      X(k0 + 1, k0 + 1) = d1;
      X(k0, k0 + 1) = 0.0;
      X(k0 + 1, k0) = 0.0;
    }
  }
  const double tiny = EPS * norm;
  int i = m;
  while (i > 0) {
    --i;
    SCH_SYNC();
    if (i == 0 || T(i, i - 1) == 0.0) {
      double z_re = T(i, i) - p, z_im = -q;
      double z = hypot(z_re, z_im);
      if (z < tiny) {
        z_re = tiny;
        z_im = 0.0;
        z = z_re;
      }
      double x_re = b_re[i], x_im = b_im[i];
      if (x_re != 0.0 || x_im != 0.0) {
        const double w_re = (z_re / z) / z, w_im = (-z_im / z) / z;
        const double r = x_re * w_re - x_im * w_im, s = x_re * w_im + x_im * w_re;
        x_re = r;
        x_im = s;
      }
      if (tid == 0) {
        X(i, k0) = x_re;
        if (pair) X(i, k0 + 1) = x_im;
      }
      for (int r = tid; r < i; r += nt) {
        const double t = T(r, i);
        b_re[r] -= t * x_re;
        b_im[r] -= t * x_im;
      }
    } else {
      const double a_re = T(i, i) - p, a_im = -q, b = T(i - 1, i), c = T(i, i - 1);
      const double r0_re = b_re[i - 1], r0_im = b_im[i - 1], r1_re = b_re[i], r1_im = b_im[i];
      double z_re = a_re * a_re - a_im * a_im - b * c, z_im = 2.0 * a_re * a_im;
      double z = hypot(z_re, z_im);
      if (z < tiny) {
        z_re = tiny;
        z_im = 0.0;
        z = z_re;
      }
      const double w_re = (z_re / z) / z, w_im = (-z_im / z) / z;
      const double x0_re = (a_re * r0_re - a_im * r0_im) - b * r1_re, x0_im = (a_re * r0_im + a_im * r0_re) - b * r1_im;
      const double x1_re = (a_re * r1_re - a_im * r1_im) - c * r0_re, x1_im = (a_re * r1_im + a_im * r1_re) - c * r0_im;
      const double y0_re = x0_re * w_re - x0_im * w_im, y0_im = x0_re * w_im + x0_im * w_re;
      const double y1_re = x1_re * w_re - x1_im * w_im, y1_im = x1_re * w_im + x1_im * w_re;
      if (tid == 0) {
        X(i - 1, k0) = y0_re;
        X(i, k0) = y1_re;
        if (pair) {
          X(i - 1, k0 + 1) = y0_im;
          X(i, k0 + 1) = y1_im;
        }
      }
      for (int r = tid; r < i - 1; r += nt) {
        const double t0 = T(r, i - 1), t1 = T(r, i);
        b_re[r] -= t0 * y0_re + t1 * y1_re;
        b_im[r] -= t0 * y0_im + t1 * y1_im;
      }
      --i;
    }
  }
}
// Complex T (conjugated entrywise when conj: the left eigenvectors' view), column k0 of X (mod.rs:622-669, 882-923)
SCH_HD inline void eigvec_cplx(MatV<const Cx> T, bool conj, MatV<Cx> X, int k0, double norm, Cx* b, int tid, int nt) {
  const Cx pk = conj ? conj_(T(k0, k0)) : T(k0, k0);
  for (int i = tid; i < k0; i += nt) b[i] = -(conj ? conj_(T(i, k0)) : T(i, k0));
  if (tid == 0) X(k0, k0) = Cx{1.0, 0.0};
  const double tiny = EPS * norm;
  for (int i = k0 - 1; i >= 0; --i) {
    SCH_SYNC();
    Cx z = (conj ? conj_(T(i, i)) : T(i, i)) - pk;
    if (absv(z) < tiny) z = Cx{tiny, 0.0};
    Cx x = b[i];
    if (!is_zero(x)) x = div_(x, z);
    if (tid == 0) X(i, k0) = x;
    for (int r = tid; r < i; r += nt) b[r] = b[r] - (conj ? conj_(T(r, i)) : T(r, i)) * x;
  }
}

}  // namespace sch
}  // namespace fb
