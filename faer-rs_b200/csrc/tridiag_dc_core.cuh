// Scalar building blocks of the divide-and-conquer eigensolver for symmetric tridiagonal matrices (tridiag_dc.cu), written
// as plain host/device functions so that the very same code is exercised on the CPU (tools/emul/tridiag_dc_host.cpp,
// tests/test_tridiag_dc_cpu.py) before it runs on a GPU.
//
// Replaces, together with tridiag_dc.cu: `evd::tridiag_evd::divide_and_conquer` (reference faer/src/linalg/evd/
// tridiag_evd.rs:270-665: Cuppen's rank-one tearing, deflation, secular equation, Gu-Eisenstat vector formation, merges as
// matmuls 595-598) and its small-size base case `qr_algorithm` (tridiag_evd.rs:8-268, implicit QL/QR sweeps).
//
// Conventions. A merge joins two solved halves: T = diag(T1, T2) + rho v v^T, v = (e_last ; sign(beta) e_first), after
// |beta| was subtracted from the two diagonal entries next to the tear. With T_i = Q_i D_i Q_i^T the merged problem is
// D + rho z z^T, z = (last row of Q_1 ; sign(beta) * first row of Q_2), normalised to |z| = 1 (rho doubles).
#pragma once
#include <cfloat>
#include <cmath>
#include <type_traits>

#ifdef __CUDACC__
#define FB_HD __host__ __device__ __forceinline__
#else
#define FB_HD inline
#endif

namespace fb {
namespace dc {

// Unit roundoff-scale tolerance and underflow threshold of the scalar type. The double-double kind (fx128) specialises this, and
// dc_sub below, in tridiag_dd.cuh; any other scalar type is rejected here.
template <class T>
struct DcLim {
  static_assert(std::is_same<T, float>::value || std::is_same<T, double>::value,
                "tridiag_dc_core.cuh: f32 / f64 only; the dd instantiation is in tridiag_dd.cuh");
  static FB_HD T eps() { return sizeof(T) == 8 ? (T)DBL_EPSILON : (T)FLT_EPSILON; }
  static FB_HD T tiny() { return sizeof(T) == 8 ? (T)DBL_MIN : (T)FLT_MIN; }
};
// a - b where the secular equation and the deflation need it to relative accuracy (differences of poles, and of a pole and a root).
// An IEEE subtraction is exact to half an ulp of the result; dd specialises it with dd_sub_accurate, because dd's own subtraction
// (faer's add(a, -b)) has an error of order 2^-106 |a| instead of 2^-106 |a - b|.
template <class T>
FB_HD T dc_sub(T a, T b) {
  return a - b;
}

// ---- implicit QL with Wilkinson shifts on a small tridiagonal block (EISPACK tql2 recurrences) -------------------------
// d[0..n): diagonal -> eigenvalues (unsorted); e[0..n): e[i] couples i and i+1 (e[n-1] unused / 0) -> destroyed.
// The rotations are reported through `rot(i, c, s)`: columns i and i+1 of the eigenvector matrix are to be updated as
//   f = z[k][i+1]; z[k][i+1] = s z[k][i] + c f; z[k][i] = c z[k][i] - s f      for every row k.
// Returns false if an eigenvalue needed more than 60 sweeps (does not happen for finite input).
template <class T, class Rot>
FB_HD bool ql_implicit(T* d, T* e, int n, Rot&& rot) {
  const T eps = DcLim<T>::eps();
  for (int l = 0; l < n; ++l) {
    int iter = 0;
    for (;;) {
      int m = l;
      for (; m < n - 1; ++m) {
        const T dd = fabs(d[m]) + fabs(d[m + 1]);
        if (fabs(e[m]) <= eps * dd) break;
      }
      if (m == l) break;
      if (++iter > 60) return false;
      T g = (d[l + 1] - d[l]) / (T(2) * e[l]);
      T r = hypot(g, T(1));
      g = d[m] - d[l] + e[l] / (g + (g >= T(0) ? fabs(r) : -fabs(r)));
      T s = T(1), c = T(1), p = T(0);
      int i = m - 1;
      for (; i >= l; --i) {
        T f = s * e[i];
        const T b = c * e[i];
        r = hypot(f, g);
        e[i + 1] = r;
        if (r == T(0)) {
          d[i + 1] -= p;
          e[m] = T(0);
          break;
        }
        s = f / r;
        c = g / r;
        g = d[i + 1] - p;
        r = (d[i] - g) * s + T(2) * c * b;
        p = s * r;
        d[i + 1] = g + p;
        g = c * r - b;
        rot(i, c, s);
      }
      if (r == T(0) && i >= l) continue;
      d[l] -= p;
      e[l] = g;
      e[m] = T(0);
    }
  }
  return true;
}

// ---- deflation scan of one merge (LAPACK dlaed2's logic) ---------------------------------------------------------------
// Input, in ascending order of d: d[0..s), z[0..s) (|z| = 1), col[0..s) = the eigenvector-matrix column each entry belongs to.
// Output:
//   k                       number of non-deflated entries
//   dl[0..k), w[0..k), cnd[0..k)   their d (ascending), z and column
//   dd[0..s-k), cdf[0..s-k)        deflated eigenvalues and their columns, in the order they were deflated
//   rot_a/rot_b/rot_c/rot_s[0..nrot)  Givens rotations (applied by the caller: columns a, b of Q, or rows a, b of the merge
//                                     matrix in reverse order): q_a' = c q_a + s q_b, q_b' = c q_b - s q_a
// `d` and `z` are modified. Returns k; *nrot_out = number of rotations.
template <class T>
FB_HD int deflate_scan(T* d, T* z, const int* col, int s, T rho, T* dl, T* w, int* cnd, T* dd, int* cdf, int* rot_a, int* rot_b,
                       T* rot_c, T* rot_s, int* nrot_out) {
  const T eps = DcLim<T>::eps();
  T dmax = T(0), zmax = T(0);
  for (int i = 0; i < s; ++i) {
    dmax = fmax(dmax, fabs(d[i]));
    zmax = fmax(zmax, fabs(z[i]));
  }
  const T tol = T(8) * eps * fmax(dmax, zmax);
  int k = 0, ndef = 0, nrot = 0;
  if (rho * zmax <= tol) {
    for (int i = 0; i < s; ++i) {
      dd[ndef] = d[i];
      cdf[ndef++] = col[i];
    }
    *nrot_out = 0;
    return 0;
  }
  int pj = -1;
  for (int j = 0; j < s; ++j) {
    if (rho * fabs(z[j]) <= tol) {
      dd[ndef] = d[j];
      cdf[ndef++] = col[j];
      continue;
    }
    if (pj < 0) {
      pj = j;
      continue;
    }
    T sn = z[pj], cs = z[j];
    const T tau = hypot(cs, sn);
    const T t = dc_sub(d[j], d[pj]);
    cs /= tau;
    sn = -sn / tau;
    if (fabs(t * cs * sn) <= tol) {
      // rotate pj into j: z[pj] becomes 0 and pj deflates
      z[j] = tau;
      z[pj] = T(0);
      rot_a[nrot] = col[pj];
      rot_b[nrot] = col[j];
      rot_c[nrot] = cs;
      rot_s[nrot] = sn;
      ++nrot;
      const T tt = d[pj] * cs * cs + d[j] * sn * sn;
      d[j] = d[pj] * sn * sn + d[j] * cs * cs;
      d[pj] = tt;
      dd[ndef] = d[pj];
      cdf[ndef++] = col[pj];
      pj = j;
    } else {
      dl[k] = d[pj];
      w[k] = z[pj];
      cnd[k++] = col[pj];
      pj = j;
    }
  }
  if (pj >= 0) {
    dl[k] = d[pj];
    w[k] = z[pj];
    cnd[k++] = col[pj];
  }
  *nrot_out = nrot;
  return k;
}

// ---- secular equation: root j of 1/rho + sum_i w_i^2 / (dl_i - lambda) = 0, dl ascending, rho > 0 ----------------------
// Returns tau and *org such that lambda_j = dl[*org] + tau with *org the nearer pole (j or j+1; k-1 for the last root), so
// that dl_i - lambda_j = (dl_i - dl[*org]) - tau is obtained without cancellation (what the vector formation needs).
// Safeguarded bisection on tau (geometric while the bracket spans more than a factor 4): the function is monotone between
// the poles, so the only stopping criterion is the bracket width, one ulp-level interval of tau.
// `ev(org, tau)` evaluates f at lambda = dl[org] + tau (the GPU passes a warp-cooperative sum, the CPU a plain loop);
// zz = sum_i w_i^2.
template <class T>
FB_HD T secular_f(const T* dl, const T* w, int k, int org, T tau, T rhoinv) {
  T f = rhoinv;
  const T dorg = dl[org];
  for (int i = 0; i < k; ++i) {
    const T del = dc_sub(dc_sub(dl[i], dorg), tau);
    f += w[i] * (w[i] / del);
  }
  return f;
}

template <class T, class Eval>
FB_HD T secular_root(const T* dl, int k, int j, T rho, T zz, Eval&& ev, int* org_out) {
  T lb, ub;
  int org;
  if (j < k - 1) {
    const T half = dc_sub(dl[j + 1], dl[j]) * T(0.5);
    const T fmid = ev(j, half);
    if (fmid > T(0)) {  // root in the left half: origin dl[j], tau in (0, half]
      org = j;
      lb = T(0);
      ub = half;
    } else {            // origin dl[j+1], tau in [-half, 0)
      org = j + 1;
      lb = -half;
      ub = T(0);
    }
  } else {
    org = k - 1;
    lb = T(0);
    ub = rho * zz;
    // f(ub) >= 0 in exact arithmetic; make sure of it numerically
    for (int it = 0; it < 8 && ev(org, ub) < T(0); ++it) ub *= T(2);
  }
  *org_out = org;
  // the open end of the bracket is a pole (tau = 0): move it inside, shrinking the ratio 2^-1, 2^-2, 2^-4, ...
  const T tiny = DcLim<T>::tiny();
  if (lb == T(0)) {
    T t = T(0), fac = T(0.5);
    for (int it = 0; it < 12; ++it) {
      const T c = ub * fac;
      if (!(c > tiny)) break;
      if (ev(org, c) < T(0)) {
        t = c;
        break;
      }
      ub = c;
      fac = fac * fac;
    }
    if (t == T(0)) return ub;  // the root is within `tiny` of the pole
    lb = t;
  } else if (ub == T(0)) {
    T t = T(0), fac = T(0.5);
    for (int it = 0; it < 12; ++it) {
      const T c = lb * fac;
      if (!(-c > tiny)) break;
      if (!(ev(org, c) < T(0))) {
        t = c;
        break;
      }
      lb = c;
      fac = fac * fac;
    }
    if (t == T(0)) return lb;
    ub = t;
  }
  // now lb, ub have the same sign, f(lb) < 0 <= f(ub)
  for (int it = 0; it < 200; ++it) {
    T mid;
    const T alb = fabs(lb), aub = fabs(ub);
    const T big = fmax(alb, aub), small = fmin(alb, aub);
    if (small > T(0) && big > T(4) * small) {
      mid = sqrt(alb) * sqrt(aub);
      if (lb < T(0)) mid = -mid;
    } else {
      mid = lb + (ub - lb) * T(0.5);
    }
    if (!(mid > lb) || !(mid < ub)) break;
    if (ev(org, mid) < T(0)) lb = mid;
    else ub = mid;
  }
  return lb + (ub - lb) * T(0.5);
}

}  // namespace dc
}  // namespace fb
