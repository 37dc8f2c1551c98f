// Double-double scalar `dd` (faer's fx128, `qd::Quad`): value = hi + lo, 16 bytes, {hi, lo} in memory. The complex kind cx128 is
// two of them, {re.hi, re.lo, im.hi, im.lo}, and is handled as the scalar kind <dd, true> (complex views in complex units on a dd*
// base), the same convention as c64 on double*.
//
// Operations (faer-traits/src/lib.rs, the fx128 impl; the algorithms are Dekker's and Knuth's):
//   add      two_sum of the high parts, the low parts added to the error, one quick_two_sum ("sloppy" add; faer's add_estimate)
//   sub      add(a, -b), as faer's SIMD loops do (DESIGN.md §7: sub_accurate below is used inside sqrt's Newton step and for the
//            differences the dd divide and conquer needs to relative accuracy, evd_dd.cu)
//   mul      FMA two_prod of the high parts, the cross products added to the error, one quick_two_sum
//   div      one correction step from hi / hi;  recip: 0 when |hi| is infinite, 1 / x otherwise
//   sqrt     one Newton step from 1 / sqrt(hi);  abs: sign flip when hi < 0;  comparisons: lexicographic on (hi, lo)
// Every FP64 step is an explicit round-to-nearest operation, so nvcc can neither contract nor reassociate it. The host build
// (plain C++ with -ffp-contract=off, tools/emul/dd_host.cpp) performs the same operations; tests/test_dd_ops_cpu.py checks that it
// reproduces the reference's quad.hpp bit for bit (tests/golden/dd_ops.npz).
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define DD_HD __host__ __device__ __forceinline__
#else
#define DD_HD inline
#endif

namespace fb {

// the dd overloads below must not hide the double ones from unqualified calls inside namespace fb
using ::fabs;
using ::sqrt;
#if !defined(__CUDACC__)
using std::isfinite;
using std::isinf;
using std::isnan;
#endif

#if defined(__CUDA_ARCH__)
DD_HD double dd_add_(double a, double b) { return __dadd_rn(a, b); }
DD_HD double dd_sub_(double a, double b) { return __dsub_rn(a, b); }
DD_HD double dd_mul_(double a, double b) { return __dmul_rn(a, b); }
DD_HD double dd_div_(double a, double b) { return __ddiv_rn(a, b); }
DD_HD double dd_fma_(double a, double b, double c) { return __fma_rn(a, b, c); }
DD_HD double dd_sqrt_(double a) { return __dsqrt_rn(a); }
#else
DD_HD double dd_add_(double a, double b) { return a + b; }
DD_HD double dd_sub_(double a, double b) { return a - b; }
DD_HD double dd_mul_(double a, double b) { return a * b; }
DD_HD double dd_div_(double a, double b) { return a / b; }
DD_HD double dd_fma_(double a, double b, double c) { return std::fma(a, b, c); }
DD_HD double dd_sqrt_(double a) { return std::sqrt(a); }
#endif

struct alignas(16) dd {
  double hi, lo;
  dd() = default;
  DD_HD constexpr dd(double h, double l) : hi(h), lo(l) {}
  DD_HD constexpr explicit dd(double h) : hi(h), lo(0.0) {}
  DD_HD constexpr explicit dd(int h) : hi((double)h), lo(0.0) {}
};

// s + e = a + b exactly (Knuth)
DD_HD double dd_two_sum(double a, double b, double& e) {
  const double s = dd_add_(a, b);
  const double bb = dd_sub_(s, a);
  e = dd_add_(dd_sub_(a, dd_sub_(s, bb)), dd_sub_(b, bb));
  return s;
}
// s + e = a - b exactly
DD_HD double dd_two_diff(double a, double b, double& e) {
  const double s = dd_sub_(a, b);
  const double bb = dd_sub_(s, a);
  e = dd_sub_(dd_sub_(a, dd_sub_(s, bb)), dd_add_(b, bb));
  return s;
}
// s + e = a + b exactly when |a| >= |b| (Dekker)
DD_HD double dd_quick_two_sum(double a, double b, double& e) {
  const double s = dd_add_(a, b);
  e = dd_sub_(b, dd_sub_(s, a));
  return s;
}

DD_HD dd operator-(dd a) { return dd(-a.hi, -a.lo); }
DD_HD dd operator+(dd a, dd b) {
  double e;
  double s = dd_two_sum(a.hi, b.hi, e);
  e = dd_add_(e, dd_add_(a.lo, b.lo));
  s = dd_quick_two_sum(s, e, e);
  return dd(s, e);
}
DD_HD dd operator-(dd a, dd b) { return a + (-b); }
DD_HD dd operator*(dd a, dd b) {
  const double p = dd_mul_(a.hi, b.hi);
  double e = dd_fma_(a.hi, b.hi, -p);
  e = dd_add_(e, dd_add_(dd_mul_(a.hi, b.lo), dd_mul_(a.lo, b.hi)));
  double s = dd_quick_two_sum(p, e, e);
  return dd(s, e);
}
// a - b with both limbs' errors kept (two two_diffs); used only by sqrt's Newton step
DD_HD dd dd_sub_accurate(dd a, dd b) {
  double s2, t2;
  double s1 = dd_two_diff(a.hi, b.hi, s2);
  const double t1 = dd_two_diff(a.lo, b.lo, t2);
  s2 = dd_add_(s2, t1);
  s1 = dd_quick_two_sum(s1, s2, s2);
  s2 = dd_add_(s2, t2);
  s1 = dd_quick_two_sum(s1, s2, s2);
  return dd(s1, s2);
}
DD_HD dd operator/(dd a, dd b) {
  const double q1 = dd_div_(a.hi, b.hi);
  const dd r = b * dd(q1);
  double s2;
  const double s1 = dd_two_diff(a.hi, r.hi, s2);
  s2 = dd_sub_(s2, r.lo);
  s2 = dd_add_(s2, a.lo);
  const double q2 = dd_div_(dd_add_(s1, s2), b.hi);
  double e;
  const double q = dd_quick_two_sum(q1, q2, e);
  return dd(q, e);
}

DD_HD dd& operator+=(dd& a, dd b) { return a = a + b; }
DD_HD dd& operator-=(dd& a, dd b) { return a = a - b; }
DD_HD dd& operator*=(dd& a, dd b) { return a = a * b; }
DD_HD dd& operator/=(dd& a, dd b) { return a = a / b; }

DD_HD bool operator==(dd a, dd b) { return a.hi == b.hi && a.lo == b.lo; }
DD_HD bool operator!=(dd a, dd b) { return !(a == b); }
DD_HD bool operator<(dd a, dd b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); }
DD_HD bool operator>(dd a, dd b) { return b < a; }
DD_HD bool operator<=(dd a, dd b) { return a.hi < b.hi || (a.hi == b.hi && a.lo <= b.lo); }
DD_HD bool operator>=(dd a, dd b) { return b <= a; }

DD_HD dd fabs(dd a) { return a.hi < 0.0 ? -a : a; }
DD_HD bool dd_is_finite(dd a) { return isfinite(a.hi) && isfinite(a.lo); }
// faer's recip for fx128: 0 when |hi| is infinite, 1 / x otherwise
DD_HD dd dd_recip(dd x) { return isinf(x.hi) ? dd(0.0, 0.0) : dd(1.0) / x; }
DD_HD dd sqrt(dd a) {
  if (a.hi == 0.0) return dd(0.0, 0.0);
  if (a.hi < 0.0) return dd(NAN, NAN);
  if (isinf(a.hi)) return dd(INFINITY, INFINITY);
  const double x = dd_div_(1.0, dd_sqrt_(a.hi));
  const dd ax(dd_mul_(a.hi, x));
  return ax + dd_sub_accurate(a, ax * ax) * dd(dd_mul_(x, 0.5));
}
// faer's mul_add for fx128: add(mul(a, b), acc)
DD_HD dd dd_mul_add(dd a, dd b, dd acc) { return a * b + acc; }

// fx128's real-field constants (faer-traits/src/lib.rs, the RealField impl for fx128): MIN_POSITIVE = (f64::MIN_POSITIVE, 0),
// sqrt_min_positive / sqrt_max_positive = sqrt(MIN_POSITIVE) / sqrt(recip(MIN_POSITIVE)), eps = Quad::EPSILON * 8 (both limbs
// scaled). Quad::EPSILON comes from the `qd` crate, whose source is not part of the reference; its value is the double-double
// unit roundoff 2^-104, so eps = 2^-101 here. The rank test is its only user and only its magnitude matters there.
DD_HD dd dd_min_positive() { return dd(2.2250738585072014e-308); }
DD_HD dd dd_sqrt_min_positive() { return sqrt(dd_min_positive()); }
DD_HD dd dd_sqrt_max_positive() { return sqrt(dd_recip(dd_min_positive())); }
DD_HD dd dd_eps() { return dd(0x1p-101); }
DD_HD dd dd_infinity() { return dd(INFINITY); }

// faer's abs_impl (faer-traits/src/lib.rs:337-352) in dd arithmetic: sqrt(re^2 + im^2) with the operands scaled by
// sqrt_min_positive or sqrt_max_positive when they are large or small. It is the modulus of a cx128 value and, as
// math_utils::hypot, fx128's hypot (lib.rs:163-165).
DD_HD dd dd_abs_impl(dd re, dd im) {
  const dd small = dd_sqrt_min_positive(), big = dd_sqrt_max_positive(), one(1.0);
  const dd ra = fabs(re), ia = fabs(im);
  if (ra > big || ia > big) {
    const dd r = re * small, i = im * small;
    return sqrt(r * r + i * i) * big;
  }
  if (ra > one || ia > one) return sqrt(re * re + im * im);
  const dd r = re * big, i = im * big;
  return sqrt(r * r + i * i) * small;
}
DD_HD dd dd_hypot(dd a, dd b) { return dd_abs_impl(a, b); }
// overloads under the libm names, so that scalar templates (tridiag_dc_core.cuh) instantiate for dd
using ::fmax;
using ::fmin;
using ::hypot;
DD_HD dd fmax(dd a, dd b) { return a < b ? b : a; }
DD_HD dd fmin(dd a, dd b) { return b < a ? b : a; }
DD_HD dd hypot(dd a, dd b) { return dd_hypot(a, b); }

#if defined(__CUDACC__)
__device__ __forceinline__ dd __ldcg(const dd* p) {
  const double2 v = ::__ldcg((const double2*)p);
  return dd(v.x, v.y);
}
#endif

// the complex double-double (cx128) arithmetic, faer's Complex<fx128>: (a.re b.re - a.im b.im, a.re b.im + a.im b.re), each
// product and sum a dd operation
struct cdd {
  dd re, im;
};
DD_HD cdd cdd_conj(cdd a) { return cdd{a.re, -a.im}; }
DD_HD cdd operator+(cdd a, cdd b) { return cdd{a.re + b.re, a.im + b.im}; }
DD_HD cdd operator-(cdd a) { return cdd{-a.re, -a.im}; }
DD_HD cdd operator*(cdd a, cdd b) { return cdd{a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }
DD_HD cdd cdd_scale(cdd a, dd s) { return cdd{a.re * s, a.im * s}; }
// |re| + |im| (faer's abs1 for cx128)
DD_HD dd cdd_abs1(cdd a) { return fabs(a.re) + fabs(a.im); }
// the modulus (faer's abs for cx128)
DD_HD dd cdd_abs(cdd a) { return dd_abs_impl(a.re, a.im); }
// faer's recip_impl (faer-traits/src/lib.rs:353-383) in dd arithmetic; small / big are fx128's sqrt_min_positive /
// sqrt_max_positive, the square roots of MIN_POSITIVE = (f64::MIN_POSITIVE, 0) and of its reciprocal
DD_HD cdd cdd_recip(cdd x) {
  const dd re = x.re, im = x.im;
  if (isnan(re.hi) || isnan(re.lo) || isnan(im.hi) || isnan(im.lo)) return cdd{dd(NAN, NAN), dd(NAN, NAN)};
  if (re == dd(0.0) && im == dd(0.0)) return cdd{dd(INFINITY, INFINITY), dd(INFINITY, INFINITY)};
  if (!dd_is_finite(re) || !dd_is_finite(im)) return cdd{dd(0.0), dd(0.0)};
  const dd mp(2.2250738585072014e-308);
  const dd small = sqrt(mp), big = sqrt(dd_recip(mp)), one(1.0);
  const dd ra = fabs(re), ia = fabs(im);
  if (ra > big || ia > big) {
    const dd r = re * small, i = im * small;
    const dd inv = dd_recip(r * r + i * i);
    return cdd{(r * inv) * small, (-i * inv) * small};
  }
  if (ra > one || ia > one) {
    const dd inv = dd_recip(re * re + im * im);
    return cdd{re * inv, -im * inv};
  }
  const dd r = re * big, i = im * big;
  const dd inv = dd_recip(r * r + i * i);
  return cdd{(r * inv) * big, (-i * inv) * big};
}
// 1 / x with x first scaled by an exact power of two that brings its larger part near 1. cdd_recip's scaling by sqrt_max_positive
// leaves |x|^-2 near MIN_POSITIVE when |x| <= 1 (and near the overflow threshold for |x| below about 2^-970), where the low limb
// falls into the subnormals and the result keeps only about 53 bits; here both limbs stay normal wherever the result can hold
// them. Zero, subnormal (the scale factor would overflow), non-finite and NaN inputs go to cdd_recip.
DD_HD cdd cdd_recip_scaled(cdd x) {
  const double mx = fmax(fabs(x.re.hi), fabs(x.im.hi));
  if (!(mx >= 0x1p-1022 && mx <= 0x1.fffffffffffffp+1023) || isnan(x.re.lo) || isnan(x.im.lo)) return cdd_recip(x);
  int e;
  frexp(mx, &e);
  const dd s(ldexp(1.0, -e));
  const dd re = x.re * s, im = x.im * s;
  const dd inv = dd_recip(re * re + im * im) * s;
  return cdd{re * inv, -(im * inv)};
}

}  // namespace fb
