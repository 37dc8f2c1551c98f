// A scalar of the kind <R, complex?> in device code: (re, im), im == 0 for the real types, with the arithmetic the pivoted
// factorizations (piv_llt.cu, colpiv_qr.cu, full_piv_lu.cu, lblt.cu) share.
//   * Functions templated on <R, CX> ignore the imaginary parts of a real kind's operands; the plain ones (cconj, csub, cscale,
//     cabs1, cabs2) compute with both parts whatever the kind. Each call site keeps the form its kernel was written with.
//   * Two rounding spellings, each kept where the reference's operation sequence needs it: the contractible form (*, +, fma)
//     and the `_rn` form, which rounds every product and sum as the reference's scalar code does.
#pragma once
#include "panel_common.cuh"

namespace fb {

template <class R>
struct Sc {
  R re, im;
};

// loads through L2 (the data may have been written by other CTAs of the same persistent kernel), and the matching store
template <class R, bool CX>
__device__ __forceinline__ Sc<R> sc_ld(const R* p) {
  return Sc<R>{__ldcg(p), CX ? __ldcg(p + 1) : R(0)};
}
template <class R, bool CX>
__device__ __forceinline__ void sc_st(R* p, Sc<R> v) {
  p[0] = v.re;
  if (CX) p[1] = v.im;
}

__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }

template <class R>
__device__ __forceinline__ Sc<R> cconj(Sc<R> a) { return Sc<R>{a.re, -a.im}; }
template <class R>
__device__ __forceinline__ Sc<R> csub(Sc<R> a, Sc<R> b) { return Sc<R>{a.re - b.re, a.im - b.im}; }
template <class R>
__device__ __forceinline__ Sc<R> cscale(Sc<R> a, R s) { return Sc<R>{a.re * s, a.im * s}; }
template <class R, bool CX>
__device__ __forceinline__ Sc<R> cadd(Sc<R> a, Sc<R> b) {
  return Sc<R>{a.re + b.re, CX ? a.im + b.im : R(0)};
}
template <class R, bool CX>
__device__ __forceinline__ Sc<R> scale(Sc<R> a, R s) {
  return Sc<R>{a.re * s, CX ? a.im * s : R(0)};
}

// a * b
template <class R, bool CX>
__device__ __forceinline__ Sc<R> cmul(Sc<R> a, Sc<R> b) {
  if (!CX) return Sc<R>{a.re * b.re, R(0)};
  return Sc<R>{a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}
template <class R, bool CX>
__device__ __forceinline__ Sc<R> cmul_rn(Sc<R> a, Sc<R> b) {
  if (!CX) return Sc<R>{mul_rn(a.re, b.re), R(0)};
  return Sc<R>{sub_rn(mul_rn(a.re, b.re), mul_rn(a.im, b.im)), add_rn(mul_rn(a.re, b.im), mul_rn(a.im, b.re))};
}
// acc + a * b, as FMAs
template <class R, bool CX>
__device__ __forceinline__ Sc<R> mul_add(Sc<R> a, Sc<R> b, Sc<R> acc) {
  acc.re = fma(a.re, b.re, acc.re);
  if (CX) {
    acc.re = fma(-a.im, b.im, acc.re);
    acc.im = fma(a.re, b.im, acc.im);
    acc.im = fma(a.im, b.re, acc.im);
  }
  return acc;
}
// acc + conj(a) * b, as FMAs
template <class R, bool CX>
__device__ __forceinline__ Sc<R> conj_mul_add(Sc<R> a, Sc<R> b, Sc<R> acc) {
  acc.re = fma(a.re, b.re, acc.re);
  if (CX) {
    acc.re = fma(a.im, b.im, acc.re);
    acc.im = fma(a.re, b.im, acc.im);
    acc.im = fma(-a.im, b.re, acc.im);
  }
  return acc;
}
// acc - a * conj(b), as FMAs
template <class R, bool CX>
__device__ __forceinline__ Sc<R> cfms_conj(Sc<R> acc, Sc<R> a, Sc<R> b) {
  acc.re = fma(-a.re, b.re, acc.re);
  if (CX) {
    acc.re = fma(-a.im, b.im, acc.re);
    acc.im = fma(a.re, b.im, acc.im);
    acc.im = fma(-a.im, b.re, acc.im);
  }
  return acc;
}

// |re| + |im|
template <class R>
__device__ __forceinline__ R cabs1(Sc<R> a) { return fabs(a.re) + fabs(a.im); }
template <class R, bool CX>
__device__ __forceinline__ R abs1_rn(Sc<R> a) {
  return CX ? add_rn(fabs(a.re), fabs(a.im)) : fabs(a.re);
}
// re^2 + im^2
template <class R>
__device__ __forceinline__ R cabs2(Sc<R> a) { return a.re * a.re + a.im * a.im; }
template <class R, bool CX>
__device__ __forceinline__ R abs2(Sc<R> a) {
  return CX ? a.re * a.re + a.im * a.im : a.re * a.re;
}
template <class R, bool CX>
__device__ __forceinline__ R cabs(Sc<R> a) { return CX ? hypot(a.re, a.im) : fabs(a.re); }

// 1 / x for the real types; faer's recip_impl (faer-traits/src/lib.rs:353-383) for the complex ones
template <class R, bool CX>
__device__ __forceinline__ Sc<R> recip_rn(Sc<R> x) {
  if (!CX) return Sc<R>{R(1) / x.re, R(0)};
  const R re = x.re, im = x.im;
  if (re != re || im != im) return Sc<R>{re + im, re + im};  // NaN
  if (re == R(0) && im == R(0)) return Sc<R>{TLim<R>::inf(), TLim<R>::inf()};
  if (!isfinite(re) || !isfinite(im)) return Sc<R>{R(0), R(0)};
  const R sml = TLim<R>::sqrt_min(), big = TLim<R>::sqrt_max();
  const R ra = fabs(re), ia = fabs(im);
  if (ra > big || ia > big) {
    const R a = mul_rn(re, sml), b = mul_rn(im, sml);
    const R inv = R(1) / add_rn(mul_rn(a, a), mul_rn(b, b));
    return Sc<R>{mul_rn(mul_rn(a, inv), sml), mul_rn(mul_rn(-b, inv), sml)};
  }
  if (ra > R(1) || ia > R(1)) {
    const R inv = R(1) / add_rn(mul_rn(re, re), mul_rn(im, im));
    return Sc<R>{mul_rn(re, inv), mul_rn(-im, inv)};
  }
  const R a = mul_rn(re, big), b = mul_rn(im, big);
  const R inv = R(1) / add_rn(mul_rn(a, a), mul_rn(b, b));
  return Sc<R>{mul_rn(mul_rn(a, inv), big), mul_rn(mul_rn(-b, inv), big)};
}

}  // namespace fb
