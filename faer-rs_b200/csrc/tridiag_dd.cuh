// The double-double (fx128) instantiation of the tridiagonal and bidiagonal scalar cores: tridiag_dc_core.cuh (divide and
// conquer), tridiag_ev.cuh (bisection) and bidiag_sv.cuh (Golub-Kahan bisection) with fx128's eps and MIN_POSITIVE, and dc_sub as
// dd_sub_accurate. Every dd user of the cores includes this header (evd_dd.cu and svd_dd.cu on the GPU, tools/emul/tridiag_dd_host.cpp
// and tools/emul/bidiag_sv_dd_host.cpp on the CPU); without it, DcLim<dd> and the Lim<dd>s do not compile.
//
// dc_sub: dd's own a - b is faer's add(a, -b), whose error is of order 2^-106 max(|a|, |b|); the deflation and the secular
// equation need d_i - d_j and d_i - lambda_j to relative accuracy for gaps down to the 2^-98 deflation tolerance.
#pragma once
#include "bidiag_sv.cuh"
#include "dd.cuh"
#include "tridiag_dc_core.cuh"
#include "tridiag_ev.cuh"

namespace fb {
namespace dc {
template <>
struct DcLim<dd> {
  static FB_HD dd eps() { return dd_eps(); }
  static FB_HD dd tiny() { return dd_min_positive(); }
};
template <>
FB_HD dd dc_sub<dd>(dd a, dd b) {
  return dd_sub_accurate(a, b);
}
}  // namespace dc
namespace tev {
template <>
struct Lim<dd> {
  static FB_HD dd eps() { return dd_eps(); }
  static FB_HD dd safmin() { return dd_min_positive(); }
};
}  // namespace tev
namespace bsv {
template <>
struct Lim<dd> {
  static FB_HD dd eps() { return dd_eps(); }
  static FB_HD dd safmin() { return dd_min_positive(); }
};
}  // namespace bsv
}  // namespace fb
