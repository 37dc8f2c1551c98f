// The per-CTA argmax record of the persistent pivot-search kernels (full_piv_lu.cu, lblt.cu): every CTA publishes its first
// maximum, and after a grid barrier every CTA reduces the records in the same way, so all CTAs take the same pivot.
#pragma once
#include "common.cuh"

namespace fb {

// per-CTA argmax record: the score and an index whose order is the reference's scan order
template <class R>
struct alignas(16) FplRec {
  R score;
  long long idx;
};

// (v2, i2) beats (v1, i1): larger score, then, between equal POSITIVE scores, the smaller index. "None" is (0, LLONG_MAX) and a
// candidate must be > 0 to replace it, so the result is the first maximum in index order with strict `>` from 0 (a 0 or NaN
// score is never chosen), whatever the combination order.
template <class R>
__device__ __forceinline__ bool fpl_better(R v2, long long i2, R v1, long long i1) {
  return v2 > v1 || (v2 == v1 && v1 > R(0) && i2 < i1);
}
template <class R>
__device__ __forceinline__ void fpl_warp_argmax(R& v, long long& i) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const R v2 = __shfl_xor_sync(0xffffffffu, v, off);
    const long long i2 = __shfl_xor_sync(0xffffffffu, i, off);
    if (fpl_better(v2, i2, v, i)) {
      v = v2;
      i = i2;
    }
  }
}

}  // namespace fb
