// The first-maximum rule of the pivot searches (colpiv_qr.cu, full_piv_lu.cu, lblt.cu) and the per-CTA argmax record of the
// persistent ones (full_piv_lu.cu, lblt.cu): every CTA publishes its first maximum, and after a grid barrier every CTA reduces the
// records in the same way, so all CTAs take the same pivot.
#pragma once
#include "common.cuh"

namespace fb {

// per-CTA argmax record: the score and an index whose order is the reference's scan order
template <class R>
struct alignas(16) FplRec {
  R score;
  long long idx;
};

// (v2, i2) beats (v1, i1): larger score, then, between equal POSITIVE scores, the smaller index. "None" is (0, the largest index)
// and a candidate must be > 0 to replace it, so the result is the first maximum in index order with strict `>` from 0 (a 0 or NaN
// score is never chosen), whatever the combination order.
template <class R, class I>
__device__ __forceinline__ bool better(R v2, I i2, R v1, I i1) {
  return v2 > v1 || (v2 == v1 && v1 > R(0) && i2 < i1);
}
template <class R>
__device__ __forceinline__ void fpl_warp_argmax(R& v, long long& i) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const R v2 = __shfl_xor_sync(0xffffffffu, v, off);
    const long long i2 = __shfl_xor_sync(0xffffffffu, i, off);
    if (better(v2, i2, v, i)) {
      v = v2;
      i = i2;
    }
  }
}
// this CTA's first maximum of (v, i) over its NWARPS warps into rec[blockIdx.x] (every thread of the CTA calls it; s_v / s_i:
// shared [NWARPS]). Contains one __syncthreads; the caller synchronises before s_v / s_i are written again.
template <int NWARPS, class R>
__device__ __forceinline__ void cta_publish(FplRec<R>* rec, R v, long long i, R* s_v, long long* s_i) {
  fpl_warp_argmax(v, i);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_v[warp] = v;
    s_i[warp] = i;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < NWARPS; ++q)
      if (better(s_v[q], s_i[q], v, i)) {
        v = s_v[q];
        i = s_i[q];
      }
    rec[blockIdx.x].score = v;
    rec[blockIdx.x].idx = i;
  }
}

}  // namespace fb
