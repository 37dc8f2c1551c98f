// Helpers shared by the cooperative "panel" kernels (QR panel, bidiagonalization, tridiagonalization): type-generic
// math spellings, numeric limits usable in device code, the grid-wide barrier, faer's scaled 2-norm accumulators
// (reductions/norm_l2.rs:18-44, 161-172) and the Householder scalars of householder.rs:59-107.
#pragma once
#include "common.cuh"

namespace fb {

__device__ __forceinline__ float t_hypot(float a, float b) { return hypotf(a, b); }
__device__ __forceinline__ double t_hypot(double a, double b) { return hypot(a, b); }
__device__ __forceinline__ float t_sqrt(float a) { return sqrtf(a); }
__device__ __forceinline__ double t_sqrt(double a) { return sqrt(a); }
__device__ __forceinline__ float t_abs(float a) { return fabsf(a); }
__device__ __forceinline__ double t_abs(double a) { return fabs(a); }
template <class T> struct TLim;
template <> struct TLim<float> {
  __device__ static float min_pos() { return 1.17549435e-38f; }
  __device__ static float eps() { return 1.1920929e-7f; }
  __device__ static float inf() { return __int_as_float(0x7f800000); }
  __device__ static float sqrt_min() { return 0x1p-63f; }  // sqrt_min_positive / sqrt_max_positive of faer's scaled norms
  __device__ static float sqrt_max() { return 0x1p63f; }
};
template <> struct TLim<double> {
  __device__ static double min_pos() { return 2.2250738585072014e-308; }
  __device__ static double eps() { return 2.220446049250313e-16; }
  __device__ static double inf() { return __longlong_as_double(0x7ff0000000000000ll); }
  __device__ static double sqrt_min() { return 0x1p-511; }
  __device__ static double sqrt_max() { return 0x1p511; }
};
// loads of data written by OTHER CTAs of the same (persistent) kernel must bypass the non-coherent L1
__device__ __forceinline__ float t_ldcg(const float* p) { return __ldcg(p); }
__device__ __forceinline__ double t_ldcg(const double* p) { return __ldcg(p); }

// Grid-wide barrier of a cooperative launch: `bar` counts arrivals monotonically, `target` = arrivals expected so far.
__device__ __forceinline__ void grid_barrier(unsigned long long* bar, unsigned long long target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1ull);
    while (*((volatile unsigned long long*)bar) < target) {
    }
    __threadfence();
  }
  __syncthreads();
}

// 16-byte vectors of T (float4 / double2) for record exchange through L2
template <class T> struct Vec16;
template <> struct Vec16<float> {
  typedef float4 type;
  static constexpr int N = 4;
  __device__ static __forceinline__ float4 zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ static __forceinline__ float get(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }
};
template <> struct Vec16<double> {
  typedef double2 type;
  static constexpr int N = 2;
  __device__ static __forceinline__ double2 zero() { return make_double2(0.0, 0.0); }
  __device__ static __forceinline__ double get(const double2& v, int e) { return e == 0 ? v.x : v.y; }
};

template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;  // xor butterfly: every lane ends with the same bits
}

constexpr int PANEL_NV = 8;  // stride of the per-CTA records published before a grid barrier

// CTA-wide fixed-order sum of NV per-thread values (NWARPS warps); thread v < NV stores the v-th sum to dst[v].
// fin: shared scratch [NWARPS][PANEL_NV]. Contains one __syncthreads; the caller's next barrier protects `fin`.
template <class T, int NV, int NWARPS>
__device__ __forceinline__ void block_publish_n(const T (&vals)[NV], T* fin, T* dst) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const T s = warp_sum(vals[v]);
    if (lane == 0) fin[warp * PANEL_NV + v] = s;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    T s = T(0);
    for (int w = 0; w < NWARPS; ++w) s += fin[w * PANEL_NV + threadIdx.x];
    dst[threadIdx.x] = s;
  }
}

// warp 0: out[v] = sum over the G CTAs of part[b][v] in a fixed order — identical bits in every CTA
template <class T, int NV>
__device__ __forceinline__ void reduce_partials(const T* part, int G, T (&out)[NV]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int v = 0; v < NV; ++v) out[v] = T(0);
  // 160 CTAs per round: five predicated records per lane, all loads issued before the first use (one L2 round trip
  // instead of five dependent ones)
  // (records are 16-byte aligned and read as 16-byte vectors: G^2 records cross the L2 per barrier grid-wide)
  typedef typename Vec16<T>::type V;
  constexpr int VEC = Vec16<T>::N, NVEC = (NV + VEC - 1) / VEC, RSTRIDE = PANEL_NV / VEC;
  const V* pv = reinterpret_cast<const V*>(part);
  for (int b0 = 0; b0 < G; b0 += 160) {
    V rec[5][NVEC];
#pragma unroll
    for (int u = 0; u < 5; ++u) {
      const int b = b0 + lane + 32 * u;
#pragma unroll
      for (int q = 0; q < NVEC; ++q) rec[u][q] = b < G ? __ldcg(&pv[(i64)b * RSTRIDE + q]) : Vec16<T>::zero();
    }
#pragma unroll
    for (int u = 0; u < 5; ++u) {
#pragma unroll
      for (int v = 0; v < NV; ++v) out[v] += Vec16<T>::get(rec[u][v / VEC], v % VEC);
    }
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) out[v] = warp_sum(out[v]);
}

__device__ __forceinline__ int pow2_ceil(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

// faer's overflow/underflow-safe 2-norm: three accumulators of (x*sml)^2, x^2, (x*big)^2 (norm_l2.rs:18-44) ...
template <class T>
struct NormAcc {
  T s, m, b;
  __device__ __forceinline__ void add(T x, T sml, T big) {
    const T xs = x * sml, xb = x * big;
    s = fma(xs, xs, s);
    m = fma(x, x, m);
    b = fma(xb, xb, b);
  }
};
// ... and the selection of norm_l2.rs:161-172
template <class T>
__device__ __forceinline__ T norm_from_acc(T a_sml, T a_med, T a_big, T sml, T big) {
  if (a_sml >= T(1)) return t_sqrt(a_sml) * big;
  if (a_med >= T(1)) return t_sqrt(a_med);
  return t_sqrt(a_big) * sml;
}

// make_householder_imp (householder.rs:59-107) on (head, |tail|): tau, 1/(head + sign*norm), the value stored in the head
template <class T>
struct HhScalars {
  T tau, inv, new_head;
  bool no_tail;
};
template <class T>
__device__ __forceinline__ HhScalars<T> make_householder_scalars(T head, T tail_norm) {
  const T min_pos = TLim<T>::min_pos();
  T head_norm = t_abs(head);
  if (head_norm < min_pos) {
    head = T(0);
    head_norm = T(0);
  }
  HhScalars<T> r;
  if (tail_norm < min_pos) {
    r.tau = TLim<T>::inf();
    r.inv = TLim<T>::inf();
    r.new_head = head;
    r.no_tail = true;
    return r;
  }
  const T norm = t_hypot(head_norm, tail_norm);
  const T sign = head_norm != T(0) ? head * (T(1) / head_norm) : T(1);
  const T signed_norm = sign * norm;
  r.inv = T(1) / (head + signed_norm);
  r.new_head = -signed_norm;
  const T tt = tail_norm * t_abs(r.inv);
  r.tau = T(0.5) * (T(1) + tt * tt);
  r.no_tail = false;
  return r;
}

}  // namespace fb
