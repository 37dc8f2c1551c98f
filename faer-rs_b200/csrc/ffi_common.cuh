// Helpers shared by the translation units of the extern "C" boundary (ffi.cu, ffi_types.cu, ffi_dd.cu and the pivoted
// factorizations): staging of matrix arguments, scalar / permutation arguments that may live on the host or on the device, the
// end-of-call sequence of the staged matrices, the statuses, and the permutations and scratch layouts the pivoted families return.
#pragma once
#include "../../include/faer_b200.h"
#include "runtime.cuh"

#include <cstdint>
#include <cstring>
#include <initializer_list>
#include <utility>
#include <vector>

namespace fb {
// (static, not an anonymous namespace: nvcc's kernel stubs of a unit that also has a global anonymous namespace must stay unambiguous)

// bytes of one element of the scalar kind <R, complex?>
template <class R, bool CX>
static constexpr size_t elem_bytes() {
  return (CX ? 2 : 1) * sizeof(R);
}

// A matrix argument of the kind <R, CX> as a device view: inputs are copied in and never back, outputs are copied back (and in
// only with `copy_in`)
template <class R, bool CX>
static StagedMat stage(FaerV0_24_MatRef m, cudaStream_t st) {
  return StagedMat(m.ptr, (i64)m.nrows, (i64)m.ncols, (i64)m.row_stride, (i64)m.col_stride, elem_bytes<R, CX>(), true, false, st);
}
template <class R, bool CX>
static StagedMat stage(FaerV0_24_MatMut m, bool copy_in, cudaStream_t st) {
  return StagedMat(m.ptr, (i64)m.nrows, (i64)m.ncols, (i64)m.row_stride, (i64)m.col_stride, elem_bytes<R, CX>(), copy_in, true, st);
}

// one scalar of the kind <R, CX> (`CX ? 2 : 1` values of R) from a host or device pointer; real parameters (T::Real) are <R, false>
template <class R, bool CX = false>
static void read_scalar(const void* p, R* out) {
  FB_ASSERT(p != nullptr, "null scalar pointer");
  if (is_device_pointer(p)) FB_CUDA_CHECK(cudaMemcpy(out, p, elem_bytes<R, CX>(), cudaMemcpyDeviceToHost));
  else memcpy((void*)out, p, elem_bytes<R, CX>());
}

static inline void finish_all(cudaStream_t st, std::initializer_list<StagedMat*> mats) {
  // the compute must be complete before input mirrors return to the pool; calls are synchronous anyway
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  for (auto* m : mats) m->finish();
}

// the statuses of the entry points, from the drivers' results
static inline FaerV0_24_LltStatus llt_status(const LltResult& r) {
  FaerV0_24_LltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LltStatus_NonPositivePivot;
    out.non_positive_pivot.index = r.non_positive_pivot_index;
  }
  return out;
}
static inline FaerV0_24_LdltStatus ldlt_status(const LdltResult& r) {
  FaerV0_24_LdltStatus out;
  memset(&out, 0, sizeof(out));
  if (r.ok) {
    out.tag = FaerV0_24_LdltStatus_Ok;
    out.ok.dynamic_regularization_count = r.dynamic_regularization_count;
  } else {
    out.tag = FaerV0_24_LdltStatus_ZeroPivot;
    out.zero_pivot.index = r.zero_pivot_index;
  }
  return out;
}
static inline FaerV0_24_PartialPivLuStatus partial_piv_lu_status(size_t transposition_count) {
  FaerV0_24_PartialPivLuStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = FaerV0_24_PartialPivLuStatus_Ok;
  out.ok.transposition_count = transposition_count;
  return out;
}
// `negative_is_unknown`: a negative rank means QrStatus::Unknown; otherwise the rank is taken as it is
static inline FaerV0_24_QrStatus qr_status(i64 rank, bool negative_is_unknown) {
  FaerV0_24_QrStatus out;
  memset(&out, 0, sizeof(out));
  if (negative_is_unknown && rank < 0) {
    out.tag = FaerV0_24_QrStatus_Unknown;
  } else {
    out.tag = FaerV0_24_QrStatus_Ok;
    out.ok.rank = (size_t)rank;
  }
  return out;
}
static inline FaerV0_24_EvdStatus evd_status(bool ok) {
  FaerV0_24_EvdStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = ok ? FaerV0_24_EvdStatus_Ok : FaerV0_24_EvdStatus_NoConvergence;
  return out;
}
static inline FaerV0_24_SvdStatus svd_status(bool ok) {
  FaerV0_24_SvdStatus out;
  memset(&out, 0, sizeof(out));
  out.tag = ok ? FaerV0_24_SvdStatus_Ok : FaerV0_24_SvdStatus_NoConvergence;
  return out;
}

// index slices (u32 / u64) <-> host int64
static inline std::vector<long long> read_perm(const void* p, size_t n, int idx_bytes) {
  std::vector<unsigned char> raw(n * (size_t)idx_bytes);
  if (n) {
    if (is_device_pointer(p)) FB_CUDA_CHECK(cudaMemcpy(raw.data(), p, raw.size(), cudaMemcpyDeviceToHost));
    else memcpy(raw.data(), p, raw.size());
  }
  std::vector<long long> out(n);
  for (size_t i = 0; i < n; ++i)
    out[i] = idx_bytes == 4 ? (long long)((const uint32_t*)raw.data())[i] : (long long)((const uint64_t*)raw.data())[i];
  return out;
}
static inline void write_perm(void* dst, const std::vector<long long>& v, int idx_bytes) {
  if (v.empty()) return;
  std::vector<unsigned char> buf(v.size() * (size_t)idx_bytes);
  for (size_t i = 0; i < v.size(); ++i) {
    if (idx_bytes == 4) ((uint32_t*)buf.data())[i] = (uint32_t)v[i];
    else ((uint64_t*)buf.data())[i] = (uint64_t)v[i];
  }
  if (is_device_pointer(dst)) FB_CUDA_CHECK(cudaMemcpy(dst, buf.data(), buf.size(), cudaMemcpyHostToDevice));
  else memcpy(dst, buf.data(), buf.size());
}
// a permutation of `n` entries that the caller hands in (PermRef::new_unchecked(fwd, bwd, min(fwd.len, bwd.len)) in the
// reference; the length used is the matrix dimension, never the slice's `len`): a null slice or an entry outside [0, n) aborts
static inline std::vector<long long> read_perm_checked(FaerV0_24_SliceRef s, size_t n, int idx_bytes) {
  FB_ASSERT(n == 0 || s.ptr != nullptr, "null permutation slice");
  std::vector<long long> p = read_perm(s.ptr, n, idx_bytes);
  for (size_t i = 0; i < n; ++i) FB_ASSERT(p[i] >= 0 && (size_t)p[i] < n, "invalid permutation entry");
  return p;
}
// fwd: the identity of `len` entries with the transpositions (i, t[i]) made in order; bwd: its inverse
static inline void perm_from_transpositions(size_t len, const std::vector<long long>& t, std::vector<long long>& fwd,
                                            std::vector<long long>& bwd) {
  fwd.resize(len);
  bwd.resize(len);
  for (size_t i = 0; i < len; ++i) fwd[i] = (long long)i;
  for (size_t i = 0; i < t.size(); ++i) std::swap(fwd[i], fwd[(size_t)t[i]]);
  for (size_t i = 0; i < len; ++i) bwd[(size_t)fwd[i]] = (long long)i;
}

// partial-pivoting LU factor scratch: StackReq::new::<I>(min(nrows, ncols)) (lu/partial_pivoting/factor.rs:224-233)
static inline FaerV0_24_Layout lu_scratch(size_t nrows, size_t ncols, size_t idx_bytes) {
  size_t size = nrows < ncols ? nrows : ncols;
  return FaerV0_24_Layout{size * idx_bytes, idx_bytes};
}
// StackReq::and: the second request placed after the first at its alignment (dyn-stack's rule for equal alignments)
static inline FaerV0_24_Layout layout_and(FaerV0_24_Layout a, size_t b_bytes) {
  const size_t al = a.align_bytes > 64 ? a.align_bytes : 64;
  const size_t off = (a.len_bytes + 63) / 64 * 64;
  return FaerV0_24_Layout{off + b_bytes, al};
}
// the transposed view: "on the right" is the transposed sequence on the left of it (householder.rs:813-854)
inline FaerV0_24_MatMut transposed(FaerV0_24_MatMut m) {
  return FaerV0_24_MatMut{m.ptr, m.ncols, m.nrows, m.col_stride, m.row_stride};
}

}  // namespace fb
