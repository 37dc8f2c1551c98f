// Row interchanges, permuted gathers and strided copies shared by the pivoted factorizations (piv_llt.cu, lblt.cu, colpiv_qr.cu,
// full_piv_lu.cu), for every scalar kind <R, complex?>. The kernels and these launchers are defined in piv_llt.cu (explicitly
// instantiated for the four kinds); the files launch the kernels only through these functions. Views in element units of the kind
// (complex: COMPLEX units on an R* base), index arrays int64 on the DEVICE. Each call is one launch on `st`.
#pragma once
#include "common.cuh"

namespace fb {

// blocks of 256 threads that cover `elems` threads of a 1-D launch
inline unsigned grid_1d(i64 elems) { return (unsigned)((elems + 255) / 256); }

// rows t and hist[t] swapped, for t = k .. k + nt - 1 in order, over columns 0..k of A
template <class R, bool CX>
void piv_laswp_t(cudaStream_t st, View<R> A, i64 k, i64 nt, const long long* hist);
// dst[i, :] = src[perm[i], :]
template <class R, bool CX>
void piv_gather_rows_t(cudaStream_t st, View<R> dst, View<const R> src, const long long* perm);
// out(i, j), i >= j: tmp(p[i], p[j]) if p[i] >= p[j], else conj(tmp(p[j], p[i])) (tmp: column-major, leading dimension ld, only
// its lower triangle is read); only the lower triangle of out is written
template <class R, bool CX>
void piv_sym_gather_t(cudaStream_t st, View<R> out, const R* tmp, i64 ld, const long long* p);
// dst = src (same shape)
template <class R, bool CX>
void piv_copy_t(cudaStream_t st, View<R> dst, View<const R> src);

}  // namespace fb
