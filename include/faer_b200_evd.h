/*
 * faer_b200_evd.h — general (non-symmetric) eigendecomposition (faer-ffi's `evd` family) of libfaer_b200.so. Included by
 * faer_b200.h; same conventions (host or device pointers, synchronous calls, abort() on precondition violations). The prototypes
 * are faer.h's, compared with it by tests/test_evd_cabi_cpu.py (tests/golden/faer_ffi_evd_prototypes.json).
 */
#ifndef LIBFAER_B200_EVD_H
#define LIBFAER_B200_EVD_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- parameter types: faer.h:106-108 (EvdFromSchurParams), 115-120 (SchurParams), 122-126 (EvdParams); HessenbergParams and
 * EvdStatus are in faer_b200.h. The two function pointers of SchurParams are host callbacks and are called on the host. ---- */
typedef struct FaerV0_24_EvdFromSchurParams {
  size_t recursion_threshold;
} FaerV0_24_EvdFromSchurParams;
typedef struct FaerV0_24_SchurParams {
  size_t (*recommended_shift_count)(size_t matrix_dimension, size_t active_block_dimension);
  size_t (*recommended_deflation_window)(size_t matrix_dimension, size_t active_block_dimension);
  size_t blocking_threshold;
  size_t nibble_threshold;
} FaerV0_24_SchurParams;
typedef struct FaerV0_24_EvdParams {
  struct FaerV0_24_HessenbergParams hessenberg;
  struct FaerV0_24_SchurParams schur;
  struct FaerV0_24_EvdFromSchurParams evd_from_schur;
} FaerV0_24_EvdParams;

/* Defaults of the reference (evd/mod.rs:74-81, evd/schur/mod.rs:26-107): recursion_threshold 64; the reference's shift-count and
 * deflation-window tables, blocking_threshold 75, nibble_threshold 50. faer.h:520-528, 532-540, 676-684. */
struct FaerV0_24_EvdFromSchurParams libfaer_v0_23_EvdFromSchurParams_c32(void);
struct FaerV0_24_EvdFromSchurParams libfaer_v0_23_EvdFromSchurParams_c64(void);
struct FaerV0_24_EvdFromSchurParams libfaer_v0_23_EvdFromSchurParams_f32(void);
struct FaerV0_24_EvdFromSchurParams libfaer_v0_23_EvdFromSchurParams_f64(void);
struct FaerV0_24_EvdParams libfaer_v0_23_EvdParams_c32(void);
struct FaerV0_24_EvdParams libfaer_v0_23_EvdParams_c64(void);
struct FaerV0_24_EvdParams libfaer_v0_23_EvdParams_f32(void);
struct FaerV0_24_EvdParams libfaer_v0_23_EvdParams_f64(void);
struct FaerV0_24_SchurParams libfaer_v0_23_SchurParams_c32(void);
struct FaerV0_24_SchurParams libfaer_v0_23_SchurParams_c64(void);
struct FaerV0_24_SchurParams libfaer_v0_23_SchurParams_f32(void);
struct FaerV0_24_SchurParams libfaer_v0_23_SchurParams_f64(void);

/* A = UR diag(S) UR^-1, UL^H A = diag(S) UL^H (csrc/schur.cu). faer-ffi/src/lib.rs:2402-2457, faer.h:2036-2118; the algorithm
 * is faer/src/linalg/evd/mod.rs:1007-1246.
 *   - UL / UR with ncols == 0: not computed; otherwise n x n. S (and S_im for the real kinds) have n entries and a positive stride.
 *   - real kinds: eigenvalue k is S[k] + i S_im[k]; a conjugate pair sits at k, k + 1 with S_im[k] > 0 = -S_im[k + 1], and its
 *     eigenvectors are column k +- i column k + 1. Complex kinds: S only, S_im is ignored.
 *   - a non-finite entry in A returns NoConvergence and writes nothing; so does reaching the reference's cap of 30 max(10, n)
 *     sweeps (outputs then hold no result). A is never written. Eigenvectors are not normalised (the reference does not either).
 *   - params: schur.recommended_shift_count(n, n), when not null, is an upper bound on the shifts of a sweep (32 real, 16
 *     complex fit the kernels). hessenberg, schur.recommended_deflation_window, schur.blocking_threshold,
 *     schur.nibble_threshold and evd_from_schur are accepted and ignored (no aggressive early deflation, no recursion);
 *     `par` and `mem` are ignored.
 *   - evd_scratch returns the size of the working copy of A; the work areas live in the library's device pool. */
struct FaerV0_24_EvdStatus libfaer_v0_23_evd_c32(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut UL, struct FaerV0_24_MatMut UR, struct FaerV0_24_VecMut S, struct FaerV0_24_VecMut S_im, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_EvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_evd_c64(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut UL, struct FaerV0_24_MatMut UR, struct FaerV0_24_VecMut S, struct FaerV0_24_VecMut S_im, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_EvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_evd_f32(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut UL, struct FaerV0_24_MatMut UR, struct FaerV0_24_VecMut S, struct FaerV0_24_VecMut S_im, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_EvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_evd_f64(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut UL, struct FaerV0_24_MatMut UR, struct FaerV0_24_VecMut S, struct FaerV0_24_VecMut S_im, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_EvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_evd_scratch_c32(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_left, enum FaerV0_24_ComputeEigenvectors compute_right, struct FaerV0_24_Par par, struct FaerV0_24_EvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_evd_scratch_c64(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_left, enum FaerV0_24_ComputeEigenvectors compute_right, struct FaerV0_24_Par par, struct FaerV0_24_EvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_evd_scratch_f32(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_left, enum FaerV0_24_ComputeEigenvectors compute_right, struct FaerV0_24_Par par, struct FaerV0_24_EvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_evd_scratch_f64(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_left, enum FaerV0_24_ComputeEigenvectors compute_right, struct FaerV0_24_Par par, struct FaerV0_24_EvdParams params);

/* extension: out[0] = sweeps, out[1] = chased windows of the last evd call of this process (tools/time_evd.py) */
void faer_b200_evd_last_sweep_counts(long long* out);

#ifdef __cplusplus
}
#endif

#endif /* LIBFAER_B200_EVD_H */
