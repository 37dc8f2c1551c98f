/*
 * faer_b200_piv_llt.h — pivoted Cholesky (faer-ffi's `piv_llt_*` family) of libfaer_b200.so. Included by faer_b200.h; same
 * conventions (host or device pointers, synchronous calls, abort() on precondition violations). The prototypes are faer.h's,
 * compared with it by tests/test_piv_llt_cabi_cpu.py (tests/golden/faer_ffi_piv_llt_prototypes.json).
 */
#ifndef LIBFAER_B200_PIV_LLT_H
#define LIBFAER_B200_PIV_LLT_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- pivoted LLT: faer-ffi/src/lib.rs (PivLltParams, PivLltStatus), faer.h:178-180, 432-453 ---- */
typedef struct FaerV0_24_PivLltParams { size_t block_size; } FaerV0_24_PivLltParams;
typedef enum FaerV0_24_PivLltStatus_Tag { FaerV0_24_PivLltStatus_Ok, FaerV0_24_PivLltStatus_NonPositivePivot, FaerV0_24_PivLltStatus_Unknown } FaerV0_24_PivLltStatus_Tag;
typedef struct FaerV0_24_PivLltStatus_FaerV0_24_Ok_Body { size_t rank; size_t transposition_count; } FaerV0_24_PivLltStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_PivLltStatus_FaerV0_24_NonPositivePivot_Body { size_t index; } FaerV0_24_PivLltStatus_FaerV0_24_NonPositivePivot_Body;
typedef struct FaerV0_24_PivLltStatus {
  FaerV0_24_PivLltStatus_Tag tag;
  union {
    FaerV0_24_PivLltStatus_FaerV0_24_Ok_Body ok;
    FaerV0_24_PivLltStatus_FaerV0_24_NonPositivePivot_Body non_positive_pivot;
  };
} FaerV0_24_PivLltStatus;

/* pivoted Cholesky P A P^T = L L^H of a positive semi-definite matrix (lower triangle read and written; csrc/piv_llt.cu).
 * faer-ffi/src/lib.rs:1076-1186 (piv_llt_*), faer.h:652-662 (PivLltParams_<T>), 5058-5520; the algorithm is
 * faer/src/linalg/cholesky/llt_pivoting/{factor.rs:47-199, solve.rs:13-41, reconstruct.rs:12-52, inverse.rs:12-54}.
 *   - PivLltParams_<T>() = {128}, the reference default. block_size == 0 aborts (the reference would not terminate); block
 *     sizes above 256 (the widest panel the GPU kernel takes) are clamped to 256, which changes results only through rounding.
 *   - factor: status, rank, transposition_count and perm_fwd / perm_bwd follow the reference exactly (same pivot sequence:
 *     first maximum of the residual diagonal, strict `>`; rank exit when the largest residual is below eps * n * max a_ii).
 *     Ok { rank, transposition_count }: columns 0..rank of the lower triangle hold L; after a rank exit (rank < n) a(rank, rank)
 *     holds the residual that ended the factorization and the rest of the lower triangle outside columns 0..rank is unspecified.
 *     NonPositivePivot { index }: index 0 for a negative or NaN diagonal entry (A untouched), j for a NaN residual at column j;
 *     perm_fwd then holds the identity with the swaps made so far, perm_bwd is unspecified, A is unspecified (index > 0).
 *     The strict upper triangle is never read or written.
 *   - solve: rhs <- A^-1 rhs (A_conj: conj(A)^-1 rhs); reconstruct / inverse: the lower triangle of A (A^-1) from the factor,
 *     the strict upper triangle of the output untouched.
 *   - permutation lengths come from A.nrows / L.nrows, never from the slices' `len` (as for the LU); `par` and `mem` are ignored. */
struct FaerV0_24_PivLltParams libfaer_v0_23_PivLltParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u32_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u32_f64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u64_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u64_f64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_PivLltParams libfaer_v0_23_PivLltParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u32_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u32_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u32_f32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u64_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u64_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u64_f32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_PivLltParams libfaer_v0_23_PivLltParams_c64(void);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u32_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u32_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u32_c64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u64_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u64_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u64_c64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_PivLltParams libfaer_v0_23_PivLltParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u32_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u32_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u32_c32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_factor_in_place_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_PivLltStatus libfaer_v0_23_piv_llt_factor_in_place_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PivLltParams params);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_solve_in_place_scratch_u64_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_solve_in_place_u64_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_reconstruct_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_reconstruct_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_piv_llt_inverse_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_piv_llt_inverse_u64_c32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

#ifdef __cplusplus
}
#endif
#endif /* LIBFAER_B200_PIV_LLT_H */
