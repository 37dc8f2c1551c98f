/*
 * faer_b200_full_piv_lu.h — full-pivoting LU (faer-ffi's `full_piv_lu_*` family) of libfaer_b200.so. Included by faer_b200.h;
 * same conventions (host or device pointers, synchronous calls, abort() on precondition violations). The prototypes are faer.h's,
 * compared with it by tests/test_full_piv_lu_cabi_cpu.py (tests/golden/faer_ffi_full_piv_lu_prototypes.json).
 */
#ifndef LIBFAER_B200_FULL_PIV_LU_H
#define LIBFAER_B200_FULL_PIV_LU_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- full-pivoting LU: faer-ffi/src/lib.rs (FullPivLuParams, FullPivLuStatus), faer.h:128-130, 287-301 ---- */
typedef struct FaerV0_24_FullPivLuParams { size_t par_threshold; } FaerV0_24_FullPivLuParams;
typedef enum FaerV0_24_FullPivLuStatus_Tag { FaerV0_24_FullPivLuStatus_Ok, FaerV0_24_FullPivLuStatus_Unknown } FaerV0_24_FullPivLuStatus_Tag;
typedef struct FaerV0_24_FullPivLuStatus_FaerV0_24_Ok_Body { size_t transposition_count; } FaerV0_24_FullPivLuStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_FullPivLuStatus {
  FaerV0_24_FullPivLuStatus_Tag tag;
  union {
    FaerV0_24_FullPivLuStatus_FaerV0_24_Ok_Body ok;
  };
} FaerV0_24_FullPivLuStatus;

/* full-pivoting LU P A Q = L U of an m x n matrix (csrc/full_piv_lu.cu). faer-ffi/src/lib.rs:2125-2325, faer.h:544-554 and
 * 2126-2970; the algorithm is faer/src/linalg/lu/full_pivoting/{factor.rs:321-538, solve.rs:21-93, reconstruct.rs:13-82,
 * inverse.rs:12-63}.
 *   - FullPivLuParams_<T>() = {256 * 512}, the reference default. `par`, `par_threshold` and `mem` are accepted and ignored.
 *   - factor: A is factored in place when |row_stride| < |col_stride|, otherwise A^T is (the reference's branch: the row of the
 *     working matrix is scaled instead of the column, and ties are broken in A's row-major order). The pivot is the first maximum
 *     of |re| + |im| in the working matrix's column-major order (strict `>`, so 0 and NaN are never chosen); the reference's SIMD
 *     search may pick another of several EXACTLY equal maxima. A maximum below the smallest normal number ends the elimination
 *     with identity transpositions. Seen from A: L unit-lower below the diagonal, U on and above it, (P A Q)[i, j] =
 *     A[row_perm_fwd[i], col_perm_fwd[j]], and Ok { transposition_count } counts the row and column swaps made.
 *   - factor_in_place_scratch(dim, block_size, ...) takes (dim, block_size) as (nrows, ncols), as faer-ffi forwards them.
 *   - solve / solve_transpose (square): rhs <- A^-1 rhs / A^-T rhs (conjugated with A_conj); reconstruct: A <- P^-1 L U Q^-1
 *     (any shape); inverse: A <- A^-1 (square).
 *   - permutation lengths come from the matrix dimensions, never from the slices' `len`. */
struct FaerV0_24_FullPivLuParams libfaer_v0_23_FullPivLuParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u32_f64(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u32_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u32_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u32_f64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u64_f64(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u64_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u64_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u64_f64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_FullPivLuParams libfaer_v0_23_FullPivLuParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u32_f32(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u32_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u32_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u32_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u32_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u32_f32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u64_f32(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u64_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u64_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u64_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u64_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u64_f32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_FullPivLuParams libfaer_v0_23_FullPivLuParams_c64(void);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u32_c64(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u32_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u32_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u32_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u32_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u32_c64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u64_c64(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u64_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u64_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u64_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u64_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u64_c64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_FullPivLuParams libfaer_v0_23_FullPivLuParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u32_c32(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u32_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u32_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u32_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u32_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u32_c32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_factor_in_place_scratch_u64_c32(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_FullPivLuStatus libfaer_v0_23_full_piv_lu_factor_in_place_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut row_perm_fwd, struct FaerV0_24_SliceMut row_perm_bwd, struct FaerV0_24_SliceMut col_perm_fwd, struct FaerV0_24_SliceMut col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_FullPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_in_place_scratch_u64_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_in_place_u64_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_solve_transpose_in_place_scratch_u64_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_solve_transpose_in_place_u64_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_reconstruct_scratch_u64_c32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_reconstruct_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_full_piv_lu_inverse_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_full_piv_lu_inverse_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef row_perm_fwd, struct FaerV0_24_SliceRef row_perm_bwd, struct FaerV0_24_SliceRef col_perm_fwd, struct FaerV0_24_SliceRef col_perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

#ifdef __cplusplus
}
#endif
#endif /* LIBFAER_B200_FULL_PIV_LU_H */
