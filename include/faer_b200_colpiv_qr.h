/*
 * faer_b200_colpiv_qr.h — column-pivoted Householder QR (faer-ffi's `colpiv_qr_*` family) of libfaer_b200.so. Included by
 * faer_b200.h; same conventions (host or device pointers, synchronous calls, abort() on precondition violations). The prototypes
 * are faer.h's, compared with it by tests/test_colpiv_qr_cabi_cpu.py (tests/golden/faer_ffi_colpiv_qr_prototypes.json).
 */
#ifndef LIBFAER_B200_COLPIV_QR_H
#define LIBFAER_B200_COLPIV_QR_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- column-pivoted QR: faer-ffi/src/lib.rs (ColPivQrParams, ColPivQrStatus), faer.h:101-104, 234-248 ---- */
typedef struct FaerV0_24_ColPivQrParams { size_t blocking_threshold; size_t par_threshold; } FaerV0_24_ColPivQrParams;
typedef enum FaerV0_24_ColPivQrStatus_Tag { FaerV0_24_ColPivQrStatus_Ok, FaerV0_24_ColPivQrStatus_Unknown } FaerV0_24_ColPivQrStatus_Tag;
typedef struct FaerV0_24_ColPivQrStatus_FaerV0_24_Ok_Body { size_t transposition_count; } FaerV0_24_ColPivQrStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_ColPivQrStatus {
  FaerV0_24_ColPivQrStatus_Tag tag;
  union {
    FaerV0_24_ColPivQrStatus_FaerV0_24_Ok_Body ok;
  };
} FaerV0_24_ColPivQrStatus;

/* column-pivoted QR A P = Q R of an m x n matrix (csrc/colpiv_qr.cu). faer-ffi/src/lib.rs:1721-1940 (colpiv_qr_*),
 * faer.h:508-518 (ColPivQrParams_<T>), 990-2030; the algorithm is faer/src/linalg/qr/col_pivoting/{factor.rs:112-388,
 * solve.rs:52-184, reconstruct.rs:16-45, inverse.rs:16-50}.
 *   - ColPivQrParams_<T>() = {48 * 48, 192 * 256}, the reference default. The GPU factorization does not depend on either field.
 *   - factor: Q_coeff is block_size x min(m, n) (block_size = Q_coeff.nrows; 0 aborts when min(m, n) > 0, the reference would not
 *     terminate). The reference's operation sequence is followed (column norms downdated, recomputed when they fall below
 *     sqrt(eps) of the last recomputed maximum or when A's row stride is not 1; first maximum, strict `>`), so perm_fwd / perm_bwd
 *     and Ok { transposition_count } match it wherever the pivots are separated by more than rounding. A holds R in its upper
 *     trapezoid and the Householder vectors below the diagonal; Q_coeff holds the T blocks, as qr_factor_in_place lays them out.
 *     An all-zero input gives NaN factors, the identity permutation and a count of 0, as in the reference.
 *   - solve / solve_transpose (square), solve_lstsq (m >= n): the unpivoted QR solves (A_conj honoured) plus one row permutation.
 *   - reconstruct: A <- Q R P^T; inverse: A <- P R^-1 Q^H.
 *   - permutation lengths come from A.ncols / R.ncols, never from the slices' `len`; `par` and `mem` are ignored. */
struct FaerV0_24_ColPivQrParams libfaer_v0_23_ColPivQrParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u32_f64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u32_f64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u32_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u32_f64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u32_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u32_f64(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u32_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u32_f64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u32_f64(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u64_f64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u64_f64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u64_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u64_f64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u64_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u64_f64(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u64_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u64_f64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u64_f64(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_ColPivQrParams libfaer_v0_23_ColPivQrParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u32_f32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u32_f32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u32_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u32_f32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u32_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u32_f32(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u32_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u32_f32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u32_f32(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u64_f32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u64_f32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u64_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u64_f32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u64_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u64_f32(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u64_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u64_f32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u64_f32(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_ColPivQrParams libfaer_v0_23_ColPivQrParams_c64(void);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u32_c64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u32_c64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u32_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u32_c64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u32_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u32_c64(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u32_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u32_c64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u32_c64(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u64_c64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u64_c64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u64_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u64_c64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u64_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u64_c64(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u64_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u64_c64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u64_c64(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_ColPivQrParams libfaer_v0_23_ColPivQrParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u32_c32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u32_c32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u32_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u32_c32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u32_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u32_c32(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u32_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u32_c32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u32_c32(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_factor_in_place_scratch_u64_c32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_ColPivQrStatus libfaer_v0_23_colpiv_qr_factor_in_place_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_ColPivQrParams params);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_in_place_scratch_u64_c32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_in_place_u64_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_transpose_in_place_scratch_u64_c32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_transpose_in_place_u64_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_scratch_u64_c32(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_solve_lstsq_in_place_u64_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_reconstruct_scratch_u64_c32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_reconstruct_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_colpiv_qr_inverse_scratch_u64_c32(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_colpiv_qr_inverse_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

#ifdef __cplusplus
}
#endif
#endif /* LIBFAER_B200_COLPIV_QR_H */
