/*
 * faer_b200_lblt.h — Bunch-Kaufman LBL^H (faer-ffi's `lblt_*` family) of libfaer_b200.so. Included by faer_b200.h; same
 * conventions (host or device pointers, synchronous calls, abort() on precondition violations). The prototypes are faer.h's,
 * compared with it by tests/test_lblt_cabi_cpu.py (tests/golden/faer_ffi_lblt_prototypes.json).
 */
#ifndef LIBFAER_B200_LBLT_H
#define LIBFAER_B200_LBLT_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- LBLT: faer-ffi/src/lib.rs:492-508 (PivotingStrategy), 576-580 (LbltStatus), 665-670 (LbltParams); faer.h:32-55, 156-160,
 * 324-338 ---- */
typedef enum FaerV0_24_PivotingStrategy {
  FaerV0_24_PivotingStrategy_Partial,
  FaerV0_24_PivotingStrategy_PartialDiag,
  FaerV0_24_PivotingStrategy_Rook,
  FaerV0_24_PivotingStrategy_RookDiag,
  FaerV0_24_PivotingStrategy_Full,
} FaerV0_24_PivotingStrategy;
typedef struct FaerV0_24_LbltParams { enum FaerV0_24_PivotingStrategy pivoting; size_t par_threshold; size_t block_size; } FaerV0_24_LbltParams;
typedef enum FaerV0_24_LbltStatus_Tag { FaerV0_24_LbltStatus_Ok, FaerV0_24_LbltStatus_Unknown } FaerV0_24_LbltStatus_Tag;
typedef struct FaerV0_24_LbltStatus_FaerV0_24_Ok_Body { size_t transposition_count; } FaerV0_24_LbltStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_LbltStatus {
  FaerV0_24_LbltStatus_Tag tag;
  union {
    FaerV0_24_LbltStatus_FaerV0_24_Ok_Body ok;
  };
} FaerV0_24_LbltStatus;

/* Bunch-Kaufman P A P^T = L B L^H of a self-adjoint (possibly indefinite) matrix, B block diagonal with 1 x 1 and 2 x 2 blocks
 * (csrc/lblt.cu). faer-ffi/src/lib.rs:1288-1420 (lblt_*), faer.h:604-612 (LbltParams_<T>), 3178-3758; the algorithm is
 * faer/src/linalg/cholesky/bunch_kaufman/{factor.rs:264-1234, solve.rs:35-104, reconstruct.rs:12-87, inverse.rs:11-42}.
 *   - LbltParams_<T>() = {PartialDiag, 128 * 128, 64}, the reference default. A `pivoting` value outside the enum aborts.
 *   - factor: the lower triangle of A holds L (unit diagonal implied) and the diagonal of B; subdiag[k] holds B's subdiagonal
 *     entry of a 2 x 2 block at (k, k+1), 0 for the other columns it writes. As in the reference, a column whose off-diagonal
 *     part is zero (and the last column of the non-Full strategies) leaves subdiag[k] unwritten: pass a zeroed subdiag.
 *     Full scales the whole matrix, strict upper triangle included, by 1 / norm_max and restores only the diagonal and
 *     subdiag; the other strategies never read or write the strict upper triangle. Ok { transposition_count }; perm_fwd /
 *     perm_bwd follow the reference's pivots.
 *   - solve: rhs <- A^-1 rhs (A_conj: conj(A)^-1 rhs); reconstruct: the lower triangle of A from the factor, the strict upper
 *     triangle the intermediate L B (zero except conj(s_j) at (j, j+1) of each 2 x 2 block); inverse: all n^2 entries.
 *   - the permutation length is min(perm_fwd.len, perm_bwd.len) and must equal the dimension; `par` and `mem` are ignored. */
struct FaerV0_24_LbltParams libfaer_v0_23_LbltParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u32_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u32_f64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u64_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u64_f64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_LbltParams libfaer_v0_23_LbltParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u32_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u32_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u32_f32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u64_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u64_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u64_f32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_LbltParams libfaer_v0_23_LbltParams_c64(void);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u32_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u32_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u32_c64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u64_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u64_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u64_c64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_LbltParams libfaer_v0_23_LbltParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u32_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u32_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u32_c32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_factor_in_place_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LbltParams params);
struct FaerV0_24_LbltStatus libfaer_v0_23_lblt_factor_in_place_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_VecMut subdiag, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LbltParams params);
struct FaerV0_24_Layout libfaer_v0_23_lblt_solve_in_place_scratch_u64_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_solve_in_place_u64_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_reconstruct_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_reconstruct_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_lblt_inverse_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_lblt_inverse_u64_c32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef diag, struct FaerV0_24_VecRef subdiag, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

#ifdef __cplusplus
}
#endif
#endif /* LIBFAER_B200_LBLT_H */
