/*
 * faer_b200_fx128.h — double-double scalars of libfaer_b200.so: faer-ffi's `matmul`, triangular solve / inverse, `llt` and
 * `partial_piv_lu` families for fx128 and cx128. Included by faer_b200.h; same conventions (host or device pointers, synchronous
 * calls, abort() on precondition violations, `Par` accepted and ignored). The prototypes are faer.h's, compared with it by
 * tests/test_fx128_cabi_cpu.py (tests/golden/faer_ffi_fx128_prototypes.json).
 *
 * Element layouts (strides count elements):
 *   fx128 = { double hi; double lo; }                        16 bytes, value hi + lo
 *   cx128 = { fx128 re; fx128 im; }                          32 bytes
 * `alpha` of matmul points to one fx128 / cx128; LltRegularization's delta and epsilon point to an fx128 for both kinds.
 */
#ifndef LIBFAER_B200_FX128_H
#define LIBFAER_B200_FX128_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

struct FaerV0_24_LltParams libfaer_v0_23_LltParams_cx128(void);
struct FaerV0_24_LltParams libfaer_v0_23_LltParams_fx128(void);
struct FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_cx128(void);
struct FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_fx128(void);
void libfaer_v0_23_inverse_triangular_lower_in_place_cx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_lower_in_place_fx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_upper_in_place_cx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_upper_in_place_fx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_lower_in_place_cx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_lower_in_place_fx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_upper_in_place_cx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_upper_in_place_fx128(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
struct FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_LltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LltParams params);
struct FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_LltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LltParams params);
struct FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_cx128(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LltParams params);
struct FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_fx128(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LltParams params);
void libfaer_v0_23_llt_inverse_cx128(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_llt_inverse_fx128(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_cx128(size_t dim, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_fx128(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_reconstruct_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_llt_reconstruct_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_cx128(size_t dim, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_fx128(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_solve_in_place_cx128(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_llt_solve_in_place_fx128(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_cx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_fx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_cx128(struct FaerV0_24_MatMut C, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A, struct FaerV0_24_MatRef B, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_fx128(struct FaerV0_24_MatMut C, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A, struct FaerV0_24_MatRef B, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_triangular_cx128(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A, enum FaerV0_24_Block A_block, struct FaerV0_24_MatRef B, enum FaerV0_24_Block B_block, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_triangular_fx128(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A, enum FaerV0_24_Block A_block, struct FaerV0_24_MatRef B, enum FaerV0_24_Block B_block, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_cx128(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_fx128(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_cx128(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_fx128(size_t dim, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u32_cx128(size_t dim, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u32_fx128(size_t dim, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u64_cx128(size_t dim, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u64_fx128(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u32_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_inverse_u32_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_inverse_u64_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_inverse_u64_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u32_cx128(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u32_fx128(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u64_cx128(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u64_fx128(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u32_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_reconstruct_u32_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_reconstruct_u64_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_reconstruct_u64_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_cx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_fx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_cx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_fx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_cx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_fx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_cx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_fx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_cx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_fx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_cx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_fx128(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_cx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_fx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_cx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_fx128(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_solve_triangular_lower_in_place_cx128(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_lower_in_place_fx128(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_upper_in_place_cx128(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_upper_in_place_fx128(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_lower_in_place_cx128(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_lower_in_place_fx128(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_upper_in_place_cx128(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_upper_in_place_fx128(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);

#ifdef __cplusplus
}
#endif

#endif /* LIBFAER_B200_FX128_H */
