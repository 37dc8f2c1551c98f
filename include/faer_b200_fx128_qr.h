/*
 * faer_b200_fx128_qr.h — double-double Householder QR of libfaer_b200.so: faer-ffi's `qr` and `apply_householder` families for
 * fx128 and cx128. Included by faer_b200.h next to faer_b200_fx128.h, whose element layouts apply (fx128 = { double hi; double
 * lo; }, cx128 = { fx128 re; fx128 im; }, strides count elements). Same conventions as the c64 / c32 entries: host or device
 * pointers with any strides (negative and row-major included), synchronous calls, abort() on precondition violations, `Par`
 * accepted and ignored, `Conj` honoured for cx128 and a no-op for fx128. `QrParams_*` returns faer's type-independent defaults
 * (factor.rs:127-136), the scratch queries the c64 formulas with 16 / 32-byte elements. The prototypes are faer.h's, compared with
 * it by tests/test_fx128_qr_cabi_cpu.py (tests/golden/faer_ffi_fx128_qr_prototypes.json); each cites the faer.h declaration and
 * the faer-ffi/src/lib.rs definition it replaces.
 */
#ifndef LIBFAER_B200_FX128_QR_H
#define LIBFAER_B200_FX128_QR_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* faer.h:668, lib.rs:672 */
struct FaerV0_24_QrParams libfaer_v0_23_QrParams_cx128(void);
/* faer.h:674, lib.rs:672 */
struct FaerV0_24_QrParams libfaer_v0_23_QrParams_fx128(void);
/* faer.h:740, lib.rs:1430 */
void libfaer_v0_23_apply_householder_on_the_left_cx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:761, lib.rs:1430 */
void libfaer_v0_23_apply_householder_on_the_left_fx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:776, lib.rs:1423 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_cx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:788, lib.rs:1423 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_fx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:806, lib.rs:1478 */
void libfaer_v0_23_apply_householder_on_the_right_cx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:827, lib.rs:1478 */
void libfaer_v0_23_apply_householder_on_the_right_fx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:842, lib.rs:1471 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_cx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:854, lib.rs:1471 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_fx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:872, lib.rs:1454 */
void libfaer_v0_23_apply_householder_transpose_on_the_left_cx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:893, lib.rs:1454 */
void libfaer_v0_23_apply_householder_transpose_on_the_left_fx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:908, lib.rs:1447 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_cx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:920, lib.rs:1447 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_fx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:938, lib.rs:1502 */
void libfaer_v0_23_apply_householder_transpose_on_the_right_cx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:959, lib.rs:1502 */
void libfaer_v0_23_apply_householder_transpose_on_the_right_fx128(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:974, lib.rs:1495 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_cx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:986, lib.rs:1495 */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_fx128(size_t dim, size_t block_size, size_t rhs_ncols);
/* faer.h:5586, lib.rs:1544 */
struct FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_QrParams params);
/* faer.h:5604, lib.rs:1544 */
struct FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_QrParams params);
/* faer.h:5622, lib.rs:1528 */
struct FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_cx128(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_QrParams params);
/* faer.h:5640, lib.rs:1528 */
struct FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_fx128(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_QrParams params);
/* faer.h:5660, lib.rs:1704 */
void libfaer_v0_23_qr_inverse_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5681, lib.rs:1704 */
void libfaer_v0_23_qr_inverse_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5696, lib.rs:1692 */
struct FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_cx128(size_t dim, size_t block_size, struct FaerV0_24_Par par);
/* faer.h:5708, lib.rs:1692 */
struct FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_fx128(size_t dim, size_t block_size, struct FaerV0_24_Par par);
/* faer.h:5716, lib.rs:1520 */
size_t libfaer_v0_23_qr_recommended_block_size_cx128(size_t nrows, size_t ncols);
/* faer.h:5722, lib.rs:1520 */
size_t libfaer_v0_23_qr_recommended_block_size_fx128(size_t nrows, size_t ncols);
/* faer.h:5738, lib.rs:1675 */
void libfaer_v0_23_qr_reconstruct_cx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5759, lib.rs:1675 */
void libfaer_v0_23_qr_reconstruct_fx128(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5776, lib.rs:1661 */
struct FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_cx128(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
/* faer.h:5791, lib.rs:1661 */
struct FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_fx128(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
/* faer.h:5812, lib.rs:1574 */
void libfaer_v0_23_qr_solve_in_place_cx128(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5836, lib.rs:1574 */
void libfaer_v0_23_qr_solve_in_place_fx128(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5854, lib.rs:1560 */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_cx128(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
/* faer.h:5869, lib.rs:1560 */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_fx128(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
/* faer.h:5890, lib.rs:1642 */
void libfaer_v0_23_qr_solve_lstsq_in_place_cx128(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5914, lib.rs:1642 */
void libfaer_v0_23_qr_solve_lstsq_in_place_fx128(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5934, lib.rs:1626 */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_cx128(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
/* faer.h:5952, lib.rs:1626 */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_fx128(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
/* faer.h:5974, lib.rs:1607 */
void libfaer_v0_23_qr_solve_transpose_in_place_cx128(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:5998, lib.rs:1607 */
void libfaer_v0_23_qr_solve_transpose_in_place_fx128(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* faer.h:6016, lib.rs:1593 */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_cx128(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
/* faer.h:6031, lib.rs:1593 */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_fx128(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);

#ifdef __cplusplus
}
#endif

#endif /* LIBFAER_B200_FX128_QR_H */
