/*
 * faer_b200_fx128_evd.h — double-double self-adjoint eigendecomposition of libfaer_b200.so: faer-ffi's `self_adjoint_evd` family
 * for fx128 and cx128. Included by faer_b200.h next to faer_b200_fx128.h, whose element layouts apply (fx128 = { double hi; double
 * lo; }, cx128 = { fx128 re; fx128 im; }, strides count elements). Same semantics as the f64 / c64 entries: only the lower
 * triangle of A is read, U with no columns asks for the eigenvalues only, S is nondecreasing (cx128: (value, 0) entries, strided in
 * complex units), non-finite input returns NoConvergence; host or device pointers with any strides, synchronous calls, abort() on
 * precondition violations, `Par` accepted and ignored. The params queries return faer's defaults (evd/mod.rs:82-90), the scratch
 * query the f64 / c64 formula with 16 / 32-byte elements. The prototypes are faer.h's, compared with it by
 * tests/test_fx128_evd_cabi_cpu.py (tests/golden/faer_ffi_fx128_evd_prototypes.json); each cites the faer.h declaration and the
 * faer-ffi/src/lib.rs definition it replaces.
 */
#ifndef LIBFAER_B200_FX128_EVD_H
#define LIBFAER_B200_FX128_EVD_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* faer.h:692, lib.rs:751 */
struct FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_cx128(void);
/* faer.h:698, lib.rs:751 */
struct FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_fx128(void);
/* faer.h:716, lib.rs:695 */
struct FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_cx128(void);
/* faer.h:722, lib.rs:695 */
struct FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_fx128(void);
/* faer.h:6050, lib.rs:2382-2400 */
struct FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_cx128(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SelfAdjointEvdParams params);
/* faer.h:6071, lib.rs:2382-2400 */
struct FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_fx128(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SelfAdjointEvdParams params);
/* faer.h:6088, lib.rs:2367-2381 */
struct FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_cx128(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_U, struct FaerV0_24_Par par, struct FaerV0_24_SelfAdjointEvdParams params);
/* faer.h:6103, lib.rs:2367-2381 */
struct FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_fx128(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_U, struct FaerV0_24_Par par, struct FaerV0_24_SelfAdjointEvdParams params);

#ifdef __cplusplus
}
#endif

#endif
