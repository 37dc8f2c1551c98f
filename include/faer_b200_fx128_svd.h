/*
 * faer_b200_fx128_svd.h — double-double singular value decomposition of libfaer_b200.so: faer-ffi's `svd` family for fx128 and
 * cx128. Included by faer_b200.h next to faer_b200_fx128.h, whose element layouts apply (fx128 = { double hi; double lo; },
 * cx128 = { fx128 re; fx128 im; }, strides count elements). Same semantics as the f64 / c64 entries: S has min(nrows, ncols) entries
 * in non-increasing order (cx128: (value, 0) entries, strided in complex units), U is nrows x {size, nrows} and V is
 * ncols x {size, ncols}, either passed with no columns is not computed (neither: the values only), non-finite input returns
 * NoConvergence, and with size == 0 a requested U / V is the identity; params.qr_ratio_threshold selects the QR-first path for
 * tall inputs; host or device pointers with any strides, synchronous calls, abort() on precondition violations, `Par` and
 * `MemAlloc` accepted and ignored. The params queries return faer's defaults (svd/mod.rs:49-58), the scratch query the f64 / c64
 * formula with 16 / 32-byte elements. The prototypes are faer.h's, compared with it by tests/test_fx128_svd_cabi_cpu.py
 * (tests/golden/faer_ffi_fx128_svd_prototypes.json); each cites the faer.h declaration and the faer-ffi/src/lib.rs definition it
 * replaces.
 */
#ifndef LIBFAER_B200_FX128_SVD_H
#define LIBFAER_B200_FX128_SVD_H

#include "faer_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* faer.h:500, lib.rs:691-694 */
struct FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_cx128(void);
/* faer.h:506, lib.rs:691-694 */
struct FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_fx128(void);
/* faer.h:704, lib.rs:744-750 */
struct FaerV0_24_SvdParams libfaer_v0_23_SvdParams_cx128(void);
/* faer.h:710, lib.rs:744-750 */
struct FaerV0_24_SvdParams libfaer_v0_23_SvdParams_fx128(void);
/* faer.h:6246, lib.rs:2345-2366 */
struct FaerV0_24_SvdStatus libfaer_v0_23_svd_cx128(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_MatMut V, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SvdParams params);
/* faer.h:6270, lib.rs:2345-2366 */
struct FaerV0_24_SvdStatus libfaer_v0_23_svd_fx128(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_MatMut V, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SvdParams params);
/* faer.h:6292, lib.rs:2327-2344 */
struct FaerV0_24_Layout libfaer_v0_23_svd_scratch_cx128(size_t nrows, size_t ncols, enum FaerV0_24_ComputeSvdVectors compute_U, enum FaerV0_24_ComputeSvdVectors compute_V, struct FaerV0_24_Par par, struct FaerV0_24_SvdParams params);
/* faer.h:6313, lib.rs:2327-2344 */
struct FaerV0_24_Layout libfaer_v0_23_svd_scratch_fx128(size_t nrows, size_t ncols, enum FaerV0_24_ComputeSvdVectors compute_U, enum FaerV0_24_ComputeSvdVectors compute_V, struct FaerV0_24_Par par, struct FaerV0_24_SvdParams params);

#ifdef __cplusplus
}
#endif

#endif
