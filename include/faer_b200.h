/*
 * faer_b200.h — C ABI of the B200-native dense backend (libfaer_b200.so).
 *
 * Drop-in for the hot-path subset of faer-ffi's generated header: same include guard, same POD layouts,
 * same symbol grammar `libfaer_v0_23_<fn>[_u32|_u64]_<dtype>` as /root/reference/faer-ffi/faer.h, so a C/C++
 * caller of faer-ffi compiles and links against this library unchanged for the entry points below.
 * Each declaration cites the reference interface it replaces (faer-ffi/src/lib.rs:LINE = Rust body,
 * faer-ffi/faer.h:LINE = generated C declaration).
 *
 * Pointer semantics (extension of the reference, which is CPU-only): every matrix/slice pointer may be
 *   - a HOST pointer  : staged to the GPU and back inside the call (the reference-facing path), or
 *   - a DEVICE pointer: operated on in place (no copies); mixed calls are allowed per argument.
 * Calls are synchronous on return, like the reference. Precondition violations abort() with a message
 * (the reference panics inside extern "C", i.e. aborts).
 * There is NO CPU fallback: without a CUDA device every compute entry point aborts.
 */
#ifndef LIBFAER_V0_24
#define LIBFAER_V0_24

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- enums: faer-ffi/src/lib.rs:59-97 ---- */
typedef enum FaerV0_24_Accum { FaerV0_24_Accum_Replace, FaerV0_24_Accum_Add } FaerV0_24_Accum;
typedef enum FaerV0_24_Conj { FaerV0_24_Conj_No, FaerV0_24_Conj_Yes } FaerV0_24_Conj;
typedef enum FaerV0_24_ParTag { FaerV0_24_ParTag_Seq, FaerV0_24_ParTag_Rayon } FaerV0_24_ParTag;
typedef enum FaerV0_24_Block {
  FaerV0_24_Block_Rectangular,
  FaerV0_24_Block_TriangularLower,
  FaerV0_24_Block_TriangularUpper,
  FaerV0_24_Block_StrictTriangularLower,
  FaerV0_24_Block_StrictTriangularUpper,
  FaerV0_24_Block_UnitTriangularLower,
  FaerV0_24_Block_UnitTriangularUpper
} FaerV0_24_Block;

/* ---- opaque scalar tags: faer-ffi/src/lib.rs:56-58 ---- */
typedef struct FaerV0_24_Scalar FaerV0_24_Scalar;
typedef struct FaerV0_24_Real FaerV0_24_Real;

/* ---- views: faer-ffi/src/lib.rs:12-58 (strides in ELEMENTS, any sign) ---- */
typedef struct FaerV0_24_MatRef { const void *ptr; size_t nrows; size_t ncols; ptrdiff_t row_stride; ptrdiff_t col_stride; } FaerV0_24_MatRef;
typedef struct FaerV0_24_MatMut { void *ptr; size_t nrows; size_t ncols; ptrdiff_t row_stride; ptrdiff_t col_stride; } FaerV0_24_MatMut;
typedef struct FaerV0_24_VecRef { const void *ptr; size_t len; ptrdiff_t stride; } FaerV0_24_VecRef;
typedef struct FaerV0_24_VecMut { void *ptr; size_t len; ptrdiff_t stride; } FaerV0_24_VecMut;
typedef struct FaerV0_24_SliceRef { const void *ptr; size_t len; } FaerV0_24_SliceRef;
typedef struct FaerV0_24_SliceMut { void *ptr; size_t len; } FaerV0_24_SliceMut;

/* ---- Par / scratch protocol: faer-ffi/src/lib.rs:76-128 ---- */
typedef struct FaerV0_24_Par { enum FaerV0_24_ParTag tag; size_t nthreads; } FaerV0_24_Par;
typedef struct FaerV0_24_Layout { size_t len_bytes; size_t align_bytes; } FaerV0_24_Layout;
typedef struct FaerV0_24_MemAlloc { void *ptr; size_t len_bytes; } FaerV0_24_MemAlloc;

/* ---- params: faer-ffi/src/lib.rs:650-688 ---- */
typedef struct FaerV0_24_LltParams { size_t recursion_threshold; size_t block_size; } FaerV0_24_LltParams;
typedef struct FaerV0_24_PartialPivLuParams { size_t recursion_threshold; size_t block_size; size_t par_threshold; } FaerV0_24_PartialPivLuParams;
typedef struct FaerV0_24_QrParams { size_t blocking_threshold; size_t par_threshold; } FaerV0_24_QrParams;

/* ---- LLT regularisation: faer-ffi/src/lib.rs:794-817 ---- */
typedef struct FaerV0_24_LltRegularization {
  const FaerV0_24_Real *dynamic_regularization_delta;
  const FaerV0_24_Real *dynamic_regularization_epsilon;
} FaerV0_24_LltRegularization;

typedef struct FaerV0_24_LdltParams { size_t recursion_threshold; size_t block_size; } FaerV0_24_LdltParams;
typedef struct FaerV0_24_LdltRegularization {
  const FaerV0_24_Real *dynamic_regularization_delta;
  const FaerV0_24_Real *dynamic_regularization_epsilon;
  struct FaerV0_24_SliceMut dynamic_regularization_signs; /* i8 */
} FaerV0_24_LdltRegularization;
typedef enum FaerV0_24_LdltStatus_Tag { FaerV0_24_LdltStatus_Ok, FaerV0_24_LdltStatus_ZeroPivot, FaerV0_24_LdltStatus_Unknown } FaerV0_24_LdltStatus_Tag;
typedef struct FaerV0_24_LdltStatus_FaerV0_24_Ok_Body { size_t dynamic_regularization_count; } FaerV0_24_LdltStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_LdltStatus_FaerV0_24_ZeroPivot_Body { size_t index; } FaerV0_24_LdltStatus_FaerV0_24_ZeroPivot_Body;
typedef struct FaerV0_24_LdltStatus {
  FaerV0_24_LdltStatus_Tag tag;
  union {
    FaerV0_24_LdltStatus_FaerV0_24_Ok_Body ok;
    FaerV0_24_LdltStatus_FaerV0_24_ZeroPivot_Body zero_pivot;
  };
} FaerV0_24_LdltStatus;

/* SVD types: faer.h:87-99 (ComputeSvdVectors, BidiagParams), 196-201 (SvdParams), 471-490 (SvdStatus); VecMut lib.rs / faer.h */
typedef enum FaerV0_24_ComputeSvdVectors { FaerV0_24_ComputeSvdVectors_No, FaerV0_24_ComputeSvdVectors_Thin, FaerV0_24_ComputeSvdVectors_Full } FaerV0_24_ComputeSvdVectors;
typedef struct FaerV0_24_BidiagParams { size_t par_threshold; } FaerV0_24_BidiagParams;
typedef struct FaerV0_24_SvdParams {
  struct FaerV0_24_BidiagParams bidiag;
  struct FaerV0_24_QrParams qr;
  size_t recursion_threshold;
  double qr_ratio_threshold;
} FaerV0_24_SvdParams;
typedef enum FaerV0_24_SvdStatus_Tag { FaerV0_24_SvdStatus_Ok, FaerV0_24_SvdStatus_NoConvergence } FaerV0_24_SvdStatus_Tag;
typedef struct FaerV0_24_SvdStatus_FaerV0_24_Ok_Body { size_t padding; } FaerV0_24_SvdStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_SvdStatus_FaerV0_24_NoConvergence_Body { size_t padding; } FaerV0_24_SvdStatus_FaerV0_24_NoConvergence_Body;
typedef struct FaerV0_24_SvdStatus {
  FaerV0_24_SvdStatus_Tag tag;
  union {
    FaerV0_24_SvdStatus_FaerV0_24_Ok_Body ok;
    FaerV0_24_SvdStatus_FaerV0_24_NoConvergence_Body no_convergence;
  };
} FaerV0_24_SvdStatus;

/* self-adjoint EVD types: faer.h:67-70 (ComputeEigenvectors), 187-194 (TridiagParams, SelfAdjointEvdParams), 260-279 (EvdStatus) */
typedef enum FaerV0_24_ComputeEigenvectors { FaerV0_24_ComputeEigenvectors_No, FaerV0_24_ComputeEigenvectors_Yes } FaerV0_24_ComputeEigenvectors;
typedef struct FaerV0_24_TridiagParams { size_t par_threshold; } FaerV0_24_TridiagParams;
typedef struct FaerV0_24_SelfAdjointEvdParams { struct FaerV0_24_TridiagParams tridiag; size_t recursion_threshold; } FaerV0_24_SelfAdjointEvdParams;
typedef enum FaerV0_24_EvdStatus_Tag { FaerV0_24_EvdStatus_Ok, FaerV0_24_EvdStatus_NoConvergence } FaerV0_24_EvdStatus_Tag;
typedef struct FaerV0_24_EvdStatus_FaerV0_24_Ok_Body { size_t padding; } FaerV0_24_EvdStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_EvdStatus_FaerV0_24_NoConvergence_Body { size_t padding; } FaerV0_24_EvdStatus_FaerV0_24_NoConvergence_Body;
typedef struct FaerV0_24_EvdStatus {
  FaerV0_24_EvdStatus_Tag tag;
  union {
    FaerV0_24_EvdStatus_FaerV0_24_Ok_Body ok;
    FaerV0_24_EvdStatus_FaerV0_24_NoConvergence_Body no_convergence;
  };
} FaerV0_24_EvdStatus;

/* ---- status unions: faer-ffi/src/lib.rs:552-629, C layout faer-ffi/faer.h:383-469 ---- */
typedef enum FaerV0_24_LltStatus_Tag { FaerV0_24_LltStatus_Ok, FaerV0_24_LltStatus_NonPositivePivot, FaerV0_24_LltStatus_Unknown } FaerV0_24_LltStatus_Tag;
typedef struct FaerV0_24_LltStatus_FaerV0_24_Ok_Body { size_t dynamic_regularization_count; } FaerV0_24_LltStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_LltStatus_FaerV0_24_NonPositivePivot_Body { size_t index; } FaerV0_24_LltStatus_FaerV0_24_NonPositivePivot_Body;
typedef struct FaerV0_24_LltStatus {
  FaerV0_24_LltStatus_Tag tag;
  union {
    FaerV0_24_LltStatus_FaerV0_24_Ok_Body ok;
    FaerV0_24_LltStatus_FaerV0_24_NonPositivePivot_Body non_positive_pivot;
  };
} FaerV0_24_LltStatus;

typedef enum FaerV0_24_PartialPivLuStatus_Tag { FaerV0_24_PartialPivLuStatus_Ok, FaerV0_24_PartialPivLuStatus_Unknown } FaerV0_24_PartialPivLuStatus_Tag;
typedef struct FaerV0_24_PartialPivLuStatus_FaerV0_24_Ok_Body { size_t transposition_count; } FaerV0_24_PartialPivLuStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_PartialPivLuStatus {
  FaerV0_24_PartialPivLuStatus_Tag tag;
  union { FaerV0_24_PartialPivLuStatus_FaerV0_24_Ok_Body ok; };
} FaerV0_24_PartialPivLuStatus;

typedef enum FaerV0_24_QrStatus_Tag { FaerV0_24_QrStatus_Ok, FaerV0_24_QrStatus_Unknown } FaerV0_24_QrStatus_Tag;
typedef struct FaerV0_24_QrStatus_FaerV0_24_Ok_Body { size_t rank; } FaerV0_24_QrStatus_FaerV0_24_Ok_Body;
typedef struct FaerV0_24_QrStatus {
  FaerV0_24_QrStatus_Tag tag;
  union { FaerV0_24_QrStatus_FaerV0_24_Ok_Body ok; };
} FaerV0_24_QrStatus;

/* =====================================================================================================
 * Hot-path entry points
 * ===================================================================================================== */

/* matmul: C = [C +] alpha * A * B.   faer-ffi/src/lib.rs:855-871, faer-ffi/faer.h:4252-4257 */
void libfaer_v0_23_matmul_f64(struct FaerV0_24_MatMut C, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                              struct FaerV0_24_MatRef B, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);

/* matmul_triangular.   faer-ffi/src/lib.rs:872-894, faer-ffi/faer.h:4306-4314 */
void libfaer_v0_23_matmul_triangular_f64(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block,
                                         enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                                         enum FaerV0_24_Block A_block, struct FaerV0_24_MatRef B,
                                         enum FaerV0_24_Block B_block, const struct FaerV0_24_Scalar *alpha,
                                         struct FaerV0_24_Par par);

/* f32 variants (3xTF32 error-compensated tensor-core kernel, fp32-level accuracy): faer.h `libfaer_v0_23_matmul_f32` /
 * `matmul_triangular_f32` (funcs! stamping, faer-ffi/src/lib.rs:313-369, 855-894); `alpha` points to a float. */
void libfaer_v0_23_matmul_f32(struct FaerV0_24_MatMut C, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                              struct FaerV0_24_MatRef B, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_triangular_f32(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block,
                                         enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                                         enum FaerV0_24_Block A_block, struct FaerV0_24_MatRef B,
                                         enum FaerV0_24_Block B_block, const struct FaerV0_24_Scalar *alpha,
                                         struct FaerV0_24_Par par);

/* c32 (interleaved complex<f32>) variants: faer-ffi/faer.h `libfaer_v0_23_matmul_c32` / `matmul_triangular_c32`
 * (same funcs! stamping, faer-ffi/src/lib.rs:313-369, 855-894); `alpha` points to a complex<float> scalar. */
void libfaer_v0_23_matmul_c32(struct FaerV0_24_MatMut C, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                              struct FaerV0_24_MatRef B, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_triangular_c32(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block,
                                         enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                                         enum FaerV0_24_Block A_block, struct FaerV0_24_MatRef B,
                                         enum FaerV0_24_Block B_block, const struct FaerV0_24_Scalar *alpha,
                                         struct FaerV0_24_Par par);

/* c64 (interleaved complex<f64>) variants: faer-ffi/faer.h `libfaer_v0_23_matmul_c64` / `matmul_triangular_c64`
 * (same funcs! stamping, faer-ffi/src/lib.rs:313-369, 855-894); `alpha` points to a complex scalar. */
void libfaer_v0_23_matmul_c64(struct FaerV0_24_MatMut C, enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                              struct FaerV0_24_MatRef B, const struct FaerV0_24_Scalar *alpha, struct FaerV0_24_Par par);
void libfaer_v0_23_matmul_triangular_c64(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block,
                                         enum FaerV0_24_Accum accum, struct FaerV0_24_MatRef A,
                                         enum FaerV0_24_Block A_block, struct FaerV0_24_MatRef B,
                                         enum FaerV0_24_Block B_block, const struct FaerV0_24_Scalar *alpha,
                                         struct FaerV0_24_Par par);

/* triangular solves, in place.   faer-ffi/src/lib.rs:896-937, faer-ffi/faer.h:6130-6143 */
void libfaer_v0_23_solve_triangular_lower_in_place_f64(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj,
                                                       struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_upper_in_place_f64(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj,
                                                       struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_lower_in_place_f64(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj,
                                                            struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_upper_in_place_f64(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj,
                                                            struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
/* f32: faer.h:6125-6215 */
void libfaer_v0_23_solve_triangular_lower_in_place_f32(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj,
                                                       struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_upper_in_place_f32(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj,
                                                       struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_lower_in_place_f32(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj,
                                                            struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_upper_in_place_f32(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj,
                                                            struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);

/* LLT.   params: faer-ffi/src/lib.rs:650-654 (+408-456), faer.h:636; scratch: lib.rs:984-995; factor: lib.rs:996-1010, faer.h:4036-4040 */
struct FaerV0_24_LltParams libfaer_v0_23_LltParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_f64(size_t dim, struct FaerV0_24_Par par,
                                                                      struct FaerV0_24_LltParams params);
struct FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_f64(struct FaerV0_24_MatMut A,
                                                                 struct FaerV0_24_LltRegularization regularization,
                                                                 struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem,
                                                                 struct FaerV0_24_LltParams params);

/* SVD (BASELINE.json configs[4]): lib.rs:2326-2366, faer.h:504 (BidiagParams), 708 (SvdParams), 6230-6268 (svd, svd_scratch);
 * semantics faer/src/linalg/svd/mod.rs:530-672. U / V passed with ncols == 0 are the reference's "None" (values only: csrc/svd.cu,
 * bisection on the bidiagonal); otherwise thin (min(nrows, ncols) columns) or full vectors (csrc/svd_vectors.cu: divide and
 * conquer + back-transforms). S receives min(nrows, ncols) values in non-increasing order. Non-finite input: NoConvergence. */
struct FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_f64(void);
struct FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_f32(void);
struct FaerV0_24_SvdParams libfaer_v0_23_SvdParams_f64(void);
struct FaerV0_24_SvdParams libfaer_v0_23_SvdParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_svd_scratch_f64(size_t nrows, size_t ncols, enum FaerV0_24_ComputeSvdVectors compute_U, enum FaerV0_24_ComputeSvdVectors compute_V, struct FaerV0_24_Par par, struct FaerV0_24_SvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_svd_scratch_f32(size_t nrows, size_t ncols, enum FaerV0_24_ComputeSvdVectors compute_U, enum FaerV0_24_ComputeSvdVectors compute_V, struct FaerV0_24_Par par, struct FaerV0_24_SvdParams params);
struct FaerV0_24_SvdStatus libfaer_v0_23_svd_f64(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_MatMut V, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SvdParams params);
struct FaerV0_24_SvdStatus libfaer_v0_23_svd_f32(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_MatMut V, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SvdParams params);

/* Self-adjoint EVD: lib.rs:2367-2400, faer.h:696, 720, 6064, 6098; semantics faer/src/linalg/evd/mod.rs:270-353 (the LOWER triangle
 * of A is read; eigenvalues in nondecreasing order). U passed with ncols == 0: eigenvalues only (csrc/evd.cu); otherwise the
 * eigenvectors too (csrc/svd_vectors.cu, tridiag_dc.cu). Any n. Non-finite input: NoConvergence. */
/* evd/hessenberg.rs:17-25 (faer.h:110-113, 600): parameters of the Hessenberg reduction (the reduction itself is reached in the
 * reference through the general EVD; here as the extension faer_b200_hessenberg_in_place_<T> below) */
typedef struct FaerV0_24_HessenbergParams {
  size_t par_threshold;
  size_t blocking_threshold;
} FaerV0_24_HessenbergParams;
struct FaerV0_24_HessenbergParams libfaer_v0_23_HessenbergParams_f64(void);
struct FaerV0_24_HessenbergParams libfaer_v0_23_HessenbergParams_f32(void);
struct FaerV0_24_HessenbergParams libfaer_v0_23_HessenbergParams_c64(void);
struct FaerV0_24_HessenbergParams libfaer_v0_23_HessenbergParams_c32(void);
struct FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_f64(void);
struct FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_f32(void);
struct FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_f64(void);
struct FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_f64(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_U, struct FaerV0_24_Par par, struct FaerV0_24_SelfAdjointEvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_f32(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_U, struct FaerV0_24_Par par, struct FaerV0_24_SelfAdjointEvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_f64(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SelfAdjointEvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_f32(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SelfAdjointEvdParams params);

/* `svd` / `self_adjoint_evd` for complex T (faer.h:6238-6268, 6043-6060; csrc/cplx_condensed.cu): same semantics as the real entry
 * points; S holds T-typed entries (value, 0), its stride counts complex elements; c32 computes in c64. */
struct FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_c64(void);
struct FaerV0_24_BidiagParams libfaer_v0_23_BidiagParams_c32(void);
struct FaerV0_24_SvdParams libfaer_v0_23_SvdParams_c64(void);
struct FaerV0_24_SvdParams libfaer_v0_23_SvdParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_svd_scratch_c64(size_t nrows, size_t ncols, enum FaerV0_24_ComputeSvdVectors compute_U, enum FaerV0_24_ComputeSvdVectors compute_V, struct FaerV0_24_Par par, struct FaerV0_24_SvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_svd_scratch_c32(size_t nrows, size_t ncols, enum FaerV0_24_ComputeSvdVectors compute_U, enum FaerV0_24_ComputeSvdVectors compute_V, struct FaerV0_24_Par par, struct FaerV0_24_SvdParams params);
struct FaerV0_24_SvdStatus libfaer_v0_23_svd_c64(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_MatMut V, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SvdParams params);
struct FaerV0_24_SvdStatus libfaer_v0_23_svd_c32(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_MatMut V, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SvdParams params);
struct FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_c64(void);
struct FaerV0_24_TridiagParams libfaer_v0_23_TridiagParams_c32(void);
struct FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_c64(void);
struct FaerV0_24_SelfAdjointEvdParams libfaer_v0_23_SelfAdjointEvdParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_c64(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_U, struct FaerV0_24_Par par, struct FaerV0_24_SelfAdjointEvdParams params);
struct FaerV0_24_Layout libfaer_v0_23_self_adjoint_evd_scratch_c32(size_t dim, enum FaerV0_24_ComputeEigenvectors compute_U, struct FaerV0_24_Par par, struct FaerV0_24_SelfAdjointEvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_c64(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SelfAdjointEvdParams params);
struct FaerV0_24_EvdStatus libfaer_v0_23_self_adjoint_evd_c32(struct FaerV0_24_MatRef A, struct FaerV0_24_MatMut U, struct FaerV0_24_VecMut S, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_SelfAdjointEvdParams params);
/* triangular inverses (faer.h:3080-3170; faer-ffi/src/lib.rs:938-980; linalg/triangular_inverse.rs): the triangle of L_inv <- the
 * inverse of the triangle of L; nothing else of L_inv is written (not its diagonal for the unit variants). csrc/reconstruct_types.cu. */
void libfaer_v0_23_inverse_triangular_lower_in_place_f64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_lower_in_place_f32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_lower_in_place_c64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_lower_in_place_c32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_upper_in_place_f64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_upper_in_place_f32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_upper_in_place_c64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_triangular_upper_in_place_c32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_lower_in_place_f64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_lower_in_place_f32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_lower_in_place_c64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_lower_in_place_c32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_upper_in_place_f64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_upper_in_place_f32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_upper_in_place_c64(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
void libfaer_v0_23_inverse_unit_triangular_upper_in_place_c32(struct FaerV0_24_MatMut L_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par);
/* reconstruct / inverse on the factors (SURVEY.md appendix C, "next" row): lib.rs:1039-1075 (llt), 1661-1720 (qr), 2059-2124 (lu);
 * semantics: cholesky/llt/reconstruct.rs:12-33 and inverse.rs:10-39 (only the LOWER triangle of the output is written),
 * lu/partial_pivoting/reconstruct.rs and inverse.rs, qr/no_pivoting/reconstruct.rs:13-39 and inverse.rs. L / U may be the packed
 * LU matrix or the split factors (the excluded parts are never read). The LU and QR inverses are the solves applied to the
 * identity (csrc/reconstruct_types.cu). */
struct FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_reconstruct_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_inverse_f64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u32_f64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u64_f64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_reconstruct_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u32_f64(size_t dim, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u64_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_inverse_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_f64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_f32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_reconstruct_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_reconstruct_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_f64(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_inverse_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* the same entry points for f32 / c64 / c32 (faer-ffi stamps them for every dtype, lib.rs:313-369; csrc/reconstruct_types.cu:
 * the compositions above on the products, solves and Householder sequences of each scalar kind) */
struct FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_reconstruct_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_inverse_f32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u32_f32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u32_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u64_f32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u64_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_f32(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_inverse_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_reconstruct_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_inverse_c64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u32_c64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u32_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u64_c64(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u64_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_c64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_reconstruct_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_c64(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_inverse_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_reconstruct_scratch_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_reconstruct_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_llt_inverse_scratch_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_inverse_c32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u32_c32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u32_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_reconstruct_scratch_u64_c32(size_t nrows, size_t ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_reconstruct_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_inverse_scratch_u64_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_inverse_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_reconstruct_scratch_c32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_reconstruct_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_inverse_scratch_c32(size_t dim, size_t block_size, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_inverse_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* f32 LLT: faer.h:636 (LltParams_f32), 4036-4048 (factor), 4180-4216 (solve); same semantics as the f64 entry points.
 * The templated leaf kernel and recursive driver of csrc/llt.cu instantiated for float. */
struct FaerV0_24_LltParams libfaer_v0_23_LltParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_f32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LltParams params);
struct FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_LltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LltParams params);
struct FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_solve_in_place_f32(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* LDLT without pivoting (SURVEY.md 8f rank 3).  types: faer.h:162-165 (LdltParams), 340-344 (VecRef), 346-381 (LdltStatus,
 * LdltRegularization);  params: lib.rs:660;  factor: lib.rs:1190-1217, faer.h:3802, 3830;  solve: lib.rs:1218-1246, faer.h:3974,
 * 4004.  Semantics: faer/src/linalg/cholesky/ldlt/factor.rs:725-767 (D on the diagonal of A, unit-lower L strictly below, strict
 * upper triangle untouched; ZeroPivot { index }), solve.rs:11-49.  dynamic_regularization_signs: i8 slice or null ptr.
 * Kernels: csrc/ldlt_f64.cu (trailing updates through spicy_matmul_f64). */
struct FaerV0_24_LdltParams libfaer_v0_23_LdltParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_factor_in_place_scratch_f64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LdltParams params);
struct FaerV0_24_LdltStatus libfaer_v0_23_ldlt_factor_in_place_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_LdltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LdltParams params);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_solve_in_place_scratch_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_solve_in_place_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* LDLT for the other dtypes and `ldlt_reconstruct` / `ldlt_inverse` (faer.h:3802-4030 stamped per dtype; lib.rs:1190-1300;
 * csrc/ldlt_types.cu: the unblocked flat-map factorization of ldlt_core.cuh for f32 / c64 / c32, compositions for the rest). The
 * regularisation scalars are T::Real, D holds T-typed entries (the real parts are used), A_conj is honoured for complex T,
 * only the LOWER triangle of the reconstruct / inverse output is written (ldlt/reconstruct.rs:9-55, inverse.rs:9-60). */
struct FaerV0_24_LdltParams libfaer_v0_23_LdltParams_f32(void);
struct FaerV0_24_LdltParams libfaer_v0_23_LdltParams_c64(void);
struct FaerV0_24_LdltParams libfaer_v0_23_LdltParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_factor_in_place_scratch_f32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LdltParams params);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_factor_in_place_scratch_c64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LdltParams params);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_factor_in_place_scratch_c32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LdltParams params);
struct FaerV0_24_LdltStatus libfaer_v0_23_ldlt_factor_in_place_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_LdltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LdltParams params);
struct FaerV0_24_LdltStatus libfaer_v0_23_ldlt_factor_in_place_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_LdltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LdltParams params);
struct FaerV0_24_LdltStatus libfaer_v0_23_ldlt_factor_in_place_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_LdltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LdltParams params);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_solve_in_place_scratch_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_solve_in_place_scratch_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_solve_in_place_scratch_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_solve_in_place_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_ldlt_solve_in_place_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_ldlt_solve_in_place_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_reconstruct_scratch_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_reconstruct_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_inverse_scratch_f64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_inverse_f64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_reconstruct_scratch_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_reconstruct_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_inverse_scratch_f32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_inverse_f32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_reconstruct_scratch_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_reconstruct_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_inverse_scratch_c64(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_inverse_c64(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_reconstruct_scratch_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_reconstruct_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_ldlt_inverse_scratch_c32(size_t dim, struct FaerV0_24_Par par);
void libfaer_v0_23_ldlt_inverse_c32(struct FaerV0_24_MatMut A_inv, struct FaerV0_24_MatRef L, struct FaerV0_24_VecRef D, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* partial-pivoting LU.   params: lib.rs:679-684, faer.h:648; scratch: lib.rs:1952-1965; factor: lib.rs:1966-1983, faer.h:4456-4461 */
/* c64 (complex<f64>, interleaved) triangular solves and LLT: faer.h:6130-6143, 636, 4036-4048 / lib.rs:896-937, 984-1038 stamped
 * for c64. `L_conj` / `A_conj` are honoured (solve with conj(T)). Regularisation parameters point to f64 (Real of c64). */
void libfaer_v0_23_solve_triangular_lower_in_place_c64(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_upper_in_place_c64(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_lower_in_place_c64(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_upper_in_place_c64(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
struct FaerV0_24_LltParams libfaer_v0_23_LltParams_c64(void);
struct FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_c64(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LltParams params);
struct FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_LltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LltParams params);
struct FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_solve_in_place_c64(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* c64 partial-pivoting LU (pivot = first row attaining the largest |re| + |im|, faer-traits abs1) and the solve on its factors
 * (`A_conj` honoured): faer.h:648, 4456-4461, 4786-4884 / lib.rs:1952-2020 stamped for c64. */
struct FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_c64(void);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_c64(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_c64(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* c32 (complex<f32>, interleaved) twins of the c64 entry points above: same faer.h / lib.rs templates stamped for c32, same
 * contracts; regularisation parameters point to f32 (Real of c32). */
void libfaer_v0_23_solve_triangular_lower_in_place_c32(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_triangular_upper_in_place_c32(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_lower_in_place_c32(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj L_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
void libfaer_v0_23_solve_unit_triangular_upper_in_place_c32(struct FaerV0_24_MatRef U, enum FaerV0_24_Conj U_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par);
struct FaerV0_24_LltParams libfaer_v0_23_LltParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_llt_factor_in_place_scratch_c32(size_t dim, struct FaerV0_24_Par par, struct FaerV0_24_LltParams params);
struct FaerV0_24_LltStatus libfaer_v0_23_llt_factor_in_place_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_LltRegularization regularization, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_LltParams params);
struct FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_solve_in_place_c32(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_c32(void);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_c32(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_c32(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

struct FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_f64(void);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_f64(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_f64(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
/* f32: the same entry points; computed in f64 on the device (the matrix is widened, factored by the f64 drivers and rounded
 * back: csrc/ffi.cu), the solves on the native f32 triangular solves. faer.h:648, 4456-4461 / lib.rs:1952-2020 for f32. */
struct FaerV0_24_PartialPivLuParams libfaer_v0_23_PartialPivLuParams_f32(void);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u32_f32(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_factor_in_place_scratch_u64_f32(size_t nrows, size_t ncols, struct FaerV0_24_Par par, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u32_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);
struct FaerV0_24_PartialPivLuStatus libfaer_v0_23_partial_piv_lu_factor_in_place_u64_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_SliceMut perm_fwd, struct FaerV0_24_SliceMut perm_bwd, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_PartialPivLuParams params);

/* Householder QR without pivoting + block-Householder sequence application, f64 and f32.
 * params: faer-ffi/src/lib.rs:671-675, faer.h:670; recommended_block_size: lib.rs:1520-1527, faer.h:5718;
 * scratch/factor: lib.rs:1528-1558, faer.h:5592-5602; apply_householder_*: lib.rs:1423-1518, faer.h:754-759.
 * Q_coeff is block_size x min(nrows, ncols): one upper-triangular T block per block of columns (tau on the diagonal,
 * faer's convention tau = (1 + |v_tail|^2)/2). Rank-deficient inputs take the reference's
 * column-skipping path (exact `rank`, +inf on the skipped T diagonals). */
struct FaerV0_24_QrParams libfaer_v0_23_QrParams_f64(void);
struct FaerV0_24_QrParams libfaer_v0_23_QrParams_f32(void);
size_t libfaer_v0_23_qr_recommended_block_size_f64(size_t nrows, size_t ncols);
size_t libfaer_v0_23_qr_recommended_block_size_f32(size_t nrows, size_t ncols);
struct FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_f64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_QrParams params);
struct FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_f32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_QrParams params);
struct FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_QrParams params);
struct FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_QrParams params);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_f64(size_t dim, size_t block_size, size_t rhs_ncols);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_f32(size_t dim, size_t block_size, size_t rhs_ncols);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_f64(size_t dim, size_t block_size, size_t rhs_ncols);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_f32(size_t dim, size_t block_size, size_t rhs_ncols);
void libfaer_v0_23_apply_householder_on_the_left_f64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_on_the_left_f32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_left_f64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_left_f32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* on the right: lib.rs:1471-1518; householder.rs:813-854 (lhs <- lhs Q  and  lhs <- lhs Q^H through the transposed view) */
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_f64(size_t dim, size_t block_size, size_t lhs_nrows);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_f64(size_t dim, size_t block_size, size_t lhs_nrows);
void libfaer_v0_23_apply_householder_on_the_right_f64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_right_f64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_f32(size_t dim, size_t block_size, size_t lhs_nrows);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_f32(size_t dim, size_t block_size, size_t lhs_nrows);
void libfaer_v0_23_apply_householder_on_the_right_f32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_right_f32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* solves on top of the factors (SURVEY.md §8f).   llt: faer-ffi/src/lib.rs:1012-1038, faer.h:4188, 4216;
 * LU: lib.rs:1985-2020, faer.h:4786, 4884. L and U are views of the factored matrix (L: unit-lower part, U: upper part). */
struct FaerV0_24_Layout libfaer_v0_23_llt_solve_in_place_scratch_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_llt_solve_in_place_f64(struct FaerV0_24_MatRef L, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs,
                                          struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
/* A^T x = b from the same factors: lib.rs:2021-2060, faer.h:4918, 4942, 4986, 5040; lu/partial_pivoting/solve.rs:55-86
 * (lower solve with U^T, unit-upper solve with L^T, rows permuted by the inverse permutation = perm_bwd). */
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_f64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_f64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u32_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_in_place_scratch_u64_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u32_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_in_place_u64_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_f32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_f32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* solves on the QR factors: faer-ffi/src/lib.rs:1560-1660 (qr_solve_in_place[_scratch] 1560-1592,
 * qr_solve_transpose_in_place[_scratch] 1593-1625, qr_solve_lstsq_in_place[_scratch] 1626-1660); faer.h:5828, 5864, 5906,
 * 5946, 5990, 6026 (f64; the f32 declarations are the neighbouring ones). Semantics: faer/src/linalg/qr/no_pivoting/solve.rs:38-76
 * (lstsq: rhs <- Q^H rhs, then the upper solve with R[..size, ..] on the first `size` rows of rhs; the solution is
 * rhs[..ncols, ..]), 96-119 (square solve), 140-176 (transpose solve). Q_basis and R are normally the same packed
 * matrix returned by qr_factor_in_place. Real types: A_conj is a no-op. */
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_f64(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_f64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_f64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_solve_lstsq_in_place_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_in_place_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_transpose_in_place_f64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_f32(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_f32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_f32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_solve_lstsq_in_place_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_in_place_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_transpose_in_place_f32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* global parallelism + allocation helpers.   faer-ffi/src/lib.rs:2521-2569, faer.h:724, 2034, 3080, 6108 */
struct FaerV0_24_Par libfaer_v0_23_get_global_par(void);
void libfaer_v0_23_set_global_par(struct FaerV0_24_Par par);
void *libfaer_v0_23_alloc(size_t size, size_t align);
void libfaer_v0_23_dealloc(void *ptr, size_t size, size_t align);

/* =====================================================================================================
 * GPU-only extensions (not in faer.h; kept in a separate namespace so faer.h layouts stay identical)
 * ===================================================================================================== */
/* Number of CUDA devices visible (0 => every compute entry point aborts). */
int faer_b200_device_count(void);
/* Stream used by subsequent calls from this process (cudaStream_t passed as void*; NULL = default stream). */
void faer_b200_set_stream(void *cuda_stream);
/* Number of kernels this library has launched since load (for bench.py's gpu_launches). */
unsigned long long faer_b200_launch_count(void);
/* Launch-phase log: between begin and end, each launch of this library stores its phase in tags[i] (i < capacity; 0 other,
 * 1 dd QR panel, 2 Householder products, 3 T-factor builds); end() returns the number of launches, which may exceed capacity. */
void faer_b200_launch_log_begin(signed char *tags, size_t capacity);
size_t faer_b200_launch_log_end(void);
/* Free the cached device workspace. */
void faer_b200_release_workspace(void);
/* Per-launch timing of the dominant kernel (the DMMA GEMM): between begin and end every GEMM launch is bracketed by
 * CUDA events on the launching stream; end() returns the summed algorithmic flop, summed kernel ms and launch count. */
void faer_b200_profile_begin(void);
void faer_b200_profile_end(double *flops, double *ms, unsigned long long *count);
/* ---- multi-GPU: one process per GPU, 1-D block-column-cyclic layout, NCCL panel broadcast (no reference
 * counterpart: faer is single-process; SURVEY.md §8e). Rank 0 obtains a 128-byte id, the caller ships it to the
 * other ranks (e.g. torch.distributed broadcast), every rank calls dist_init (collective). A_local is the DEVICE
 * column-major n x (local columns) matrix holding the block columns b with b % nranks == rank, in increasing b.
 * The returned status is this rank's view (only the owner of a failing panel sees NonPositivePivot): reduce it
 * over the ranks with the caller's process group. Works without dist_init as a single-rank run. */
int faer_b200_dist_unique_id(void *out128);
int faer_b200_dist_init(int rank, int nranks, const void *id128);
void faer_b200_dist_finalize(void);
struct FaerV0_24_LltStatus faer_b200_dist_llt_factor_in_place_f64(void *A_local, size_t ld, size_t n, size_t nb,
                                                                  struct FaerV0_24_LltRegularization regularization,
                                                                  int lookahead);
/* Distributed P A = L U (square). perm_fwd / perm_inv: HOST int64[n], identical on every rank. Returns the
 * transposition count. Pivots are identical to the single-GPU entry point's. */
size_t faer_b200_dist_partial_piv_lu_factor_in_place_f64(void *A_local, size_t ld, size_t n, size_t nb,
                                                         long long *perm_fwd, long long *perm_inv, int lookahead);
/* Distributed Householder QR without pivoting (SURVEY.md 8e: the owner factors its block column, broadcasts the factored panel
 * and its T block, every rank applies the block reflector to its own columns). nrows >= ncols; the layout's block width is the
 * Householder block size `block_size` (the reference's Q_coeff.nrows, qr/no_pivoting/factor.rs:258-301). Q_coeff: DEVICE,
 * block_size x ncols column-major with leading dimension block_size, replicated (every rank ends with all T blocks).
 * Returns ncols, or -1 (on every rank) when a block is rank-deficient: use the single-GPU entry point for such inputs.
 * `flags` bit 1: purely local run that ignores an existing communicator. */
long long faer_b200_dist_qr_factor_in_place_f64(void *A_local, size_t ld, size_t nrows, size_t ncols, size_t block_size,
                                                void *Q_coeff, int flags);
long long faer_b200_dist_qr_factor_in_place_f32(void *A_local, size_t ld, size_t nrows, size_t ncols, size_t block_size,
                                                void *Q_coeff, int flags);
/* ---- reduction to bidiagonal form A = U B V^H (nrows >= ncols). faer-ffi does not export this stage on its own (it is
 * reached through libfaer_v0_23_svd_*, faer-ffi/src/lib.rs:2345-2366 -> faer/src/linalg/svd/mod.rs:326-431); the entry
 * mirrors the Rust function it replaces, faer::linalg::svd::bidiag::bidiag_in_place (faer/src/linalg/svd/bidiag.rs:47-54):
 * B on A's diagonal / superdiagonal, left reflectors below the diagonal with H_left (bl x ncols) holding their T blocks,
 * right reflectors right of the superdiagonal with H_right (br x (ncols-1)). Any layout (views that are not column-major go through a
 * compact column-major copy). */
void faer_b200_bidiag_in_place_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut H_left, struct FaerV0_24_MatMut H_right);
void faer_b200_bidiag_in_place_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut H_left, struct FaerV0_24_MatMut H_right);
/* complex T: the functional unblocked sequences of csrc/cplx_condensed_core.cuh (any layout) */
void faer_b200_bidiag_in_place_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut H_left, struct FaerV0_24_MatMut H_right);
void faer_b200_bidiag_in_place_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut H_left, struct FaerV0_24_MatMut H_right);
/* ---- reduction to tridiagonal form A = Q T Q^H of a self-adjoint matrix (lower triangle read and written). Reached in the reference through libfaer_v0_23_self_adjoint_evd_* (faer-ffi/src/lib.rs:2382-2400 ->
 * faer/src/linalg/evd/mod.rs); mirrors faer::linalg::evd::tridiag::tridiag_in_place (faer/src/linalg/evd/tridiag.rs:274-280):
 * T on A's diagonal / subdiagonal, reflectors below the subdiagonal, `householder` (b x (n-1)) holds their T blocks. */
void faer_b200_tridiag_in_place_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
void faer_b200_tridiag_in_place_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
void faer_b200_tridiag_in_place_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
void faer_b200_tridiag_in_place_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
/* ---- reduction to upper Hessenberg form A = Q H Q^H (general square matrix). faer-ffi exports only the parameter structs of this
 * stage (FaerV0_24_HessenbergParams, faer.h:110-113); the entry mirrors faer::linalg::evd::hessenberg::hessenberg_in_place (faer/src/linalg/evd/hessenberg.rs:549-567):
 * H in the entries (i, j) with i <= j + 1, the reflectors of Q = H_0 ... H_{n-2} below the subdiagonal, `householder` (b x (n-1))
 * holds their T blocks. Functional (the unblocked flat-map sequence of csrc/cplx_condensed_core.cuh; real dtypes run it on (x, 0)). */
void faer_b200_hessenberg_in_place_f64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
void faer_b200_hessenberg_in_place_f32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
void faer_b200_hessenberg_in_place_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
void faer_b200_hessenberg_in_place_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut householder);
/* "spicy" matmul: C[row_idx[i], col_idx[j]] (+)= alpha * (A diag(D) B)[i, j] for the (i, j) that C_block keeps (block structure
 * of the PRODUCT). Mirrors faer::linalg::matmul::internal::spicy_matmul (faer/src/linalg/matmul/internal/mod.rs:45-58), which
 * faer-ffi does not export (it is an internal of LDLT and of the sparse supernodal Cholesky): row_idx / col_idx may be NULL
 * (then C has A.nrows rows / B.ncols columns), D (A.ncols entries) may be NULL; host or device pointers. Real f64. */
void faer_b200_spicy_matmul_f64(struct FaerV0_24_MatMut C, enum FaerV0_24_Block C_block, const unsigned long long *row_idx,
                                size_t nrow_idx, const unsigned long long *col_idx, size_t ncol_idx, enum FaerV0_24_Accum accum,
                                struct FaerV0_24_MatRef A, struct FaerV0_24_MatRef B, const double *D,
                                const struct FaerV0_24_Scalar *alpha);
/* Inner seam: the type-erased product call faer makes at matmul/mod.rs:1373-1411 (DstKind::Full), matmul/triangular.rs:641-680
 * (DstKind::Lower / Upper) and matmul/internal/mod.rs:143-201 (row / column scatter + diagonal scaling) into
 * `private_gemm_x86::gemm`, with that function's parameter list: a Rust build of faer can swap the backend at those three call
 * sites by forwarding the arguments unchanged (the crate's enums are translated to the constants below; INTEGRATION.md shows it).
 *   dst[row_idx[i], col_idx[j]] (+)= alpha * sum_k conj?(lhs[i, k]) * diag[k * diag_stride] * conj?(rhs[k, j])
 * for the (i, j) that dst_kind keeps (Lower: i >= j, Upper: i <= j; both include the diagonal, as the reference asks the backend
 * for the inclusive trapezoid, triangular.rs:633-640). row_idx / col_idx / diag may be NULL. Strides in elements. Pointers may be
 * host or device pointers. `instr_set` and `n_threads` are accepted and ignored. Index scatter and diagonal scaling: f64. */
enum FaerB200_GemmDType { FaerB200_GemmDType_F32 = 0, FaerB200_GemmDType_F64 = 1, FaerB200_GemmDType_C32 = 2, FaerB200_GemmDType_C64 = 3 };
enum FaerB200_GemmIType { FaerB200_GemmIType_U32 = 0, FaerB200_GemmIType_U64 = 1 };
enum FaerB200_GemmDstKind { FaerB200_GemmDstKind_Lower = 0, FaerB200_GemmDstKind_Upper = 1, FaerB200_GemmDstKind_Full = 2 };
void faer_b200_gemm(int dtype, int itype, int instr_set, size_t m, size_t n, size_t k, void *dst, ptrdiff_t dst_rs, ptrdiff_t dst_cs,
                    const void *row_idx, const void *col_idx, int dst_kind, int accum /* 0 Replace, 1 Add */, const void *lhs,
                    ptrdiff_t lhs_rs, ptrdiff_t lhs_cs, bool conj_lhs, const void *diag, ptrdiff_t diag_stride, const void *rhs,
                    ptrdiff_t rhs_rs, ptrdiff_t rhs_cs, bool conj_rhs, const void *alpha, size_t n_threads);
/* Run-time options (initial values from the environment variable in brackets). Returns 0, or -1 for an unknown name.
 *   "gemm_ws"        [FAER_B200_GEMM_WS]        0 never / 1 heuristic (default) / 2 always use the TMA-fed warp-specialised
 *                                                f64 GEMM (csrc/gemm_f64_ws.cuh) where the operands qualify, 128 x 64 tiles /
 *                                                3 always, 128 x 128 tiles (spicy_matmul: as 1)
 *   "f64_gemm_mode"  [FAER_B200_F64_GEMM_MODE]  0 native f64 tensor op (default) / 1 int8-sliced wgmma products for large  
 *                                                unstructured matmuls (csrc/gemm_f64_sliced.cuh states the accuracy contract) */
int faer_b200_set_option(const char *name, long long value);
long long faer_b200_get_option(const char *name);
/* Version string. */
const char *faer_b200_version(void);

/* complex (c64 / c32, interleaved) Householder QR without pivoting, the block-Householder sequence applications and the QR solves:
 * the same faer.h / lib.rs templates as the f64 / f32 entry points above stamped for c64 / c32 (qr/no_pivoting/factor.rs:11-301 with
 * the exact rank of the reference's column-skipping path, householder.rs:724-854, qr/no_pivoting/solve.rs:38-176). The conjugation
 * arguments (`householder_conj`, `A_conj`) are honoured. */
struct FaerV0_24_QrParams libfaer_v0_23_QrParams_c64(void);
struct FaerV0_24_QrParams libfaer_v0_23_QrParams_c32(void);
size_t libfaer_v0_23_qr_recommended_block_size_c64(size_t nrows, size_t ncols);
size_t libfaer_v0_23_qr_recommended_block_size_c32(size_t nrows, size_t ncols);
struct FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_c64(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_QrParams params);
struct FaerV0_24_Layout libfaer_v0_23_qr_factor_in_place_scratch_c32(size_t nrows, size_t ncols, size_t block_size, struct FaerV0_24_Par par, struct FaerV0_24_QrParams params);
struct FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_c64(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_QrParams params);
struct FaerV0_24_QrStatus libfaer_v0_23_qr_factor_in_place_c32(struct FaerV0_24_MatMut A, struct FaerV0_24_MatMut Q_coeff, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem, struct FaerV0_24_QrParams params);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_c64(size_t dim, size_t block_size, size_t rhs_ncols);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_left_scratch_c32(size_t dim, size_t block_size, size_t rhs_ncols);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_c64(size_t dim, size_t block_size, size_t rhs_ncols);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_left_scratch_c32(size_t dim, size_t block_size, size_t rhs_ncols);
void libfaer_v0_23_apply_householder_on_the_left_c64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_on_the_left_c32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_left_c64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_left_c32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_c64(size_t dim, size_t block_size, size_t lhs_nrows);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_on_the_right_scratch_c32(size_t dim, size_t block_size, size_t lhs_nrows);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_c64(size_t dim, size_t block_size, size_t lhs_nrows);
struct FaerV0_24_Layout libfaer_v0_23_apply_householder_transpose_on_the_right_scratch_c32(size_t dim, size_t block_size, size_t lhs_nrows);
void libfaer_v0_23_apply_householder_on_the_right_c64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_on_the_right_c32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_right_c64(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_apply_householder_transpose_on_the_right_c32(struct FaerV0_24_MatRef householder_basis, struct FaerV0_24_MatRef householder_factor, enum FaerV0_24_Conj householder_conj, struct FaerV0_24_MatMut lhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_c64(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_lstsq_in_place_scratch_c32(size_t nrows, size_t ncols, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_c64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_in_place_scratch_c32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_c64(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_qr_solve_transpose_in_place_scratch_c32(size_t dim, size_t block_size, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_qr_solve_lstsq_in_place_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_lstsq_in_place_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_in_place_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_in_place_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_transpose_in_place_c64(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_qr_solve_transpose_in_place_c32(struct FaerV0_24_MatRef Q_basis, struct FaerV0_24_MatRef Q_coeff, struct FaerV0_24_MatRef R, enum FaerV0_24_Conj A_conj, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

/* complex partial-pivoting LU: the transpose solve (lu/partial_pivoting/solve.rs:55-86; `A_conj` honoured, `perm_bwd` is the one read) */
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u32_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_c64(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
struct FaerV0_24_Layout libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_scratch_u64_c32(size_t dim, size_t rhs_ncols, struct FaerV0_24_Par par);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u32_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_c64(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);
void libfaer_v0_23_partial_piv_lu_solve_transpose_in_place_u64_c32(struct FaerV0_24_MatRef L, struct FaerV0_24_MatRef U, enum FaerV0_24_Conj A_conj, struct FaerV0_24_SliceRef perm_fwd, struct FaerV0_24_SliceRef perm_bwd, struct FaerV0_24_MatMut rhs, struct FaerV0_24_Par par, struct FaerV0_24_MemAlloc mem);

#ifdef __cplusplus
}
#endif

/* pivoted Cholesky (piv_llt_*): declared in its own header */
#include "faer_b200_piv_llt.h"
/* column-pivoted QR (colpiv_qr_*): declared in its own header */
#include "faer_b200_colpiv_qr.h"
/* full-pivoting LU (full_piv_lu_*): declared in its own header */
#include "faer_b200_full_piv_lu.h"
/* Bunch-Kaufman LBLT (lblt_*): declared in its own header */
#include "faer_b200_lblt.h"
#include "faer_b200_evd.h"
#include "faer_b200_fx128.h"
#include "faer_b200_fx128_qr.h"
#include "faer_b200_fx128_evd.h"
#include "faer_b200_fx128_svd.h"

#endif /* LIBFAER_V0_24 */
