// P1 + driver: in-place lower Cholesky (LLT), f64 and f32 (one templated leaf kernel and recursive driver).
//
// Reference: faer/src/linalg/cholesky/llt/factor.rs:68-97 -> ldlt/factor.rs:367-498
// (`cholesky_recursion_right_looking`: for each block column: factor A00, A10 <- A10 * L00^-H,
//  A11(lower) -= A10 * A10^H), leaf recurrence ldlt/factor.rs:7-177 / 299-366:
//     a_ij <- fma(-conj(a_jk), a_ik, a_ij)  for k = 0..j-1 (in k order),
//     d = Re(a_jj); [regularise]; fail with Err(j) if !(d > 0); l_jj = sqrt(d); fail if l_jj == 0 or non-finite;
//     column j (INCLUDING the diagonal entry) is multiplied by recip(l_jj).
//
// GPU mapping: recursive blocked driver on the host stream; the <=128-wide diagonal block is factored by ONE CTA that
// keeps it in shared memory and works through it in 32-column panels without a CTA barrier per column (potf2_kernel).
// The panel solve is G3 and the trailing update is the lower-masked DMMA GEMM (G2). A device status word carries the
// first failing column / the regularisation count and is read back once per factorisation.
#include <atomic>

#include "gemm_f32.cuh"
#include "linalg_f64.cuh"

namespace fb {

namespace {

constexpr int POTF2_MAX = 128;
constexpr int POTF2_W = 32;                             // panel width: one diagonal-block row per lane
constexpr int POTF2_PANEL_WARPS = POTF2_MAX / POTF2_W;  // warps that factor a panel, 32 rows each
constexpr int POTF2_WARPS = 8;
constexpr int POTF2_THREADS = POTF2_WARPS * 32;
constexpr int POTF2_TN = 4;                             // trailing update: columns per warp tile

__device__ __forceinline__ double recip_rn(double x) { return __drcp_rn(x); }
__device__ __forceinline__ float recip_rn(float x) { return __frcp_rn(x); }
template <class T>
struct __align__(2 * sizeof(T)) Pair {
  T x, y;
};

// scalar-type dispatch of the two building blocks the recursion calls (G3 solve, lower-masked GEMM)
inline void solve_lower(cudaStream_t st, VCD tri, bool unit, VD rhs) { solve_lower_triangular_in_place_f64(st, tri, unit, rhs); }
inline void solve_lower(cudaStream_t st, VCF tri, bool unit, VF rhs) { solve_lower_triangular_in_place_f32(st, tri, unit, rhs); }
// dst(lower) -= a * a^H
inline void gemm_lower_update(cudaStream_t st, VD dst, VCD a) { gemm_f64(st, dst, TRI_LOWER, 1, a, RECT, a.t(), RECT, -1.0); }
inline void gemm_lower_update(cudaStream_t st, VF dst, VCF a) { gemm_f32(st, dst, TRI_LOWER, 1, a, RECT, a.t(), RECT, -1.0f); }

// One CTA factors an n <= 128 diagonal block held in shared memory, S[c * POTF2_MAX + i] = a_ic, in 32-column panels:
//   1. warps 0-3 factor the panel: warp w holds the panel's rows p0 + 32w + lane in registers (warp 0: the diagonal
//      block's rows), and every one of them also holds the diagonal block's rows and factors that block itself, warp
//      synchronously: the pivot comes from lane c by shuffle, the column of L travels through a warp-private buffer.
//      Warps 1-3 thereby run the forward substitution of the rows below the diagonal block without waiting for warp 0;
//   2. all warps apply the panel to the trailing lower triangle (32 FMAs per element).
// Three CTA barriers per panel instead of one per column. The arithmetic is the reference leaf's, element by element:
// a_ic <- fma(-l_ck, l_ik, a_ic) for k = 0..c-1 in ascending order, l_xk = (updated a_xk) * recip_rn(sqrt(d_k)), and
// the diagonal entry is scaled with the rest of its column; the four warps compute the diagonal block's bits
// identically, so the pivot decisions are the same in all of them and every branch below is warp- or CTA-uniform.
// info[0]: first failing global column (or -1), info[1]: regularisation count. On a failure at column f, columns < f
// hold L and the rest of A is left as it was; the count is not added.
template <class T>
__global__ void __launch_bounds__(POTF2_THREADS, 1) potf2_kernel(T* __restrict__ A, i64 rs, i64 cs, int n, i64 j0,
                                                                  int regularize, T eps, T delta,
                                                                  long long* __restrict__ info) {
  extern __shared__ __align__(16) unsigned char potf2_smem[];
  T* S = reinterpret_cast<T*>(potf2_smem);  // columns 0 .. roundup(n, 32) - 1
  __shared__ __align__(16) T colv[POTF2_PANEL_WARPS][2][2 * POTF2_W];
  __shared__ int s_fail, s_count;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (info[0] >= 0) return;  // an earlier block already failed (uniform across the CTA)

  // the whole block in flight at once, zero-filled outside the lower triangle
  const int ncol = (n + POTF2_W - 1) & ~(POTF2_W - 1);
  for (int e = tid; e < ncol * POTF2_MAX; e += POTF2_THREADS) {
    const int i = e % POTF2_MAX, c = e / POTF2_MAX;
    const bool ok = i < n && c <= i;
    const T* src = ok ? A + (i64)i * rs + (i64)c * cs : A;
    if constexpr (sizeof(T) == 8) cp_async_8(S + e, src, ok ? 8 : 0);
    else cp_async_4(S + e, src, ok ? 4 : 0);
  }
  cp_async_commit();
  cp_async_wait<0>();
  if (tid == 0) {
    s_fail = -1;
    s_count = 0;
  }
  __syncthreads();

  for (int p0 = 0; p0 < n; p0 += POTF2_W) {
    T* P = S + p0 * POTF2_MAX;  // the panel's first column
    const int wp = min(POTF2_W, n - p0);
    const int r = p0 + POTF2_W * warp + lane;  // this lane's row of the panel
    const bool factors = warp < POTF2_PANEL_WARPS && p0 + POTF2_W * warp < n;
    T ad[POTF2_W], ar[POTF2_W];  // row p0 + lane of the diagonal block, row r of the panel
    if (factors) {
#pragma unroll
      for (int c = 0; c < POTF2_W; ++c) {
        ad[c] = P[c * POTF2_MAX + p0 + lane];
        ar[c] = P[c * POTF2_MAX + r];
      }
    }
    __syncthreads();  // every copy of the diagonal block is read before warp 0 overwrites it with L

    if (factors) {
      int cnt = 0, fail = -1;
      T dn = ad[0];  // lane c: the diagonal entry of column c, updated through column c - 1
      // One rolled iteration per column, so that the loop stays in the instruction cache: fully unrolled over the 32
      // columns the kernel was ~8k instructions, and inside the LLT step, where the bulk update keeps L2 busy, its
      // instruction fetches made it 3x slower than on an idle GPU. ad[k] / ar[k] hold column c + k, and each column's
      // update also shifts the rows down by one slot (ad[k] <- fma(., ., ad[k + 1])), so the current column is always
      // slot 0 and every register index stays a compile-time constant.
#pragma unroll 1
      for (int c = 0; c < wp; ++c) {
        // pivot (reference ldlt/factor.rs:122-160); d is the same in every lane
        T d = __shfl_sync(0xffffffffu, dn, c);
        if (regularize) {
          if (d <= eps) {  // LLT: sign == +1
            d = delta;
            ++cnt;
          }
        }
        T inv = T(0);
        bool bad = !(d > T(0));
        if (!bad) {
          const T sd = sqrt(d);
          if (sd == T(0) || !isfinite(sd)) bad = true;
          else inv = recip_rn(sd);  // correctly rounded reciprocal = T(1) / sd bit for bit, without the division's slow path
        }
        if (bad) {
          fail = p0 + c;
          break;
        }
        // NB: like the reference, the stored diagonal is (unregularised a_cc) * recip(l_cc)
        // (ldlt/factor.rs:161-175 scales the whole column, diagonal included, and `diag` is a local copy).
        const T ld = ad[0] * inv, lr = ar[0] * inv;
        if (r >= p0 + c && r < n) P[c * POTF2_MAX + r] = lr;
        // l of diagonal-block row `lane` goes to slot W - 1 + lane - c: the entry of column c + 1 + k is slot W + k
        T* cv = colv[warp][c & 1];  // double-buffered: column c + 1 writes the other half
        cv[POTF2_W - 1 + lane - c] = ld;
        __syncwarp();
        dn = fma(-ld, ld, ad[1]);  // lane c + 1's own l: the next pivot does not wait for the buffer
        const int live = wp - 1 - c;  // columns of the panel after c; slots from `live` on are never read again
        const Pair<T>* cp = reinterpret_cast<const Pair<T>*>(cv + POTF2_W);
#pragma unroll
        for (int q = 0; q < POTF2_W / 2; ++q) {
          if (q % 4 == 0 && 2 * q >= live) break;  // warp-uniform, in steps of 8 slots
          const Pair<T> l2 = cp[q];
          ad[2 * q] = fma(-l2.x, ld, ad[2 * q + 1]);
          ar[2 * q] = fma(-l2.x, lr, ar[2 * q + 1]);
          if (2 * q + 2 < POTF2_W) {
            ad[2 * q + 1] = fma(-l2.y, ld, ad[2 * q + 2]);
            ar[2 * q + 1] = fma(-l2.y, lr, ar[2 * q + 2]);
          }
        }
      }
      if (tid == 0) {
        s_count += cnt;
        s_fail = fail;
      }
    }
    __syncthreads();
    if (s_fail >= 0) break;

    // trailing update of columns [p0 + 32, n): warp tiles of 4 columns x 128 rows, row slots below the diagonal only
    for (int cg = p0 + POTF2_W + POTF2_TN * warp; cg < n; cg += POTF2_TN * POTF2_WARPS) {
      T acc[4][POTF2_TN];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int j = 0; j < POTF2_TN; ++j) acc[a][j] = S[(cg + j) * POTF2_MAX + 32 * a + lane];
#pragma unroll
      for (int k = 0; k < POTF2_W; ++k) {
        const T* Lk = P + k * POTF2_MAX;
        T lc[POTF2_TN];
#pragma unroll
        for (int j = 0; j < POTF2_TN; ++j) lc[j] = Lk[cg + j];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          if (32 * a + 31 >= cg && 32 * a < n) {  // warp-uniform: the slot meets the lower triangle
            const T li = Lk[32 * a + lane];
#pragma unroll
            for (int j = 0; j < POTF2_TN; ++j) acc[a][j] = fma(-lc[j], li, acc[a][j]);
          }
        }
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
        if (32 * a + 31 >= cg && 32 * a < n)
#pragma unroll
          for (int j = 0; j < POTF2_TN; ++j) S[(cg + j) * POTF2_MAX + 32 * a + lane] = acc[a][j];
    }
    __syncthreads();
  }

  const int fail = s_fail;
  const int done = fail >= 0 ? fail : n;  // columns of L to store
  for (int e = tid; e < done * POTF2_MAX; e += POTF2_THREADS) {
    const int i = e % POTF2_MAX, c = e / POTF2_MAX;
    if (i >= c && i < n) A[(i64)i * rs + (i64)c * cs] = S[e];
  }
  if (tid == 0) {
    if (fail >= 0) info[0] = j0 + fail;
    else if (s_count) info[1] += s_count;
  }
}

// potf2_kernel on the block; the shared-memory opt-in is set once per device
template <class T>
void potf2(cudaStream_t stream, View<T> A, i64 j0, int regularize, T eps, T delta, long long* d_info) {
  static std::atomic<unsigned long long> opted{0};
  int dev = 0;
  FB_CUDA_CHECK(cudaGetDevice(&dev));
  FB_ASSERT(dev < 64, "device index out of range");
  if (!(opted.load() >> dev & 1)) {
    FB_CUDA_CHECK(cudaFuncSetAttribute(potf2_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(POTF2_MAX * POTF2_MAX * sizeof(T))));
    opted.fetch_or(1ull << dev);
  }
  const int n = (int)A.nrows;
  const size_t smem = (size_t)((n + POTF2_W - 1) / POTF2_W * POTF2_W) * POTF2_MAX * sizeof(T);
  potf2_kernel<T><<<1, POTF2_THREADS, smem, stream>>>(A.ptr, A.rs, A.cs, n, j0, regularize, eps, delta, d_info);
  FB_CUDA_CHECK(cudaGetLastError());
  note_launch();
}

template <class T>
struct LltCtx {
  cudaStream_t stream;
  int regularize;
  T eps, delta;
  long long* d_info;
  i64 nb;  // leaf (diagonal block) size, <= POTF2_MAX
};

// Recursive blocked LLT. Same dataflow as the reference's right-looking recursion (factor A00, solve the panel,
// update the trailing lower triangle, continue) but split in HALVES instead of fixed 128-wide steps, so that
// almost all flops are DMMA GEMMs with a large contracted dimension (k = n/2, n/4, ...): the trailing matrix is
// read/written O(log n) times instead of n/128 times. Leaves (<= nb) are the single-CTA potf2 kernel.
template <class T>
void llt_rec(const LltCtx<T>& ctx, View<T> A, i64 j0) {
  const i64 n = A.nrows;
  if (n <= ctx.nb) {
    potf2<T>(ctx.stream, A, j0, ctx.regularize, ctx.eps, ctx.delta, ctx.d_info);
    return;
  }
  // split at a multiple of the leaf size closest to n/2
  i64 n1 = ((n / 2 + ctx.nb - 1) / ctx.nb) * ctx.nb;
  if (n1 >= n) n1 = ((n - 1) / ctx.nb) * ctx.nb;
  const i64 n2 = n - n1;
  View<T> A11 = A.sub(0, 0, n1, n1), A21 = A.sub(n1, 0, n2, n1), A22 = A.sub(n1, n1, n2, n2);
  llt_rec(ctx, A11, j0);
  // conj(L11) X = A21^T   (reference ldlt/factor.rs:421-426)
  solve_lower(ctx.stream, cv(A11), false, A21.t());
  // A22(lower) += -1 * A21 * A21^H   (reference ldlt/factor.rs:435-446)
  gemm_lower_update(ctx.stream, A22, cv(A21));
  llt_rec(ctx, A22, j0 + n1);
}

}  // namespace

namespace {
// the recursive driver with its own status word (one read-back per factorisation)
template <class T>
LltResult llt_recursive_in_place(cudaStream_t stream, View<T> A, T reg_delta, T reg_eps, LltParams params) {
  LltResult res{true, 0, 0};
  const int regularize = (reg_delta > T(0) && reg_eps > T(0)) ? 1 : 0;
  i64 nb = (i64)params.block_size;
  if (nb <= 0 || nb > POTF2_MAX) nb = POTF2_MAX;

  long long* d_info = (long long*)ws_alloc(2 * sizeof(long long));
  long long h_info[2] = {-1, 0};
  FB_CUDA_CHECK(cudaMemcpyAsync(d_info, h_info, sizeof(h_info), cudaMemcpyHostToDevice, stream));

  LltCtx<T> ctx{stream, regularize, reg_eps, reg_delta, d_info, nb};
  llt_rec<T>(ctx, A, 0);

  FB_CUDA_CHECK(cudaMemcpyAsync(h_info, d_info, sizeof(h_info), cudaMemcpyDeviceToHost, stream));
  FB_CUDA_CHECK(cudaStreamSynchronize(stream));
  ws_free(d_info);
  if (h_info[0] >= 0) {
    res.ok = false;
    res.non_positive_pivot_index = (size_t)h_info[0];
  } else {
    res.dynamic_regularization_count = (size_t)h_info[1];
  }
  return res;
}
}  // namespace

// Device-side variant for callers that own the status word (multi-GPU driver): no synchronisation, no read-back.
// d_info[0] must hold -1 (or the first failing column of an earlier block), d_info[1] the regularisation count.
void llt_cholesky_device_f64(cudaStream_t stream, VD A, double reg_delta, double reg_eps, long long* d_info, i64 j0) {
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  if (A.nrows == 0) return;
  const int regularize = (reg_delta > 0.0 && reg_eps > 0.0) ? 1 : 0;
  LltCtx<double> ctx{stream, regularize, reg_eps, reg_delta, d_info, POTF2_MAX};
  llt_rec<double>(ctx, A, j0);
}

LltResult llt_cholesky_in_place_f64(cudaStream_t stream, VD A, double reg_delta, double reg_eps, LltParams params) {
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  const i64 n = A.nrows;
  LltResult res{true, 0, 0};
  if (n == 0) return res;
  // Large column-major problems: right-looking block-column driver with two-stream look-ahead (dist.cu run on a
  // single rank): the panel chain (potf2 + solves of block column k+1) overlaps the trailing update of step k.
  if (A.rs == 1 && n >= lookahead_min_n()) {
    // block width: with the trailing update of a step as ONE structured launch, 512-wide blocks while the trailing matrix
    // is large, then 256, then 128 in the tail keep the panel chain short (dist.cu: llt_block_bounds); FAER_B200_NB
    // overrides the 512 / 256 tiers with one width
    if (lookahead_block()) return dist_llt_f64(A.ptr, A.cs, n, lookahead_block(), reg_delta, reg_eps, /*lookahead | local*/ 3);
    return dist_llt_f64(A.ptr, A.cs, n, 256, reg_delta, reg_eps, /*lookahead | local | wide head*/ 7);
  }
  return llt_recursive_in_place<double>(stream, A, reg_delta, reg_eps, params);
}

// f32: the same leaf kernel and recursive driver instantiated for float (trailing updates on the 3xTF32 GEMM — wgmma for large
// products —, panel solves on the f32 triangular solve). The look-ahead block-column drivers (dist.cu) are f64-only.
LltResult llt_cholesky_in_place_f32(cudaStream_t stream, VF A, float reg_delta, float reg_eps, LltParams params) {
  FB_ASSERT(A.nrows == A.ncols, "LLT needs a square matrix");
  if (A.nrows == 0) return LltResult{true, 0, 0};
  return llt_recursive_in_place<float>(stream, A, reg_delta, reg_eps, params);
}

}  // namespace fb
