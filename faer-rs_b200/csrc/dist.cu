// Multi-GPU (one process per GPU) 1-D block-column-cyclic factorizations with NCCL panel broadcast over NVLink.
//
// The reference is a single-process CPU library (SURVEY.md §2b: no collective anywhere), so this file has no reference
// counterpart; it distributes the SAME factorizations (llt.cu / lu_f64.cu kernels) the single-GPU entry points
// use. SURVEY.md §8e: block column b (width nb) is owned by rank b % P; at step k the owner factors panel k,
// broadcasts it (plus the pivots for LU) and every rank updates only its own block columns — one exchange per panel,
// no reduction on the data path. Look-ahead: the owner of panel k+1 updates and factors it on a high-priority
// stream and starts its broadcast while the other trailing updates of step k are still running.
//
// NCCL is resolved at run time with dlopen("libnccl.so.2") (the copy torch already loaded in a torch process), so
// libfaer_b200.so has no link-time NCCL dependency and single-GPU users never touch it.
//
// The same block-column drivers run the large single-GPU factorizations (P = 1, no communicator). Three single-GPU
// refinements live here as well:
//   * SM partitioning with CUDA green contexts (`ensure_green_streams`): the LU panel chain gets its own SMs, the
//     trailing updates an urgent and a bulk stream on the rest (`lu_local_partitioned_f64`);
//   * on one GPU the LLT trailing update of a step is ONE structured launch instead of one per block column;
//   * host-resident matrices are streamed through the LLT (`llt_host_pipelined_f64`): uploads, factorization and
//     downloads of finished panels overlap.
#include <cuda.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

namespace {

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;
ncclComm_t g_comm = nullptr;
int g_rank = 0, g_nranks = 1;
cudaStream_t g_panel_stream = nullptr;  // high priority: panel factorization + broadcast
cudaStream_t g_main_stream = nullptr;   // trailing updates
cudaStream_t g_side_stream = nullptr;   // high priority: the LLT's look-ahead column update below its diagonal block

bool load_nccl() {
  if (g_nccl.handle) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    fprintf(stderr, "faer_b200: cannot dlopen libnccl.so.2: %s\n", dlerror());
    return false;
  }
  g_nccl.handle = h;
#define LOAD(field, sym)                                            \
  *(void**)(&g_nccl.field) = dlsym(h, sym);                         \
  if (!g_nccl.field) {                                              \
    fprintf(stderr, "faer_b200: libnccl lacks %s\n", sym);          \
    return false;                                                   \
  }
  LOAD(GetUniqueId, "ncclGetUniqueId")
  LOAD(CommInitRank, "ncclCommInitRank")
  LOAD(CommDestroy, "ncclCommDestroy")
  LOAD(Broadcast, "ncclBroadcast")
  LOAD(GroupStart, "ncclGroupStart")
  LOAD(GroupEnd, "ncclGroupEnd")
  LOAD(GetErrorString, "ncclGetErrorString")
#undef LOAD
  return true;
}

#define FB_NCCL_CHECK(x)                                                                            \
  do {                                                                                              \
    ncclResult_t r_ = (x);                                                                          \
    if (r_ != ncclSuccess) {                                                                        \
      fprintf(stderr, "faer_b200: NCCL error %s at %s:%d\n", g_nccl.GetErrorString(r_), __FILE__, __LINE__); \
      abort();                                                                                      \
    }                                                                                               \
  } while (0)

// pack / unpack a (rows x cols) sub-block of a column-major matrix (ld) to / from a contiguous buffer
void pack(cudaStream_t st, double* dst, const double* src, i64 ld, i64 rows, i64 cols) {
  if (rows == 0 || cols == 0) return;
  FB_CUDA_CHECK(cudaMemcpy2DAsync(dst, (size_t)rows * 8, src, (size_t)ld * 8, (size_t)rows * 8, (size_t)cols,
                                  cudaMemcpyDeviceToDevice, st));
}

inline i64 nblocks(i64 n, i64 nb) { return (n + nb - 1) / nb; }
// number of local columns of rank r
inline i64 local_cols(i64 n, i64 nb, int P, int r) {
  i64 cnt = 0;
  for (i64 b = r; b < nblocks(n, nb); b += P) cnt += std::min(nb, n - b * nb);
  return cnt;
}
// local column offset of global block column b (owned by this rank)
inline i64 local_off(i64 b, i64 nb, int P) { return (b / P) * nb; }

}  // namespace

// the panel (high priority) / trailing-update (low priority) stream pair, also used for single-rank look-ahead
static void ensure_streams() {
  if (g_panel_stream) return;
  int lo = 0, hi = 0;
  FB_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  FB_CUDA_CHECK(cudaStreamCreateWithPriority(&g_panel_stream, cudaStreamNonBlocking, hi));
  FB_CUDA_CHECK(cudaStreamCreateWithPriority(&g_main_stream, cudaStreamNonBlocking, lo));
  FB_CUDA_CHECK(cudaStreamCreateWithPriority(&g_side_stream, cudaStreamNonBlocking, hi));
}

// ---- SM partitioning for the single-GPU look-ahead (CUDA green contexts) ------------------------------------------
// The panel chain (potf2 / TRSM leaves / small GEMMs / the cooperative LU panel) is latency-bound and must not queue
// behind the trailing-update GEMM, whose CTAs fill every SM: a pending panel CTA otherwise waits for whole SMs to drain
// (a 64x64x1024 GEMM tile holds its SM for a long time). A green context pins the panel stream to its own `P` SMs and the update
// stream to the rest. FAER_B200_GREEN_SMS=P (multiple of 8; 0 = off) selects the partition size.
static cudaStream_t g_green_panel = nullptr, g_green_main = nullptr, g_green_urgent = nullptr;
static int g_green_state = 0;      // 0 = not tried, 1 = active, -1 = unavailable / off
static int g_green_panel_sms = 0;  // SMs of the panel partition when active

static int green_sms_wanted() {
  static int v = -1;
  if (v < 0) {
    // default 16 (a 16-SM panel partition + cluster panel next to the trailing updates); 0 switches the partitioned
    // drivers off
    const char* e = getenv("FAER_B200_GREEN_SMS");
    v = e ? atoi(e) : 16;
    if (v < 0) v = 0;
  }
  return v;
}

static bool ensure_green_streams() {
  if (g_green_state) return g_green_state > 0;
  g_green_state = -1;
  const int want = green_sms_wanted();
  if (want <= 0) return false;
#define FB_DRV(name)                                                                                         \
  decltype(&name) p_##name = nullptr;                                                                       \
  {                                                                                                          \
    void* f_ = nullptr;                                                                                      \
    cudaDriverEntryPointQueryResult q_;                                                                      \
    if (cudaGetDriverEntryPoint(#name, &f_, cudaEnableDefault, &q_) != cudaSuccess || !f_) {                 \
      fprintf(stderr, "faer_b200: green contexts unavailable (%s missing); look-ahead uses plain streams\n", #name); \
      return false;                                                                                          \
    }                                                                                                        \
    p_##name = (decltype(&name))f_;                                                                          \
  }
#define FB_DRV_OK(call)                                                                                      \
  {                                                                                                          \
    const CUresult r_ = (call);                                                                              \
    if (r_ != CUDA_SUCCESS) {                                                                                \
      fprintf(stderr, "faer_b200: %s failed (%d); look-ahead uses plain streams\n", #call, (int)r_);         \
      return false;                                                                                          \
    }                                                                                                        \
  }
  FB_DRV(cuDeviceGet)
  FB_DRV(cuDeviceGetDevResource)
  FB_DRV(cuDevSmResourceSplitByCount)
  FB_DRV(cuDevResourceGenerateDesc)
  FB_DRV(cuGreenCtxCreate)
  FB_DRV(cuGreenCtxStreamCreate)
  int dev = 0;
  FB_CUDA_CHECK(cudaGetDevice(&dev));
  FB_CUDA_CHECK(cudaFree(0));  // primary context up
  CUdevice cudev;
  FB_DRV_OK(p_cuDeviceGet(&cudev, dev));
  CUdevResource all, grp[1], rem;
  FB_DRV_OK(p_cuDeviceGetDevResource(cudev, &all, CU_DEV_RESOURCE_TYPE_SM));
  unsigned int ngrp = 1;
  // MAX_POTENTIAL_CLUSTER_SIZE: keep the panel group inside as few GPCs as possible so that a 16-CTA cluster fits
  if (p_cuDevSmResourceSplitByCount(grp, &ngrp, &all, &rem, CU_DEV_SM_RESOURCE_SPLIT_MAX_POTENTIAL_CLUSTER_SIZE,
                                    (unsigned int)want) != CUDA_SUCCESS) {
    ngrp = 1;
    FB_DRV_OK(p_cuDevSmResourceSplitByCount(grp, &ngrp, &all, &rem, 0, (unsigned int)want));
  }
  if (ngrp < 1 || rem.type != CU_DEV_RESOURCE_TYPE_SM || rem.sm.smCount == 0) {
    fprintf(stderr, "faer_b200: SM split produced no remainder; look-ahead uses plain streams\n");
    return false;
  }
  CUdevResourceDesc d_panel, d_main;
  FB_DRV_OK(p_cuDevResourceGenerateDesc(&d_panel, &grp[0], 1));
  FB_DRV_OK(p_cuDevResourceGenerateDesc(&d_main, &rem, 1));
  CUgreenCtx g_panel, g_main;
  FB_DRV_OK(p_cuGreenCtxCreate(&g_panel, d_panel, cudev, CU_GREEN_CTX_DEFAULT_STREAM));
  FB_DRV_OK(p_cuGreenCtxCreate(&g_main, d_main, cudev, CU_GREEN_CTX_DEFAULT_STREAM));
  int lo = 0, hi = 0;
  FB_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CUstream s_panel, s_main, s_urgent;
  FB_DRV_OK(p_cuGreenCtxStreamCreate(&s_panel, g_panel, CU_STREAM_NON_BLOCKING, hi));
  FB_DRV_OK(p_cuGreenCtxStreamCreate(&s_main, g_main, CU_STREAM_NON_BLOCKING, lo));
  FB_DRV_OK(p_cuGreenCtxStreamCreate(&s_urgent, g_main, CU_STREAM_NON_BLOCKING, hi));
#undef FB_DRV
#undef FB_DRV_OK
  g_green_panel = (cudaStream_t)s_panel;
  g_green_main = (cudaStream_t)s_main;
  g_green_urgent = (cudaStream_t)s_urgent;
  g_green_panel_sms = (int)grp[0].sm.smCount;
  g_green_state = 1;
  return true;
}

// ---- host-resident input: stream the matrix through the factorization ------------------------------------------------
// The C ABI accepts host pointers (the reference is a CPU library). Copy-in / factor / copy-out would leave the GPU idle
// during 2 x 2.1 GB of PCIe traffic at n = 16384; instead the block columns are uploaded in order on their own stream
// (only the part on / below the diagonal blocks: the strict upper triangle is never read), the right-looking driver
// waits for column j only at its first touch, and every finished panel goes home on a third stream at once.
struct LltHostPipe {
  double* host;
  i64 host_ld;
  cudaStream_t s_d2h;
  std::vector<cudaEvent_t> up;  // up[j]: block column j is resident on the device
};
static LltHostPipe* g_llt_pipe = nullptr;

// Block-column boundaries of the single-GPU LLT drivers. Uniform width nb while the trailing updates bound the schedule; in
// the tail (remaining order <= FAER_B200_LLT_TAIL, default 6144) the panel chain does — potf2 + the 128-wide TRSM / SYRK
// inside a 256-block + the panel solve's leaves; 128-wide blocks have no inner recursion and half the leaves — so the
// blocks narrow to 128 there. P > 1 keeps uniform blocks (ownership is b % P).
// `wide_head` (the device-resident driver at its default width): while the remaining order exceeds FAER_B200_LLT_HEAD
// (default 8192) the blocks are 512 wide: contracting k = 512 per update halves how often the SYRK pays its per-tile
// fixed cost and how often the trailing matrix crosses HBM, while a step's trailing update (~ m^2) still hides the
// longer 512-wide panel chain. At n = 16384 every boundary from 6144 to 10240 measured the same within noise
// (profiles/r08_bench_parent_vs_branch.json).
static std::vector<i64> llt_block_bounds(i64 n, i64 nb, bool uniform, bool wide_head = false) {
  static i64 tail = -1, head = -1;
  if (tail < 0) {
    const char* e = getenv("FAER_B200_LLT_TAIL");
    tail = e ? atoll(e) : 6144;
    const char* h = getenv("FAER_B200_LLT_HEAD");
    head = h ? atoll(h) : 8192;
  }
  std::vector<i64> b0;
  for (i64 c = 0; c < n;) {
    b0.push_back(c);
    i64 w = nb;
    if (!uniform && nb > 128 && n - c <= tail) w = 128;
    else if (!uniform && wide_head && n - c > head) w = 512;
    c += std::min<i64>(w, n - c);
  }
  b0.push_back(n);
  return b0;
}

i64 lookahead_min_n() {
  static i64 v = -1;
  if (v < 0) {
    const char* e = getenv("FAER_B200_LOOKAHEAD_MIN_N");
    v = e ? atoll(e) : 4096;
    if (v == 0) v = (i64)1 << 62;
  }
  return v;
}
i64 lookahead_block() {
  static i64 v = -1;
  if (v < 0) {
    const char* e = getenv("FAER_B200_NB");
    v = e ? atoll(e) : 0;  // 0 = caller's default (LLT 512 / 256 / 128, see llt_block_bounds; LU 512 up to n = 20000, then 1024)
    if (v < 0 || (v & 1)) v = 0;
  }
  return v;
}

bool dist_ready() { return g_comm != nullptr; }
int dist_rank() { return g_rank; }
int dist_nranks() { return g_nranks; }

int dist_unique_id(void* out128) {
  if (!load_nccl()) return -1;
  ncclUniqueId id;
  FB_NCCL_CHECK(g_nccl.GetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  memcpy(out128, &id, 128);
  return 0;
}

int dist_init(int rank, int nranks, const void* id128) {
  FB_ENTRY();
  if (!load_nccl()) return -1;
  if (g_comm) return 0;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  FB_NCCL_CHECK(g_nccl.CommInitRank(&g_comm, nranks, id, rank));
  g_rank = rank;
  g_nranks = nranks;
  ensure_streams();
  return 0;
}

void dist_finalize() {
  if (g_comm) {
    g_nccl.CommDestroy(g_comm);
    g_comm = nullptr;
  }
  if (g_panel_stream) cudaStreamDestroy(g_panel_stream), g_panel_stream = nullptr;
  if (g_main_stream) cudaStreamDestroy(g_main_stream), g_main_stream = nullptr;
  if (g_side_stream) cudaStreamDestroy(g_side_stream), g_side_stream = nullptr;
  g_rank = 0;
  g_nranks = 1;
}

// -----------------------------------------------------------------------------------------------------------------
// Distributed LLT. A_local: column-major n x local_cols (ld = ld_local >= n): the block columns this rank owns, in
// increasing global order. On return the lower triangle of the global matrix holds L (strict upper part untouched).
// Works for P == 1 too (no communicator needed) — the same code path the multi-GPU runs use, so results do not depend
// on P: every output element receives its rank-nb updates in the same order k = 0, 1, ...
// -----------------------------------------------------------------------------------------------------------------
LltResult dist_llt_f64(double* A_local, i64 ld, i64 n, i64 nb, double reg_delta, double reg_eps, int lookahead) {
  FB_ENTRY();
  // `lookahead` bit 0: two-stream look-ahead; bit 1: purely local run (ignore the communicator even if one exists);
  // bit 2: 512-wide leading blocks (llt_block_bounds' wide_head; single GPU, device-resident matrix, look-ahead only)
  const bool local_only = (lookahead & 2) != 0;
  const bool wide_head = (lookahead & 4) != 0;
  lookahead &= 1;
  const int P = (g_comm && !local_only) ? g_nranks : 1, me = (g_comm && !local_only) ? g_rank : 0;
  LltResult res{true, 0, 0};
  if (n == 0) return res;
  FB_ASSERT(nb > 0 && nb % 2 == 0, "block size must be positive and even");
  if (lookahead) ensure_streams();
  LltHostPipe* pipe = (P == 1 && lookahead) ? g_llt_pipe : nullptr;  // host-resident matrix streamed through (see below)
  // Single GPU: the chain (sp, high priority) and the bulk update (sm) share every SM. A wide bulk CTA fills its SM (384
  // threads x 168 registers, ~225 KB of shared memory), so a chain kernel starts only as bulk CTAs end; that is why the
  // bulk CTAs are short-lived. Giving the chain SMs of its own (green-context partitions) measured 1.2-2.5x slower at
  // n = 16384: potf2 takes ~95 us per launch alone as in the step, while the panel solve, the column update and the bulk
  // lose SMs (profiles/r13_llt_chain_*.json, H100 SXM at 700 W).
  cudaStream_t sp = lookahead ? g_panel_stream : current_stream();
  cudaStream_t sm = lookahead ? g_main_stream : current_stream();
  const bool two_streams = sp != sm && lookahead;
  if (!two_streams) sm = sp;
  // Single GPU: the look-ahead update of block column k+1 is split. Its diagonal block is updated on sp, and the part
  // below it on the side stream ss, where it runs beside the diagonal block's factorization (potf2 alone is ~95 us per
  // 128 columns); sp joins ss before the panel solve. Same kernels on the same operands, so the factor is unchanged.
  // In the 128-wide tail the chain, not the trailing update, sets the step time.
  cudaStream_t ss = (two_streams && P == 1) ? g_side_stream : sp;
  // order after whatever the caller enqueued on the current stream
  cudaEvent_t ev_start, ev_fork, ev_join;
  bool join_pending = false;
  FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming));
  FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
  FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
  FB_CUDA_CHECK(cudaEventRecord(ev_start, current_stream()));
  FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_start, 0));
  if (two_streams) FB_CUDA_CHECK(cudaStreamWaitEvent(sm, ev_start, 0));

  const std::vector<i64> b0 = llt_block_bounds(n, nb, /*uniform*/ P > 1 || !lookahead, wide_head && P == 1 && !pipe);
  const i64 nblk = (i64)b0.size() - 1;
  auto col_off = [&](i64 b) { return P == 1 ? b0[(size_t)b] : local_off(b, nb, P) ; };  // local column of block b (owned)
  i64 wmax = 0;
  for (i64 k = 0; k < nblk; ++k) wmax = std::max(wmax, b0[(size_t)k + 1] - b0[(size_t)k]);
  // two panel buffers (double buffering for look-ahead)
  double* W[2];
  W[0] = (double*)ws_alloc((size_t)n * wmax * 8);
  W[1] = (double*)ws_alloc((size_t)n * wmax * 8);
  long long* d_info = (long long*)ws_alloc(4 * sizeof(long long));
  long long h_info[2] = {-1, 0};
  FB_CUDA_CHECK(cudaMemcpyAsync(d_info, h_info, sizeof(h_info), cudaMemcpyHostToDevice, sp));
  std::vector<cudaEvent_t> ev_bcast((size_t)nblk), ev_used((size_t)nblk);
  for (i64 k = 0; k < nblk; ++k) {
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_bcast[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_used[(size_t)k], cudaEventDisableTiming));
  }

  auto factor_and_bcast = [&](i64 k) {
    // runs on sp. Panel k: rows k0..n of block column k.
    const i64 k0 = b0[(size_t)k], kb = b0[(size_t)k + 1] - k0, rows = n - k0;
    const int owner = (int)(k % P);
    double* Wk = W[k & 1];
    cudaStream_t packed_on = sp;  // the stream that completes W_k
    if (k >= 2) FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_used[(size_t)(k - 2)], 0));  // buffer reuse
    if (owner == me) {
      double* pk = A_local + col_off(k) * ld + k0;
      VD diag{pk, kb, kb, 1, ld};
      llt_cholesky_device_f64(sp, diag, reg_delta, reg_eps, d_info, k0);
      if (join_pending) {  // the look-ahead update below the diagonal block (ss)
        FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_join, 0));
        join_pending = false;
      }
      if (rows > kb) {
        VD below{pk + kb, rows - kb, kb, 1, ld};
        solve_lower_triangular_in_place_f64(sp, cv(diag), false, below.t());
      }
      // split look-ahead (ss != sp): sp packs only the rows the next diagonal-block update reads, ss the rest (the rows
      // its own update below that block and the trailing update read)
      const i64 head = (ss != sp && k + 1 < nblk) ? b0[(size_t)k + 2] - k0 : rows;
      FB_CUDA_CHECK(cudaMemcpy2DAsync(Wk, (size_t)rows * 8, pk, (size_t)ld * 8, (size_t)head * 8, (size_t)kb,
                                      cudaMemcpyDeviceToDevice, sp));
      if (head < rows) {
        FB_CUDA_CHECK(cudaEventRecord(ev_fork, sp));
        FB_CUDA_CHECK(cudaStreamWaitEvent(ss, ev_fork, 0));
        FB_CUDA_CHECK(cudaMemcpy2DAsync(Wk + head, (size_t)rows * 8, pk + head, (size_t)ld * 8, (size_t)(rows - head) * 8,
                                        (size_t)kb, cudaMemcpyDeviceToDevice, ss));
        packed_on = ss;
      }
    }
    if (P > 1) FB_NCCL_CHECK(g_nccl.Broadcast(Wk, Wk, (size_t)rows * kb, ncclDouble, owner, g_comm, sp));
    FB_CUDA_CHECK(cudaEventRecord(ev_bcast[(size_t)k], packed_on));
    if (pipe) {  // block column k is final: send it home while the factorization goes on
      FB_CUDA_CHECK(cudaStreamWaitEvent(pipe->s_d2h, ev_bcast[(size_t)k], 0));
      FB_CUDA_CHECK(cudaMemcpy2DAsync(pipe->host + k0 * pipe->host_ld + k0, (size_t)pipe->host_ld * 8,
                                      A_local + k0 * ld + k0, (size_t)ld * 8, (size_t)rows * 8, (size_t)kb,
                                      cudaMemcpyDeviceToHost, pipe->s_d2h));
    }
  };

  auto update_block_col = [&](cudaStream_t st, i64 k, i64 j, cudaStream_t st_below) {
    // block column j (> k, owned by me) -= W_k[rows >= j0] * W_k[rows of block j]^T; the part below the diagonal block
    // on st_below (ordered after st's work so far, joined by the panel solve of block j)
    if (pipe && k == 0) FB_CUDA_CHECK(cudaStreamWaitEvent(st, pipe->up[(size_t)j], 0));  // first touch of column j
    const i64 k0 = b0[(size_t)k], kb = b0[(size_t)k + 1] - k0, rows_k = n - k0;
    const i64 j0 = b0[(size_t)j], jb = b0[(size_t)j + 1] - j0;
    const double* Wk = W[k & 1];
    double* pj = A_local + col_off(j) * ld + j0;
    VCD Wj{Wk + (j0 - k0), jb, kb, 1, rows_k};                       // rows of block j in the panel
    VD djj{pj, jb, jb, 1, ld};
    const i64 below = n - j0 - jb;
    if (below > 0 && st_below != st) {
      FB_CUDA_CHECK(cudaEventRecord(ev_fork, st));
      FB_CUDA_CHECK(cudaStreamWaitEvent(st_below, ev_fork, 0));
    }
    gemm_f64(st, djj, TRI_LOWER, 1, Wj, RECT, Wj.t(), RECT, -1.0);    // diagonal block: lower triangle only
    if (below > 0) {
      VCD Wb{Wk + (j0 - k0) + jb, below, kb, 1, rows_k};
      VD dbj{pj + jb, below, jb, 1, ld};
      gemm_f64(st_below, dbj, 1, Wb, Wj.t(), -1.0);
      if (st_below != st) {
        FB_CUDA_CHECK(cudaEventRecord(ev_join, st_below));
        join_pending = true;
      }
    }
  };

  if (pipe) FB_CUDA_CHECK(cudaStreamWaitEvent(sp, pipe->up[0], 0));
  factor_and_bcast(0);
  for (i64 k = 0; k < nblk; ++k) {
    // trailing updates of step k need panel k
    if (two_streams) FB_CUDA_CHECK(cudaStreamWaitEvent(sm, ev_bcast[(size_t)k], 0));
    const i64 kn = k + 1;
    if (kn < nblk) {
      if ((int)(kn % P) == me) {
        // look-ahead: bring block column k+1 up to date first (on the panel stream), then factor + broadcast it
        // block column k+1 has received updates 0..k-1 on sm; order sp after them
        if (two_streams && k >= 1) FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_used[(size_t)(k - 1)], 0));
        update_block_col(sp, k, kn, ss);
      }
      factor_and_bcast(kn);
    }
    if (P == 1 && k + 2 < nblk && !(pipe && k == 0)) {
      // single GPU: every remaining block column in ONE structured launch (lower-triangular destination: tiles above
      // the diagonal exit at once) instead of one launch per block column — no per-launch tail, better L2 reuse
      const i64 k0 = b0[(size_t)k], kb = b0[(size_t)k + 1] - k0, rows_k = n - k0, j0 = b0[(size_t)k + 2];
      VCD Wr{W[k & 1] + (j0 - k0), n - j0, kb, 1, rows_k};
      VD dst{A_local + j0 * ld + j0, n - j0, n - j0, 1, ld};
      gemm_f64(sm, dst, TRI_LOWER, 1, Wr, RECT, Wr.t(), RECT, -1.0);
    } else {
      for (i64 j = k + 2; j < nblk; ++j)
        if ((int)(j % P) == me) update_block_col(sm, k, j, sm);
    }
    FB_CUDA_CHECK(cudaEventRecord(ev_used[(size_t)k], sm));
  }
  if (two_streams) {
    FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_used[(size_t)(nblk - 1)], 0));
  }
  FB_CUDA_CHECK(cudaMemcpyAsync(h_info, d_info, sizeof(h_info), cudaMemcpyDeviceToHost, sp));
  FB_CUDA_CHECK(cudaStreamSynchronize(sp));
  if (two_streams) FB_CUDA_CHECK(cudaStreamSynchronize(sm));
  if (pipe) FB_CUDA_CHECK(cudaStreamSynchronize(pipe->s_d2h));
  for (i64 k = 0; k < nblk; ++k) {
    cudaEventDestroy(ev_bcast[(size_t)k]);
    cudaEventDestroy(ev_used[(size_t)k]);
  }
  cudaEventDestroy(ev_start);
  cudaEventDestroy(ev_fork);
  cudaEventDestroy(ev_join);
  ws_free(d_info);
  ws_free(W[1]);
  ws_free(W[0]);
  // the status word lives on the owners; combine across ranks (tiny host-side exchange through a broadcast per rank
  // would need another collective: instead every owner's failure is propagated through the panel data itself — a
  // failed panel is NaN-free but the failing rank reports; callers reduce the status with their own process group).
  if (h_info[0] >= 0) {
    res.ok = false;
    res.non_positive_pivot_index = (size_t)h_info[0];
  } else {
    res.dynamic_regularization_count = (size_t)h_info[1];
  }
  return res;
}

// -----------------------------------------------------------------------------------------------------------------
// Distributed LU with partial pivoting (square n x n), same layout. Step k: the owner factors panel k (all rows
// k0.., our recursive panel LU => pivots identical to the single-GPU path: the pivot search only ever looks at the
// panel's own, fully updated columns), broadcasts the factored panel + its kb transpositions; every rank applies the
// row swaps to ALL its other columns (left ones too: final L is fully permuted, LAPACK/faer convention), then
// U_kj = L_kk^-1 A_kj and A_(k+1:, j) -= L_(k+1:, k) U_kj on its own block columns j > k.
// -----------------------------------------------------------------------------------------------------------------
// LLT of a HOST column-major matrix (lower triangle), transfers overlapped with the factorization (see LltHostPipe).
LltResult llt_host_pipelined_f64(double* hostA, i64 host_ld, i64 n, i64 nb, double reg_delta, double reg_eps) {
  FB_ENTRY();
  static cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  if (!s_h2d) {
    FB_CUDA_CHECK(cudaStreamCreateWithFlags(&s_h2d, cudaStreamNonBlocking));
    FB_CUDA_CHECK(cudaStreamCreateWithFlags(&s_d2h, cudaStreamNonBlocking));
  }
  // the same block boundaries as dist_llt_f64, which waits for block column j at its first touch
  const std::vector<i64> b0 = llt_block_bounds(n, nb, /*uniform*/ false);
  const i64 nblk = (i64)b0.size() - 1;
  double* dA = (double*)ws_alloc((size_t)n * n * 8);
  LltHostPipe pipe;
  pipe.host = hostA;
  pipe.host_ld = host_ld;
  pipe.s_d2h = s_d2h;
  pipe.up.resize((size_t)nblk);
  for (i64 j = 0; j < nblk; ++j) {
    const i64 j0 = b0[(size_t)j], jb = b0[(size_t)j + 1] - j0;
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&pipe.up[(size_t)j], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaMemcpy2DAsync(dA + j0 * n + j0, (size_t)n * 8, hostA + j0 * host_ld + j0, (size_t)host_ld * 8,
                                    (size_t)(n - j0) * 8, (size_t)jb, cudaMemcpyHostToDevice, s_h2d));
    FB_CUDA_CHECK(cudaEventRecord(pipe.up[(size_t)j], s_h2d));
  }
  g_llt_pipe = &pipe;
  const LltResult r = dist_llt_f64(dA, n, n, nb, reg_delta, reg_eps, /*lookahead | local*/ 3);
  g_llt_pipe = nullptr;
  FB_CUDA_CHECK(cudaStreamSynchronize(s_h2d));
  for (i64 j = 0; j < nblk; ++j) cudaEventDestroy(pipe.up[(size_t)j]);
  ws_free(dA);
  return r;
}

// Single-GPU right-looking block-column LU on a partitioned GPU (green contexts; same stream roles as the LLT driver):
//   sp  panel partition          : recursive panel LU of block column k+1 (cooperative pivot-search kernel + its glue)
//   su  update partition, urgent : row swaps + U_k,k+1 = L_kk^-1 A_k,k+1 + trailing update of block column k+1
//   sm  update partition, bulk   : the same for block columns k+2.. (k+2 first) and the row swaps of the left columns
// The panel kernel is latency-bound (one grid barrier per column) and, as a cooperative launch, could not start while
// trailing-update CTAs occupied every SM; on its own partition it overlaps with the GEMMs completely.
static void lu_local_partitioned_f64(double* A, i64 ld, i64 n, i64 nb, int* d_trans) {
  cudaStream_t sp = g_green_panel, su = g_green_urgent, sm = g_green_main;
  cudaEvent_t ev_start;
  FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming));
  FB_CUDA_CHECK(cudaEventRecord(ev_start, current_stream()));
  FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_start, 0));
  FB_CUDA_CHECK(cudaStreamWaitEvent(su, ev_start, 0));
  FB_CUDA_CHECK(cudaStreamWaitEvent(sm, ev_start, 0));
  std::vector<i64> b0;
  for (i64 c = 0; c < n; c += std::min<i64>(nb, n - c)) b0.push_back(c);
  b0.push_back(n);
  const i64 nblk = (i64)b0.size() - 1;
  LuWorkspace* wp = lu_ws_create(sp, nb, g_green_panel_sms);
  lu_ws_set_big_stream(wp, su);  // big recursion nodes run on the update partition
  // leaves on a thread-block cluster (DSMEM exchange) inside the panel partition
  lu_ws_set_cluster(wp, g_green_panel_sms >= 16 ? 16 : 8);
  LuWorkspace* wu = lu_ws_create(su, nb);
  LuWorkspace* wm = lu_ws_create(sm, nb);
  std::vector<cudaEvent_t> ev_panel((size_t)nblk), ev_ready((size_t)nblk), ev_first((size_t)nblk);
  for (i64 k = 0; k < nblk; ++k) {
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_panel[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_ready[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_first[(size_t)k], cudaEventDisableTiming));
  }
  auto factor_panel = [&](i64 k) {  // on sp
    const i64 k0 = b0[(size_t)k], kb = b0[(size_t)k + 1] - k0, rows = n - k0;
    VD panel{A + k0 * ld + k0, rows, kb, 1, ld};
    lu_factor_window_f64(wp, panel, 0, kb, d_trans + k0);
    FB_CUDA_CHECK(cudaEventRecord(ev_panel[(size_t)k], sp));
  };
  // swaps (+ TRSM / GEMM if `right`) of step k on the columns [c0, c1)
  auto update_cols = [&](LuWorkspace* w, cudaStream_t st, i64 k, i64 c0, i64 c1, bool right) {
    if (c1 <= c0) return;
    const i64 k0 = b0[(size_t)k], kb = b0[(size_t)k + 1] - k0, rows = n - k0;
    VD cols{A + c0 * ld + k0, rows, c1 - c0, 1, ld};
    lu_apply_transpositions_f64(w, cols, d_trans + k0, kb);
    if (right) {
      VCD L11{A + k0 * ld + k0, kb, kb, 1, ld};
      VD top = cols.sub(0, 0, kb, c1 - c0);
      solve_lower_triangular_in_place_f64(st, L11, true, top);
      if (rows > kb) {
        VCD L21{A + k0 * ld + k0 + kb, rows - kb, kb, 1, ld};
        gemm_f64(st, cols.sub(kb, 0, rows - kb, c1 - c0), 1, L21, cv(top), -1.0);
      }
    }
  };
  factor_panel(0);
  for (i64 k = 0; k < nblk; ++k) {
    const i64 k0 = b0[(size_t)k];
    const i64 kn = k + 1;
    if (kn < nblk) {
      const i64 c0 = b0[(size_t)kn], c1 = b0[(size_t)kn + 1];
      FB_CUDA_CHECK(cudaStreamWaitEvent(su, ev_panel[(size_t)k], 0));
      if (k >= 1) FB_CUDA_CHECK(cudaStreamWaitEvent(su, ev_first[(size_t)(k - 1)], 0));
      update_cols(wu, su, k, c0, c1, true);
      FB_CUDA_CHECK(cudaEventRecord(ev_ready[(size_t)kn], su));
      FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_ready[(size_t)kn], 0));
      factor_panel(kn);
    }
    FB_CUDA_CHECK(cudaStreamWaitEvent(sm, ev_panel[(size_t)k], 0));
    if (k + 2 < nblk) {
      const i64 c2 = b0[(size_t)k + 2], c3 = b0[(size_t)k + 3];
      update_cols(wm, sm, k, c2, c3, true);  // the next urgent column first
      FB_CUDA_CHECK(cudaEventRecord(ev_first[(size_t)k], sm));
      update_cols(wm, sm, k, c3, n, true);
    }
    update_cols(wm, sm, k, 0, k0, false);  // the left columns only receive the row swaps
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(sp));
  FB_CUDA_CHECK(cudaStreamSynchronize(su));
  FB_CUDA_CHECK(cudaStreamSynchronize(sm));
  for (i64 k = 0; k < nblk; ++k) {
    cudaEventDestroy(ev_panel[(size_t)k]);
    cudaEventDestroy(ev_ready[(size_t)k]);
    cudaEventDestroy(ev_first[(size_t)k]);
  }
  cudaEventDestroy(ev_start);
  lu_ws_destroy(wm);
  lu_ws_destroy(wu);
  lu_ws_destroy(wp);
}

size_t dist_lu_f64(double* A_local, i64 ld, i64 n, i64 nb, long long* perm_fwd, long long* perm_inv, int lookahead) {
  FB_ENTRY();
  // `lookahead` bit 0: two-stream look-ahead; bit 1: purely local run (ignore the communicator even if one exists)
  const bool local_only = (lookahead & 2) != 0;
  lookahead &= 1;
  const int P = (g_comm && !local_only) ? g_nranks : 1, me = (g_comm && !local_only) ? g_rank : 0;
  for (i64 i = 0; i < n; ++i) perm_fwd[i] = i;
  size_t n_trans = 0;
  if (n == 0) return 0;
  FB_ASSERT(nb > 0 && nb % 2 == 0, "block size must be positive and even");
  // the partition pays off where the panel chain is exposed (moderate n); for large n the schedule is bound by the
  // trailing updates and giving 16 SMs away costs more than it saves: plain look-ahead there
  if (lookahead && P == 1 && n <= 24576 && ensure_green_streams()) {
    int* d_trans = (int*)ws_alloc((size_t)n * sizeof(int));
    lu_local_partitioned_f64(A_local, ld, n, nb, d_trans);
    std::vector<int> h_trans((size_t)n);
    FB_CUDA_CHECK(cudaMemcpy(h_trans.data(), d_trans, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
    ws_free(d_trans);
    for (i64 i = 0; i < n; ++i) {
      const int t = h_trans[(size_t)i];
      if (t != 0) {
        std::swap(perm_fwd[i], perm_fwd[i + t]);
        ++n_trans;
      }
    }
    for (i64 i = 0; i < n; ++i) perm_inv[perm_fwd[i]] = i;
    return n_trans;
  }
  // Stream roles (P >= 1). With an SM partition (green contexts) the panel chain owns its SMs:
  //   sp  panel factorization (cluster kernels; big recursion nodes go to su)     su  look-ahead column update (urgent)
  //   sm  bulk trailing updates                                                   sb  the NCCL broadcast (plain stream)
  // Without a partition (FAER_B200_GREEN_SMS=0 or no look-ahead) sp = su = sb is the high-priority stream.
  if (lookahead) ensure_streams();
  const bool part = lookahead && ensure_green_streams();
  cudaStream_t sp = part ? g_green_panel : (lookahead ? g_panel_stream : current_stream());
  cudaStream_t su = part ? g_green_urgent : sp;
  cudaStream_t sm = part ? g_green_main : (lookahead ? g_main_stream : current_stream());
  cudaStream_t sb = part ? g_panel_stream : sp;
  const bool two_streams = sp != sm && lookahead;
  if (!two_streams) sm = sp;
  cudaEvent_t ev_start;
  FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming));
  FB_CUDA_CHECK(cudaEventRecord(ev_start, current_stream()));
  for (cudaStream_t st : {sp, su, sm, sb})
    if (st != current_stream()) FB_CUDA_CHECK(cudaStreamWaitEvent(st, ev_start, 0));

  const i64 nblk = nblocks(n, nb);
  const i64 ncols_loc = local_cols(n, nb, P, me);
  constexpr int NW = 3;  // panel buffers in flight
  double* W[NW];
  for (int i = 0; i < NW; ++i) W[i] = (double*)ws_alloc((size_t)n * nb * 8);
  int* d_trans = (int*)ws_alloc((size_t)n * sizeof(int));
  LuWorkspace* wp = lu_ws_create(sp, nb, part ? g_green_panel_sms : 0);
  if (part) {
    lu_ws_set_big_stream(wp, su);
    lu_ws_set_cluster(wp, g_green_panel_sms >= 16 ? 16 : 8);
  }
  LuWorkspace* wu = (su != sp) ? lu_ws_create(su, nb) : wp;
  LuWorkspace* wm = two_streams ? lu_ws_create(sm, nb) : wp;
  std::vector<cudaEvent_t> ev_fact((size_t)nblk), ev_bcast((size_t)nblk), ev_used((size_t)nblk), ev_first((size_t)nblk),
      ev_ready((size_t)nblk);
  for (i64 k = 0; k < nblk; ++k) {
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_fact[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_bcast[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_used[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_first[(size_t)k], cudaEventDisableTiming));
    FB_CUDA_CHECK(cudaEventCreateWithFlags(&ev_ready[(size_t)k], cudaEventDisableTiming));
  }
  // number of local columns that belong to blocks with index < b
  auto cols_before = [&](i64 b) {
    i64 cnt = 0;
    for (i64 q = me; q < b && q < nblk; q += P) cnt += std::min(nb, n - q * nb);
    return cnt;
  };

  // panel k: factored by its owner on sp (in place), packed into W[k % NW], broadcast on sb. The buffer is free once
  // every local update of step k - NW is done (ev_used on sm; the urgent update of that step precedes it on su).
  auto factor_and_bcast = [&](i64 k) {
    const i64 k0 = k * nb, kb = std::min(nb, n - k0), rows = n - k0;
    const int owner = (int)(k % P);
    double* Wk = W[k % NW];
    if (owner == me) {
      double* pk = A_local + local_off(k, nb, P) * ld + k0;
      VD panel{pk, rows, kb, 1, ld};
      lu_factor_window_f64(wp, panel, 0, kb, d_trans + k0);
      if (k >= NW) {
        FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_used[(size_t)(k - NW)], 0));
        if (su != sp && k - NW + 1 < nblk) FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_ready[(size_t)(k - NW + 1)], 0));
      }
      pack(sp, Wk, pk, ld, rows, kb);
      FB_CUDA_CHECK(cudaEventRecord(ev_fact[(size_t)k], sp));
    }
    if (P > 1) {
      if (sb != sp) {
        if (owner == me) FB_CUDA_CHECK(cudaStreamWaitEvent(sb, ev_fact[(size_t)k], 0));
        else if (k >= NW) {
          FB_CUDA_CHECK(cudaStreamWaitEvent(sb, ev_used[(size_t)(k - NW)], 0));
          if (k - NW + 1 < nblk) FB_CUDA_CHECK(cudaStreamWaitEvent(sb, ev_ready[(size_t)(k - NW + 1)], 0));
        }
      } else if (owner != me && k >= NW) {
        FB_CUDA_CHECK(cudaStreamWaitEvent(sb, ev_used[(size_t)(k - NW)], 0));
      }
      FB_NCCL_CHECK(g_nccl.GroupStart());
      FB_NCCL_CHECK(g_nccl.Broadcast(Wk, Wk, (size_t)rows * kb, ncclDouble, owner, g_comm, sb));
      FB_NCCL_CHECK(g_nccl.Broadcast(d_trans + k0, d_trans + k0, (size_t)kb, ncclInt32, owner, g_comm, sb));
      FB_NCCL_CHECK(g_nccl.GroupEnd());
      FB_CUDA_CHECK(cudaEventRecord(ev_bcast[(size_t)k], sb));
    } else {
      FB_CUDA_CHECK(cudaEventRecord(ev_bcast[(size_t)k], sp));
    }
  };

  // swaps (+ TRSM/GEMM if `right`) of step k on the local column range [c0, c1)
  auto update_cols = [&](LuWorkspace* w, cudaStream_t st, i64 k, i64 c0, i64 c1, bool right) {
    if (c1 <= c0) return;
    const i64 k0 = k * nb, kb = std::min(nb, n - k0), rows = n - k0;
    const double* Wk = W[k % NW];
    VD cols{A_local + c0 * ld + k0, rows, c1 - c0, 1, ld};
    lu_apply_transpositions_f64(w, cols, d_trans + k0, kb);
    if (right) {
      VCD L11{Wk, kb, kb, 1, rows};
      VD top = cols.sub(0, 0, kb, c1 - c0);
      solve_lower_triangular_in_place_f64(st, L11, true, top);
      if (rows > kb) {
        VCD L21{Wk + kb, rows - kb, kb, 1, rows};
        gemm_f64(st, cols.sub(kb, 0, rows - kb, c1 - c0), 1, L21, cv(top), -1.0);
      }
    }
  };

  factor_and_bcast(0);
  for (i64 k = 0; k < nblk; ++k) {
    const i64 kb = std::min(nb, n - k * nb);
    const i64 left_end = cols_before(k);                                // blocks < k
    const i64 right_begin = left_end + (((int)(k % P) == me) ? kb : 0);  // skip the panel itself on its owner
    i64 sm_right_begin = right_begin;
    const i64 kn = k + 1;
    if (kn < nblk) {
      if ((int)(kn % P) == me) {
        const i64 cb = cols_before(kn);
        const i64 knb = std::min(nb, n - kn * nb);
        if (two_streams) {
          FB_CUDA_CHECK(cudaStreamWaitEvent(su, ev_bcast[(size_t)k], 0));
          // block k+1 received step k-1's update on the bulk stream (first thing it did in that step)
          if (k >= 1) FB_CUDA_CHECK(cudaStreamWaitEvent(su, ev_first[(size_t)(k - 1)], 0));
        }
        update_cols(wu, su, k, cb, cb + knb, true);
        FB_CUDA_CHECK(cudaEventRecord(ev_ready[(size_t)kn], su));
        if (su != sp) FB_CUDA_CHECK(cudaStreamWaitEvent(sp, ev_ready[(size_t)kn], 0));
        sm_right_begin = cb + knb;  // block k+1 is my first block to the right of k
      } else {
        FB_CUDA_CHECK(cudaEventRecord(ev_ready[(size_t)kn], su));  // nothing urgent here: keeps the event defined
      }
      factor_and_bcast(kn);
    }
    if (two_streams) FB_CUDA_CHECK(cudaStreamWaitEvent(sm, ev_bcast[(size_t)k], 0));
    // bulk: my block k+2 first (its owner's urgent stream needs it next), then the rest, then the left columns (swaps only)
    i64 first_end = sm_right_begin;
    if (k + 2 < nblk && (int)((k + 2) % P) == me) {
      const i64 cb2 = cols_before(k + 2);
      first_end = cb2 + std::min(nb, n - (k + 2) * nb);
    }
    update_cols(wm, sm, k, sm_right_begin, first_end, true);
    FB_CUDA_CHECK(cudaEventRecord(ev_first[(size_t)k], sm));
    update_cols(wm, sm, k, first_end, ncols_loc, true);
    update_cols(wm, sm, k, 0, left_end, false);
    FB_CUDA_CHECK(cudaEventRecord(ev_used[(size_t)k], sm));
  }
  std::vector<int> h_trans((size_t)n);
  FB_CUDA_CHECK(cudaStreamSynchronize(sb));
  FB_CUDA_CHECK(cudaStreamSynchronize(sp));
  FB_CUDA_CHECK(cudaStreamSynchronize(su));
  FB_CUDA_CHECK(cudaStreamSynchronize(sm));
  FB_CUDA_CHECK(cudaMemcpy(h_trans.data(), d_trans, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  for (i64 i = 0; i < n; ++i) {
    const int t = h_trans[(size_t)i];
    if (t != 0) {
      std::swap(perm_fwd[i], perm_fwd[i + t]);
      ++n_trans;
    }
  }
  for (i64 i = 0; i < n; ++i) perm_inv[perm_fwd[i]] = i;
  for (i64 k = 0; k < nblk; ++k) {
    cudaEventDestroy(ev_fact[(size_t)k]);
    cudaEventDestroy(ev_bcast[(size_t)k]);
    cudaEventDestroy(ev_used[(size_t)k]);
    cudaEventDestroy(ev_first[(size_t)k]);
    cudaEventDestroy(ev_ready[(size_t)k]);
  }
  cudaEventDestroy(ev_start);
  if (wm != wp) lu_ws_destroy(wm);
  if (wu != wp) lu_ws_destroy(wu);
  lu_ws_destroy(wp);
  ws_free(d_trans);
  for (int i = NW - 1; i >= 0; --i) ws_free(W[i]);
  return n_trans;
}

// ---- distributed Householder QR without pivoting (SURVEY.md 8e: "QR: broadcast (V panel, T)") ----------------------------------
// A (m x n, m >= n) in the 1-D block-column-cyclic layout with block width = the Householder block size bs: at step k the owner
// factors its block column below the diagonal with the single-GPU driver (qr.cu: same panel kernels, same T blocks as a
// single-GPU run with this block size), the factored panel (V below the diagonal, R on / above it) and its T block are broadcast
// (two ncclBroadcast per block), and every rank applies (I - V T^-H V^H) to its own columns to the right. Q_coeff (bs x n,
// leading dimension bs, DEVICE memory) is replicated: every rank ends with all T blocks. No look-ahead yet: the panel and
// the updates alternate on the caller's stream. A rank-deficient block stops the run on every rank (returns -1): the
// reference's column skipping crosses block boundaries, which the single-GPU general driver handles and this one does not.
// `flags` bit 1: purely local run (ignore the communicator), as for the LLT / LU drivers.
template <class T>
static i64 dist_qr_impl(T* A_local, i64 ld, i64 m, i64 n, i64 bs, T* Q_coeff, int flags) {
  FB_ENTRY();
  const bool local_only = (flags & 2) != 0;
  const int P = (g_comm && !local_only) ? g_nranks : 1, me = (g_comm && !local_only) ? g_rank : 0;
  FB_ASSERT(m >= n, "distributed QR: nrows >= ncols");
  FB_ASSERT(bs > 0, "block size must be positive");
  if (n == 0) return 0;
  cudaStream_t st = current_stream();
  const ncclDataType_t dt = sizeof(T) == 8 ? ncclDouble : ncclFloat;
  const i64 nblk = nblocks(n, bs), my_cols = local_cols(n, bs, P, me);
  T* W = P > 1 ? (T*)ws_alloc((size_t)m * (size_t)bs * sizeof(T)) : nullptr;
  T* tmp = (T*)ws_alloc((size_t)bs * (size_t)std::max<i64>(my_cols, 1) * sizeof(T));
  int* d_status = (int*)ws_alloc(sizeof(int));
  i64 result = n;
  for (i64 k = 0; k < nblk; ++k) {
    const i64 j0 = k * bs, jb = std::min(bs, n - j0), rows = m - j0;
    const int owner = (int)(k % P);
    T* Tk = Q_coeff + j0 * bs;  // bs x jb block of the replicated factor (the jb x jb T block in its first rows)
    View<T> Hk{Tk, jb, jb, 1, bs};
    View<const T> V;
    int status = 0;
    if (owner == me) {
      T* pk = A_local + local_off(k, bs, P) * ld + j0;
      View<T> panel{pk, rows, jb, 1, ld};
      const i64 r = qr_in_place<T>(st, panel, Hk);  // synchronises st
      status = r < jb ? 1 : 0;
      if (P > 1) {
        FB_CUDA_CHECK(cudaMemcpy2DAsync(W, (size_t)rows * sizeof(T), pk, (size_t)ld * sizeof(T), (size_t)rows * sizeof(T), (size_t)jb,
                                        cudaMemcpyDeviceToDevice, st));
        V = View<const T>{W, rows, jb, 1, rows};
      } else {
        V = View<const T>{pk, rows, jb, 1, ld};
      }
    } else {
      V = View<const T>{W, rows, jb, 1, rows};
    }
    if (P > 1) {
      FB_CUDA_CHECK(cudaMemcpyAsync(d_status, &status, sizeof(int), cudaMemcpyHostToDevice, st));
      FB_NCCL_CHECK(g_nccl.Broadcast(d_status, d_status, 1, ncclInt32, owner, g_comm, st));
      FB_NCCL_CHECK(g_nccl.Broadcast(W, W, (size_t)rows * (size_t)jb, dt, owner, g_comm, st));
      FB_NCCL_CHECK(g_nccl.Broadcast(Tk, Tk, (size_t)bs * (size_t)jb, dt, owner, g_comm, st));
      FB_CUDA_CHECK(cudaMemcpyAsync(&status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
      FB_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    if (status) {
      result = -1;
      break;
    }
    // my columns to the right of block k: local storage is ordered by block index, so they are the tail of A_local
    i64 t0 = 0;
    for (i64 b = me; b <= k; b += P) t0 += std::min(bs, n - b * bs);
    if (my_cols > t0)
      apply_block_householder_on_the_left<T>(st, V, cview(Hk), View<T>{A_local + t0 * ld + j0, rows, my_cols - t0, 1, ld}, true, tmp);
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(d_status);
  ws_free(tmp);
  if (W) ws_free(W);
  return result;
}
i64 dist_qr_f64(double* A_local, i64 ld, i64 m, i64 n, i64 bs, double* Q_coeff, int flags) {
  return dist_qr_impl<double>(A_local, ld, m, n, bs, Q_coeff, flags);
}
i64 dist_qr_f32(float* A_local, i64 ld, i64 m, i64 n, i64 bs, float* Q_coeff, int flags) {
  return dist_qr_impl<float>(A_local, ld, m, n, bs, Q_coeff, flags);
}


}  // namespace fb
