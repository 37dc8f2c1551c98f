// Process-wide runtime state: stream, launch counter, device workspace pool, host<->device staging.
#include "runtime.cuh"

#include <cstring>
#include <mutex>
#include <vector>

namespace fb {

unsigned long long g_launch_count = 0;
int g_launch_tag = LAUNCH_OTHER;
signed char* g_launch_log = nullptr;
size_t g_launch_log_len = 0, g_launch_log_cap = 0;

namespace {
cudaStream_t g_stream = nullptr;
std::mutex g_pool_mutex;
struct PoolBlock {
  void* ptr;
  size_t bytes;
  bool in_use;
};
std::vector<PoolBlock> g_pool;
bool g_checked_device = false;
}  // namespace

cudaStream_t current_stream() { return g_stream; }
void set_current_stream(cudaStream_t s) { g_stream = s; }

namespace {
int g_device_sms = 0;
}  // namespace
int stream_sms(cudaStream_t) {
  if (g_device_sms == 0) {
    int dev = 0;
    FB_CUDA_CHECK(cudaGetDevice(&dev));
    FB_CUDA_CHECK(cudaDeviceGetAttribute(&g_device_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  return g_device_sms;
}

namespace {
struct OptDef {
  const char* name;
  const char* env;
  long long dflt;
};
const OptDef g_opt_defs[OPT_COUNT] = {{"gemm_ws", "FAER_B200_GEMM_WS", 1}, {"f64_gemm_mode", "FAER_B200_F64_GEMM_MODE", 0}};
long long g_opt_vals[OPT_COUNT];
bool g_opt_init = false;
void opts_init() {
  if (g_opt_init) return;
  for (int i = 0; i < OPT_COUNT; ++i) {
    const char* e = getenv(g_opt_defs[i].env);
    g_opt_vals[i] = e ? atoll(e) : g_opt_defs[i].dflt;
  }
  g_opt_init = true;
}
}  // namespace
long long get_option(int opt) {
  opts_init();
  return g_opt_vals[opt];
}
bool set_option_by_name(const char* name, long long value) {
  opts_init();
  for (int i = 0; i < OPT_COUNT; ++i)
    if (strcmp(name, g_opt_defs[i].name) == 0) {
      g_opt_vals[i] = value;
      return true;
    }
  return false;
}
long long get_option_by_name(const char* name) {
  opts_init();
  for (int i = 0; i < OPT_COUNT; ++i)
    if (strcmp(name, g_opt_defs[i].name) == 0) return g_opt_vals[i];
  return -1;
}

std::recursive_mutex& entry_mutex() {
  static std::recursive_mutex m;
  return m;
}

void require_device() {
  if (g_checked_device) return;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    fprintf(stderr,
            "faer_b200: no CUDA device available (%s). This backend has no CPU fallback; refusing to compute.\n",
            e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    abort();
  }
  g_checked_device = true;
}

void* ws_alloc(size_t bytes) {
  if (bytes == 0) bytes = 256;
  bytes = (bytes + 255) & ~(size_t)255;
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  int best = -1;
  for (int i = 0; i < (int)g_pool.size(); ++i) {
    if (!g_pool[i].in_use && g_pool[i].bytes >= bytes) {
      if (best < 0 || g_pool[i].bytes < g_pool[best].bytes) best = i;
    }
  }
  if (best >= 0 && g_pool[best].bytes <= 2 * bytes + (1 << 20)) {
    g_pool[best].in_use = true;
    return g_pool[best].ptr;
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    // drop cached free blocks and retry once
    for (auto it = g_pool.begin(); it != g_pool.end();) {
      if (!it->in_use) {
        cudaFree(it->ptr);
        it = g_pool.erase(it);
      } else {
        ++it;
      }
    }
    (void)cudaGetLastError();
    FB_CUDA_CHECK(cudaMalloc(&p, bytes));
  }
  g_pool.push_back(PoolBlock{p, bytes, true});
  return p;
}

void* stream_scratch(cudaStream_t stream, size_t bytes) {
  struct Slot {
    cudaStream_t st;
    void* p;
    size_t bytes;
    bool used;
  };
  static Slot slots[16];
  Slot* s = nullptr;
  for (auto& c : slots)
    if (c.used && c.st == stream) s = &c;
  if (!s)
    for (auto& c : slots)
      if (!c.used) {
        c.used = true;
        c.st = stream;
        c.p = nullptr;
        c.bytes = 0;
        s = &c;
        break;
      }
  if (!s) {
    FB_CUDA_CHECK(cudaStreamSynchronize(slots[0].st));
    slots[0].st = stream;
    s = &slots[0];
  }
  if (bytes > s->bytes) {
    if (s->p) {
      FB_CUDA_CHECK(cudaStreamSynchronize(stream));
      FB_CUDA_CHECK(cudaFree(s->p));
    }
    FB_CUDA_CHECK(cudaMalloc(&s->p, bytes));
    s->bytes = bytes;
  }
  return s->p;
}

void ws_free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  for (auto& b : g_pool)
    if (b.ptr == p) {
      b.in_use = false;
      return;
    }
  FB_ASSERT(false, "ws_free of unknown pointer");
}

void ws_release_all() {
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  for (auto it = g_pool.begin(); it != g_pool.end();) {
    if (!it->in_use) {
      cudaFree(it->ptr);
      it = g_pool.erase(it);
    } else {
      ++it;
    }
  }
}

namespace {
bool g_prof = false;
struct ProfRec { cudaEvent_t e0, e1; double flops; };
std::vector<ProfRec> g_prof_recs;
cudaEvent_t g_prof_pending = nullptr;
}  // namespace
bool profiling_enabled() { return g_prof; }
void profile_begin() {
  g_prof_recs.clear();
  g_prof = true;
}
void profile_record_start(cudaStream_t st) {
  if (!g_prof) return;
  FB_CUDA_CHECK(cudaEventCreate(&g_prof_pending));
  FB_CUDA_CHECK(cudaEventRecord(g_prof_pending, st));
}
void profile_record_stop(cudaStream_t st, double flops) {
  if (!g_prof || !g_prof_pending) return;
  ProfRec r;
  r.e0 = g_prof_pending;
  g_prof_pending = nullptr;
  FB_CUDA_CHECK(cudaEventCreate(&r.e1));
  FB_CUDA_CHECK(cudaEventRecord(r.e1, st));
  r.flops = flops;
  g_prof_recs.push_back(r);
}
void profile_end(double* flops, double* ms, unsigned long long* count) {
  g_prof = false;
  double f = 0, t = 0;
  for (auto& r : g_prof_recs) {
    FB_CUDA_CHECK(cudaEventSynchronize(r.e1));
    float m = 0;
    FB_CUDA_CHECK(cudaEventElapsedTime(&m, r.e0, r.e1));
    t += m;
    f += r.flops;
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  *flops = f;
  *ms = t;
  *count = g_prof_recs.size();
  g_prof_recs.clear();
}

bool is_device_pointer(const void* p) {
  if (!p) return false;
  cudaPointerAttributes attr;
  cudaError_t e = cudaPointerGetAttributes(&attr, p);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

// ---- staging -------------------------------------------------------------------------------------
StagedMat::StagedMat(const void* host_or_dev, i64 nrows, i64 ncols, i64 rs, i64 cs, size_t elem, bool copy_in,
                     bool copy_out, cudaStream_t stream)
    : orig_((void*)host_or_dev), nrows_(nrows), ncols_(ncols), rs_(rs), cs_(cs), elem_(elem), copy_out_(copy_out),
      stream_(stream) {
  dev_ptr_ = orig_;
  dev_rs_ = rs;
  dev_cs_ = cs;
  if (nrows == 0 || ncols == 0 || is_device_pointer(host_or_dev)) {
    staged_ = false;
    return;
  }
  staged_ = true;
  char* base = (char*)orig_;
  if (rs == 1 && cs >= nrows) {
    mode_ = 1;  // column-major rectangle
    i64 ld = (nrows + 1) & ~(i64)1;
    buf_ = ws_alloc((size_t)ld * ncols * elem);
    dev_ptr_ = buf_;
    dev_rs_ = 1;
    dev_cs_ = ld;
    if (copy_in)
      FB_CUDA_CHECK(cudaMemcpy2DAsync(buf_, (size_t)ld * elem, base, (size_t)cs * elem, (size_t)nrows * elem,
                                      (size_t)ncols, cudaMemcpyHostToDevice, stream));
  } else if (cs == 1 && rs >= ncols) {
    mode_ = 2;  // row-major rectangle
    i64 ld = (ncols + 1) & ~(i64)1;
    buf_ = ws_alloc((size_t)ld * nrows * elem);
    dev_ptr_ = buf_;
    dev_rs_ = ld;
    dev_cs_ = 1;
    if (copy_in)
      FB_CUDA_CHECK(cudaMemcpy2DAsync(buf_, (size_t)ld * elem, base, (size_t)rs * elem, (size_t)ncols * elem,
                                      (size_t)nrows, cudaMemcpyHostToDevice, stream));
  } else {
    mode_ = 3;  // arbitrary strides: mirror the spanned address range (always copied in, so that the
                // untouched gaps are written back unchanged)
    i64 lo = 0, hi = 0;
    i64 r = (nrows - 1) * rs, c = (ncols - 1) * cs;
    if (r < 0) lo += r; else hi += r;
    if (c < 0) lo += c; else hi += c;
    span_lo_ = lo;
    span_elems_ = hi - lo + 1;
    buf_ = ws_alloc((size_t)span_elems_ * elem);
    FB_CUDA_CHECK(cudaMemcpyAsync(buf_, base + lo * (i64)elem, (size_t)span_elems_ * elem, cudaMemcpyHostToDevice,
                                  stream));
    dev_ptr_ = (char*)buf_ - lo * (i64)elem;
  }
}

void StagedMat::finish() {
  if (!staged_ || done_) return;
  done_ = true;
  char* base = (char*)orig_;
  if (copy_out_) {
    if (mode_ == 1)
      FB_CUDA_CHECK(cudaMemcpy2DAsync(base, (size_t)cs_ * elem_, buf_, (size_t)dev_cs_ * elem_, (size_t)nrows_ * elem_,
                                      (size_t)ncols_, cudaMemcpyDeviceToHost, stream_));
    else if (mode_ == 2)
      FB_CUDA_CHECK(cudaMemcpy2DAsync(base, (size_t)rs_ * elem_, buf_, (size_t)dev_rs_ * elem_, (size_t)ncols_ * elem_,
                                      (size_t)nrows_, cudaMemcpyDeviceToHost, stream_));
    else {
      // general strides: the mirror covers the whole spanned address range, but only the view's OWN elements go back —
      // another output of the same call may live in the gaps (e.g. A = buf[0::2], Q_coeff = buf[1::2]) and must not be
      // overwritten with the stale bytes this mirror was filled with
      std::vector<char> tmp((size_t)span_elems_ * elem_);
      FB_CUDA_CHECK(cudaMemcpyAsync(tmp.data(), buf_, tmp.size(), cudaMemcpyDeviceToHost, stream_));
      FB_CUDA_CHECK(cudaStreamSynchronize(stream_));
      for (i64 j = 0; j < ncols_; ++j)
        for (i64 i = 0; i < nrows_; ++i) {
          const i64 off = (i * rs_ + j * cs_) * (i64)elem_;
          memcpy(base + off, tmp.data() + (off - span_lo_ * (i64)elem_), elem_);
        }
    }
    FB_CUDA_CHECK(cudaStreamSynchronize(stream_));
  }
  ws_free(buf_);
  buf_ = nullptr;
}

StagedMat::~StagedMat() {
  if (staged_ && !done_) {
    // not finished explicitly: release without copying back
    FB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    ws_free(buf_);
  }
}

}  // namespace fb
