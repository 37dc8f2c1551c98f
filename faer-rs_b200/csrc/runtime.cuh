// Runtime plumbing shared by the C ABI: current stream, device check, staging of host views.
#pragma once
#include "common.cuh"
#include "linalg_f64.cuh"

#include <mutex>

namespace fb {

cudaStream_t current_stream();
void set_current_stream(cudaStream_t s);
// abort()s with a clear message if no CUDA device is usable (there is no CPU fallback).
void require_device();
// Every compute entry point of the C ABI holds this lock for the whole call. The library keeps per-process state
// (current stream, workspace pool, per-stream scratch, packed-operand workspaces, SM partitions, launch counter) and one
// GPU runs one factorization at a time anyway, so concurrent callers (the reference's entry points are reentrant) are
// serialised instead of racing. Recursive: entry points may call each other.
std::recursive_mutex& entry_mutex();
#define FB_ENTRY()                                                              \
  std::lock_guard<std::recursive_mutex> fb_entry_lock_(::fb::entry_mutex()); \
  ::fb::require_device()
bool is_device_pointer(const void* p);
// Run-time options (C ABI: faer_b200_set_option / faer_b200_get_option; initial values from the environment):
//   gemm_ws        FAER_B200_GEMM_WS        0 = never use the TMA / warp-specialised f64 GEMM, 1 = heuristic (default), 2 = always
//                                           (128 x 64 tiles), 3 = always (128 x 128 tiles)
//   f64_gemm_mode  FAER_B200_F64_GEMM_MODE  0 = native f64 tensor op (DMMA; default), 1 = int8-sliced wgmma products for  
//                                           large unstructured `matmul`s (opt-in; accuracy contract in gemm_f64_sliced.cuh)
enum Option : int { OPT_GEMM_WS = 0, OPT_F64_GEMM_MODE = 1, OPT_COUNT };
long long get_option(int opt);
bool set_option_by_name(const char* name, long long value);
long long get_option_by_name(const char* name);
// SMs a kernel launched on `st` may use: the device's SM count (cached), for every stream, including those of dist.cu's
// green-context partitions. Persistent kernels size their grids with it.
int stream_sms(cudaStream_t st);

// Optional per-launch timing of the dominant kernel (bench.py roofline): CUDA events around each GEMM launch.
bool profiling_enabled();
void profile_begin();
void profile_record_start(cudaStream_t st);
void profile_record_stop(cudaStream_t st, double flops);
void profile_end(double* flops, double* ms, unsigned long long* count);

// A matrix argument of the C ABI. Device pointers are used in place; host pointers are mirrored in device
// memory (H2D on construction if `copy_in`, D2H in finish() if `copy_out`).
class StagedMat {
 public:
  StagedMat(const void* host_or_dev, i64 nrows, i64 ncols, i64 rs, i64 cs, size_t elem, bool copy_in, bool copy_out,
            cudaStream_t stream);
  ~StagedMat();
  StagedMat(const StagedMat&) = delete;
  StagedMat& operator=(const StagedMat&) = delete;
  template <class T>
  View<T> view() const { return View<T>{(T*)dev_ptr_, nrows_, ncols_, dev_rs_, dev_cs_}; }
  bool staged() const { return staged_; }
  // copy back (if requested) and release the mirror; the stream must already be idle w.r.t. the compute,
  // or finish() must be called after the compute was enqueued on the same stream (copies are stream-ordered).
  void finish();

 private:
  void* orig_;
  i64 nrows_, ncols_, rs_, cs_;
  size_t elem_;
  bool copy_out_;
  cudaStream_t stream_;
  bool staged_ = false, done_ = false;
  int mode_ = 0;
  void* buf_ = nullptr;
  void* dev_ptr_ = nullptr;
  i64 dev_rs_ = 0, dev_cs_ = 0;
  i64 span_lo_ = 0, span_elems_ = 0;
};

}  // namespace fb
