// Measures the f64 roofline denominators on the box: the issue-bound throughput of every f64 DMMA shape sm_90a has
// (m8n8k4, m16n8k4, m16n8k8, m16n8k16; burst and ~2 s sustained), the DFMA peak, and, as sanity yardsticks only (never on
// the product path), cuBLAS DGEMM at a few sizes and cuBLAS DSYRK at the shape of LLT's largest trailing update.
// Every launch is checked: a launch that fails (e.g. too many registers for the block size) is reported, not timed.
// Build: make -C faer-rs_b200 tools/peaks     Run: tools/peaks [json_out]
#include <cublas_v2.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
#define CB(x) do { cublasStatus_t s = (x); if (s != CUBLAS_STATUS_SUCCESS) { printf("cuBLAS error %d line %d\n", (int)s, __LINE__); exit(1);} } while (0)

// SHAPE: 0 = m8n8k4, 1 = m16n8k4, 2 = m16n8k8, 3 = m16n8k16. NACC independent accumulator chains per warp.
template <int SHAPE>
struct Dmma;
template <>
struct Dmma<0> {
  static constexpr int M = 8, N = 8, K = 4, NC = 2;
  static constexpr const char* name = "m8n8k4";
  __device__ static void run(double* c, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
  }
};
template <>
struct Dmma<1> {
  static constexpr int M = 16, N = 8, K = 4, NC = 4;
  static constexpr const char* name = "m16n8k4";
  __device__ static void run(double* c, double a, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a), "d"(b), "d"(b));
  }
};
template <>
struct Dmma<2> {
  static constexpr int M = 16, N = 8, K = 8, NC = 4;
  static constexpr const char* name = "m16n8k8";
  __device__ static void run(double* c, double a, double b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a), "d"(b), "d"(a), "d"(b), "d"(b), "d"(a));
  }
};
template <>
struct Dmma<3> {
  static constexpr int M = 16, N = 8, K = 16, NC = 4;
  static constexpr const char* name = "m16n8k16";
  __device__ static void run(double* c, double a, double b) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
        "{%0,%1,%2,%3};\n"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a), "d"(b), "d"(a), "d"(b), "d"(a), "d"(b), "d"(a), "d"(b), "d"(b), "d"(a), "d"(b), "d"(a));
  }
};

template <int SHAPE, int NACC>
__global__ void dmma_peak(double* out, int iters) {
  using D = Dmma<SHAPE>;
  double c[NACC][D::NC];
  double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
#pragma unroll
  for (int i = 0; i < NACC; ++i)
#pragma unroll
    for (int e = 0; e < D::NC; ++e) c[i][e] = 0.0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) D::run(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NACC; ++i)
#pragma unroll
    for (int e = 0; e < D::NC; ++e) s += c[i][e];
  if (s == 123.456) out[0] = s;
}

template <int NACC>
__global__ void dfma_peak(double* out, int iters) {
  double c[NACC];
  double a = 1.0 + threadIdx.x * 1e-9, b = 1e-9;
#pragma unroll
  for (int i = 0; i < NACC; ++i) c[i] = i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) c[i] = fma(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NACC; ++i) s += c[i];
  if (s == 123.456) out[0] = s;
}

// best of `reps` timed calls of f (after one untimed call); a negative result means f's launch failed
template <class F>
float time_ms(F f, int reps) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  f();
  if (cudaGetLastError() != cudaSuccess) return -1.f;
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    CK(cudaEventRecord(e0));
    f();
    CK(cudaGetLastError());
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
  return best;
}

constexpr int NACC = 8;  // independent chains per warp (latency hiding comes from NACC x warps per SM)

struct ShapeResult {
  const char* name;
  double burst, sustained;
};

template <int SHAPE>
ShapeResult measure_shape(int sms, double* out) {
  using D = Dmma<SHAPE>;
  const int iters = 160000 / D::K;  // same k-depth of work per chain for every shape
  const double flop_per_warp = 2.0 * D::M * D::N * D::K * (double)NACC * iters;
  double best = 0;
  int best_warps = 0;
  for (int warps : {4, 8, 16}) {
    const float ms = time_ms([&] { dmma_peak<SHAPE, NACC><<<sms, warps * 32>>>(out, iters); }, 5);
    if (ms < 0) {
      printf("DMMA %-8s %2d warps/SM: launch failed\n", D::name, warps);
      continue;
    }
    const double tf = flop_per_warp * warps * sms / (ms * 1e-3) / 1e12;
    printf("DMMA %-8s %2d warps/SM, %d chains/warp: %8.3f ms  %6.2f TFLOP/s\n", D::name, warps, NACC, ms, tf);
    if (tf > best) { best = tf; best_warps = warps; }
  }
  // sustained (~2 s back to back) at the best burst configuration: the power-limited figure
  double sustained = 0;
  if (best_warps) {
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    float total = 0;
    int reps = 0;
    while (total < 2000.f && reps < 100000) {
      for (int i = 0; i < 10; ++i) dmma_peak<SHAPE, NACC><<<sms, best_warps * 32>>>(out, iters);
      CK(cudaGetLastError());
      reps += 10;
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      CK(cudaEventElapsedTime(&total, e0, e1));
    }
    sustained = flop_per_warp * best_warps * sms * reps / (total * 1e-3) / 1e12;
    printf("DMMA %-8s sustained over %.0f ms (%d warps/SM): %.2f TFLOP/s\n", D::name, total, best_warps, sustained);
    CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
  }
  return {D::name, best, sustained};
}

int main(int argc, char** argv) {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  int sms = prop.multiProcessorCount;
  printf("device: %s, %d SMs, %.0f MHz max\n", prop.name, sms, prop.clockRate / 1e3);
  double* out; CK(cudaMalloc(&out, 1024));
  std::vector<ShapeResult> dmma;
  dmma.push_back(measure_shape<0>(sms, out));
  dmma.push_back(measure_shape<1>(sms, out));
  dmma.push_back(measure_shape<2>(sms, out));
  dmma.push_back(measure_shape<3>(sms, out));
  double best_dfma = 0;
  const int iters = 20000;
  for (int warps : {8, 16, 32}) {
    float ms = time_ms([&] { dfma_peak<16><<<sms, warps * 32>>>(out, iters); }, 5);
    if (ms < 0) {
      printf("DFMA 16 acc, %2d warps/SM: launch failed\n", warps);
      continue;
    }
    double flops = 2.0 * 32 * 16.0 * iters * warps * sms;
    double tf = flops / (ms * 1e-3) / 1e12;
    printf("DFMA 16 acc, %2d warps/SM: %.3f ms  %.2f TFLOP/s\n", warps, ms, tf);
    if (tf > best_dfma) best_dfma = tf;
  }
  // cuBLAS yardsticks
  cublasHandle_t h; CB(cublasCreate(&h));
  std::vector<std::pair<int, double>> cub;
  for (int n : {4096, 8192, 16384}) {
    double *A, *B, *C;
    size_t bytes = (size_t)n * n * 8;
    CK(cudaMalloc(&A, bytes)); CK(cudaMalloc(&B, bytes)); CK(cudaMalloc(&C, bytes));
    CK(cudaMemset(A, 0, bytes)); CK(cudaMemset(B, 0, bytes));
    double one = 1.0, zero = 0.0;
    float ms = time_ms([&] { CB(cublasDgemm(h, CUBLAS_OP_N, CUBLAS_OP_N, n, n, n, &one, A, n, B, n, &zero, C, n)); }, n >= 16384 ? 2 : 4);
    double tf = 2.0 * n * (double)n * n / (ms * 1e-3) / 1e12;
    printf("cuBLAS DGEMM n=%d: %.3f ms  %.2f TFLOP/s\n", n, ms, tf);
    cub.push_back({n, tf});
    CK(cudaFree(A)); CK(cudaFree(B)); CK(cudaFree(C));
  }
  // DSYRK C(lower) = C - P P^T at the shape of LLT's largest trailing update (n = 16128, k = 256); flop = n (n + 1) k
  double syrk_tf = 0, syrk_ms = 0;
  {
    const int n = 16128, k = 256;
    double *P, *C;
    CK(cudaMalloc(&P, (size_t)n * k * 8)); CK(cudaMalloc(&C, (size_t)n * n * 8));
    CK(cudaMemset(P, 0, (size_t)n * k * 8)); CK(cudaMemset(C, 0, (size_t)n * n * 8));
    double minus_one = -1.0, one = 1.0;
    syrk_ms = time_ms([&] { CB(cublasDsyrk(h, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N, n, k, &minus_one, P, n, &one, C, n)); }, 10);
    syrk_tf = (double)n * (n + 1.0) * k / (syrk_ms * 1e-3) / 1e12;
    printf("cuBLAS DSYRK lower n=%d k=%d: %.3f ms  %.2f TFLOP/s\n", n, k, syrk_ms, syrk_tf);
    CK(cudaFree(P)); CK(cudaFree(C));
  }
  CB(cublasDestroy(h));
  if (argc > 1) {
    FILE* f = fopen(argv[1], "w");
    fprintf(f, "{\"gpu\": \"%s\", \"sms\": %d, \"dmma_tflops\": {", prop.name, sms);
    for (size_t i = 0; i < dmma.size(); ++i)
      fprintf(f, "%s\"%s\": {\"burst\": %.3f, \"sustained\": %.3f}", i ? ", " : "", dmma[i].name, dmma[i].burst, dmma[i].sustained);
    fprintf(f, "}, \"dfma_tflops\": %.3f, \"cublas_dgemm_tflops\": {", best_dfma);
    for (size_t i = 0; i < cub.size(); ++i) fprintf(f, "%s\"%d\": %.3f", i ? ", " : "", cub[i].first, cub[i].second);
    fprintf(f, "}, \"cublas_dsyrk_n16128_k256\": {\"ms\": %.4f, \"tflops\": %.3f}}\n", syrk_ms, syrk_tf);
    fclose(f);
  }
  return 0;
}
