// Measured int32 ALU peak (SURVEY 8d: "P_int32 measured on the GPU ... a committed microbenchmark of
// independent IADD3 / VIMNMX chains over all SMs").  Measurement infrastructure for bench.py's
// int32 roofline; not on the alignment path.
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int CHAINS = 8;
constexpr int ITERS = 4096;

// kind 0: add chains; 1: max chains; 2: add+max alternating (the DP's own mix)
template <int KIND>
__global__ void __launch_bounds__(256) int32_chain_kernel(int32_t* out, int32_t seed) {
  int32_t a[CHAINS], b[CHAINS];
#pragma unroll
  for (int k = 0; k < CHAINS; ++k) {
    a[k] = seed + (int32_t)threadIdx.x * (k + 1);
    b[k] = seed * (k + 3) - (int32_t)blockIdx.x;
  }
#pragma unroll 1
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int k = 0; k < CHAINS; ++k) {
      if (KIND == 0) {
        asm volatile("add.s32 %0, %0, %1;" : "+r"(a[k]) : "r"(b[k]));
        asm volatile("add.s32 %0, %0, %1;" : "+r"(b[k]) : "r"(a[k]));
      } else if (KIND == 1) {
        asm volatile("max.s32 %0, %0, %1;" : "+r"(a[k]) : "r"(b[k]));
        asm volatile("min.s32 %0, %0, %1;" : "+r"(b[k]) : "r"(a[k]));
      } else {
        asm volatile("add.s32 %0, %0, %1;" : "+r"(a[k]) : "r"(b[k]));
        asm volatile("max.s32 %0, %0, %1;" : "+r"(b[k]) : "r"(a[k]));
      }
    }
  }
  int32_t acc = 0;
#pragma unroll
  for (int k = 0; k < CHAINS; ++k) acc ^= a[k] ^ b[k];
  if (acc == 0x7fffffff) out[0] = acc;  // never true in practice; keeps the chains alive
}

template <int KIND>
float run_kind(int sms, int32_t* d_out) {
  const int grid = sms * 16;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  int32_chain_kernel<KIND><<<grid, 256>>>(d_out, 12345);  // warm-up
  float best = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    cudaEventRecord(e0);
    int32_chain_kernel<KIND><<<grid, 256>>>(d_out, 12345 + rep);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  const double ops = (double)grid * 256.0 * ITERS * CHAINS * 2.0;
  return (float)(ops / (best * 1e-3) / 1e12);  // tera lane-ops / s
}

}  // namespace

extern "C" int32_t b2a_util_int32_peak(int32_t device_id, float* tops_add, float* tops_minmax,
                                       float* tops_mixed) {
  if (cudaSetDevice(device_id) != cudaSuccess) return -2;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess) return -2;
  int32_t* d_out = nullptr;
  if (cudaMalloc(&d_out, 64) != cudaSuccess) return -3;
  const float a = run_kind<0>(prop.multiProcessorCount, d_out);
  const float b = run_kind<1>(prop.multiProcessorCount, d_out);
  const float c = run_kind<2>(prop.multiProcessorCount, d_out);
  cudaFree(d_out);
  if (cudaGetLastError() != cudaSuccess) return -3;
  if (tops_add) *tops_add = a;
  if (tops_minmax) *tops_minmax = b;
  if (tops_mixed) *tops_mixed = c;
  return 0;
}
