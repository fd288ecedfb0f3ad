// Kernels and launches of the batched pair HMM (lane logic: b2a_pairhmm.cuh; entry points: b2a_engine.cu).
#include <cuda_runtime.h>

#include <algorithm>

#include "b2a_pairhmm.cuh"

namespace b2a {
namespace {

constexpr int kPhmmWarps = 4;  // warps per CTA

// persistent warps: each takes the tier's pairs from the counter; the emission tables sit in shared memory
template <int C>
__global__ void __launch_bounds__(kPhmmWarps * 32) pairhmm_kernel(PairHmmArgs a, uint32_t* __restrict__ ctr) {
  __shared__ double emit[4 * 256];
  for (uint32_t k = threadIdx.x; k < 4 * a.n_classes; k += blockDim.x) emit[k] = a.emit[k];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint64_t w = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  PairHmmRec* rec = a.rec + w * a.rec_stride;
  double* cols = a.cols + w * a.cols_stride;
  for (;;) {
    uint32_t t = 0;
    if (lane == 0) t = atomicAdd(ctr, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= a.n_tasks) break;
    const uint32_t p = a.tasks[t];
    const uint64_t xo = a.x_off[p], yo = a.y_off[p];
    const PairHmmSeq s{a.seq + xo, a.cls ? a.cls + xo : nullptr, a.seq + yo, a.cls ? a.cls + yo : nullptr, a.x_len[p],
                       a.y_len[p]};
    const double r = pairhmm_warp<C>(a.g, emit, a.n_classes, s, rec, cols, lane);
    if (lane == 0) a.prob[p] = r;
  }
}

template <int C>
cudaError_t grid_of(int num_sms, uint32_t n_tasks, int* ctas) {
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pairhmm_kernel<C>, kPhmmWarps * 32, 0);
  if (e != cudaSuccess) return e;
  const uint64_t need = ((uint64_t)n_tasks + kPhmmWarps - 1) / kPhmmWarps;
  *ctas = (int)std::max<uint64_t>(1, std::min<uint64_t>(need, (uint64_t)std::max(per_sm, 1) * num_sms));
  return cudaSuccess;
}

}  // namespace

cudaError_t pairhmm_grid(int tier, int num_sms, uint32_t n_tasks, int* ctas, int* warps_per_cta) {
  *warps_per_cta = kPhmmWarps;
  switch (tier) {
    case PT_C1: return grid_of<1>(num_sms, n_tasks, ctas);
    case PT_C2: return grid_of<2>(num_sms, n_tasks, ctas);
    case PT_C4: return grid_of<4>(num_sms, n_tasks, ctas);
    case PT_C5: return grid_of<5>(num_sms, n_tasks, ctas);
    case PT_C8:
    case PT_STRIP: return grid_of<8>(num_sms, n_tasks, ctas);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_pairhmm(int tier, const PairHmmArgs& a, int ctas, int warps_per_cta, uint32_t* ctr,
                           cudaStream_t st) {
  if (!a.n_tasks) return cudaSuccess;
  const int threads = warps_per_cta * 32;
  switch (tier) {
    case PT_C1: pairhmm_kernel<1><<<ctas, threads, 0, st>>>(a, ctr); break;
    case PT_C2: pairhmm_kernel<2><<<ctas, threads, 0, st>>>(a, ctr); break;
    case PT_C4: pairhmm_kernel<4><<<ctas, threads, 0, st>>>(a, ctr); break;
    case PT_C5: pairhmm_kernel<5><<<ctas, threads, 0, st>>>(a, ctr); break;
    case PT_C8:
    case PT_STRIP: pairhmm_kernel<8><<<ctas, threads, 0, st>>>(a, ctr); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace b2a
