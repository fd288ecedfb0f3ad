// Kernels and launches of the batched edit distances (lane logic: b2a_distance.cuh; entry points: b2a_engine.cu).
#include <cuda_runtime.h>

#include <algorithm>

#include "b2a_distance.cuh"

namespace b2a {
namespace {

constexpr uint32_t kDistSmem = 96 * 1024;  // dynamic shared memory a distance CTA may ask for (match masks)
constexpr int kThreadCta = 128;            // threads per CTA of the thread-per-pair tiers, when the masks fit

__global__ void __launch_bounds__(256) dist_translate_kernel(uint8_t* __restrict__ blob, uint64_t n,
                                                             const uint8_t* __restrict__ codemap) {
  __shared__ uint8_t map[256];
  map[threadIdx.x] = codemap[threadIdx.x];
  __syncthreads();
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x * 4;
  for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    if (i + 4 <= n) {
      uint32_t v = *reinterpret_cast<uint32_t*>(blob + i);
      v = (uint32_t)map[v & 0xFF] | ((uint32_t)map[(v >> 8) & 0xFF] << 8) | ((uint32_t)map[(v >> 16) & 0xFF] << 16) |
          ((uint32_t)map[v >> 24] << 24);
      *reinterpret_cast<uint32_t*>(blob + i) = v;
    } else {
      for (uint64_t b = i; b < n; ++b) blob[b] = map[blob[b]];
    }
  }
}

// one thread per pair; TIER in DT_REGS1 .. DT_BAND8
template <int TIER>
__global__ void __launch_bounds__(kThreadCta) lev_thread_kernel(DistArgs a) {
  extern __shared__ uint64_t peq[];
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.n_tasks) return;
  const uint32_t p = a.tasks[t];
  const DistPair d = dist_pair(a.codes, a.x_off[p], a.x_len[p], a.y_off[p], a.y_len[p], a.k);
  uint64_t* mine = peq + threadIdx.x;
  uint32_t r;
  if constexpr (TIER == DT_BAND4)
    r = lev_band<4>(d, mine, blockDim.x, a.sigma);
  else if constexpr (TIER == DT_BAND8)
    r = lev_band<8>(d, mine, blockDim.x, a.sigma);
  else
    r = lev_regs<TIER - DT_REGS1 + 1>(d, mine, blockDim.x, a.sigma);
  a.dist[p] = r;
}

// persistent warps: each takes DT_WARP pairs from the counter and owns `bnd_words` boundary words
__global__ void __launch_bounds__(256) lev_warp_kernel(DistArgs a, uint32_t* __restrict__ bnd, uint64_t bnd_words,
                                                       uint32_t* __restrict__ ctr) {
  extern __shared__ uint64_t peq[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint64_t* mine = peq + (size_t)wid * 32 * a.sigma;
  uint32_t* my_bnd = bnd + ((uint64_t)blockIdx.x * (blockDim.x >> 5) + wid) * bnd_words;
  for (;;) {
    uint32_t t = 0;
    if (lane == 0) t = atomicAdd(ctr, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= a.n_tasks) break;
    const uint32_t p = a.tasks[t];
    const DistPair d = dist_pair(a.codes, a.x_off[p], a.x_len[p], a.y_off[p], a.y_len[p], a.k);
    const uint32_t r = lev_warp<32>(d, mine, a.sigma, my_bnd, lane);
    if (lane == 0) a.dist[p] = r;
    __syncwarp();
  }
}

// one warp per pair over every pair of equal lengths
__global__ void __launch_bounds__(256) hamming_kernel(DistArgs a, uint64_t n_pairs) {
  const int lane = threadIdx.x & 31;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t p = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_pairs; p += nwarps) {
    const uint32_t L = a.x_len[p];
    if (L != a.y_len[p]) continue;
    const uint32_t r = hamming_coop<32>(a.codes + a.x_off[p], a.codes + a.y_off[p], L, lane);
    if (lane == 0) a.dist[p] = r;
  }
}

template <int TIER>
cudaError_t launch_thread_tier(const DistArgs& a, int words, cudaStream_t st) {
  const uint32_t per_thread = (uint32_t)a.sigma * (uint32_t)words * 8;
  int threads = (int)std::min<uint32_t>(kThreadCta, kDistSmem / per_thread);
  if (threads >= 32) threads &= ~31;
  const uint32_t smem = per_thread * (uint32_t)threads;
  cudaError_t e = cudaFuncSetAttribute(lev_thread_kernel<TIER>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDistSmem);
  if (e != cudaSuccess) return e;
  lev_thread_kernel<TIER><<<(a.n_tasks + threads - 1) / threads, threads, smem, st>>>(a);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_dist_translate(uint8_t* blob, uint64_t bytes, const uint8_t* codemap, int num_sms, cudaStream_t st) {
  if (!bytes) return cudaSuccess;
  const uint64_t want = (bytes / 4 + 255) / 256;
  dist_translate_kernel<<<(unsigned)std::min<uint64_t>(std::max<uint64_t>(want, 1), (uint64_t)num_sms * 8), 256, 0, st>>>(
      blob, bytes, codemap);
  return cudaGetLastError();
}

cudaError_t launch_lev_thread(int tier, const DistArgs& a, cudaStream_t st) {
  if (!a.n_tasks) return cudaSuccess;
  switch (tier) {
    case DT_REGS1: return launch_thread_tier<DT_REGS1>(a, 1, st);
    case DT_REGS1 + 1: return launch_thread_tier<DT_REGS1 + 1>(a, 2, st);
    case DT_REGS1 + 2: return launch_thread_tier<DT_REGS1 + 2>(a, 3, st);
    case DT_REGS1 + 3: return launch_thread_tier<DT_REGS1 + 3>(a, 4, st);
    case DT_BAND4: return launch_thread_tier<DT_BAND4>(a, 4, st);
    case DT_BAND8: return launch_thread_tier<DT_BAND8>(a, 8, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t lev_warp_grid(int sigma, int num_sms, uint32_t n_tasks, int* ctas, int* warps_per_cta) {
  const uint32_t per_warp = (uint32_t)sigma * 32 * 8;
  const int wpc = (int)std::max<uint32_t>(1, std::min<uint32_t>(8, kDistSmem / per_warp));
  cudaError_t e = cudaFuncSetAttribute(lev_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDistSmem);
  if (e != cudaSuccess) return e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lev_warp_kernel, wpc * 32, (size_t)per_warp * wpc);
  if (e != cudaSuccess) return e;
  const uint64_t need = ((uint64_t)n_tasks + wpc - 1) / wpc;
  *ctas = (int)std::max<uint64_t>(1, std::min<uint64_t>(need, (uint64_t)std::max(per_sm, 1) * num_sms));
  *warps_per_cta = wpc;
  return cudaSuccess;
}

cudaError_t launch_lev_warp(const DistArgs& a, int ctas, int warps_per_cta, uint32_t* bnd, uint64_t bnd_words,
                            uint32_t* ctr, cudaStream_t st) {
  if (!a.n_tasks) return cudaSuccess;
  const size_t smem = (size_t)a.sigma * 32 * 8 * warps_per_cta;
  lev_warp_kernel<<<ctas, warps_per_cta * 32, smem, st>>>(a, bnd, bnd_words, ctr);
  return cudaGetLastError();
}

cudaError_t launch_hamming(const DistArgs& a, uint64_t n_pairs, int num_sms, cudaStream_t st) {
  if (!n_pairs) return cudaSuccess;
  const uint64_t want = (n_pairs + 7) / 8;
  hamming_kernel<<<(unsigned)std::min<uint64_t>(want, (uint64_t)num_sms * 16), 256, 0, st>>>(a, n_pairs);
  return cudaGetLastError();
}

}  // namespace b2a
