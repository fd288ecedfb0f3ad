// Kernels and launches of the batched Myers pattern matching (lane logic: b2a_myers.cuh; entry points:
// b2a_engine.cu).
#include <cuda_runtime.h>

#include <algorithm>

#include "b2a_myers.cuh"

namespace b2a {
namespace {

constexpr uint32_t kMyersSmem = 96 * 1024;  // dynamic shared memory a CTA may ask for (match masks)
constexpr int kThreadCta = 128;             // threads per CTA of the thread-per-pair tier, when the masks fit

// the pair's hits start at hit_off[p] in pass 2; pass 1 writes no hits
__device__ __forceinline__ void myers_store(const MyersArgs& a, uint32_t p, const MyersResult& r) {
  if (a.hit_off) return;
  a.best_end[p] = r.best_end;
  a.best_dist[p] = r.best_dist;
  if (a.count) a.count[p] = r.count;
}

// one thread per pair; TIER in MT_REGS1 .. MT_REGS1 + 3
template <int TIER>
__global__ void __launch_bounds__(kThreadCta) myers_thread_kernel(MyersArgs a) {
  extern __shared__ uint64_t peq[];
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.n_tasks) return;
  const uint32_t p = a.tasks[t];
  const DistPair d = myers_pair(a.codes, a.x_off[p], a.x_len[p], a.y_off[p], a.y_len[p]);
  const uint64_t o = a.hit_off ? a.hit_off[p] : 0;
  const MyersResult r = myers_regs<TIER - MT_REGS1 + 1>(d, peq + threadIdx.x, blockDim.x, a.sigma, a.match, a.k,
                                                        a.hit_off ? a.hit_end + o : nullptr, a.hit_dist + o);
  myers_store(a, p, r);
}

// persistent warps: each takes MT_WARP pairs from the counter and owns `bnd_words` boundary words
__global__ void __launch_bounds__(256) myers_warp_kernel(MyersArgs a, uint32_t* __restrict__ bnd, uint64_t bnd_words,
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
    const DistPair d = myers_pair(a.codes, a.x_off[p], a.x_len[p], a.y_off[p], a.y_len[p]);
    const uint64_t o = a.hit_off ? a.hit_off[p] : 0;
    const MyersResult r = myers_warp<32>(d, mine, a.sigma, a.match, my_bnd, lane, a.k,
                                         a.hit_off ? a.hit_end + o : nullptr, a.hit_dist + o);
    if (lane == 0) myers_store(a, p, r);
    __syncwarp();
  }
}

// a warp's tasks that go on to pass 2 take their slots with one atomic per tier present in the warp
__global__ void __launch_bounds__(256) myers_select_kernel(const uint32_t* __restrict__ order, MyersSegs seg,
                                                           const uint32_t* __restrict__ count, uint32_t* __restrict__ out,
                                                           uint32_t* __restrict__ n_out) {
  const uint32_t n_all = seg.at[MT_COUNT];
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const uint32_t p = i < n_all ? order[i] : 0;
  const bool keep = i < n_all && count[p] != 0;
  int tier = MT_REGS1;
  while (tier + 1 < MT_COUNT && i >= seg.at[tier + 1]) ++tier;
  const uint32_t kept = __ballot_sync(0xffffffffu, keep);
  if (!kept) return;
  const uint32_t same = __match_any_sync(0xffffffffu, tier) & kept;
  if (!keep) return;
  const int leader = __ffs(same) - 1;
  uint32_t base = 0;
  if (lane == leader) base = atomicAdd(&n_out[tier], (uint32_t)__popc(same));
  base = __shfl_sync(same, base, leader);
  out[seg.at[tier] + base + __popc(same & ((1u << lane) - 1u))] = p;
}

template <int TIER>
cudaError_t launch_thread_tier(const MyersArgs& a, int words, cudaStream_t st) {
  const uint32_t per_thread = (uint32_t)a.sigma * (uint32_t)words * 8;
  int threads = (int)std::min<uint32_t>(kThreadCta, kMyersSmem / per_thread);
  if (threads >= 32) threads &= ~31;
  const uint32_t smem = per_thread * (uint32_t)threads;
  cudaError_t e = cudaFuncSetAttribute(myers_thread_kernel<TIER>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)kMyersSmem);
  if (e != cudaSuccess) return e;
  myers_thread_kernel<TIER><<<(a.n_tasks + threads - 1) / threads, threads, smem, st>>>(a);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_myers_thread(int tier, const MyersArgs& a, cudaStream_t st) {
  if (!a.n_tasks) return cudaSuccess;
  switch (tier) {
    case MT_REGS1: return launch_thread_tier<MT_REGS1>(a, 1, st);
    case MT_REGS1 + 1: return launch_thread_tier<MT_REGS1 + 1>(a, 2, st);
    case MT_REGS1 + 2: return launch_thread_tier<MT_REGS1 + 2>(a, 3, st);
    case MT_REGS1 + 3: return launch_thread_tier<MT_REGS1 + 3>(a, 4, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t myers_warp_grid(int sigma, int num_sms, uint32_t n_tasks, int* ctas, int* warps_per_cta) {
  const uint32_t per_warp = (uint32_t)sigma * 32 * 8;
  const int wpc = (int)std::max<uint32_t>(1, std::min<uint32_t>(8, kMyersSmem / per_warp));
  cudaError_t e = cudaFuncSetAttribute(myers_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMyersSmem);
  if (e != cudaSuccess) return e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, myers_warp_kernel, wpc * 32, (size_t)per_warp * wpc);
  if (e != cudaSuccess) return e;
  const uint64_t need = ((uint64_t)n_tasks + wpc - 1) / wpc;
  *ctas = (int)std::max<uint64_t>(1, std::min<uint64_t>(need, (uint64_t)std::max(per_sm, 1) * num_sms));
  *warps_per_cta = wpc;
  return cudaSuccess;
}

cudaError_t launch_myers_warp(const MyersArgs& a, int ctas, int warps_per_cta, uint32_t* bnd, uint64_t bnd_words,
                              uint32_t* ctr, cudaStream_t st) {
  if (!a.n_tasks) return cudaSuccess;
  const size_t smem = (size_t)a.sigma * 32 * 8 * warps_per_cta;
  myers_warp_kernel<<<ctas, warps_per_cta * 32, smem, st>>>(a, bnd, bnd_words, ctr);
  return cudaGetLastError();
}

cudaError_t launch_myers_select(const uint32_t* order, MyersSegs seg, const uint32_t* count, uint32_t* out,
                                uint32_t* n_out, cudaStream_t st) {
  const uint32_t n_all = seg.at[MT_COUNT];
  if (!n_all) return cudaSuccess;
  myers_select_kernel<<<(n_all + 255) / 256, 256, 0, st>>>(order, seg, count, out, n_out);
  return cudaGetLastError();
}

}  // namespace b2a
