// Host entry points of the K1 instantiations (one translation unit per (G, R)
// shape, see b2a_fill_inst.cu) so nvcc can build them in parallel.
#pragma once
#include <cuda_runtime.h>

#include "b2a_fill.cuh"

namespace b2a {

typedef cudaError_t (*FillLaunchFn)(int flags, const FillParams& prm, uint32_t ntasks, int num_sms,
                                    cudaStream_t stream, int* grid_out, int dry);

struct FillLaunch {
  int G, R;
  // launches the variant for `flags`; smem/grid are computed inside. Returns the grid used.
  // dry != 0: nothing is launched, *grid_out = the warps of this variant resident on the whole GPU.
  FillLaunchFn launch;
  // the F_NOTB variants (score-only batches), built for the shapes choose_shape picks; null for the others
  FillLaunchFn launch_notb;
  // the recomputed-traceback fills (F_CKPT pass and F_REFILL windows), warp-per-pair shapes only; null for the others
  FillLaunchFn launch_recompute = nullptr;
};

#define B2A_DECLARE_FILL(G, R)                                                                  \
  cudaError_t launch_fill_##G##_##R(int flags, const FillParams& prm, uint32_t ntasks,          \
                                    int num_sms, cudaStream_t stream, int* grid_out, int dry);
#define B2A_DECLARE_FILL_NOTB(G, R)                                                             \
  cudaError_t launch_fill_notb_##G##_##R(int flags, const FillParams& prm, uint32_t ntasks,     \
                                         int num_sms, cudaStream_t stream, int* grid_out, int dry);
#define B2A_DECLARE_FILL_RECOMPUTE(G, R)                                                        \
  cudaError_t launch_fill_recompute_##G##_##R(int flags, const FillParams& prm, uint32_t ntasks, \
                                              int num_sms, cudaStream_t stream, int* grid_out, int dry);

B2A_DECLARE_FILL(1, 16)
B2A_DECLARE_FILL(1, 8)
B2A_DECLARE_FILL(1, 20)
B2A_DECLARE_FILL(2, 16)
B2A_DECLARE_FILL(2, 20)
B2A_DECLARE_FILL(4, 16)
B2A_DECLARE_FILL(8, 16)
B2A_DECLARE_FILL(8, 20)
B2A_DECLARE_FILL(32, 8)
B2A_DECLARE_FILL(32, 16)
B2A_DECLARE_FILL_NOTB(1, 16)
B2A_DECLARE_FILL_NOTB(8, 16)
B2A_DECLARE_FILL_NOTB(8, 20)
B2A_DECLARE_FILL_NOTB(32, 8)
B2A_DECLARE_FILL_NOTB(32, 16)
B2A_DECLARE_FILL_RECOMPUTE(32, 8)
B2A_DECLARE_FILL_RECOMPUTE(32, 16)

}  // namespace b2a
