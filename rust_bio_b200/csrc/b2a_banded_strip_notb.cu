// The score-only (F_NOTB) twins of the strip-wavefront fill (b2a_banded_strip.cuh), one per flag set the engine
// selects, in a translation unit of their own so that they compile in parallel with b2a_engine.cu.
#include <cuda_runtime.h>

#define B2A_BANDED_NO_KERNELS  // b2a_engine.cu defines the K4 / K3 kernels
#include "b2a_banded_strip.cuh"

namespace b2a {

cudaError_t launch_banded_strip_fill_notb(int flags, unsigned grid, size_t smem, cudaStream_t st, const StripParams& sp) {
  switch (flags) {
#define B2A_KSN_CASE1(F)                                                                                                       \
  case (F) | F_NOTB:                                                                                                           \
    if (smem > 48 * 1024) {                                                                                                    \
      const cudaError_t ce = cudaFuncSetAttribute(banded_strip_fill_kernel<(F) | F_NOTB>,                                      \
                                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                     \
      if (ce != cudaSuccess) return ce;                                                                                        \
    }                                                                                                                          \
    banded_strip_fill_kernel<(F) | F_NOTB><<<grid, KS_WARPS * 32, smem, st>>>(sp);                                             \
    return cudaGetLastError();
#define B2A_KSN_CASE(F) B2A_KSN_CASE1(F) B2A_KSN_CASE1((F) | F_LUT)
    B2A_KSN_CASE(0)
    B2A_KSN_CASE(F_TRACK_ROWS)
    B2A_KSN_CASE(F_CLIPX)
    B2A_KSN_CASE(F_CLIPY)
    B2A_KSN_CASE(F_TRACK_ROWS | F_CLIPX)
    B2A_KSN_CASE(F_TRACK_ROWS | F_CLIPY)
    B2A_KSN_CASE(F_CLIPX | F_CLIPY)
    B2A_KSN_CASE(F_TRACK_ROWS | F_CLIPX | F_CLIPY)
    B2A_KSN_CASE(F_TRACK_COLS)
    B2A_KSN_CASE(F_TRACK_COLS | F_TRACK_ROWS)
    B2A_KSN_CASE(F_TRACK_COLS | F_CLIPX)
    B2A_KSN_CASE(F_TRACK_COLS | F_CLIPY)
    B2A_KSN_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPX)
    B2A_KSN_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPY)
    B2A_KSN_CASE(F_TRACK_COLS | F_CLIPX | F_CLIPY)
    B2A_KSN_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPX | F_CLIPY)
#undef B2A_KSN_CASE
#undef B2A_KSN_CASE1
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace b2a
