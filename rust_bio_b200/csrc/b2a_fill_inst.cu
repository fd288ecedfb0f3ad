// One (G, R) shape of the K1 fill kernel: compile with -DB2A_G=<G> -DB2A_R=<R>.  With -DB2A_NOTB the same
// flag cases are instantiated with F_NOTB added (score-only batches) as launch_fill_notb_<G>_<R>, in a
// translation unit of their own so that the build stays parallel.  With -DB2A_RECOMPUTE (warp-per-pair shapes) the
// recomputed-traceback fills are instantiated as launch_fill_recompute_<G>_<R>: the F_NOTB | F_CKPT pass over the flag
// cases of a recomputing batch (F_PACKREL or explicit trackers, F_YSTREAM), and the tracker-free F_REFILL fills.
#include "b2a_fill_launch.h"

#ifndef B2A_G
#error "compile with -DB2A_G=... -DB2A_R=..."
#endif

#if defined(B2A_RECOMPUTE)
#define B2A_LAUNCH_NAME launch_fill_recompute_
#elif defined(B2A_NOTB)
#define B2A_LAUNCH_NAME launch_fill_notb_
#else
#define B2A_LAUNCH_NAME launch_fill_
#endif

namespace b2a {

namespace {

template <int FLAGS>
cudaError_t go(const FillParams& prm, uint32_t ntasks, int num_sms, cudaStream_t stream,
               int* grid_out, int dry) {
  auto kern = fill_kernel<B2A_G, B2A_R, FLAGS>;
  constexpr int FILL_WARPS = fill_warps_of(B2A_G, B2A_R);
  const uint32_t lut_bytes = (FLAGS & F_LUT) ? lut_smem_bytes(prm.sc.alpha) : 0u;
  const size_t smem = 64 + lut_bytes + (size_t)FILL_WARPS * prm.smem_seq_bytes;
  cudaError_t err =
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return err;
  int per_sm = 0;
  err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, FILL_WARPS * 32, smem);
  if (err != cudaSuccess) return err;
  if (per_sm < 1) return cudaErrorLaunchOutOfResources;
  if (dry) {  // no launch: how many warps of this kernel are resident on the whole GPU
    if (grid_out) *grid_out = num_sms * per_sm * FILL_WARPS;
    return cudaSuccess;
  }
  const uint32_t want = (ntasks + FILL_WARPS - 1) / FILL_WARPS;
  uint32_t grid = (uint32_t)(num_sms * per_sm);
  if (grid > want) grid = want;
  if (prm.task_limit) grid = (want + prm.task_limit - 1) / prm.task_limit;  // every warp retires after task_limit tasks
  if (grid < 1) grid = 1;
  if (grid_out) *grid_out = (int)grid;
  kern<<<grid, FILL_WARPS * 32, smem, stream>>>(prm);
  return cudaGetLastError();
}

}  // namespace

#define B2A_CAT2(a, b, c) a##b##_##c
#define B2A_CAT(a, b, c) B2A_CAT2(a, b, c)

cudaError_t B2A_CAT(B2A_LAUNCH_NAME, B2A_G, B2A_R)(int flags, const FillParams& prm, uint32_t ntasks,
                                                   int num_sms, cudaStream_t stream, int* grid_out, int dry) {
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
#if defined(B2A_RECOMPUTE)
  static_assert(B2A_G == 32, "the recomputed traceback is a warp-per-pair form");
#define B2A_CASE(F) case (F): return go<(F)>(prm, ntasks, num_sms, stream, grid_out, dry);
#define B2A_PASS1(F) B2A_CASE(F_NOTB | F_CKPT | F_YSTREAM | (F))
#define B2A_REFILL(F) B2A_CASE(F_REFILL | F_YSTREAM | (F))
  switch (flags) {
    B2A_PASS1(0)
    B2A_PASS1(F_TRACK_ROWS)
    B2A_PASS1(F_TRACK_ROWS | F_PACKREL)
    B2A_PASS1(ALL)
    B2A_PASS1(ALL | F_PACKREL)
    B2A_PASS1(ALL | F_RELU)
    B2A_PASS1(ALL | F_PACKREL | F_RELU)
    B2A_PASS1(F_LUT)
    B2A_PASS1(F_LUT | F_TRACK_ROWS)
    B2A_PASS1(F_LUT | F_TRACK_ROWS | F_PACKREL)
    B2A_PASS1(F_LUT | ALL)
    B2A_PASS1(F_LUT | ALL | F_PACKREL)
    B2A_PASS1(F_LUT | ALL | F_RELU)
    B2A_PASS1(F_LUT | ALL | F_PACKREL | F_RELU)
    B2A_REFILL(0)
    B2A_REFILL(F_CLIPX)
    B2A_REFILL(F_CLIPX | F_RELU)
    B2A_REFILL(F_LUT)
    B2A_REFILL(F_LUT | F_CLIPX)
    B2A_REFILL(F_LUT | F_CLIPX | F_RELU)
    default: return cudaErrorInvalidValue;
  }
#else
#ifdef B2A_NOTB
  constexpr int NOTB = F_NOTB;
#else
  constexpr int NOTB = 0;
#endif
  // the warp-per-pair shape also has every case with y read from the arena (F_YSTREAM: y longer than its staging)
#if B2A_G == 32
#define B2A_CASE(F)                                                                    \
  case (NOTB | (F)): return go<(NOTB | (F))>(prm, ntasks, num_sms, stream, grid_out, dry); \
  case (NOTB | F_YSTREAM | (F)): return go<(NOTB | F_YSTREAM | (F))>(prm, ntasks, num_sms, stream, grid_out, dry);
#elif B2A_G == 1
  // the thread-per-pair shape finishes each pair's matrix in the fill (F_FINISH) wherever its row trackers are final
  // at column n, i.e. without F_PACKREL: those cases exist only in the finishing form
#define B2A_FIN(F) (((F) & F_PACKREL) ? (F) : ((F) | F_FINISH))
#define B2A_CASE(F) \
  case (NOTB | B2A_FIN(F)): return go<(NOTB | B2A_FIN(F))>(prm, ntasks, num_sms, stream, grid_out, dry);
#else
#define B2A_CASE(F) \
  case (NOTB | (F)): return go<(NOTB | (F))>(prm, ntasks, num_sms, stream, grid_out, dry);
#endif
  switch (flags) {
    B2A_CASE(0)
    B2A_CASE(F_TRACK_ROWS)
    B2A_CASE(F_TRACK_ROWS | F_PACKTRK)
    B2A_CASE(ALL)
    B2A_CASE(ALL | F_PACKTRK)
    B2A_CASE(ALL | F_RELU)
    B2A_CASE(ALL | F_PACKTRK | F_RELU)
    B2A_CASE(F_LUT)
    B2A_CASE(F_LUT | F_TRACK_ROWS)
    B2A_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK)
    B2A_CASE(F_LUT | ALL)
    B2A_CASE(F_LUT | ALL | F_PACKTRK)
    B2A_CASE(F_LUT | ALL | F_RELU)
    B2A_CASE(F_LUT | ALL | F_PACKTRK | F_RELU)
    B2A_CASE(F_TRACK_ROWS | F_PACKTRK | F_BND8)
    B2A_CASE(ALL | F_PACKTRK | F_BND8)
    B2A_CASE(ALL | F_PACKTRK | F_RELU | F_BND8)
    B2A_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK | F_BND8)
    B2A_CASE(F_LUT | ALL | F_PACKTRK | F_BND8)
    B2A_CASE(F_LUT | ALL | F_PACKTRK | F_RELU | F_BND8)
    B2A_CASE(F_TRACK_ROWS | F_PACKREL)
    B2A_CASE(ALL | F_PACKREL)
    B2A_CASE(ALL | F_PACKREL | F_RELU)
    B2A_CASE(F_LUT | F_TRACK_ROWS | F_PACKREL)
    B2A_CASE(F_LUT | ALL | F_PACKREL)
    B2A_CASE(F_LUT | ALL | F_PACKREL | F_RELU)
    default: return cudaErrorInvalidValue;
  }
#endif
}

}  // namespace b2a
