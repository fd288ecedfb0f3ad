// CPU simulation of the pair-HMM kernels (test tool, not a product path): the lane logic of b2a_pairhmm.cuh --
// pairhmm_warp<C> for every C the kernels instantiate -- compiled for the host with the host log1p, on the 32
// emulated lanes of b2a_sim.cpp, with the gap cache the engine builds.  Test tool only (tests/test_pairhmm.py).
#include "b2a_sim.cpp"
#include "../../rust_bio_b200/csrc/b2a_pairhmm.cuh"

extern "C" {

// gap[4]: prob_gap_x, prob_gap_y, prob_gap_x_extend, prob_gap_y_extend; max_edit_dist: UINT64_MAX = None.
// force_tier < 0: each pair runs the tier the engine picks; else every pair with DP runs tier force_tier's C (strips
// of 32 * C columns whenever len_y is above them).  Returns 0, 1 / 2 / 3 when the gap cache asserts, -1 on a lane
// disagreement.
int sim_pairhmm(const double* gap, int free_start, int free_end, uint64_t max_edit_dist, const double* emit,
                uint32_t n_classes, const uint8_t* blob, const uint8_t* cls, const uint64_t* xo, const uint32_t* xl,
                const uint64_t* yo, const uint32_t* yl, uint64_t n, int force_tier, double* out, int32_t* tier_out) {
  PairHmmGap g;
  const int bad = pairhmm_gap_cache(gap[0], gap[1], gap[2], gap[3], free_start != 0, free_end != 0, max_edit_dist, &g);
  if (bad) return bad;
  for (uint64_t p = 0; p < n; ++p) {
    const uint32_t m = xl[p], nn = yl[p];
    int t = pairhmm_tier(m, nn);
    tier_out[p] = t;
    if (t == PT_DONE) {
      out[p] = pairhmm_empty(m, nn, free_end != 0);
      continue;
    }
    if (force_tier > 0) t = force_tier;
    const PairHmmSeq s{blob + xo[p], cls ? cls + xo[p] : nullptr, blob + yo[p], cls ? cls + yo[p] : nullptr, m, nn};
    std::vector<PairHmmRec> rec(m);
    std::vector<double> cols(3 * (size_t)m);
    double got[32];
    LaneFibers::run([&](int lane) {
      switch (t) {
        case PT_C1: got[lane] = pairhmm_warp<1>(g, emit, n_classes, s, rec.data(), cols.data(), lane); break;
        case PT_C2: got[lane] = pairhmm_warp<2>(g, emit, n_classes, s, rec.data(), cols.data(), lane); break;
        case PT_C4: got[lane] = pairhmm_warp<4>(g, emit, n_classes, s, rec.data(), cols.data(), lane); break;
        case PT_C5: got[lane] = pairhmm_warp<5>(g, emit, n_classes, s, rec.data(), cols.data(), lane); break;
        default: got[lane] = pairhmm_warp<8>(g, emit, n_classes, s, rec.data(), cols.data(), lane); break;
      }
    });
    for (int l = 1; l < 32; ++l)  // every lane returns the pair's result
      if (std::memcmp(&got[l], &got[0], 8) != 0) return -1;
    out[p] = got[0];
  }
  return 0;
}

}  // extern "C"
