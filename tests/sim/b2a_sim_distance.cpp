// CPU simulation of the edit-distance kernels (test tool, not a product path): the lane logic of b2a_distance.cuh --
// lev_regs, lev_band, lev_warp<32> and hamming_coop<32> -- compiled for the host, the warp functions on the 32
// emulated lanes of b2a_sim.cpp.  The blob is rewritten into alphabet codes as the engine does, in a 16-byte aligned
// copy with the engine's 16 bytes of slack.  Test tool only (tests/test_distance.py).
#include "b2a_sim.cpp"
#include "../../rust_bio_b200/csrc/b2a_distance.cuh"

namespace {

struct AlignedBlob {
  std::vector<uint64_t> words;  // 8-byte (and, through the allocator, 16-byte) aligned storage
  uint8_t* p = nullptr;
  AlignedBlob(const uint8_t* src, uint64_t bytes, const uint8_t* map) : words((bytes + 32 + 15) / 8 + 2, 0) {
    p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(words.data()) + 15) & ~(uintptr_t)15);
    for (uint64_t i = 0; i < bytes; ++i) p[i] = map ? map[src[i]] : src[i];
  }
};

uint32_t run_warp(const DistPair& d, int sigma) {
  std::vector<uint64_t> peq((size_t)sigma * 32);
  std::vector<uint32_t> bnd(d.N / 16 + 2);
  uint32_t got[32];
  LaneFibers::run([&](int lane) { got[lane] = lev_warp<32>(d, peq.data(), sigma, bnd.data(), lane); });
  for (int l = 1; l < 32; ++l)
    if (got[l] != got[0]) std::abort();  // every lane returns the pair's result
  return got[0];
}

}  // namespace

extern "C" {

// force_tier: -1 the engine's choice (dist_tier); DT_WARP the warp tier for every pair that needs DP; DT_BAND4 /
// DT_BAND8 the band for every bounded pair it can hold (else the engine's choice).  tier_out: the tier each pair ran.
int sim_levenshtein(const uint8_t* blob, uint64_t blob_bytes, const uint64_t* xo, const uint32_t* xl,
                    const uint64_t* yo, const uint32_t* yl, uint64_t n, uint32_t k, int force_tier, uint32_t* out,
                    int32_t* tier_out) {
  bool present[256] = {false};
  for (uint64_t i = 0; i < blob_bytes; ++i) present[blob[i]] = true;
  uint8_t map[256];
  int sigma = 0;
  for (int c = 0; c < 256; ++c) map[c] = present[c] ? (uint8_t)sigma++ : 0xFF;
  if (!sigma) sigma = 1;
  const AlignedBlob codes(blob, blob_bytes, map);
  for (uint64_t p = 0; p < n; ++p) {
    uint32_t v = 0;
    int t = dist_tier(xl[p], yl[p], k, &v);
    const DistPair d = dist_pair(codes.p, xo[p], xl[p], yo[p], yl[p], k);
    if (t != DT_DONE && force_tier == DT_WARP) t = DT_WARP;
    if (t != DT_DONE && k != DIST_NONE && (force_tier == DT_BAND4 || force_tier == DT_BAND8) &&
        band_words(d.kk) <= (force_tier == DT_BAND4 ? 4 : 8))
      t = force_tier;
    std::vector<uint64_t> peq((size_t)sigma * 8);
    switch (t) {
      case DT_DONE: break;
      case DT_REGS1: v = lev_regs<1>(d, peq.data(), 1, sigma); break;
      case DT_REGS1 + 1: v = lev_regs<2>(d, peq.data(), 1, sigma); break;
      case DT_REGS1 + 2: v = lev_regs<3>(d, peq.data(), 1, sigma); break;
      case DT_REGS1 + 3: v = lev_regs<4>(d, peq.data(), 1, sigma); break;
      case DT_BAND4: v = lev_band<4>(d, peq.data(), 1, sigma); break;
      case DT_BAND8: v = lev_band<8>(d, peq.data(), 1, sigma); break;
      case DT_WARP: v = run_warp(d, sigma); break;
      default: return -1;
    }
    out[p] = v;
    tier_out[p] = t;
  }
  return 0;
}

// pairs of unequal lengths get 0xFFFFFFFF
int sim_hamming(const uint8_t* blob, uint64_t blob_bytes, const uint64_t* xo, const uint32_t* xl, const uint64_t* yo,
                const uint32_t* yl, uint64_t n, uint32_t* out) {
  const AlignedBlob bytes(blob, blob_bytes, nullptr);
  for (uint64_t p = 0; p < n; ++p) {
    if (xl[p] != yl[p]) {
      out[p] = DIST_NONE;
      continue;
    }
    uint32_t got[32];
    LaneFibers::run([&](int lane) { got[lane] = hamming_coop<32>(bytes.p + xo[p], bytes.p + yo[p], xl[p], lane); });
    for (int l = 1; l < 32; ++l)
      if (got[l] != got[0]) return -1;
    out[p] = got[0];
  }
  return 0;
}

}  // extern "C"
