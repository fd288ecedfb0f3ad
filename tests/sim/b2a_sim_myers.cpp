// CPU simulation of the pattern-matching kernels (test tool, not a product path): the lane logic of b2a_myers.cuh --
// myers_regs<1..4> and myers_warp<32> -- compiled for the host, the warp function on the 32 emulated lanes of
// b2a_sim.cpp.  The blob is rewritten into alphabet codes as the engine does, and the call's ambiguity rows and
// wildcards become a relation over those codes as the engine builds it.  Test tool only (tests/test_myers.py).
#include "b2a_sim.cpp"
#include "../../rust_bio_b200/csrc/b2a_myers.cuh"

namespace {

struct AlignedCodes {
  std::vector<uint64_t> words;
  uint8_t* p = nullptr;
  AlignedCodes(const uint8_t* src, uint64_t bytes, const uint8_t* map) : words((bytes + 32 + 15) / 8 + 2, 0) {
    p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(words.data()) + 15) & ~(uintptr_t)15);
    for (uint64_t i = 0; i < bytes; ++i) p[i] = map[src[i]];
  }
};

bool bit(const uint8_t* row, int t) { return (row[t >> 3] >> (t & 7)) & 1; }

}  // namespace

extern "C" {

// force_warp: every pair that needs DP runs the warp tier.  hit_off == nullptr: pass 1 (best_end, best_dist, count,
// tier per pair); else pass 2, each pair's hits written at hit_off[p] of hit_end / hit_dist.
int sim_myers(const uint8_t* blob, uint64_t blob_bytes, const uint64_t* xo, const uint32_t* xl, const uint64_t* yo,
              const uint32_t* yl, uint64_t n, const uint8_t* ambig, const uint8_t* wildcards, uint32_t k,
              int force_warp, uint32_t* best_end, uint32_t* best_dist, uint32_t* count, int32_t* tier_out,
              const uint64_t* hit_off, uint32_t* hit_end, uint32_t* hit_dist) {
  bool present[256] = {false};
  for (uint64_t i = 0; i < blob_bytes; ++i) present[blob[i]] = true;
  uint8_t map[256];
  std::vector<int> syms;
  for (int c = 0; c < 256; ++c) {
    map[c] = present[c] ? (uint8_t)syms.size() : 0xFF;
    if (present[c]) syms.push_back(c);
  }
  if (syms.empty()) syms.push_back(0);
  const int sigma = (int)syms.size();
  const AlignedCodes codes(blob, blob_bytes, map);
  std::vector<uint32_t> rel_off(sigma + 1, 0);
  std::vector<uint8_t> rel, wild;
  for (int a = 0; a < sigma; ++a) {
    rel_off[a] = (uint32_t)rel.size();
    for (int b = 0; ambig && b < sigma; ++b)
      if (b != a && bit(ambig + 32 * syms[a], syms[b])) rel.push_back((uint8_t)b);
  }
  rel_off[sigma] = (uint32_t)rel.size();
  for (int b = 0; wildcards && b < sigma; ++b)
    if (bit(wildcards, syms[b])) wild.push_back((uint8_t)b);
  MyersMatch mm{nullptr, nullptr, nullptr, 0};
  if (!rel.empty() || !wild.empty()) mm = MyersMatch{rel_off.data(), rel.data(), wild.data(), (int)wild.size()};
  for (uint64_t p = 0; p < n; ++p) {
    int t = myers_tier(xl[p], yl[p]);
    if (t != MT_DONE && force_warp) t = MT_WARP;
    const DistPair d = myers_pair(codes.p, xo[p], xl[p], yo[p], yl[p]);
    uint32_t* he = hit_off ? hit_end + hit_off[p] : nullptr;
    uint32_t* hd = hit_off ? hit_dist + hit_off[p] : nullptr;
    std::vector<uint64_t> peq((size_t)sigma * 4);
    MyersResult r{DIST_NONE, DIST_NONE, 0};
    switch (t) {
      case MT_DONE: break;
      case MT_REGS1: r = myers_regs<1>(d, peq.data(), 1, sigma, mm, k, he, hd); break;
      case MT_REGS1 + 1: r = myers_regs<2>(d, peq.data(), 1, sigma, mm, k, he, hd); break;
      case MT_REGS1 + 2: r = myers_regs<3>(d, peq.data(), 1, sigma, mm, k, he, hd); break;
      case MT_REGS1 + 3: r = myers_regs<4>(d, peq.data(), 1, sigma, mm, k, he, hd); break;
      case MT_WARP: {
        std::vector<uint64_t> wpeq((size_t)sigma * 32);
        std::vector<uint32_t> bnd(d.N / 16 + 2);
        MyersResult got[32];
        LaneFibers::run([&](int lane) {
          got[lane] = myers_warp<32>(d, wpeq.data(), sigma, mm, bnd.data(), lane, k, he, hd);
        });
        for (int l = 1; l < 32; ++l)  // every lane returns the pair's result
          if (got[l].best_end != got[0].best_end || got[l].best_dist != got[0].best_dist || got[l].count != got[0].count)
            return -1;
        r = got[0];
        break;
      }
      default: return -1;
    }
    if (!hit_off) {
      best_end[p] = r.best_end;
      best_dist[p] = r.best_dist;
      count[p] = r.count;
      tier_out[p] = t;
    }
  }
  return 0;
}

}  // extern "C"
