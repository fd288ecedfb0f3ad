// Batched Myers pattern matching (bio::pattern_matching::myers): the semi-global search of a pattern x in a text y,
// D[0][j] = 0 (the text is free at both ends), read off row m at every text column.  Per pair: the first end of
// minimal distance, and the ends whose distance is <= k in ascending order.
//
// The column step, the text reader and the warp tier's strip scheme are those of the edit distance
// (b2a_distance.cuh); what differs is the top row's horizontal input (0 here, +1 there), the per-column result on
// row m, and match masks that may carry the pattern side's ambiguities and the text's wildcards.  As there, the lane
// logic is B2A_HD so that tests/sim compiles the very code the GPU runs; the kernels are in b2a_myers.cu.
#pragma once
#include "b2a_distance.cuh"

namespace b2a {

// Tiers, picked per pair by the host from the pattern length (myers_tier); the numbering of dist_tier's tiers that
// apply here, so that the register tier shares its masks' layout.
enum : int {
  MT_DONE = 0,      // answered without DP: an empty pattern (a panic) or an empty text
  MT_REGS1 = 1,     // MT_REGS1 + w - 1: thread per pair, w = ceil(P / 64) words in registers (w <= 4)
  MT_WARP = 5,      // warp per pair, 32-word strips
  MT_COUNT
};

inline int myers_tier(uint32_t m, uint32_t n) {
  if (m == 0 || n == 0) return MT_DONE;
  const uint32_t words = (m + 63) / 64;
  return words <= (uint32_t)DIST_REGS_WORDS ? MT_REGS1 + (int)words - 1 : MT_WARP;
}

// The pattern is always x, the text y (the roles do not swap as the symmetric distance's do).
B2A_HD DistPair myers_pair(const uint8_t* codes, uint64_t xo, uint32_t m, uint64_t yo, uint32_t n) {
  DistPair d;
  d.pat = codes + xo, d.P = m, d.txt = codes + yo, d.N = n, d.kk = DIST_NONE;
  return d;
}

// The match relation over the batch's codes.  rel_off == nullptr: a code matches itself only.  Otherwise pattern code
// a also matches the text codes rel[rel_off[a] .. rel_off[a + 1]), and every text code in wild[0 .. n_wild) matches
// every pattern code.
struct MyersMatch {
  const uint32_t* rel_off;
  const uint8_t* rel;
  const uint8_t* wild;
  int n_wild;
};

// What a pair's search gives: the first end (0-based) of the least distance (DIST_NONE for both when the text is
// empty), and how many ends have a distance <= k.
struct MyersResult {
  uint32_t best_end, best_dist, count;
};

// The match masks of pattern rows [r0, r1) into one word per code: m[c * stride] for code c (zeroed first).
B2A_HD void myers_masks(const uint8_t* pat, uint32_t r0, uint32_t r1, const MyersMatch& mm, uint64_t* m, int stride,
                        int sigma) {
  for (int c = 0; c < sigma; ++c) m[c * stride] = 0;
  if (!mm.rel_off) {
    for (uint32_t i = r0; i < r1; ++i) m[pat[i] * stride] |= 1ull << (i - r0);
    return;
  }
  for (uint32_t i = r0; i < r1; ++i) {
    const uint32_t a = pat[i];
    const uint64_t bit = 1ull << (i - r0);
    m[a * stride] |= bit;
    for (uint32_t e = mm.rel_off[a]; e < mm.rel_off[a + 1]; ++e) m[mm.rel[e] * stride] |= bit;
  }
  for (int w = 0; w < mm.n_wild; ++w) m[mm.wild[w] * stride] = ~0ull;
}

// Row m's value at column j (1-based) into the result; with `hit_end` the hit is also written at the count's slot.
B2A_HD void myers_column(MyersResult& r, uint32_t j, uint32_t v, uint32_t k, uint32_t* hit_end, uint32_t* hit_dist) {
  if (v < r.best_dist) r.best_dist = v, r.best_end = j - 1;  // strict: the first end of the least distance
  if (v <= k) {
    if (hit_end) hit_end[r.count] = j - 1, hit_dist[r.count] = v;
    ++r.count;
  }
}

// Tier 1: thread per pair, the pattern's NW words in registers.  peq: this thread's sigma * NW match masks,
// peq[(c * NW + w) * stride].
template <int NW>
B2A_HD MyersResult myers_regs(const DistPair& d, uint64_t* peq, int stride, int sigma, const MyersMatch& mm,
                              uint32_t k, uint32_t* hit_end, uint32_t* hit_dist) {
  for (int w = 0; w < NW; ++w) {  // (NW = ceil(P / 64): every word holds rows)
    const uint32_t r0 = (uint32_t)w * 64, r1 = r0 + 64 < d.P ? r0 + 64 : d.P;
    myers_masks(d.pat, r0, r1, mm, peq + (size_t)w * stride, NW * stride, sigma);
  }
  uint64_t pv[NW], mv[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) pv[w] = ~0ull, mv[w] = 0;
  const uint64_t hlast = last_row_mask(d.P);
  MyersResult r{DIST_NONE, DIST_NONE, 0};
  uint32_t score = d.P;  // D[P][0]
  TextReader rd(d.txt);
  for (uint32_t j = 1; j <= d.N; ++j) {
    const uint64_t* e = peq + (size_t)rd.next() * NW * stride;
    int h = 0;  // semi-global boundary: D[0][j] = 0
#pragma unroll
    for (int w = 0; w < NW; ++w) h = myers_step(pv[w], mv[w], e[w * stride], h, w == NW - 1 ? hlast : 1ull << 63);
    score += h;
    myers_column(r, j, score, k, hit_end, hit_dist);
  }
  return r;
}

// Tier 2: warp per pair, lev_warp's diagonal wavefront over 2048-row strips (see there) with the semi-global top
// row: lane 0 of strip 0 takes 0 as its horizontal input.  The owner lane of the last strip meets the columns in
// ascending order and produces row m's values.  The result is valid in every lane.
template <int W>
B2A_HD MyersResult myers_warp(const DistPair& d, uint64_t* peq, int sigma, const MyersMatch& mm, uint32_t* bnd,
                              int lane, uint32_t k, uint32_t* hit_end, uint32_t* hit_dist) {
  const uint32_t P = d.P, N = d.N, nw = (P + 63) / 64;
  const uint32_t nstrips = (nw + DIST_STRIP_WORDS - 1) / DIST_STRIP_WORDS;
  const int owner = (int)((nw - 1) % DIST_STRIP_WORDS);
  MyersResult r{DIST_NONE, DIST_NONE, 0};
  uint32_t score = P;
  for (uint32_t s = 0; s < nstrips; ++s) {
    const uint32_t w = s * DIST_STRIP_WORDS + (uint32_t)lane;
    const bool last = s + 1 == nstrips;
    const uint32_t r0 = w < nw ? w * 64 : P, r1 = w < nw && r0 + 64 < P ? r0 + 64 : P;
    myers_masks(d.pat, r0, r1, mm, peq + lane, 32, sigma);
    const uint64_t hmask = w == nw - 1 ? last_row_mask(P) : 1ull << 63;
    uint64_t pv = ~0ull, mv = 0;
    int hup = 0;
    uint32_t rd = 0, wr = 0;
    Coop<W>::sync();
    for (uint32_t t = 0; t < N + DIST_STRIP_WORDS - 1; ++t) {
      const int64_t j = (int64_t)t - lane;
      const bool valid = j >= 0 && j < (int64_t)N;
      int hin = hup;
      if (lane == 0 && s > 0 && valid) {
        if ((j & 15) == 0) rd = bnd[j >> 4];
        hin = (int)((rd >> (2 * (j & 15))) & 3u) - 1;
      }
      int hout = 0;
      if (valid) {
        const uint32_t c = d.txt[j];
        hout = myers_step(pv, mv, peq[c * 32 + lane], hin, hmask);
        if (last && lane == owner) {
          score += hout;
          myers_column(r, (uint32_t)j + 1, score, k, hit_end, hit_dist);
        }
        if (!last && lane == DIST_STRIP_WORDS - 1) {
          wr |= (uint32_t)(hout + 1) << (2 * (j & 15));
          if ((j & 15) == 15 || j == (int64_t)N - 1) {
            bnd[j >> 4] = wr;
            wr = 0;
          }
        }
      }
      hup = Coop<W>::up(hout, 1);
      if (lane == 0) hup = 0;  // (lane 0 reads its input from the boundary; strip 0's is the 0 of row 0)
    }
    Coop<W>::sync();  // lane 31's boundary words are visible to lane 0 of the next strip
  }
  r.best_end = (uint32_t)Coop<W>::from((int32_t)r.best_end, owner);
  r.best_dist = (uint32_t)Coop<W>::from((int32_t)r.best_dist, owner);
  r.count = (uint32_t)Coop<W>::from((int32_t)r.count, owner);
  return r;
}

}  // namespace b2a

#if defined(__CUDACC__)
#include <cuda_runtime.h>
namespace b2a {

// Launches of b2a_myers.cu.  tasks: pair indices of one tier.  Pass 1 (hit_off == nullptr) writes best_end,
// best_dist and, with `count`, the number of ends <= k per pair; pass 2 (hit_off set) writes each pair's hits at
// hit_off[p].  Results are per pair, in caller order.
struct MyersArgs {
  const uint8_t* codes;
  const uint64_t* x_off;
  const uint32_t* x_len;
  const uint64_t* y_off;
  const uint32_t* y_len;
  const uint32_t* tasks;
  uint32_t n_tasks;
  uint32_t k;
  int sigma;
  MyersMatch match;
  uint32_t* best_end;
  uint32_t* best_dist;
  uint32_t* count;
  const uint64_t* hit_off;
  uint32_t* hit_end;
  uint32_t* hit_dist;
};
// tier: MT_REGS1 .. MT_REGS1 + 3 (thread per pair)
cudaError_t launch_myers_thread(int tier, const MyersArgs& a, cudaStream_t st);
// persistent warps over the MT_WARP tasks: `bnd` holds warps * bnd_words boundary words, ctr one zeroed counter
cudaError_t myers_warp_grid(int sigma, int num_sms, uint32_t n_tasks, int* ctas, int* warps_per_cta);
cudaError_t launch_myers_warp(const MyersArgs& a, int ctas, int warps_per_cta, uint32_t* bnd, uint64_t bnd_words,
                              uint32_t* ctr, cudaStream_t st);
// pass 2's task lists: `order` holds the tasks of tier t at [seg.at[t], seg.at[t + 1]) for t = 1 .. MT_COUNT - 1;
// those whose pair has a nonzero count go to the same segment of `out`, and their number to n_out[t] (zeroed by the
// caller).  Their order within a segment is arbitrary: each pair writes its hits at its own offset.
struct MyersSegs {
  uint32_t at[MT_COUNT + 1];
};
cudaError_t launch_myers_select(const uint32_t* order, MyersSegs seg, const uint32_t* count, uint32_t* out,
                                uint32_t* n_out, cudaStream_t st);

}  // namespace b2a
#endif
