// Batched edit distance (bio::alignment::distance): unit-cost Levenshtein by Myers/Hyyrö bit-parallel column steps,
// bounded Levenshtein (Ukkonen's cutoff at word granularity, as in edlib: Šošić & Šikić 2017) and Hamming.
//
// The lane logic lives here as B2A_HD functions so that tests/sim compiles the very code the GPU runs; the kernels and
// their launches are in b2a_distance.cu.  The sequences arrive as codes of the batch's compacted alphabet (sigma
// symbols, one byte each: the engine rewrites the uploaded blob through its codemap before the Levenshtein kernels).
//
// Words are 64 bits: on sm_90 a 64-bit add is one IADD3 pair with carry and every logical op is one LOP3 per half,
// so a 64-row word costs what two 32-row words with an explicit carry chain cost, in half the loop trips.
// The pattern (rows) is the shorter sequence of a pair, the text (columns) the longer; the distance is symmetric.
#pragma once
#include "b2a_coop.cuh"

namespace b2a {

constexpr uint32_t DIST_NONE = 0xFFFFFFFFu;  // B2A_DIST_NONE: unbounded (k), or None (bounded result)
constexpr int DIST_REGS_WORDS = 4;          // tier 1: the whole pattern in registers, up to 256 rows
constexpr int DIST_STRIP_WORDS = 32;        // tier 3: one word per lane, 2048-row strips

// Tiers, picked per pair by the host from the lengths and the bound (dist_tier).
enum : int {
  DT_DONE = 0,                 // answered without DP: an empty side, or |m - n| above the bound
  DT_REGS1 = 1,                // DT_REGS1 + w - 1: thread per pair, w = ceil(P / 64) words in registers (w <= 4)
  DT_BAND4 = DT_REGS1 + DIST_REGS_WORDS,  // thread per pair, sliding window of 4 words (bounded only)
  DT_BAND8,                    // ... of 8 words (bounds up to 223)
  DT_WARP,                     // warp per pair, 32-word strips
  DT_COUNT
};

// Words of a sliding window that must hold every row of diagonals [j - k, j + k] at any column: rows j-k .. j+k
// meet at most floor(2k / 64) + 2 words.
inline int band_words(uint32_t k) { return (int)(2ull * k / 64) + 2; }

// The tier of one pair (x of length m, y of length n) under bound k (DIST_NONE: unbounded).  DT_DONE sets *done.
inline int dist_tier(uint32_t m, uint32_t n, uint32_t k, uint32_t* done) {
  const uint32_t P = m < n ? m : n, N = m < n ? n : m;
  const uint32_t kk = k < N ? k : N;  // simd::bounded_levenshtein bounds by min(k, max(|x|, |y|))
  if (N - P > kk) {                   // d >= |m - n|
    *done = DIST_NONE;
    return DT_DONE;
  }
  if (P == 0) {
    *done = N;  // N <= kk here
    return DT_DONE;
  }
  const uint32_t words = (P + 63) / 64;
  if (words <= (uint32_t)DIST_REGS_WORDS) return DT_REGS1 + (int)words - 1;
  if (k != DIST_NONE) {
    if (band_words(kk) <= 4) return DT_BAND4;
    if (band_words(kk) <= 8) return DT_BAND8;
  }
  return DT_WARP;
}

// One Myers/Hyyrö column step on a 64-row word (vertical deltas +1 = pv bit, -1 = mv bit) for a text symbol whose
// match mask over the word's rows is `eq`; `hin` is the horizontal delta entering the word's top row, the return
// value the one leaving the row `hmask` selects (bit 63, or the pattern's last row in its last word).
B2A_HD int myers_step(uint64_t& pv, uint64_t& mv, uint64_t eq, int hin, uint64_t hmask) {
  const uint64_t hneg = hin < 0 ? 1ull : 0ull, hpos = hin > 0 ? 1ull : 0ull;
  const uint64_t xv = eq | mv;
  eq |= hneg;
  const uint64_t xh = (((eq & pv) + pv) ^ pv) | eq;
  uint64_t ph = mv | ~(xh | pv);
  uint64_t mh = pv & xh;
  const int hout = ((ph & hmask) ? 1 : 0) - ((mh & hmask) ? 1 : 0);
  ph = (ph << 1) | hpos;
  mh = (mh << 1) | hneg;
  pv = mh | ~(xv | ph);
  mv = ph & xv;
  return hout;
}

B2A_HD uint64_t last_row_mask(uint32_t P) { return 1ull << ((P - 1) & 63); }

B2A_HD int popc64(uint64_t v) {
#if defined(__CUDA_ARCH__)
  return __popcll(v);
#else
  return __builtin_popcountll(v);
#endif
}

// Pattern and text of a pair: the shorter side is the pattern.
struct DistPair {
  const uint8_t* pat;
  const uint8_t* txt;
  uint32_t P, N, kk;  // kk = min(k, N), or DIST_NONE
};

B2A_HD DistPair dist_pair(const uint8_t* codes, uint64_t xo, uint32_t m, uint64_t yo, uint32_t n, uint32_t k) {
  DistPair d;
  if (m <= n) {
    d.pat = codes + xo, d.P = m, d.txt = codes + yo, d.N = n;
  } else {
    d.pat = codes + yo, d.P = n, d.txt = codes + xo, d.N = m;
  }
  d.kk = k == DIST_NONE ? DIST_NONE : (k < d.N ? k : d.N);
  return d;
}

// d <= kk, or a lower bound above kk: D[P][N] >= D[P][j] - (N - j) since neighbours on a row differ by at most one
B2A_HD bool over_bound(int64_t score, uint32_t N, uint32_t j_done, uint32_t kk) {
  return kk != DIST_NONE && score - (int64_t)(N - j_done) > (int64_t)kk;
}

// The text one column at a time, read 16 bytes per load from 16-byte aligned addresses (the engine's blob carries 16
// bytes of slack past its end, so the last aligned chunk is always inside the allocation).
struct TextReader {
  const uint8_t* p;  // the next 16-byte chunk
  uint64_t lo = 0, hi = 0;
  uint32_t i;  // byte of the current chunk to return next (16: load the next chunk)
  B2A_HD explicit TextReader(const uint8_t* txt) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(txt);
    p = reinterpret_cast<const uint8_t*>(a & ~(uintptr_t)15);
    i = (uint32_t)(a & 15);
    load();
  }
  B2A_HD void load() {
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    lo = (uint64_t)v.x | ((uint64_t)v.y << 32);
    hi = (uint64_t)v.z | ((uint64_t)v.w << 32);
    p += 16;
  }
  B2A_HD uint32_t next() {
    if (i == 16) {
      load();
      i = 0;
    }
    const uint32_t c = (uint32_t)((i < 8 ? lo >> (8 * i) : hi >> (8 * (i - 8))) & 0xFFu);
    ++i;
    return c;
  }
};

// Tier 1: thread per pair, the pattern's NW words in registers.  peq: this thread's sigma * NW match masks,
// peq[(c * NW + w) * stride].  Returns the distance, or DIST_NONE when it is above kk.
template <int NW>
B2A_HD uint32_t lev_regs(const DistPair& d, uint64_t* peq, int stride, int sigma) {
  for (int c = 0; c < sigma * NW; ++c) peq[c * stride] = 0;
  for (uint32_t i = 0; i < d.P; ++i) peq[(d.pat[i] * NW + (int)(i >> 6)) * stride] |= 1ull << (i & 63);
  uint64_t pv[NW], mv[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) pv[w] = ~0ull, mv[w] = 0;
  const uint64_t hlast = last_row_mask(d.P);
  int64_t score = d.P;
  TextReader rd(d.txt);
  for (uint32_t j = 1; j <= d.N; ++j) {
    const uint64_t* e = peq + (size_t)rd.next() * NW * stride;
    int h = 1;  // global boundary: D[0][j] = j
#pragma unroll
    for (int w = 0; w < NW; ++w) h = myers_step(pv[w], mv[w], e[w * stride], h, w == NW - 1 ? hlast : 1ull << 63);
    score += h;
    if ((j & 15) == 0 && over_bound(score, d.N, j, d.kk)) return DIST_NONE;
  }
  if (d.kk != DIST_NONE && score > (int64_t)d.kk) return DIST_NONE;
  return (uint32_t)score;
}

// Tier 2 (bounded only): thread per pair, a window of at most NWB words that slides down the pattern so that it
// holds every row of diagonals [j - kk, j + kk] at column j (requires band_words(kk) <= NWB and |P - N| <= kk).
// A word entering at the bottom starts with all vertical deltas +1 from the score of the word above it; above the
// top word the horizontal input is +1.  Both are upper bounds, so a cell whose true value is <= kk (its optimal path
// stays within the diagonals, hence within the window) is exact and one above kk is computed above kk: D[P][N] <= kk
// is decided exactly.  Once every cell of the window is above kk no path of cost <= kk crosses the column: None.
// peq: a ring of NWB word slots, peq[(c * NWB + slot) * stride], refilled from the pattern as words enter.
template <int NWB>
B2A_HD uint32_t lev_band(const DistPair& d, uint64_t* peq, int stride, int sigma) {
  const uint32_t P = d.P, kk = d.kk, nw = (P + 63) / 64;
  uint64_t pv[NWB], mv[NWB];
#pragma unroll
  for (int s = 0; s < NWB; ++s) pv[s] = ~0ull, mv[s] = 0;
  uint32_t lo = 0;    // top word of the window
  int cnt = 0;        // words in the window
  int32_t bsc = 0;    // value of the bottom row of the window's bottom word (row 0 before any word)
  uint32_t next = 0;  // the next word to enter
  TextReader rd(d.txt);
  for (uint32_t j = 1; j <= d.N; ++j) {
    const uint32_t c = rd.next();
    // leave: a word whose rows all lie above diagonal j - kk (the band moves one row per column: one word at most)
    if (cnt > 0 && (uint64_t)(lo + 1) * 64 + kk < j) {
#pragma unroll
      for (int s = 0; s + 1 < NWB; ++s) pv[s] = pv[s + 1], mv[s] = mv[s + 1];
      ++lo;
      --cnt;
    }
    if (cnt == 0) lo = next;
    // enter: words whose top row is at or above j + kk
    while (next < nw && (uint64_t)next * 64 + 1 <= (uint64_t)j + kk) {
      const int slot = (int)(next & (NWB - 1));
      for (int a = 0; a < sigma; ++a) peq[(a * NWB + slot) * stride] = 0;
      const uint32_t r0 = next * 64, r1 = r0 + 64 < P ? r0 + 64 : P;
      for (uint32_t i = r0; i < r1; ++i) peq[(d.pat[i] * NWB + slot) * stride] |= 1ull << (i - r0);
      bsc += (int32_t)(r1 - r0);  // D[r1][j-1] <= D[r0][j-1] + (r1 - r0)
#pragma unroll
      for (int s = 0; s < NWB; ++s) {  // (selects on every slot: the arrays stay in registers)
        pv[s] = s == cnt ? ~0ull : pv[s];
        mv[s] = s == cnt ? 0ull : mv[s];
      }
      ++cnt;
      ++next;
    }
    int h = 1;
#pragma unroll
    for (int s = 0; s < NWB; ++s) {
      if (s < cnt) {
        const uint32_t w = lo + (uint32_t)s;
        const uint64_t eq = peq[(c * NWB + (w & (NWB - 1))) * stride];
        h = myers_step(pv[s], mv[s], eq, h, w == nw - 1 ? last_row_mask(P) : 1ull << 63);
      }
    }
    bsc += h;  // h left the bottom word's bottom row
    if ((j & 7) == 0) {
      // every cell of the window above kk?  Walk up from the bottom row: a word's least cell is >= its bottom value
      // minus (height - 1), and the value above its top row is the bottom value minus the sum of its vertical deltas
      int64_t v = bsc;
      bool all_over = true;
#pragma unroll
      for (int s = NWB - 1; s >= 0; --s) {
        if (s < cnt) {
          const uint32_t w = lo + (uint32_t)s, height = w == nw - 1 ? P - w * 64 : 64;
          const uint64_t rows = height == 64 ? ~0ull : (1ull << height) - 1;
          all_over = all_over && v - (int64_t)(height - 1) > (int64_t)kk;
          v -= (int64_t)popc64(pv[s] & rows) - (int64_t)popc64(mv[s] & rows);
        }
      }
      if (all_over) return DIST_NONE;
    }
  }
  // at column N the window's bottom word is the last one (its top row <= P <= N + kk) and bsc = D'[P][N]
  if (bsc > (int32_t)kk) return DIST_NONE;
  return (uint32_t)bsc;
}

// Tier 3: warp per pair.  Lane l owns word 32 s + l of strip s and runs column t - l at step t (a diagonal
// wavefront): the horizontal delta leaving its bottom row reaches lane l + 1 by a shuffle for the next step.  Lane 0
// takes the previous strip's bottom-row deltas from `bnd` (2 bits per column, 16 columns per word), lane 31 writes
// them for the next strip; a column's word is read by lane 0 before lane 31 of the same strip rewrites it, so one
// buffer of ceil(N / 16) words serves every strip.  peq: this warp's match masks, peq[c * 32 + lane].
// Returns the distance (valid in every lane), or DIST_NONE when it is above kk.
template <int W>
B2A_HD uint32_t lev_warp(const DistPair& d, uint64_t* peq, int sigma, uint32_t* bnd, int lane) {
  const uint32_t P = d.P, N = d.N, nw = (P + 63) / 64;
  const uint32_t nstrips = (nw + DIST_STRIP_WORDS - 1) / DIST_STRIP_WORDS;
  const int owner = (int)((nw - 1) % DIST_STRIP_WORDS);  // lane of the last word, in the last strip
  int64_t score = P;
  bool over = false;
  for (uint32_t s = 0; s < nstrips && !over; ++s) {
    const uint32_t w = s * DIST_STRIP_WORDS + (uint32_t)lane;
    const bool last = s + 1 == nstrips;
    for (int a = 0; a < sigma; ++a) peq[a * 32 + lane] = 0;
    if (w < nw) {
      const uint32_t r0 = w * 64, r1 = r0 + 64 < P ? r0 + 64 : P;
      for (uint32_t i = r0; i < r1; ++i) peq[d.pat[i] * 32 + lane] |= 1ull << (i - r0);
    }
    const uint64_t hmask = w == nw - 1 ? last_row_mask(P) : 1ull << 63;
    uint64_t pv = ~0ull, mv = 0;
    int hup = 1;          // horizontal input from lane - 1 (lane 0: from the strip above)
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
        if (last && lane == owner) score += hout;
        if (!last && lane == DIST_STRIP_WORDS - 1) {
          wr |= (uint32_t)(hout + 1) << (2 * (j & 15));
          if ((j & 15) == 15 || j == (int64_t)N - 1) {
            bnd[j >> 4] = wr;
            wr = 0;
          }
        }
      }
      hup = Coop<W>::up(hout, 1);
      if (lane == 0) hup = 1;  // (lane 0 reads its input from the boundary; strip 0's is the +1 of row 0)
      if (last && d.kk != DIST_NONE && (t & 31) == 31) {
        const int64_t jo = (int64_t)t - owner;  // the owner's last column
        const bool ex = lane == owner && jo >= 0 && over_bound(score, N, (uint32_t)(jo + 1), d.kk);
        if (Coop<W>::ballot(ex)) {
          over = true;
          break;
        }
      }
    }
    Coop<W>::sync();  // lane 31's boundary words are visible to lane 0 of the next strip
  }
  const int32_t fin = Coop<W>::from((int32_t)score, owner);
  if (over || (d.kk != DIST_NONE && fin > (int64_t)d.kk)) return DIST_NONE;
  return (uint32_t)fin;
}

// Four byte lanes compared at once: 0xFF in each byte where a and b differ.
B2A_HD uint32_t vcmpne4(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __vcmpne4(a, b);
#else
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i)
    if (((a >> (8 * i)) & 0xFFu) != ((b >> (8 * i)) & 0xFFu)) r |= 0xFFu << (8 * i);
  return r;
#endif
}

// Four bytes at any address, from two aligned loads (reads up to 7 bytes past p: the blob's slack covers it).
B2A_HD uint32_t load4(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3) * 8;
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(q[0], q[1], sh);
#else
  return sh ? (q[0] >> sh) | (q[1] << (32 - sh)) : q[0];
#endif
}

// Hamming distance of two sequences of length L by the W lanes of one pair (W = 32: a warp); valid in every lane.
template <int W>
B2A_HD uint32_t hamming_coop(const uint8_t* x, const uint8_t* y, uint32_t L, int lane) {
  unsigned long long cnt = 0;
  const uint32_t chunks = (L + 3) / 4;
  for (uint32_t q = (uint32_t)lane; q < chunks; q += W) {
    uint32_t diff = vcmpne4(load4(x + 4 * q), load4(y + 4 * q)) & 0x01010101u;
    const uint32_t left = L - 4 * q;
    if (left < 4) diff &= (1u << (8 * left)) - 1u;
    cnt += (unsigned long long)Coop<W>::popc(diff);
  }
  return (uint32_t)Coop<W>::all_sum(cnt);
}

}  // namespace b2a

#if defined(__CUDACC__)
#include <cuda_runtime.h>
namespace b2a {

// Launches of b2a_distance.cu.  codes: the blob as alphabet codes (Levenshtein) or bytes (Hamming); tasks: pair
// indices of one tier; dist: per pair, in caller order.
struct DistArgs {
  const uint8_t* codes;
  const uint64_t* x_off;
  const uint32_t* x_len;
  const uint64_t* y_off;
  const uint32_t* y_len;
  const uint32_t* tasks;
  uint32_t n_tasks;
  uint32_t k;
  int sigma;
  uint32_t* dist;
};
// the blob rewritten in place through a 256-entry byte map
cudaError_t launch_dist_translate(uint8_t* blob, uint64_t bytes, const uint8_t* codemap, int num_sms, cudaStream_t st);
// tier: DT_REGS1 .. DT_BAND8 (thread per pair)
cudaError_t launch_lev_thread(int tier, const DistArgs& a, cudaStream_t st);
// persistent warps over the DT_WARP tasks: `bnd` holds warps * bnd_words boundary words, ctr one zeroed counter
cudaError_t lev_warp_grid(int sigma, int num_sms, uint32_t n_tasks, int* ctas, int* warps_per_cta);
cudaError_t launch_lev_warp(const DistArgs& a, int ctas, int warps_per_cta, uint32_t* bnd, uint64_t bnd_words,
                            uint32_t* ctr, cudaStream_t st);
// every pair whose lengths agree (the host marks the others)
cudaError_t launch_hamming(const DistArgs& a, uint64_t n_pairs, int num_sms, cudaStream_t st);

}  // namespace b2a
#endif
