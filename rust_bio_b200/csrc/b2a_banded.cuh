// K4 + K3: banded::Aligner on the device, one warp per pair in both kernels.
//
// Reference rust-bio 4.0.1:
//   sparse::find_kmer_matches          src/alignment/sparse.rs:337-402
//   sparse::sdpkpp + PrevPtr           sparse.rs:145-295   (prefix-max of bit_tree.rs:45-99)
//   Band::{add_kmer,add_entry,add_gap,set_boundaries,create_*,num_cells}   banded.rs:1047-1380
//   banded::Aligner::compute_alignment banded.rs:406-869
// The banded DP is full of order-dependent quirks (rolling arrays keep leftovers from earlier
// columns, eager traceback writes that later stores overwrite, a walk that may stop on an untouched
// cell outside the band), so K3 replays the column loop literally -- but on GPU-sized state:
//   * the reference's (m+1)(n+1) u16 traceback (10 MB for 500x10,000, re-zeroed per call) becomes
//     band cells + row 0 + row m + column 0 + column n; every other cell is a constant START;
//   * k-mer matches come from a rolling-hash table of the shorter sequence (exact: verified bytes);
//   * the Fenwick tree over coordinates 0..n becomes a Fenwick tree over the (<= #matches) distinct
//     end coordinates -- the same prefix-max, since only inserted coordinates can ever answer.
// All per-pair state lives in one HBM scratch slab per pair (BandedSlab).
#pragma once
#include "b2a_common.cuh"
#include "b2a_coop.cuh"

namespace b2a {

constexpr uint64_t BANDED_MAX_CELLS = 5000000ull;  // banded.rs:104
constexpr int32_t BANDED_DEFAULT_MATCH_SCORE = 2;  // banded.rs:105
constexpr int K3_FAST_ROWS = 5;
// geometry of the strip-wavefront fill (b2a_banded_strip.cuh): 8 lanes per pair, KS_R rows per lane
#ifndef B2A_KS_R
#define B2A_KS_R 16
#endif
constexpr int KS_G = 8, KS_R = B2A_KS_R, KS_ROWS = KS_G * KS_R, KS_TBW = KS_R / 4;
static_assert(KS_R == 8 || KS_R == 16, "rows per lane of the strip fill: 8 or 16");
constexpr uint32_t KS_ROWS_LOG2 = KS_R == 16 ? 7u : 6u, KS_R_LOG2 = KS_R == 16 ? 4u : 3u;
constexpr uint32_t KS_TAB = 4;  // u32 per strip-table entry: first column of the window, traceback offset (uint4), steps stored, 0  // rows per lane of the register-resident K3 loop: bands up to ~160 rows per column

struct BandedParams {
  const uint8_t* blob;
  const uint64_t* x_off;
  const uint32_t* x_len;
  const uint64_t* y_off;
  const uint32_t* y_len;
  const uint8_t* codemap;  // symbol -> LUT code (LUT mode)
  const int32_t* lut;      // alpha*alpha plain scores, or null
  DevScoring sc;           // clip presets already applied
  int32_t has_match_scores;
  uint32_t k, w;
  uint32_t cap_matches;    // per pair
  uint64_t n_pairs;
  uint32_t pair_lo;        // first pair of this wave
  // per-pair slabs
  uint8_t* slab;           // K4 slab base (wave-relative pair index * slab_stride)
  uint64_t slab_stride;
  uint32_t* ranges;        // [(n_pad+1) * 2] per pair, wave arena: ranges_off[p]
  const uint64_t* ranges_off;
  uint64_t* num_cells;     // [n_pairs] out (K4), in (K3)
  uint32_t* k4_status;     // [n_pairs] 0 ok, 1 too many matches
  // caller-supplied band inputs (banded.rs:294-401); null = found on the device
  const uint64_t* hint_match_off;  // [n_pairs + 1] into hint_match_xy pairs, or null
  const uint32_t* hint_match_xy;   // (xpos, ypos) per match
  const uint64_t* hint_path_off;   // [n_pairs + 1] into hint_path_idx, or null (custom_with_match_path)
  const uint32_t* hint_path_idx;
  int32_t allowed_mismatches;      // custom_with_expanded_matches: >= 0 expands the matches, -1 = None
  int32_t use_lcskpp_union;        // custom_with_expanded_matches
  // strip-wavefront fill (b2a_banded_strip.cuh)
  int32_t strip_ok;        // bit 0: the batch's scoring suits it (host check): K4 may mark pairs strip-eligible (bit 9);
                           // bit 1: also pairs whose band holds cells of column n (global mode)
  int32_t redo_pass;       // K3 column-loop kernels: 0 = the pairs K4 did not mark for the strip path, 1 = the pairs the
                           // strip path handed back (bit 10)
  uint32_t* band_cols;     // [n_pairs * 3] out (K4): first / last non-empty band column, strip columns
  const uint8_t* strip;    // strip areas of the sub-wave (finish pass), or null
  const uint64_t* strip_off;
  // K3 state
  uint8_t* fill;           // K3 slab arena
  const uint64_t* fill_off;  // per pair byte offset of the K3 slab
  int32_t filter_clips;
  // outputs (caller order)
  int32_t* score;
  uint32_t* xstart;
  uint32_t* xend;
  uint32_t* ystart;
  uint32_t* yend;
  uint32_t* n_ops;
  uint64_t* ops_src;
  uint32_t* clip_len;
  uint32_t* status;
  uint32_t* err_flag;
  uint8_t* ops_scratch;
  const uint64_t* ops_off;  // per pair: end of its ops region (ops are written backwards)
};

B2A_HD uint64_t sat_sub64(uint64_t a, uint64_t b) { return a > b ? a - b : 0; }
B2A_HD uint64_t umin64(uint64_t a, uint64_t b) { return a < b ? a : b; }
B2A_HD uint64_t umax64(uint64_t a, uint64_t b) { return a > b ? a : b; }

// ------------------------------------------------------------------ heap sort on 64-bit keys
B2A_HD void sift_down(uint64_t* a, uint64_t start, uint64_t end) {
  uint64_t root = start;
  for (;;) {
    uint64_t child = 2 * root + 1;
    if (child > end) break;
    if (child + 1 <= end && a[child] < a[child + 1]) child += 1;
    if (a[root] < a[child]) {
      const uint64_t t = a[root];
      a[root] = a[child];
      a[child] = t;
      root = child;
    } else {
      break;
    }
  }
}
B2A_HD void heap_sort_u64(uint64_t* a, uint64_t n) {
  if (n < 2) return;
  for (uint64_t s = (n - 2) / 2 + 1; s-- > 0;) sift_down(a, s, n - 1);
  for (uint64_t end = n - 1; end > 0; --end) {
    const uint64_t t = a[0];
    a[0] = a[end];
    a[end] = t;
    sift_down(a, 0, end - 1);
  }
}

// ------------------------------------------------------------------ K4 slab layout
struct PrevPtrD {  // sparse.rs:145-153, compared lexicographically (plane, score, d, id, x, y)
  uint32_t plane, score, d, id, x, y;
};
B2A_HD bool prev_ge(const PrevPtrD& b, const PrevPtrD& a) {  // b >= a
  if (b.plane != a.plane) return b.plane > a.plane;
  if (b.score != a.score) return b.score > a.score;
  if (b.d != a.d) return b.d > a.d;
  if (b.id != a.id) return b.id > a.id;
  if (b.x != a.x) return b.x > a.x;
  return b.y >= a.y;
}

struct K4Slab {
  uint64_t* matches;   // cap: (x << 32) | y, sorted
  uint64_t* table;     // H entries: (hash_hi32 << 32) | (pos + 1); 0 = empty
  uint64_t* events;    // 2*cap: (x << 40) | (y << 16)... see pack_event
  uint32_t* ev_id;     // unused (ids are packed in events)
  uint32_t* dp_score;  // cap
  int32_t* dp_prev;    // cap
  PrevPtrD* fen;       // cap + 2
  uint32_t* ycoord;    // cap: sorted distinct end-y coordinates
  uint32_t* path;      // cap
  uint32_t H;
};

B2A_HD uint64_t k4_slab_bytes(uint32_t cap, uint32_t short_len) {
  uint32_t H = 16;
  while (H < 2 * (short_len + 1)) H <<= 1;
  uint64_t b = 0;
  b += (uint64_t)cap * 8;          // matches
  b += (uint64_t)H * 8;            // table
  b += (uint64_t)2 * cap * 8 * 2;  // events (two u64 per event)
  b += (uint64_t)cap * 4 * 2;      // dp
  b += (uint64_t)(cap + 2) * sizeof(PrevPtrD);
  b += (uint64_t)cap * 4 * 2;      // ycoord, path
  b += (uint64_t)cap * 4 * 2;      // path continues (a union path holds up to 2*cap entries), lcskpp path
  return (b + 255) & ~255ull;
}

// ------------------------------------------------------------------ cooperative sort of 64-bit keys
// Bitonic network in its all-ascending form (first step of a merge compares i with its mirror i ^ (k-1), the
// rest with i ^ j): every compare-exchange leaves the smaller key at the lower index, so the virtual +inf
// padding up to the next power of two never moves and pairs that reach past n are simply skipped.
template <int W>
B2A_HD void coop_sort_u64(int lane, uint64_t* a, uint64_t n) {
  using C = Coop<W>;
  if (n < 2) return;
  auto step = [&](uint64_t mask) {
    for (uint64_t i = (uint64_t)lane; i < n; i += W) {
      const uint64_t j = i ^ mask;
      if (j > i && j < n) {
        const uint64_t u = a[i], v = a[j];
        if (u > v) {
          a[i] = v;
          a[j] = u;
        }
      }
    }
    C::sync();
  };
  for (uint64_t k = 2; (k >> 1) < n; k <<= 1) {
    step(k - 1);
    for (uint64_t j = k >> 2; j > 0; j >>= 1) step(j);
  }
}

// ------------------------------------------------------------------ Band (ranges as u32 pairs)
// W cooperating lanes: every loop over columns is strided over the lanes.  lo() is a minimum and hi() a maximum,
// so the order in which the reference's add_kmer/add_entry/add_gap calls touch a column does not matter; a
// sync after each loop keeps two lanes from updating one column at the same time.
template <int W>
struct BandD {
  using C = Coop<W>;
  uint32_t* r;  // r[2j] = start, r[2j+1] = end
  uint64_t rows, cols;
  int lane = 0;
  bool oob = false;  // a column index past the matrix: the reference panics on ranges[j] (caller-supplied matches)
  // the columns this lane has touched since init (every other column still holds Band::new's sentinel): the passes
  // over the finished band -- num_cells, the K3 eligibility checks -- only visit [first, last] of the whole warp
  uint64_t tmin = ~0ull, tmax = 0;
  B2A_HD void touched(uint64_t& first, uint64_t& last) const {  // first > last: nothing touched
    long long a = tmin == ~0ull ? (long long)0x8000000000000000ull : -(long long)tmin;  // min as a max of negatives
    long long b = tmin == ~0ull ? (long long)0x8000000000000000ull : (long long)tmax;
    a = C::all_max(a);
    b = C::all_max(b);
    if (a == (long long)0x8000000000000000ull) {
      first = 1;
      last = 0;
    } else {
      first = (uint64_t)(-a);
      last = (uint64_t)b;
    }
  }
  B2A_HD void init(uint64_t m, uint64_t n) {  // Band::new, banded.rs:1061-1067
    rows = m + 1;
    cols = n + 1;
    for (uint64_t j = (uint64_t)lane; j < cols; j += W) {
      r[2 * j] = (uint32_t)(m + 1);
      r[2 * j + 1] = 0;
    }
    C::sync();
  }
  B2A_HD void lo(uint64_t j, uint64_t v) {
    if (j >= cols) {
      oob = true;
      return;
    }
    if ((uint64_t)r[2 * j] > v) r[2 * j] = (uint32_t)v;
    tmin = j < tmin ? j : tmin;
    tmax = j > tmax ? j : tmax;
  }
  B2A_HD void hi(uint64_t j, uint64_t v) {
    if (j >= cols) {
      oob = true;
      return;
    }
    if ((uint64_t)r[2 * j + 1] < v) r[2 * j + 1] = (uint32_t)v;
    tmin = j < tmin ? j : tmin;
    tmax = j > tmax ? j : tmax;
  }
  B2A_HD void add_kmer(uint64_t r0, uint64_t c0, uint64_t k, uint64_t w) {  // banded.rs:1071-1107
    if (k == 0) return;
    {
      const uint64_t i = sat_sub64(r0, w);
      for (uint64_t j = sat_sub64(c0, w) + (uint64_t)lane; j < umin64(c0 + w + 1, cols); j += W) lo(j, i);
    }
    {
      const uint64_t i0 = sat_sub64(r0, w), j0 = umin64(c0 + w, cols);
      for (uint64_t j = j0 + (uint64_t)lane; j < umin64(c0 + k + w, cols); j += W) lo(j, i0 + (j - j0));
    }
    C::sync();
    {
      // the reference walks j down from J0 = sat_sub(c0+k-1, w) to sat_sub(c0, w), i down from r0+w+k beside it
      const uint64_t i0 = r0 + w + k, J0 = sat_sub64(c0 + k - 1, w), jb = sat_sub64(c0, w);
      for (uint64_t j = jb + (uint64_t)lane; j < J0; j += W) hi(j, umin64(i0 - (J0 - j), rows));
    }
    {
      const uint64_t i = umin64(r0 + w + k, rows);
      for (uint64_t j = sat_sub64(c0 + k - 1, w) + (uint64_t)lane; j < umin64(c0 + k + w, cols); j += W) hi(j, i);
    }
    C::sync();
  }
  B2A_HD void add_entry(uint64_t r0, uint64_t c0, uint64_t w) {  // banded.rs:1111-1120
    const uint64_t istart = sat_sub64(r0, w), iend = umin64(r0 + w + 1, rows);
    for (uint64_t j = sat_sub64(c0, w) + (uint64_t)lane; j < umin64(c0 + w + 1, cols); j += W) {
      lo(j, istart);
      hi(j, iend);
    }
    C::sync();
  }
  // L consecutive add_entry calls along a diagonal, (r0 + u, c0 + u) for u = 0..L-1 (a run of matches that each
  // continue the previous one, banded.rs:1354-1357), in closed form per column: the entries covering column j are
  // u in [j - c0 - w, j - c0 + w] clipped to the run, their lowest start is the first one's and their highest end
  // the last one's.
  B2A_HD void add_entry_run(uint64_t r0, uint64_t c0, uint64_t L, uint64_t w) {
    if (L == 0) return;
    const uint64_t jb = sat_sub64(c0, w), je = umin64(c0 + (L - 1) + w + 1, cols);
    for (uint64_t j = jb + (uint64_t)lane; j < je; j += W) {
      const uint64_t u_lo = sat_sub64(j, c0 + w);                      // j <= c0 + u + w
      const uint64_t u_hi = umin64(L - 1, j + w >= c0 ? j + w - c0 : 0);  // c0 + u - w <= j
      if (j + w < c0 || u_lo > u_hi) continue;
      lo(j, sat_sub64(r0 + u_lo, w));
      hi(j, umin64(r0 + u_hi + w + 1, rows));
    }
    C::sync();
  }
  // banded.rs:1123-1137, u32 arithmetic.  Returns false where the reference would divide by zero.
  B2A_HD bool add_gap(uint32_t s0, uint32_t s1, uint32_t e0, uint32_t e1, uint64_t w) {
    const uint32_t nrows = e0 - s0, ncols = e1 - s1;
    if (nrows > ncols) {
      for (uint32_t rr = s0; rr < e0; ++rr) {
        const uint32_t den = e0 - s0;
        if (den == 0) return false;
        const uint32_t c = s1 + (e1 - s1) * (rr - s0) / den;
        add_entry(rr, c, w);
      }
    } else {
      for (uint32_t c = s1; c < e1; ++c) {
        const uint32_t den = e1 - s1;
        if (den == 0) return false;
        const uint32_t rr = s0 + (e0 - s0) * (c - s1) / den;
        add_entry(rr, c, w);
      }
    }
    return true;
  }
  B2A_HD bool set_boundaries(uint32_t st0, uint32_t st1, uint32_t en0, uint32_t en1, uint64_t k, uint64_t w,
                             const DevScoring& sc) {  // banded.rs:1150-1276
    const uint64_t lazy = 2 * k;
    bool ok = true;
    {
      const uint64_t rr = st0, c = st1;
      if (!(rr == 0 && c == 0)) {
        int32_t to_start = rr > 0 ? sc.xclip_prefix : 0;
        to_start += c > 0 ? sc.yclip_prefix : 0;
        if (to_start == 0) {
          const uint64_t d = umin64(lazy, umin64(rr, c));
          add_kmer(rr - d, c - d, d, w);
          ok &= add_gap((uint32_t)sat_sub64(rr, lazy), (uint32_t)sat_sub64(c, lazy), (uint32_t)(rr - d),
                        (uint32_t)(c - d), w);
        } else {
          const int32_t diag = rr > c ? sc.xclip_prefix : (rr < c ? sc.yclip_prefix : 0);
          if (diag == 0) {
            const uint64_t d = umin64(rr, c);
            add_kmer(rr - d, c - d, d, w);
            const uint32_t a0 = (uint32_t)sat_sub64(rr, lazy), a1 = (uint32_t)sat_sub64(c, lazy);
            const uint32_t b0 = (uint32_t)(rr - d), b1 = (uint32_t)(c - d);
            if (a0 <= b0 && a1 <= b1) ok &= add_gap(a0, a1, b0, b1, w);
          } else {
            ok &= add_gap(0u, 0u, st0, st1, w);
          }
        }
      }
    }
    {
      const uint64_t rr = (uint64_t)en0 + k, c = (uint64_t)en1 + k;
      if (rr > rows || c > cols) {  // rows - rr underflows in the reference (caller-supplied matches only)
        oob = true;
        return ok;
      }
      if (!(rr == rows && c == cols)) {
        int32_t from_end = rr == rows ? 0 : sc.xclip_suffix;
        from_end += c == cols ? 0 : sc.yclip_suffix;
        if (from_end == 0) {
          const uint64_t d = umin64(lazy, umin64(rows - rr, cols - c));
          add_kmer(rr, c, d, w);
          const uint64_t r1 = umin64(rows, rr + d) - 1, c1 = umin64(cols, c + d) - 1;
          const uint64_t r2 = umin64(rows, rr + lazy), c2 = umin64(cols, c + lazy);
          if (r1 <= r2 && c1 <= c2) ok &= add_gap((uint32_t)r1, (uint32_t)c1, (uint32_t)r2, (uint32_t)c2, w);
        } else {
          const uint64_t dr = rows - rr, dc = cols - c;
          const int32_t diag = dr > dc ? sc.xclip_suffix : (dr < dc ? sc.yclip_suffix : 0);
          if (diag == 0) {
            const uint64_t d = umin64(dr, dc);
            add_kmer(rr, c, d, w);
            const uint64_t r1 = umin64(rows, rr + d) - 1, c1 = umin64(cols, c + d) - 1;
            const uint64_t r2 = umin64(rows, rr + lazy), c2 = umin64(cols, c + lazy);
            if (r1 <= r2 && c1 <= c2) ok &= add_gap((uint32_t)r1, (uint32_t)c1, (uint32_t)r2, (uint32_t)c2, w);
          } else {
            ok &= add_gap((uint32_t)rr, (uint32_t)c, (uint32_t)rows, (uint32_t)cols, w);
          }
        }
      }
    }
    return ok;
  }
  B2A_HD void full_matrix() {  // banded.rs:1369-1372
    for (uint64_t j = (uint64_t)lane; j < cols; j += W) {
      r[2 * j] = 0;
      r[2 * j + 1] = (uint32_t)rows;
    }
    tmin = 0;
    tmax = cols - 1;
    C::sync();
  }
  B2A_HD uint64_t num_cells() const {  // banded.rs:1374-1380 (untouched columns are empty)
    unsigned long long cells = 0;
    uint64_t a, b;
    touched(a, b);
    for (uint64_t j = a + (uint64_t)lane; j <= b && j < cols; j += W) cells += sat_sub64(r[2 * j + 1], r[2 * j]);
    return C::all_sum(cells);
  }
  B2A_HD bool any_oob() const { return C::ballot(oob) != 0u; }
};

// ------------------------------------------------------------------ k-mer matches (exact)
constexpr uint64_t HASH_B = 0x9E3779B97F4A7C15ull | 1ull;
constexpr uint32_t KF_BITS = 1u << 15;  // bit filter over the hashed k-mers, per warp (4 KB of shared memory)
constexpr uint32_t K4_SHARED_WORDS = 2u + KF_BITS / 32u;  // band_create_d's `shared_u32`: two scratch words + the filter

// all (i, j) with x[i..i+k] == y[j..j+k] as (i << 32 | j), sorted; returns count or ~0 on overflow.
// Each lane hashes / probes a contiguous run of positions with its own rolling hash; table slots are claimed
// with a compare-and-swap and matches appended through a counter, in any order: the table layout and the
// append order do not matter, the result is the sorted set.
template <int W>
B2A_HD uint64_t find_kmer_matches_d(int lane, const uint8_t* x, uint64_t m, const uint8_t* y, uint64_t n, uint64_t k,
                                    uint64_t* table, uint32_t H, uint64_t* out, uint64_t cap, uint32_t* counter,
                                    uint64_t* hbuf, uint64_t hbuf_entries, uint32_t* filter /* KF_BITS / 32 words */) {
  using C = Coop<W>;
  const uint64_t nx = sat_sub64(m + 1, k), ny = sat_sub64(n + 1, k);
  if (nx == 0 || ny == 0 || k == 0) return 0;
  const bool hash_x = m <= n;  // hash the shorter one
  const uint8_t* hs = hash_x ? x : y;
  const uint8_t* ps = hash_x ? y : x;
  const uint64_t nh = hash_x ? nx : ny, np = hash_x ? ny : nx;
  for (uint32_t s = (uint32_t)lane; s < H; s += W) table[s] = 0;
  for (uint32_t s = (uint32_t)lane; s < KF_BITS / 32u; s += W) filter[s] = 0;
  if (lane == 0) *counter = 0;
  C::sync();
  uint64_t bk = 1;  // B^(k-1)
  for (uint64_t t = 1; t < k; ++t) bk *= HASH_B;
  auto mix = [](uint64_t h) { return h ^ (h >> 29); };
  const uint32_t mask = H - 1;
  {
    const uint64_t seg = (nh + W - 1) / W, lo = umin64(nh, seg * (uint64_t)lane), hi = umin64(nh, lo + seg);
    if (lo < hi) {
      uint64_t h = 0;
      for (uint64_t t = 0; t < k; ++t) h = h * HASH_B + (uint64_t)(hs[lo + t] + 1);
      for (uint64_t i = lo; i < hi; ++i) {
        const uint64_t hm = mix(h);
        uint32_t slot = (uint32_t)hm & mask;
        const uint64_t entry = ((hm >> 32) << 32) | (i + 1);
        while (!C::claim(&table[slot], entry)) slot = (slot + 1) & mask;
        const uint32_t bit = (uint32_t)(hm >> 17) & (KF_BITS - 1u);
        C::or_u32(&filter[bit >> 5], 1u << (bit & 31u));
        if (i + 1 < hi) h = (h - (uint64_t)(hs[i] + 1) * bk) * HASH_B + (uint64_t)(hs[i + k] + 1);
      }
    }
  }
  C::sync();
  // Probe.  A lane rolls its hash over a contiguous run of positions.  Nearly all of them (a read against a long
  // reference: 95 %) have no partner, so a position first asks a bit filter over the hashed k-mers (KF_BITS bits per
  // warp in shared memory, 1.4 % false positives at 469 k-mers): one shared load instead of a walk down a chain of the
  // open-addressing table -- a walk the whole warp sits through whenever ONE of its lanes takes it.  The positions
  // that pass are compacted (ballot + popcount) into a queue in the event scratch (free until sdpkpp) and the table
  // walks are then dealt out over the lanes entry by entry, so the few real matches (they sit in the runs of two
  // lanes) no longer serialise the warp either.  Candidates (equal upper hash halves) are appended unverified; the
  // byte comparison follows, one candidate per lane.
  {
    const uint64_t seg = (np + W - 1) / W, lo = umin64(np, seg * (uint64_t)lane), hi = umin64(np, lo + seg);
    const uint32_t Q = (uint32_t)(hbuf_entries / 2);  // queue capacity in (hash, position) entries, >= 2 W
    uint32_t qn = 0;
    auto drain = [&]() {
      for (uint32_t e = (uint32_t)lane; e < qn; e += W) {
        const uint64_t hm = hbuf[2 * e], j = hbuf[2 * e + 1];
        uint32_t slot = (uint32_t)hm & mask;
        for (;;) {
          const uint64_t en = table[slot];
          if ((uint32_t)en == 0u) break;  // (the low half is position + 1: never 0 in a used slot)
          if ((uint32_t)(en >> 32) == (uint32_t)(hm >> 32)) {
            const uint64_t i = (en & 0xffffffffull) - 1;
            const uint32_t at = C::fetch_add(counter, 1u);
            if (at < cap) out[at] = hash_x ? ((i << 32) | j) : ((j << 32) | i);
          }
          slot = (slot + 1) & mask;
        }
      }
    };
    uint64_t h = 0;
    if (lo < hi)
      for (uint64_t t = 0; t < k; ++t) h = h * HASH_B + (uint64_t)(ps[lo + t] + 1);
    for (uint64_t r = 0; r < seg; ++r) {
      const uint64_t j = lo + r;
      const bool valid = j < hi;
      uint64_t hm = 0;
      bool pass = false;
      if (valid) {
        hm = mix(h);
        const uint32_t bit = (uint32_t)(hm >> 17) & (KF_BITS - 1u);
        pass = ((filter[bit >> 5] >> (bit & 31u)) & 1u) != 0u;
        if (j + 1 < hi) h = (h - (uint64_t)(ps[j] + 1) * bk) * HASH_B + (uint64_t)(ps[j + k] + 1);
      }
      const uint32_t bal = C::ballot(pass);
      if (pass) {
        const uint32_t at = qn + (uint32_t)C::popc(bal & ((1u << lane) - 1u));
        hbuf[2ull * at] = hm;
        hbuf[2ull * at + 1] = j;
      }
      qn += (uint32_t)C::popc(bal);
      if (qn + (uint32_t)W > Q) {  // the next position could overflow the queue (Q >= 2 W: checked by the caller)
        C::sync();
        drain();
        C::sync();
        qn = 0;
      }
    }
    C::sync();
    drain();
  }
  C::sync();
  const uint64_t cand = *counter;
  C::sync();
  if (cand > cap) return ~0ull;
  // verify the candidates byte by byte; a false one (a 32-bit hash collision) is struck out and sorts to the end
  uint32_t bad = 0;
  for (uint64_t c = (uint64_t)lane; c < cand; c += W) {
    const uint64_t mt = out[c];
    const uint64_t i = hash_x ? (mt >> 32) : (mt & 0xffffffffull), j = hash_x ? (mt & 0xffffffffull) : (mt >> 32);
    bool same = true;
    for (uint64_t t = 0; t < k; ++t)
      if (hs[i + t] != ps[j + t]) {
        same = false;
        break;
      }
    if (!same) {
      out[c] = ~0ull;
      ++bad;
    }
  }
  const uint64_t nbad = (uint64_t)C::all_sum((unsigned long long)bad);
  C::sync();
  coop_sort_u64<W>(lane, out, cand);
  return cand - nbad;
}

// ------------------------------------------------------------------ sdpkpp, sparse.rs:188-295
// events are two u64: key0 = (x << 32 | y), key1 = id; sorted by (x, y, id).
B2A_HD uint32_t lower_bound_u32(const uint32_t* a, uint32_t n, uint32_t v) {  // first index with a[i] >= v
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// returns path length (path[] = indices into matches), 0 if no matches
// lcs = true runs sparse::lcskpp (sparse.rs:67-143) on the same machinery: unit scores, no gap term, and a
// prefix-max tree over (score, id) tuples -- PrevPtrD{0, score, 0, id, 0, 0} compares exactly like that tuple.
// The sorts and the array set-up are spread over the W lanes; the event loop itself (each event reads what the
// previous ones wrote into the tree) is sequential work of lane 0.  Every lane returns the path length.
template <int W>
B2A_HD uint32_t sdpkpp_d(int lane, const uint64_t* matches, uint32_t nm, uint32_t k, uint32_t match_score,
                         int32_t gap_open, int32_t gap_extend, uint64_t* ev /*4*nm u64*/, uint32_t* dp_score,
                         int32_t* dp_prev, PrevPtrD* fen, uint32_t* ycoord, uint32_t* path, uint32_t* shared_u32,
                         bool lcs = false) {
  using C = Coop<W>;
  if (nm == 0) return 0;
  if (lcs) match_score = 1;
  const uint32_t go = (uint32_t)(-gap_open), ge = (uint32_t)(-gap_extend);
  // events sorted lexicographically by (x, y, id): pack (x, y) in one key and sort pairs by two passes:
  // sort by combined 64-bit key (x << 32 | y) with id as tie-break -> id < 2*nm <= 2^31; use a stable
  // trick: key = (x,y) and secondary array; simplest exact way: sort 128-bit items by heap sort on
  // an index permutation is costly, so encode id into a second heap sort pass:
  //   ends (id < nm) sort before starts (id >= nm) at equal (x, y); among equal (x, y, kind) ids are
  //   unique per match and (x, y) is unique per match for starts and for ends, so (x, y, kind) is a
  //   total order: key = (x << 33) | (y << 1) | kind needs 65 bits when x,y use 32 -> lengths are
  //   limited to 2^24 by the engine, so x,y < 2^25 and the key fits.
  uint64_t* tmp = ev + 2ull * nm;  // scratch half
  for (uint32_t idx = (uint32_t)lane; idx < nm; idx += W) {
    const uint64_t x = matches[idx] >> 32, y = matches[idx] & 0xffffffffull;
    ev[2 * idx] = (x << 33) | (y << 1) | 1ull;              // start (id = idx + nm)
    ev[2 * idx + 1] = ((x + k) << 33) | ((y + k) << 1);     // end   (id = idx)
    tmp[idx] = y + k;
    dp_score[idx] = 0;
    dp_prev[idx] = 0;
  }
  C::sync();
  coop_sort_u64<W>(lane, ev, 2ull * nm);
  coop_sort_u64<W>(lane, tmp, nm);
  // distinct end-y coordinates, ascending (the only indices ever set in the prefix-max tree)
  uint32_t ny = 0;
  if (lane == 0) {
    for (uint32_t t = 0; t < nm; ++t)
      if (ny == 0 || ycoord[ny - 1] != (uint32_t)tmp[t]) ycoord[ny++] = (uint32_t)tmp[t];
    shared_u32[0] = ny;
  }
  C::sync();
  ny = shared_u32[0];
  for (uint32_t t = (uint32_t)lane; t <= ny + 1; t += W) fen[t] = PrevPtrD{0, 0, 0, 0, 0, 0};
  C::sync();
  // everything an event needs that does not depend on earlier events is looked up by all lanes up front: its
  // match, the tree rank of its coordinate and (for an end) the match one step up the diagonal.  The sorted y
  // scratch is free again, and `path` is not written before the backtrack.
  uint32_t* ev_p = reinterpret_cast<uint32_t*>(tmp);  // [2 nm] match index of the event
  uint32_t* ev_aux = ev_p + 2ull * nm;                // [2 nm] start: #coordinates <= y; end: diagonal predecessor
  uint32_t* rank_end = path;                          // [nm]   1-based tree position of the match's end coordinate
  for (uint64_t e = (uint64_t)lane; e < 2ull * nm; e += W) {
    const uint64_t key = ev[e];
    const bool is_start = (key & 1ull) != 0;
    const uint32_t e0 = (uint32_t)(key >> 33), e1 = (uint32_t)((key >> 1) & 0xffffffffull);
    const uint64_t want = is_start ? (((uint64_t)e0 << 32) | e1) : (((uint64_t)(e0 - k) << 32) | (e1 - k));
    uint32_t lo = 0, hi = nm;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) / 2;
      if (matches[mid] < want) lo = mid + 1;
      else hi = mid;
    }
    ev_p[e] = lo;
    if (is_start) {
      ev_aux[e] = lower_bound_u32(ycoord, ny, e1 + 1);
    } else {
      uint32_t found = 0xFFFFFFFFu;
      if (e0 > k && e1 > k) {
        const uint64_t cw = ((uint64_t)(e0 - k - 1) << 32) | (e1 - k - 1);
        uint32_t l2 = 0, h2 = nm;
        while (l2 < h2) {
          const uint32_t mid = (l2 + h2) / 2;
          if (matches[mid] < cw) l2 = mid + 1;
          else h2 = mid;
        }
        if (l2 < nm && matches[l2] == cw) found = l2;
      }
      ev_aux[e] = found;
      rank_end[lo] = lower_bound_u32(ycoord, ny, e1) + 1;
    }
  }
  C::sync();
  uint32_t np = 0;
  // The event loop: each event reads what earlier ones wrote into the prefix-max tree, so events run one after
  // the other -- but a Fenwick query touches its <= log2(ny)+1 nodes independently of each other (the index chain
  // idx -= lowbit(idx) does not depend on the loaded values), and so does an update.  Lane l takes the l-th node
  // of the chain; a query is then two warp maxima, an update one predicated store per lane.  The PrevPtr order
  // (plane, score, d, id, x, y) is decided by (plane, score, d, id) alone: id is unique per entry.  Everything
  // else of an event is the same arithmetic in every lane; lane 0 stores dp.
  uint32_t best_score = k;
  int32_t best_idx = 0;
  auto dp_gt = [](uint32_t s1, int32_t p1, uint32_t s2, int32_t p2) {  // (s1,p1) > (s2,p2)
    return s1 != s2 ? s1 > s2 : p1 > p2;
  };
  const long long flip = (long long)0x8000000000000000ull;  // unsigned order through a signed maximum
  for (uint64_t e = 0; e < 2ull * nm; ++e) {
    const uint64_t key = ev[e];
    const bool is_start = (key & 1ull) != 0;
    const uint32_t e0 = (uint32_t)(key >> 33), e1 = (uint32_t)((key >> 1) & 0xffffffffull);
    const uint32_t p = ev_p[e];
    if (is_start) {
      uint32_t dps = k * match_score;
      int32_t dpp = -1;
      // max_col_dp.get(j): prefix max over inserted coordinates <= e1; node l of the chain in lane l
      PrevPtrD mine{0, 0, 0, 0, 0, 0};
      {
        uint32_t idx = ev_aux[e];  // number of coordinates <= e1; Fenwick positions are 1-based
        for (int t = 0; t < lane && idx; ++t) idx &= idx - 1u;
        if (W == 1) {  // sequential build: walk the whole chain
          while (idx > 0) {
            if (prev_ge(fen[idx], mine)) mine = fen[idx];
            idx &= idx - 1u;
          }
        } else if (idx > 0) {
          mine = fen[idx];
        }
      }
      PrevPtrD best = mine;
      if (W > 1) {
        const long long k1 = (long long)(((uint64_t)mine.plane << 32) | mine.score) ^ flip;
        const long long m1 = C::all_max(k1);
        const long long k2 = k1 == m1 ? (long long)((((uint64_t)mine.d << 32) | mine.id) ^ (uint64_t)flip) : flip;
        const long long m2 = C::all_max(k2);
        const uint32_t who = C::ballot(k1 == m1 && k2 == m2);
        int src = 0;
        while (!((who >> src) & 1u)) ++src;
        best.plane = (uint32_t)(((uint64_t)(m1 ^ flip)) >> 32);
        best.score = (uint32_t)((uint64_t)(m1 ^ flip) & 0xffffffffull);
        best.d = (uint32_t)(((uint64_t)(m2 ^ flip)) >> 32);
        best.id = (uint32_t)((uint64_t)(m2 ^ flip) & 0xffffffffull);
        best.x = (uint32_t)C::from((int32_t)mine.x, src);
        best.y = (uint32_t)C::from((int32_t)mine.y, src);
      }
      if (best.score > 0) {
        if (lcs) {  // dp[p] = (k + best_value, best_position), sparse.rs:111-113
          dps = k + best.score;
          dpp = (int32_t)best.id;
        } else {
          const uint32_t g0 = e0 - best.x, g1 = e1 - best.y;
          const uint32_t gap = g0 > g1 ? g0 : g1;
          const uint32_t pen = gap > 0 ? go + gap * ge : 0;
          const uint32_t sum = best.score + k * match_score;
          const uint32_t ns = sum > pen ? sum - pen : 0;
          if (dp_gt(ns, (int32_t)best.id, dps, dpp)) {
            dps = ns;
            dpp = (int32_t)best.id;
          }
        }
        if (dp_gt(dps, (int32_t)p, best_score, best_idx)) {
          best_score = dps;
          best_idx = (int32_t)p;
        }
      }
      if (lane == 0) {
        dp_score[p] = dps;
        dp_prev[p] = dpp;
      }
    } else {
      uint32_t dps = dp_score[p];
      int32_t dpp = dp_prev[p];
      {
        const uint32_t l2 = ev_aux[e];  // the match at (x - 1, y - 1), sparse.rs:267-275
        if (l2 != 0xFFFFFFFFu) {
          const uint32_t cs = dp_score[l2] + match_score;
          if (dp_gt(cs, (int32_t)l2, dps, dpp)) {
            dps = cs;
            dpp = (int32_t)l2;
          }
          if (dp_gt(dps, (int32_t)p, best_score, best_idx)) {
            best_score = dps;
            best_idx = (int32_t)p;
          }
        }
      }
      if (lane == 0) {
        dp_score[p] = dps;
        dp_prev[p] = dpp;
      }
      PrevPtrD pf;
      pf.d = lcs ? 0u : e0 + e1;
      pf.plane = lcs ? 0u : dps + pf.d * ge;
      pf.score = dps;
      pf.id = p;
      pf.x = lcs ? 0u : e0;
      pf.y = lcs ? 0u : e1;
      uint32_t idx = rank_end[p];  // 1-based rank of this coordinate; node l of the update chain in lane l
      for (int t = 0; t < lane && idx <= ny; ++t) idx += idx & (0u - idx);
      if (W == 1) {
        while (idx <= ny) {
          if (prev_ge(pf, fen[idx])) fen[idx] = pf;
          idx += idx & (0u - idx);
        }
      } else if (idx <= ny) {
        if (prev_ge(pf, fen[idx])) fen[idx] = pf;
      }
    }
    C::sync();  // the tree and dp as this event left them are what the next one reads
  }
  if (lane == 0) {
  int32_t pm = best_idx;
  while (pm >= 0 && np < nm) {
    path[np++] = (uint32_t)pm;
    pm = dp_prev[pm];
  }
  for (uint32_t a = 0, b = np ? np - 1 : 0; a < b; ++a, --b) {
    const uint32_t t = path[a];
    path[a] = path[b];
    path[b] = t;
  }
  shared_u32[0] = np;
  }
  C::sync();
  np = shared_u32[0];
  C::sync();  // shared_u32 may be reused by the caller
  return np;
}

// ------------------------------------------------------------------ sparse::expand_kmer_matches, sparse.rs:404-498
// The reference's two hash maps keyed by diagonal hold "the previous (next) match on this diagonal in processing
// order"; with the matches sorted that is the predecessor (successor) in (diagonal, x) order, found here by
// binary search in a sorted key array.  matches: sorted (x << 32 | y), expanded in place; returns the new count,
// ~0 if more than cap, ~1 where the reference would panic (a position outside the sequences).
B2A_HD uint64_t expand_kmer_matches_d(const uint8_t* s1, uint64_t l1, const uint8_t* s2, uint64_t l2, uint64_t k,
                                      uint64_t* matches, uint64_t nm, uint64_t cap, uint64_t allowed,
                                      uint64_t* dk /* cap u64 */) {
  auto diag_of = [](uint64_t mt) -> uint64_t {
    return (uint64_t)(uint32_t)((uint32_t)(mt >> 32) - (uint32_t)mt + 0x80000000u);
  };
  auto lower = [](const uint64_t* a, uint64_t n, uint64_t v) -> uint64_t {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
      const uint64_t mid = (lo + hi) / 2;
      if (a[mid] < v) lo = mid + 1;
      else hi = mid;
    }
    return lo;
  };
  for (uint64_t i = 0; i < nm; ++i) {
    const uint64_t x = matches[i] >> 32, y = matches[i] & 0xffffffffull;
    if (x > l1 || y > l2) return ~1ull;
    dk[i] = (diag_of(matches[i]) << 32) | x;
  }
  heap_sort_u64(dk, nm);
  uint64_t cnt = nm;
  for (uint64_t i = 0; i < nm; ++i) {  // extend to the left, 417-448
    const int64_t x = (int64_t)(matches[i] >> 32), y = (int64_t)(matches[i] & 0xffffffffull);
    const uint64_t dg = diag_of(matches[i]);
    const uint64_t q = lower(dk, nm, (dg << 32) | (uint64_t)x);
    int64_t last_x;  // x of the last match along this diagonal (the pair is on the diagonal: compare x only)
    if (q > 0 && (dk[q - 1] >> 32) == dg) last_x = (int64_t)(dk[q - 1] & 0xffffffffull);
    else last_x = x - (x < y ? x : y) - 1;
    uint64_t n_mis = 0;
    int64_t cx = x - 1, cy = y - 1;
    for (;;) {
      if (last_x >= cx) break;
      n_mis += s1[cx] == s2[cy] ? 0 : 1;
      if (n_mis > allowed) break;
      if (cnt >= cap) return ~0ull;
      matches[cnt++] = ((uint64_t)cx << 32) | (uint64_t)cy;
      cx -= 1;
      cy -= 1;
    }
  }
  heap_sort_u64(matches, cnt);
  const uint64_t nl = cnt;  // the left-expanded set; extend each of its members to the right, 450-494
  for (uint64_t i = 0; i < nl; ++i) dk[i] = (diag_of(matches[i]) << 32) | (matches[i] >> 32);
  heap_sort_u64(dk, nl);
  for (uint64_t i = 0; i < nl; ++i) {
    const uint64_t x = matches[i] >> 32, y = matches[i] & 0xffffffffull;
    const uint64_t dg = diag_of(matches[i]);
    const uint64_t q = lower(dk, nl, (dg << 32) | x) + 1;
    uint64_t next_x;
    if (q < nl && (dk[q] >> 32) == dg) {
      next_x = dk[q] & 0xffffffffull;
    } else {
      const uint64_t a = l1 - x, b = l2 - y, mn = a < b ? a : b;
      next_x = x + sat_sub64(mn, k - 1);
    }
    uint64_t n_mis = 0;
    uint64_t cx = x + 1, cy = y + 1;
    for (;;) {
      if (cx >= next_x) break;
      if (cx + k - 1 >= l1 || cy + k - 1 >= l2) return ~1ull;  // index out of bounds in the reference
      n_mis += s1[cx + k - 1] == s2[cy + k - 1] ? 0 : 1;
      if (n_mis > allowed) break;
      if (cnt >= cap) return ~0ull;
      matches[cnt++] = (cx << 32) | cy;
      cx += 1;
      cy += 1;
    }
  }
  heap_sort_u64(matches, cnt);
  return cnt;
}

// ------------------------------------------------------------------ K4: Band::create* for one pair
struct BandHintsD {
  const uint32_t* mxy = nullptr;  // caller's matches (xpos, ypos); null: find them (Band::create)
  uint64_t n_matches = 0;
  const uint32_t* pidx = nullptr;  // caller's path (custom_with_match_path); null: sdpkpp [union lcskpp]
  uint64_t n_path = 0;
  bool have_path = false;
  int32_t allowed_mismatches = -1;
  int32_t use_lcskpp_union = 0;
};

// W cooperating lanes build one pair's band (W = 32: one warp; W = 1: the host logic build).  `shared_u32` is
// K4_SHARED_WORDS words all lanes can read and write (shared memory on the device): two scratch words + the k-mer bit filter.
// returns status: 0 ok, 1 too many matches (capacity), 2 reference would panic (divide by zero),
// 3 reference would panic on the caller's matches/path (not sorted, index out of range, outside the matrix)
template <int W>
B2A_HD uint32_t band_create_d(int lane, const uint8_t* x, uint64_t m, const uint8_t* y, uint64_t n, uint32_t k,
                              uint32_t w, const DevScoring& sc, int32_t has_match_scores, uint8_t* slab,
                              uint32_t cap, uint32_t* ranges, uint64_t* cells_out, uint32_t* shared_u32,
                              const BandHintsD& hint = BandHintsD{}, uint32_t* touched_out = nullptr) {
  using C = Coop<W>;
  const uint64_t short_len = m <= n ? m : n;
  uint32_t H = 16;
  while (H < 2 * (short_len + 1)) H <<= 1;
  uint64_t* matches = reinterpret_cast<uint64_t*>(slab);
  uint64_t* table = matches + cap;
  uint64_t* ev = table + H;
  uint32_t* dp_score = reinterpret_cast<uint32_t*>(ev + 4ull * cap);
  int32_t* dp_prev = reinterpret_cast<int32_t*>(dp_score + cap);
  PrevPtrD* fen = reinterpret_cast<PrevPtrD*>(dp_prev + cap);
  uint32_t* ycoord = reinterpret_cast<uint32_t*>(fen + cap + 2);
  uint32_t* path = ycoord + cap;          // 2 * cap entries
  uint32_t* path2 = path + 2ull * cap;    // cap entries (lcskpp path)
  BandD<W> band;
  band.r = ranges;
  band.lane = lane;
  band.init(m, n);
  *cells_out = 0;
  uint64_t nm64;
  if (hint.mxy) {
    if (hint.n_matches > cap) return 1;
    for (uint64_t i = (uint64_t)lane; i < hint.n_matches; i += W)
      matches[i] = ((uint64_t)hint.mxy[2 * i] << 32) | (uint64_t)hint.mxy[2 * i + 1];
    nm64 = hint.n_matches;
    C::sync();
  } else {
    // (the probe queue lives in the event scratch, 4 * cap u64: a capacity below 32 matches would not hold one round
    //  of a warp's positions -- such a pair reports a capacity overflow and the wave is redone with a larger one)
    if (4ull * cap < 4ull * (uint64_t)W) return 1;
    nm64 = find_kmer_matches_d<W>(lane, x, m, y, n, k, table, H, matches, cap, shared_u32, ev, 4ull * cap, shared_u32 + 2);
    if (nm64 == ~0ull) return 1;
  }
  // sdpkpp, lcskpp and expand_kmer_matches assert strictly ascending matches (sparse.rs:77-82, 213-218, 411-416)
  auto sorted = [&](uint64_t cnt) {
    bool ok = true;
    for (uint64_t i = 1 + (uint64_t)lane; i < cnt; i += W)
      if (!(matches[i - 1] < matches[i])) ok = false;
    return C::ballot(!ok) == 0u;
  };
  if (hint.allowed_mismatches >= 0) {  // custom_with_expanded_matches, banded.rs:346-349
    if (!sorted(nm64)) return 3;
    if (lane == 0) {  // a rare entry point: sequential
      const uint64_t got = expand_kmer_matches_d(x, m, y, n, k, matches, nm64, cap, (uint64_t)hint.allowed_mismatches, ev);
      shared_u32[0] = got >= ~1ull ? (got == ~0ull ? 0xFFFFFFFFu : 0xFFFFFFFEu) : (uint32_t)got;
    }
    C::sync();
    const uint32_t got = shared_u32[0];
    C::sync();
    if (got == 0xFFFFFFFFu) return 1;
    if (got == 0xFFFFFFFEu) return 3;
    nm64 = got;
  }
  const uint32_t nm = (uint32_t)nm64;
  uint32_t status = 0;
  if (nm == 0) {
    band.full_matrix();  // banded.rs:1309-1313, 1341-1344
  } else {
    uint32_t np;
    if (hint.have_path) {  // custom_with_match_path: the path is used as given (391-401)
      if (hint.n_path == 0 || hint.n_path > 2ull * cap) return hint.n_path == 0 ? 3 : 1;
      bool bad = false;
      for (uint64_t t = (uint64_t)lane; t < hint.n_path; t += W) {
        if (hint.pidx[t] >= nm) bad = true;
        else path[t] = hint.pidx[t];
      }
      if (C::ballot(bad) != 0u) return 3;
      np = (uint32_t)hint.n_path;
      C::sync();
    } else {
      if (!sorted(nm)) return 3;
      const int32_t ms = has_match_scores ? sc.match_score : BANDED_DEFAULT_MATCH_SCORE;  // 1315-1318
      if (hint.use_lcskpp_union) {  // sparse::sdpkpp_union_lcskpp_path, sparse.rs:297-330
        const uint32_t nl = sdpkpp_d<W>(lane, matches, nm, k, 1u, 0, 0, ev, dp_score, dp_prev, fen, ycoord, path2,
                                        shared_u32, true);
        uint32_t* sp = path + cap;  // the sdpkpp path, parked in the upper half while the union is assembled
        const uint32_t ns = sdpkpp_d<W>(lane, matches, nm, k, (uint32_t)ms, sc.gap_open, sc.gap_extend, ev, dp_score,
                                        dp_prev, fen, ycoord, sp, shared_u32);
        if (lane == 0) {
          auto bsearch = [&](uint32_t v, bool& found) -> uint32_t {
            const uint32_t q = lower_bound_u32(path2, nl, v);
            found = q < nl && path2[q] == v;
            return q;
          };
          bool f0 = false, f1 = false;
          const uint32_t i0 = bsearch(sp[0], f0), i1 = bsearch(sp[ns - 1], f1);
          const uint32_t pre = f0 ? i0 : 0u, post = f1 ? i1 + 1 : nl;
          uint32_t q = 0;
          for (uint32_t t = 0; t < pre; ++t) path[q++] = path2[t];
          for (uint32_t t = 0; t < ns; ++t) path[q++] = sp[t];  // q <= pre + t < cap + t: never overtakes sp
          for (uint32_t t = post; t < nl; ++t) path[q++] = path2[t];
          shared_u32[0] = q;
        }
        C::sync();
        np = shared_u32[0];
        C::sync();
      } else {
        np = sdpkpp_d<W>(lane, matches, nm, k, (uint32_t)ms, sc.gap_open, sc.gap_extend, ev, dp_score, dp_prev, fen,
                         ycoord, path, shared_u32);
      }
    }
    // create_from_match_path, banded.rs:1330-1367
    const uint64_t first = matches[path[0]], last = matches[path[np - 1]];
    if (!band.set_boundaries((uint32_t)(first >> 32), (uint32_t)first, (uint32_t)(last >> 32), (uint32_t)last, k, w, sc))
      status = 2;
    bool has_prev = false;
    uint32_t p0 = 0, p1 = 0;
    for (uint32_t t = 0; t < np;) {
      const uint64_t cur = matches[path[t]];
      const uint32_t c0 = (uint32_t)(cur >> 32), c1 = (uint32_t)cur;
      if (has_prev && c0 == p0 + 1 && c1 == p1 + 1) {
        // a run of matches that each continue the previous one: add_entry((prev.0 + k, prev.1 + k)) per member
        uint32_t L = 1;
        while (t + L < np) {
          const uint64_t nx = matches[path[t + L]];
          if ((uint32_t)(nx >> 32) != c0 + L || (uint32_t)nx != c1 + L) break;
          ++L;
        }
        band.add_entry_run((uint64_t)p0 + k, (uint64_t)p1 + k, L, w);
        p0 = c0 + (L - 1);
        p1 = c1 + (L - 1);
        t += L;
      } else {
        if (has_prev)
          if (!band.add_gap(p0 + (k - 1), p1 + (k - 1), c0, c1, w)) status = 2;
        band.add_kmer(c0, c1, k, w);
        p0 = c0;
        p1 = c1;
        t += 1;
      }
      has_prev = true;
    }
  }
  if (band.any_oob()) return 3;
  *cells_out = band.num_cells();
  if (touched_out) {
    uint64_t a, b;
    band.touched(a, b);
    touched_out[0] = (uint32_t)a;
    touched_out[1] = (uint32_t)b;
  }
  return status;
}

// ------------------------------------------------------------------ K3: compute_alignment for one pair
// K3 slab of one pair (byte offsets; every array starts 16-byte aligned)
struct K3Layout {
  uint64_t colstart, S, Sn, Ly, Lx, row0, rowm, col0, coln, cells, total;
};
B2A_HD uint64_t al16(uint64_t v) { return (v + 15) & ~15ull; }
B2A_HD K3Layout k3_layout(uint64_t m, uint64_t n, uint64_t ncells) {
  K3Layout L;
  uint64_t b = 0;
  L.colstart = b; b = al16(b + (n + 2) * 4);
  L.S = b;        b = al16(b + 6 * (m + 1) * 4);   // S[2], I[2], D[2]
  L.Sn = b;       b = al16(b + (m + 1) * 4);
  L.Ly = b;       b = al16(b + (m + 1) * 4);
  L.Lx = b;       b = al16(b + (n + 1) * 4);
  L.row0 = b;     b = al16(b + (n + 1) * 2);
  L.rowm = b;     b = al16(b + (n + 1) * 2);
  L.col0 = b;     b = al16(b + (m + 1) * 2);
  L.coln = b;     b = al16(b + (m + 1) * 2);
  L.cells = b;    b = al16(b + ncells * 2);
  L.total = (b + 255) & ~255ull;
  return L;
}
// score_only: the slab of a score-only call has no interior cells (the region `cells` is empty)
B2A_HD uint64_t k3_slab_bytes(uint64_t m, uint64_t n, uint64_t cells, bool score_only = false) {
  // a refused band (> MAX_CELLS) needs no state at all
  return cells > BANDED_MAX_CELLS ? 256 : k3_layout(m, n, score_only ? 0 : cells).total;
}

struct BandedOut {
  int32_t score;
  uint32_t xstart, xend, ystart, yend, xlen, ylen, n_ops, status;
  uint32_t clip[4];
};

// ---------------------------------------------------------------------------------------------------------
// The register-resident column loop of K3.
//
// The literal loop keeps the reference's rolling S/I/D arrays in the slab and gives one band row of a column
// to each lane, 32 rows at a time: ~245 instructions per cell-lane (loads, stores, 64-bit indexing, a 5-step
// scan per 32 rows) plus ~600 per column of one-lane sections and barriers.  Here a lane owns R CONSECUTIVE rows
// and carries what the next column needs of them in registers -- S and D of the previous column, the s-bits of
// the previous column's cell (the D-open nibble), the row tracker Sn -- so a column costs one pass over R rows per
// lane, one prefix maximum over the lanes for the vertical I chain, and no S/I/D traffic at all; the one-lane
// sections become uniform register arithmetic.  The traceback cells, Sn/Ly, Lx and the border rows are written
// exactly as before, and the last column's S and I are left in the slab for the end-of-matrix passes.
//
// Rows are owned in blocks of R: row i belongs to block i / R, block B to lane B % W; a lane holds one block at
// a time and moves on to block B + W when B has fallen out of the sliding window (the band of the column plus
// the row above it).  It applies to pairs (banded_fast_ok) whose band
//   * never needs more than W blocks in one column (band height up to ~W*R rows: 160 for R = 5),
//   * has non-decreasing starts and ends over consecutive non-empty columns (then every value the reference
//     reads from outside the previous column's band is MIN_SCORE: the rows below were reset, banded.rs:676-680,
//     the row above was set, 556-561 -- no leftovers of older columns are ever visible), and
//   * has only the Band::new sentinel as empty columns;
// every other pair runs the literal loop.  All 300 sampled pairs of BASELINE config 4 qualify.
// [jlo, jhi]: the columns the band construction touched (every other column is a Band::new sentinel and passes)
template <int W, int R>
B2A_HD bool banded_fast_ok(int lane, const uint32_t* rng, uint64_t m, uint64_t n, uint64_t jlo = 0,
                           uint64_t jhi = ~0ull) {
  using C = Coop<W>;
  if (W != 32 || m < 2 || n < 2 || m >= (1u << 24) || n >= (1u << 24)) return false;
  bool ok = true;
  const uint64_t jend = jhi < n ? jhi + 1 : n;  // one past the touched range: it still looks back at column jhi
  for (uint64_t j = jlo + (uint64_t)lane; j <= jend; j += W) {
    const uint64_t s = rng[2 * j], e = rng[2 * j + 1];
    if (s >= e) {
      if (!(s == m + 1 && e == 0)) ok = false;
      continue;
    }
    const uint64_t lo = umax64(1, s), hi = umin64(e, m);
    if (lo < hi) {
      const uint64_t f = umax64(lo - 1, 1);
      if ((hi - 1) / R - f / R + 1 > (uint64_t)W) ok = false;
    }
    if (j >= 1) {
      const uint64_t ps = rng[2 * (j - 1)], pe = rng[2 * (j - 1) + 1];
      if (ps < pe && (s < ps || e < pe)) ok = false;
    }
  }
  return C::ballot(!ok) == 0u;
}

// Pairs for the strip-wavefront fill (b2a_banded_strip.cuh): the conditions of banded_fast_ok that make every read
// outside the previous column's band a MIN_SCORE (monotone starts and ends, Band::new sentinels only) -- without
// its height limit, the rows are not held in a sliding window there -- plus: the band's columns are one run (the
// strips find their column windows by binary search), and column n is empty (the last column's extra Sn terms,
// banded.rs:590-596, stay with the literal loops).  out3 = {first, last non-empty column, sum over the band's
// columns 1..n-1 of the KS_ROWS-row strips they touch}.
template <int W>
B2A_HD bool banded_strip_ok(int lane, const uint32_t* rng, uint64_t m, uint64_t n, uint32_t* out3, uint64_t jlo = 0,
                            uint64_t jhi = ~0ull, bool last_column_ok = false) {
  using C = Coop<W>;
  if (W != 32 || m < 2 || n < 2 || m >= (1u << 24) || n >= (1u << 24)) return false;
  bool ok = true;
  uint32_t c0 = 0xFFFFFFFFu, c1 = 0, cnt = 0, scols = 0;
  const uint64_t jend = jhi < n ? jhi + 1 : n;
  for (uint64_t j = jlo + (uint64_t)lane; j <= jend; j += W) {
    const uint64_t s = rng[2 * j], e = rng[2 * j + 1];
    if (s >= e) {
      if (!(s == m + 1 && e == 0)) ok = false;
      continue;
    }
    ++cnt;
    c0 = (uint32_t)j < c0 ? (uint32_t)j : c0;
    c1 = (uint32_t)j > c1 ? (uint32_t)j : c1;
    if (j == n && !last_column_ok) ok = false;  // (the finish pass runs the literal loop on column n when allowed)
    if (j >= 1) {
      const uint64_t ps = rng[2 * (j - 1)], pe = rng[2 * (j - 1) + 1];
      if (ps < pe && (s < ps || e < pe)) ok = false;
      const uint64_t lo = umax64(1, s), hi = umin64(e, m);  // interior rows lo .. hi-1
      if (lo < hi && j < n) scols += (uint32_t)((hi - 2) / KS_ROWS - (lo - 1) / KS_ROWS + 1);
    }
  }
  for (int d = 16; d; d >>= 1) {
    // (butterfly by rotation: every lane ends with the totals)
    const uint32_t oc0 = (uint32_t)C::from((int32_t)c0, (lane + d) % W), oc1 = (uint32_t)C::from((int32_t)c1, (lane + d) % W);
    const uint32_t ocnt = (uint32_t)C::from((int32_t)cnt, (lane + d) % W), osc = (uint32_t)C::from((int32_t)scols, (lane + d) % W);
    c0 = oc0 < c0 ? oc0 : c0;
    c1 = oc1 > c1 ? oc1 : c1;
    cnt += ocnt;
    scols += osc;
  }
  if (C::ballot(!ok) != 0u) return false;
  if (cnt == 0 || cnt != c1 - c0 + 1) return false;
  out3[0] = c0;
  out3[1] = c1;
  out3[2] = scols;
  return true;
}

B2A_HD int32_t count_trailing_ones(uint32_t v) {  // number of consecutive set bits from bit 0
#if defined(__CUDA_ARCH__)
  return v == 0xFFFFFFFFu ? 32 : __ffs((int)~v) - 1;
#else
  int32_t c = 0;
  while (c < 32 && ((v >> c) & 1u)) ++c;
  return c;
#endif
}

// SCORES: no interior cell is stored (`cells` may be null); column n's cells, the border rows, Sn/Ly and Lx are as above
template <int W, int R, class ScoreFn, bool SCORES = false>
B2A_HD void banded_columns_fast(const int lane, const uint8_t* x, const int32_t m, const uint8_t* y, const int32_t n,
                                const DevScoring& sc, ScoreFn score, const uint32_t* rng, const uint32_t* colstart,
                                const int32_t* S0arr /* column 0's S */, int32_t* Sfin, int32_t* Ifin, int32_t* Sn,
                                uint32_t* Ly, uint32_t* Lx, uint16_t* row0, uint16_t* rowm, const uint16_t* col0,
                                uint16_t* coln, uint16_t* cells) {
  using C = Coop<W>;
  static_assert(W == 32 || W == 1, "lanes of one warp");
  const int32_t go = sc.gap_open, ge = sc.gap_extend;
  const int32_t xp = sc.xclip_prefix, xs = sc.xclip_suffix, yp = sc.yclip_prefix, ys = sc.yclip_suffix;
  const int32_t gs = imax(ge, go);
  constexpr int32_t NEG = -(1 << 30);  // "no contribution" in the transformed I chain
  const int prev_lane = (lane + W - 1) % W;
  // lane state: the block of R rows this lane holds
  int32_t blk = -1;
  int32_t Sp[R], Dp[R], Snr[R];
  uint32_t psb[R];
  int32_t xr[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    Sp[r] = Dp[r] = Snr[r] = MIN_SCORE;
    psb[r] = 0;
    xr[r] = 0;
  }
  // uniform state (every lane holds the same values)
  int32_t S0_prev = S0arr[0];   // S(0, j-1), MIN_SCORE when row 0 was not in the band there
  int32_t Sm_prev = S0arr[m];   // S[m] as the previous column left it
  int32_t Dm_prev = MIN_SCORE;  // D(m, j-1)
  int32_t Sn0 = Sn[0], Snm = Sn[m];
  bool all_fresh = false;       // an empty column has passed: nothing of older columns is visible any more
  bool last_empty = false;      // column n is empty
  for (int32_t j = 1; j <= n; ++j) {
    const int32_t s = (int32_t)rng[2 * j], e = (int32_t)rng[2 * j + 1];
    if (s >= e) {
      // a run of empty columns: only row m's x-suffix-clip nibble is written (banded.rs:655-661 with i_end = 0)
      const int32_t jc = j + lane;
      const bool emp = jc <= n && rng[2 * jc] >= rng[2 * jc + 1];
      const uint32_t bal = C::ballot(emp);
      const int32_t run = count_trailing_ones(bal);  // >= 1: this column is empty
      if (lane < run) rowm[jc] = (uint16_t)((rowm[jc] & ~0x0F00u) | (TB_XCLIP_SUFFIX << 8));
      S0_prev = Sm_prev = Dm_prev = MIN_SCORE;
      all_fresh = true;
      j += run - 1;
      last_empty = j >= n;
      continue;
    }
    const bool last = j == n;
    const int32_t lo = s > 1 ? s : 1, hi_main = e < m ? e : m;
    const int32_t q = (int32_t)y[j - 1];
    // ------------------------------------------------------------------ row 0 (banded.rs:519-553), uniform
    int32_t S0_cur = MIN_SCORE;
    uint32_t sb0 = 0;
    if (s == 0) {
      int32_t D0;
      uint32_t db;
      if (j == 1) {
        D0 = go;
        db = TB_START;
      } else {
        const int32_t d_score = go + ge * (j - 1), c_score = yp + go;
        if (d_score > c_score) {
          D0 = d_score;
          db = TB_DEL;
        } else {
          D0 = c_score;
          db = TB_YCLIP_PREFIX;
        }
      }
      if (D0 > yp) {
        S0_cur = D0;
        sb0 = TB_DEL;
      } else {
        S0_cur = yp;
        sb0 = TB_YCLIP_PREFIX;
      }
      if (S0_cur + ys > Sn0) {
        Sn0 = S0_cur + ys;
        if (lane == 0) {
          Sn[0] = Sn0;
          Ly[0] = (uint32_t)(n - j);
          row0[n] = (uint16_t)((row0[n] & ~0x0F00u) | (TB_YCLIP_SUFFIX << 8));
        }
      }
      // (the eager write above lands on this very cell when j == n; the reference's put() then overwrites it)
      if (lane == 0) row0[j] = (uint16_t)((db << 4) | (sb0 << 8));
    }
    const int32_t xclip_score = xp + imax(last ? imax(yp, Sn0) : yp, go + ge * (j - 1));
    // carries into the first band row: the row above it in THIS column (banded.rs:556-561: MIN_SCORE unless it is row 0)
    int32_t cS = s == 0 ? S0_cur : MIN_SCORE, cI = MIN_SCORE, cSn = MIN_SCORE;
    uint32_t csb = s == 0 ? sb0 : 0u;
    if (last) {
      cSn = lo - 1 == 0 ? Sn0 : Sn[lo - 1];
      if (lo - 1 >= 1) csb = ((uint32_t)coln[lo - 1] >> 8) & 15u;  // column n's cells exist outside the band too
    }
    int32_t trk_val = MIN_SCORE, trk_i = 0;
    bool trk_hit = false;
    // values of row m-1 in this column (for the cell of row m), valid when hi_main == m
    int32_t rS = cS, rI = cI, rSn = cSn, rSup = MIN_SCORE;
    uint32_t rsb = csb;
    if (lo < hi_main) {
      // ---------------------------------------------------------------- the lane's block for this column
      const int32_t f = lo - 1 > 1 ? lo - 1 : 1;
      const int32_t Blo = f / R;
      const int32_t k = (lane - Blo % W + W) % W;  // position of this lane's block in the window, lowest block first
      const int32_t nblk = Blo + k;
      if (nblk != blk || all_fresh) {
        blk = nblk;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int32_t i = blk * R + r;
          const bool real = i >= 1 && i <= m;
          Sp[r] = MIN_SCORE;
          psb[r] = 0;
          if (j == 1 && real) {  // the previous column is column 0: its S and cells are in the slab
            Sp[r] = S0arr[i];
            psb[r] = ((uint32_t)col0[i] >> 8) & 15u;
          }
          Dp[r] = MIN_SCORE;
          Snr[r] = real ? Sn[i] : MIN_SCORE;
          xr[r] = (int32_t)x[real ? i - 1 : 0];  // rows beyond x repeat a real symbol: the score function only ever sees sequence bytes
        }
      }
      // ---------------------------------------------------------------- per row: everything that does not need I
      int32_t A[R], best_d[R], m_score[R], ycs[R];
      uint32_t db[R];
      bool inw[R];
      const int32_t up_S = C::from(Sp[R - 1], prev_lane);  // S(i-1, j-1) of this lane's first row
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int32_t i = blk * R + r;
        inw[r] = i >= lo && i < hi_main;
        int32_t sup = r == 0 ? up_S : Sp[r - 1];
        if (i == 1) sup = S0_prev;  // row 0 is not a lane row
        m_score[r] = sup + score((uint8_t)xr[r], (uint8_t)q);
        const int32_t d_score = Dp[r] + ge, s_open = Sp[r] + go;
        if (d_score > s_open) {
          best_d[r] = d_score;
          db[r] = TB_DEL;
        } else {
          best_d[r] = s_open;
          db[r] = psb[r];
        }
        ycs[r] = yp + go + ge * (i - 1);
        A[r] = imax(imax(imax(MIN_SCORE, m_score[r]), imax(best_d[r], xclip_score)), ycs[r]);
      }
      // ---------------------------------------------------------------- the vertical chain: I(i) - gs*i is a
      // running maximum (see banded_compute_d); rows outside the band contribute nothing, the first band row is
      // seeded literally from the row above it
      const int32_t up_A = C::from(A[R - 1], prev_lane);
      const int32_t up_Sn = last ? C::from(Snr[R - 1], prev_lane) : MIN_SCORE;
      int32_t u[R];
      {
        int32_t run_max = NEG;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int32_t i = blk * R + r;
          int32_t t = NEG;
          if (inw[r]) {
            if (i == lo) {
              int32_t bi = imax(cI + ge, cS + go);
              if (last) bi = imax(bi, cSn + go);
              t = bi - gs * i;
            } else {
              const int32_t aprev = r == 0 ? up_A : A[r - 1];
              const int32_t snprev = r == 0 ? up_Sn : Snr[r - 1];
              t = (last ? imax(aprev, snprev) : aprev) + go - gs * i;
            }
          }
          run_max = imax(run_max, t);
          u[r] = run_max;
        }
      }
      int32_t excl;
      {
        int32_t v = u[R - 1];  // inclusive scan over the lanes in window order (lane of the lowest block first)
        for (int d = 1; d < W; d <<= 1) {
          const int32_t t = C::from(v, (lane + W - d) % W);
          if (k >= d) v = imax(v, t);
        }
        excl = C::from(v, prev_lane);
        if (k == 0) excl = NEG;
      }
      // ---------------------------------------------------------------- the cells, literally
      int32_t best[R], best_i[R], sncur[R];
      uint32_t sb[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int32_t i = blk * R + r;
        best_i[r] = imax(u[r], excl) + gs * i;
        int32_t b = MIN_SCORE;
        uint32_t c = TB_START;
        if (m_score[r] > b) {
          b = m_score[r];
          c = (xr[r] == q) ? TB_MATCH : TB_SUBST;
        }
        if (best_i[r] > b) {
          b = best_i[r];
          c = TB_INS;
        }
        if (best_d[r] > b) {
          b = best_d[r];
          c = TB_DEL;
        }
        if (xclip_score > b) {
          b = xclip_score;
          c = TB_XCLIP_PREFIX;
        }
        if (ycs[r] > b) {
          b = ycs[r];
          c = TB_YCLIP_PREFIX;
        }
        best[r] = b;
        sb[r] = c;
        sncur[r] = Snr[r];
        if (inw[r] && b + ys > Snr[r]) {  // row tracker, banded.rs:650-654 (eager write of (i, n)'s s-bits)
          sncur[r] = b + ys;
          Sn[i] = sncur[r];
          Ly[i] = (uint32_t)(n - j);
          if (!last) coln[i] = (uint16_t)((coln[i] & ~0x0F00u) | (TB_YCLIP_SUFFIX << 8));
        }
      }
      // the I nibble needs the final values of the row above
      const int32_t up_best = C::from(best[R - 1], prev_lane), up_bi = C::from(best_i[R - 1], prev_lane);
      const uint32_t up_sb = (uint32_t)C::from((int32_t)sb[R - 1], prev_lane);
      const int32_t up_sncur = last ? C::from(sncur[R - 1], prev_lane) : MIN_SCORE;
      uint16_t* const wbase = last ? coln : cells;
      const uint32_t woff = (last || SCORES) ? 0u : colstart[j] - (uint32_t)s;  // cell (i, j) = wbase[woff + i]
      int32_t lane_trk_val = MIN_SCORE, lane_trk_i = 0;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int32_t i = blk * R + r;
        if (!inw[r]) continue;
        int32_t pS, pI, pSn;
        uint32_t psbc;
        if (i == lo) {
          pS = cS;
          pI = cI;
          pSn = cSn;
          psbc = csb;
        } else if (r == 0) {
          pS = up_best;
          pI = up_bi;
          pSn = up_sncur;
          psbc = up_sb;
        } else {
          pS = best[r - 1];
          pI = best_i[r - 1];
          pSn = sncur[r - 1];
          psbc = sb[r - 1];
        }
        uint32_t ib;
        {
          const int32_t i_score = pI + ge, s_score = pS + go;
          int32_t bl;
          if (i_score > s_score) {
            bl = i_score;
            ib = TB_INS;
          } else {
            bl = s_score;
            ib = psbc;
          }
          if (last && pSn + go > bl) ib = TB_YCLIP_SUFFIX;
        }
        if (!SCORES || last) wbase[woff + (uint32_t)i] = (uint16_t)(ib | (db[r] << 4) | (sb[r] << 8));
        if (last) {  // the end-of-matrix passes read column n's S and I from the slab
          Sfin[i] = best[r];
          Ifin[i] = best_i[r];
        }
        if (best[r] + xs > lane_trk_val) {  // this lane's rows ascend: a strict > keeps the first
          lane_trk_val = best[r] + xs;
          lane_trk_i = i;
        }
      }
      {  // first row with the highest S + xs (lowest row wins ties), banded.rs:645-649
        long long key = lane_trk_val > MIN_SCORE
                            ? (long long)((unsigned long long)(long long)lane_trk_val << 32) +
                                  (long long)(0xFFFFFFFFu - (uint32_t)lane_trk_i)
                            : (long long)0x8000000000000000ull;
        key = C::all_max(key);
        if (key != (long long)0x8000000000000000ull) {
          trk_val = (int32_t)(key >> 32);
          trk_i = (int32_t)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFll));
          trk_hit = true;  // trk_val > MIN_SCORE == the tracker's value at the start of the column
        }
      }
      if (hi_main == m) {  // row m-1 of this column and S(m-1, j-1), for the cell of row m
        const int32_t rr = (m - 1) % R, owner = ((m - 1) / R) % W;
        int32_t vS = best[0], vI = best_i[0], vSn = sncur[0], vSup = Sp[0];
        uint32_t vsb = sb[0];
#pragma unroll
        for (int r = 1; r < R; ++r)
          if (r == rr) {
            vS = best[r];
            vI = best_i[r];
            vSn = sncur[r];
            vSup = Sp[r];
            vsb = sb[r];
          }
        rS = C::from(vS, owner);
        rI = C::from(vI, owner);
        rSn = C::from(vSn, owner);
        rSup = C::from(vSup, owner);
        rsb = (uint32_t)C::from((int32_t)vsb, owner);
      }
      // roll the lane state forward: what column j+1 reads of this column
#pragma unroll
      for (int r = 0; r < R; ++r) {
        Sp[r] = inw[r] ? best[r] : MIN_SCORE;
        Dp[r] = inw[r] ? best_d[r] : MIN_SCORE;
        psb[r] = inw[r] ? sb[r] : 0u;
        Snr[r] = sncur[r];
      }
      all_fresh = false;
    } else {
      // no interior rows in this column (row 0 and / or row m only)
      if (hi_main == m && e == m + 1) {  // row m's neighbours: row m-1 is the (unowned or fresh) row above
        const int32_t owner = ((m - 1) / R) % W, rr = (m - 1) % R;
        int32_t vSup = Sp[0];
#pragma unroll
        for (int r = 1; r < R; ++r)
          if (r == rr) vSup = Sp[r];
        const int32_t have = (blk == (m - 1) / R && !all_fresh) ? 1 : 0;
        const int32_t got = C::from(vSup, owner), has = C::from(have, owner);
        rSup = has ? got : MIN_SCORE;
        if (m - 1 == 0) rSup = S0_prev;
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        Sp[r] = Dp[r] = MIN_SCORE;
        psb[r] = 0;
      }
    }
    // ------------------------------------------------------------------ the column tracker and row m, uniform
    int32_t Sm = MIN_SCORE;  // S[m] of this column: reset at the start of every column (banded.rs:556-561)
    if (trk_hit) {
      Sm = trk_val;
      if (lane == 0) {
        Lx[j] = (uint32_t)(m - trk_i);
        rowm[j] = (uint16_t)((rowm[j] & ~0x0F00u) | (TB_XCLIP_SUFFIX << 8));
      }
    }
    int32_t Dm_cur = MIN_SCORE;
    const int32_t hi = e;
    if ((s > 1 ? s : 1) < hi && hi == m + 1) {  // the cell of row m: it starts from the column tracker
      const int32_t i = m;
      const int32_t p = (int32_t)x[i - 1];
      uint32_t ib, dbm, sbm;
      if (m - 1 == 0) rSup = S0_prev;
      const int32_t m_sc = rSup + score((uint8_t)p, (uint8_t)q);
      const int32_t i_score = rI + ge;
      int32_t s_score = rS + go;
      int32_t bi;
      if (i_score > s_score) {
        bi = i_score;
        ib = TB_INS;
      } else {
        bi = s_score;
        ib = rsb;
      }
      if (last) {
        const int32_t clip_score = rSn + go;
        if (clip_score > bi) {
          bi = clip_score;
          ib = TB_YCLIP_SUFFIX;
        }
      }
      const int32_t d_score = Dm_prev + ge;
      s_score = Sm_prev + go;
      int32_t bd;
      if (d_score > s_score) {
        bd = d_score;
        dbm = TB_DEL;
      } else {
        bd = s_score;
        dbm = ((uint32_t)rowm[j - 1] >> 8) & 15u;  // s-bits of (m, j-1) as stored so far
      }
      sbm = TB_XCLIP_SUFFIX;
      int32_t b = Sm;
      if (m_sc > b) {
        b = m_sc;
        sbm = (p == q) ? TB_MATCH : TB_SUBST;
      }
      if (bi > b) {
        b = bi;
        sbm = TB_INS;
      }
      if (bd > b) {
        b = bd;
        sbm = TB_DEL;
      }
      if (xclip_score > b) {
        b = xclip_score;
        sbm = TB_XCLIP_PREFIX;
      }
      const int32_t yclip_score = yp + go + ge * (i - 1);
      if (yclip_score > b) {
        b = yclip_score;
        sbm = TB_YCLIP_PREFIX;
      }
      Sm = b;
      Dm_cur = bd;
      // (S[i] + xs > S[m] with i == m never holds: xs <= 0)
      if (Sm + ys > Snm) {  // banded.rs:650-654 at i == m: the eager write goes to (m, n) ...
        Snm = Sm + ys;
        if (lane == 0) {
          Sn[m] = Snm;
          Ly[m] = (uint32_t)(n - j);
          rowm[n] = (uint16_t)((rowm[n] & ~0x0F00u) | (TB_YCLIP_SUFFIX << 8));
        }
      }
      if (lane == 0) {  // ... and the cell's own put() follows it (so at j == n the put wins)
        if (last) Ifin[m] = bi;
        rowm[j] = (uint16_t)(ib | (dbm << 4) | (sbm << 8));
      }
    }
    if (Sm + ys > Snm) {  // banded.rs:662-666
      Snm = Sm + ys;
      if (lane == 0) {
        Sn[m] = Snm;
        Ly[m] = (uint32_t)(n - j);
        rowm[n] = (uint16_t)((rowm[n] & ~0x0F00u) | (TB_YCLIP_SUFFIX << 8));
      }
    }
    if (e < m + 1) {
      if (lane == 0) rowm[j] = (uint16_t)((rowm[j] & ~0x0F00u) | (TB_XCLIP_SUFFIX << 8));
      Sm = MIN_SCORE;
    }
    if (last) {
      if (lane == 0) {
        Sfin[m] = Sm;
        if (s == 0) {
          Sfin[0] = S0_cur;
          Ifin[0] = MIN_SCORE;
        }
        if (e < m) Sfin[e] = MIN_SCORE;  // the row just below the band keeps its (reset) MIN_SCORE, banded.rs:689
      }
    }
    S0_prev = s == 0 ? S0_cur : MIN_SCORE;
    Sm_prev = Sm;
    Dm_prev = Dm_cur;
    C::sync();  // Sn / column-n cells written by one lane are read by others in later columns
  }
  // an empty last column leaves S[m] = MIN_SCORE behind (banded.rs:556-561); the slab may still hold column 0's
  if (last_empty && lane == 0) Sfin[m] = MIN_SCORE;
  C::sync();
}

// compute_alignment for one pair by W cooperating lanes (banded.rs:406-869).
//
// The column loop keeps the reference's arrays (rolling S/I/D with their leftovers, Sn/Ly/Lx, the eager
// traceback writes) in the pair's slab and performs the same reads and writes per column; only the inner
// loop over the band rows of one column is spread over the lanes, 32 rows at a time:
//   * everything that comes from column j-1 (M, D, the clip terms) is independent per row;
//   * the vertical chain I(i) = max(I(i-1)+ge, S(i-1)+go [, Sn(i-1)+go in the last column]) is a prefix
//     maximum: with A(i) = S(i) without its I term, S(i-1) = max(A(i-1), I(i-1)), hence
//     I(i) = max(I(i-1) + gs, A(i-1) + go) with gs = max(ge, go), i.e. I(i) - gs*i is a running maximum
//     of A(i-1) + go - gs*i -- exact integer arithmetic, no saturation anywhere;
//   * with the values known, every strict comparison of the reference (which source wins S, I from
//     extension or open, the Sn/Ly row tracker) is re-evaluated literally per row from the final
//     neighbours' values, and the column tracker S[m]/Lx is an arg-max with the lowest row winning ties.
// Row m of a column, row 0, column 0, the end-of-matrix passes and the walk are sequential work of lane 0.
// FASTR > 0 selects the register-resident column loop (FASTR rows per lane, see below); the caller must have
// checked banded_fast_ok<W, FASTR> for the pair.  FASTR == 0 is the literal loop.
// PHASE: 0 = the whole alignment; 1 = everything up to the final score (left in S[n % 2][m]); 2 = the walk only, on
// the state phase 1 left in the slab (the strip path walks one pair per LANE in a kernel of its own: the walk is
// sequential per pair, and a warp whose other 31 lanes wait for lane 0 issues 32 times the instructions).
// SCORES (score-only calls): score, xend, yend and status only.  No interior cell (1 <= i <= m-1, 1 <= j <= n-1) is
// stored or read -- the slab has no `cells` region, the strip area no traceback -- and a read of one returns START
// without touching memory; row 0, row m, column 0, column n, Sn/Ly/Lx and the end-of-matrix passes are as above.
// xend / yend are set only by the suffix-clip moves, whose codes sit on row m and column n, and the walk never
// increases i or j: it stops on the first cell with i < m and j < n, before reading it (DESIGN.md §2).  It writes no
// ops (ops_end may be null), no starts and no clip lengths.
template <int W, class ScoreFn, int FASTR = 0, int PHASE = 0, bool SCORES = false>
B2A_HD void banded_compute_d(int lane, const uint8_t* x, uint64_t m, const uint8_t* y, uint64_t n,
                             const DevScoring& sc, ScoreFn score, const uint32_t* rng, uint64_t num_cells,
                             uint8_t* slab, bool filter_clips, uint8_t* ops_end, BandedOut& out,
                             const uint8_t* strip_area = nullptr, const uint32_t* cols3 = nullptr, bool* redo = nullptr) {
  using C = Coop<W>;
  constexpr bool STRIP = FASTR < 0;  // the finish pass of the strip-wavefront fill (b2a_banded_strip.cuh)
  out.status = 0;
  out.n_ops = 0;
  for (int q = 0; q < 4; ++q) out.clip[q] = 0;
  if (num_cells > BANDED_MAX_CELLS) {  // banded.rs:407-420
    out.score = MIN_SCORE;
    out.xstart = out.xend = out.ystart = out.yend = out.xlen = out.ylen = 0;
    return;
  }
  out.xlen = (uint32_t)m;
  out.ylen = (uint32_t)n;
  const K3Layout L = k3_layout(m, n, SCORES ? 0 : num_cells);
  uint32_t* colstart = reinterpret_cast<uint32_t*>(slab + L.colstart);
  int32_t* S0 = reinterpret_cast<int32_t*>(slab + L.S);
  int32_t* Sarr[2] = {S0, S0 + (m + 1)};
  int32_t* Iarr[2] = {S0 + 2 * (m + 1), S0 + 3 * (m + 1)};
  int32_t* Darr[2] = {S0 + 4 * (m + 1), S0 + 5 * (m + 1)};
  int32_t* Sn = reinterpret_cast<int32_t*>(slab + L.Sn);
  uint32_t* Ly = reinterpret_cast<uint32_t*>(slab + L.Ly);
  uint32_t* Lx = reinterpret_cast<uint32_t*>(slab + L.Lx);
  uint16_t* row0 = reinterpret_cast<uint16_t*>(slab + L.row0);
  uint16_t* rowm = reinterpret_cast<uint16_t*>(slab + L.rowm);
  uint16_t* col0 = reinterpret_cast<uint16_t*>(slab + L.col0);
  uint16_t* coln = reinterpret_cast<uint16_t*>(slab + L.coln);
  uint16_t* cells = reinterpret_cast<uint16_t*>(slab + L.cells);
  int64_t kc0 = 1, kc1 = 0;  // STRIP: the band's interior columns, clipped to [1, n-1]
  if (STRIP) {
    kc0 = cols3[0] > 1u ? (int64_t)cols3[0] : 1;
    kc1 = (int64_t)cols3[1] < (int64_t)n - 1 ? (int64_t)cols3[1] : (int64_t)n - 1;
  }
  if constexpr (PHASE != 2) {
  // init (banded.rs:423-438): only the cells that can ever be non-START are stored
  if (!STRIP && !SCORES) {
    uint32_t acc = 0;  // exclusive prefix sum of the column heights
    for (uint64_t b = 0; b <= n; b += W) {
      const uint64_t j = b + (uint64_t)lane;
      const uint32_t h = j <= n ? (uint32_t)sat_sub64(rng[2 * j + 1], rng[2 * j]) : 0u;
      uint32_t inc = h;
      for (int d = 1; d < W; d <<= 1) {
        const uint32_t t = (uint32_t)C::up((int32_t)inc, d);
        if (lane >= d) inc += t;
      }
      if (j <= n) colstart[j] = acc + inc - h;
      acc += (uint32_t)C::from((int32_t)inc, W - 1);
    }
    if (lane == 0) colstart[n + 1] = acc;
  }
  for (int kk = 0; kk < 2; ++kk)
    for (uint64_t i = (uint64_t)lane; i <= m; i += W) {
      Sarr[kk][i] = MIN_SCORE;
      Iarr[kk][i] = MIN_SCORE;
      Darr[kk][i] = MIN_SCORE;
    }
  for (uint64_t i = (uint64_t)lane; i <= m; i += W) {
    if (!STRIP || i == 0 || i == m) {  // (the strip fill has written the rows 1..m-1 of these three)
      Sn[i] = MIN_SCORE;
      Ly[i] = 0;
      coln[i] = 0;
    }
    col0[i] = 0;
  }
  for (uint64_t j = (uint64_t)lane; j <= n; j += W) {
    Lx[j] = 0;
    if (STRIP && j >= 1) {
      // the strip path's finish pass: row m of every column starts as the x-suffix-clip nibble the column loop leaves
      // there (655-661 / 671-674), and row 0's cells 1..n-1 get their final value in one store -- the closed-form
      // s-bits of the border pass (725-731) and, where row 0 is in the band, the d-bits of its cell (518-554)
      rowm[j] = (uint16_t)(TB_XCLIP_SUFFIX << 8);
      uint32_t c0v = 0;
      if (j < n) {
        const bool in0 = (int64_t)j >= kc0 && (int64_t)j <= kc1 && rng[2 * j] == 0 && rng[2 * j + 1] > 0;
        const int32_t d_score = sc.gap_open + sc.gap_extend * ((int32_t)j - 1);
        c0v = ((in0 ? row0_dbits(sc, (int32_t)j) : 0u) << 4) |
              ((d_score > sc.yclip_prefix ? (uint32_t)TB_DEL : (uint32_t)TB_YCLIP_PREFIX) << 8);
      }
      row0[j] = (uint16_t)c0v;
    } else {
      row0[j] = 0;
      rowm[j] = 0;
    }
  }
  C::sync();
  }
  // traceback cell access: pointer for writes (nullptr = a cell the reference never writes there),
  // value for reads (untouched cells read as 0 = START in every nibble)
  auto cellp = [&](uint64_t i, uint64_t j) -> uint16_t* {
    if (i == 0) return &row0[j];
    if (i == m) return &rowm[j];
    if (j == 0) return &col0[i];
    if (j == n) return &coln[i];
    if (STRIP || SCORES) return nullptr;  // interior cells live in the 4-bit traceback (or nowhere), nothing writes them here
    const uint64_t s = rng[2 * j], e = rng[2 * j + 1];
    if (i >= s && i < e) return &cells[colstart[j] + (i - s)];
    return nullptr;
  };
  // STRIP: the strip fill's per-strip table, boundary row m-1 and 4-bit traceback (KsLayout, b2a_banded_strip.cuh)
  const uint32_t* ks_tab = nullptr;
  const int32_t* ks_bnd = nullptr;  // int4 {4*S, 4*I + 2, column-tracker key, 0} per column, index j - kc0 + 1
  const uint32_t* ks_tb = nullptr;
  const uint8_t* ks_last = nullptr;  // int2 {4*S, D} of column n-1 per row (rows of its band), for column n's literal pass
  if (STRIP) {
    const uint64_t ns = m >= 2 ? (m - 1 + KS_ROWS - 1) / KS_ROWS : 0;
    const uint64_t o_tab = 0, o_bnd = al16(ns * KS_TAB * 4),
                   o_last = al16(o_bnd + (uint64_t)((kc1 >= kc0 ? kc1 - kc0 + 1 : 0) + 2) * 16), o_tb = al16(o_last + (m + 1) * 8);
    ks_last = strip_area + o_last;
    ks_tab = reinterpret_cast<const uint32_t*>(strip_area + o_tab);
    ks_bnd = reinterpret_cast<const int32_t*>(strip_area + o_bnd);
    ks_tb = reinterpret_cast<const uint32_t*>(strip_area + o_tb);
  }
  // the 4-bit nibble of an interior cell (1 <= i <= m-1, 1 <= j <= n-1) of the band, 16 = outside the band
  auto ks_nib = [&](uint64_t i, uint64_t j) -> uint32_t {
    const uint64_t s = rng[2 * j], e = rng[2 * j + 1];
    if (!(i >= s && i < e)) return 16u;
    const uint32_t st = (uint32_t)((i - 1) >> KS_ROWS_LOG2), rem = (uint32_t)((i - 1) & (uint64_t)(KS_ROWS - 1)),
                   l = rem >> KS_R_LOG2, r = rem & (uint32_t)(KS_R - 1);
    const uint32_t ja = ks_tab[KS_TAB * st], off = ks_tab[KS_TAB * st + 1];
    const uint32_t t = (uint32_t)j - ja + l;
    const uint32_t word = ks_tb[((size_t)off + ((size_t)(t >> 3) * KS_TBW + (r >> 2)) * KS_G + l) * 4 + (r & 3u)];
    return (word >> (4u * (7u - (t & 7u)))) & 15u;
  };
  auto ks_sbits = [&](uint64_t i, uint64_t j, uint32_t nb) -> uint32_t {
    switch (nb & 3u) {
      case NB_DIAG: return x[i - 1] == y[j - 1] ? (uint32_t)TB_MATCH : (uint32_t)TB_SUBST;
      case NB_INS: return TB_INS;
      case NB_DEL: return TB_DEL;
      default:  // one of the two prefix clips: the x clip is tested first and keeps ties (banded.rs:631-642)
        return xclip_score(sc, (int32_t)j) >= sc.yclip_prefix + sc.gap_open + sc.gap_extend * ((int32_t)i - 1)
                   ? (uint32_t)TB_XCLIP_PREFIX
                   : (uint32_t)TB_YCLIP_PREFIX;
    }
  };
  auto sbits_at = [&](uint64_t i, uint64_t j) -> uint32_t {
    if (SCORES && i >= 1 && i < m && j >= 1 && j < n) return 0u;
    if (STRIP && i >= 1 && i < m && j >= 1 && j < n) {
      const uint32_t nb = ks_nib(i, j);
      return nb == 16u ? 0u : ks_sbits(i, j, nb);
    }
    uint16_t* p = cellp(i, j);
    return p ? ((uint32_t)*p >> 8) & 15u : 0u;
  };
  // one field of a cell (0: i-bits, 1: d-bits, 2: s-bits); in the 4-bit traceback "came from S of the neighbour"
  // resolves to that neighbour's s-bits (untouched cells read as START)
  auto rd_part = [&](uint64_t i, uint64_t j, int part) -> uint32_t {
    if (SCORES && i >= 1 && i < m && j >= 1 && j < n) return 0u;
    if (STRIP && i >= 1 && i < m && j >= 1 && j < n) {
      const uint32_t nb = ks_nib(i, j);
      if (nb == 16u) return 0u;
      if (part == 2) return ks_sbits(i, j, nb);
      if (part == 0) return (nb & NB_IEXT) ? (uint32_t)TB_INS : sbits_at(i - 1, j);
      return (nb & NB_DEXT) ? (uint32_t)TB_DEL : sbits_at(i, j - 1);
    }
    uint16_t* p = cellp(i, j);
    return p ? ((uint32_t)*p >> (4 * part)) & 15u : 0u;
  };
  auto rd = [&](uint64_t i, uint64_t j) -> uint32_t {
    return rd_part(i, j, 0) | (rd_part(i, j, 1) << 4) | (rd_part(i, j, 2) << 8);
  };
  auto set_s = [&](uint64_t i, uint64_t j, uint32_t v) {
    uint16_t* p = cellp(i, j);
    if (p) *p = (uint16_t)((*p & ~0x0F00u) | (v << 8));
  };
  auto set_i = [&](uint64_t i, uint64_t j, uint32_t v) {
    uint16_t* p = cellp(i, j);
    if (p) *p = (uint16_t)((*p & ~0x000Fu) | v);
  };
  auto put = [&](uint64_t i, uint64_t j, uint32_t c) {
    uint16_t* p = cellp(i, j);
    if (p) *p = (uint16_t)c;
  };
  const int32_t go = sc.gap_open, ge = sc.gap_extend;
  const int32_t xp = sc.xclip_prefix, xs = sc.xclip_suffix, yp = sc.yclip_prefix, ys = sc.yclip_suffix;
  const int32_t gs = imax(ge, go);  // slope of the I chain (the banded aligner opens a gap at go alone)
  int32_t* const Sfin = Sarr[n % 2];
  if constexpr (PHASE != 2) {
  if (lane == 0) {  // j = 0, banded.rs:440-509
    int32_t* S = Sarr[0];
    int32_t* I = Iarr[0];
    const uint64_t i_start = rng[0], i_end = rng[1];
    if (i_start == 0) S[0] = 0;
    for (uint64_t i = umax64(1, i_start); i < i_end; ++i) {
      uint32_t ib, sb = TB_START;
      if (i == 1) {
        I[i] = go;
        ib = TB_START;
      } else {
        const int32_t i_score = go + ge * ((int32_t)i - 1), c_score = xp + go;
        if (i_score > c_score) {
          I[i] = i_score;
          ib = TB_INS;
        } else {
          I[i] = c_score;
          ib = TB_XCLIP_PREFIX;
        }
      }
      if (i == m) sb = TB_XCLIP_SUFFIX;
      if (I[i] > S[i]) {
        S[i] = I[i];
        sb = TB_INS;
      }
      if (xp > S[i]) {
        S[i] = xp;
        sb = TB_XCLIP_PREFIX;
      }
      if (S[i] + xs > S[m]) {
        S[m] = S[i] + xs;
        Lx[0] = (uint32_t)(m - i);
        set_s(m, 0, TB_XCLIP_SUFFIX);
      }
      put(i, 0, ib | (TB_START << 4) | (sb << 8));
    }
    for (uint64_t i = i_end; i < umin64(m + 1, rng[2 * umin64(n, 1) + 1]); ++i) {
      S[i] = MIN_SCORE;
      I[i] = MIN_SCORE;
    }
    if (i_end < m + 1) S[m] = MIN_SCORE;
    if (yp > ys) {
      Sn[0] = yp;
      set_s(0, n, TB_YCLIP_PREFIX);
    } else {
      Sn[0] = ys;
      Ly[0] = (uint32_t)n;
      set_s(0, n, TB_YCLIP_SUFFIX);
    }
  }
  C::sync();
  uint64_t lit_from = 1;  // first column of the literal loop below
  if constexpr (FASTR > 0) {
    banded_columns_fast<W, FASTR, ScoreFn, SCORES>(lane, x, (int32_t)m, y, (int32_t)n, sc, score, rng, colstart, Sarr[0],
                                                   Sarr[n % 2], Iarr[n % 2], Sn, Ly, Lx, row0, rowm, col0, coln, cells);
  } else if constexpr (FASTR < 0) {
    // ---------------------------------------------------------------------------------------------------------
    // Finish pass of the strip-wavefront fill: what the column loop (banded.rs:511-681) does outside the interior
    // cells 1..m-1 x 1..n-1 -- row 0's cells and its Sn/Ly seed, row m's cells (they start from the column tracker the
    // fill hands over in the boundary row), and the x-suffix-clip nibble every column leaves in row m.
    const int32_t mi = (int32_t)m;
    const bool coln_empty = rng[2 * n] >= rng[2 * n + 1];
    int32_t Sm_last = MIN_SCORE, Dm_last = MIN_SCORE;  // S / D of (m, n-1), for column n's pass (lane 0)
    // (row 0's cells and row m's x-suffix-clip nibbles were written by the initialisation above)
    if (lane == 0 && kc0 <= kc1 && rng[2 * kc0] == 0 && rng[2 * kc0 + 1] > 0) {
      // S(0, j) never increases with j: only the first row-0 column can raise Sn[0] (547-552)
      const int32_t S0c = imax(row0_D(sc, (int32_t)kc0), yp);
      if (S0c + ys > Sn[0]) {
        Sn[0] = S0c + ys;
        Ly[0] = (uint32_t)(n - (uint64_t)kc0);
        row0[n] = (uint16_t)((row0[n] & ~0x0F00u) | (TB_YCLIP_SUFFIX << 8));
      }
    }
    // row m is in the band where a column's end is m + 1: ends do not decrease, so that is a suffix of the band's columns
    int64_t jm0 = kc1 + 1;
    {
      int64_t a = kc0, b = kc1 + 1;
      while (a < b) {
        const int64_t mid = (a + b) >> 1;
        if (rng[2 * mid + 1] == (uint32_t)(m + 1)) b = mid;
        else a = mid + 1;
      }
      jm0 = a;
    }
    if (lane == 0) {
      // (S, I)(m-1, j) from the boundary row the strip fill left, MIN_SCORE outside the band; 32-bit column arithmetic
      const int32_t k0 = (int32_t)kc0, k1 = (int32_t)kc1, m1 = mi - 1;
      const bool xs_live = xs > DEAD_CLIP;
      auto bnd_SI = [&](int32_t j, int32_t& S_, int32_t& I_) {
        S_ = I_ = MIN_SCORE;
        if (j == 0) {
          S_ = Sarr[0][m1];
          return;
        }
        if (!((int32_t)rng[2 * j] <= m1 && (int32_t)rng[2 * j + 1] > m1)) return;
        const int32_t vs = ks_bnd[4 * (j - k0 + 1)], vi = ks_bnd[4 * (j - k0 + 1) + 1];
        S_ = vs <= -(1 << 29) ? MIN_SCORE : vs >> 2;
        I_ = vi <= -(1 << 29) ? MIN_SCORE : vi >> 2;
      };
      int32_t Sm_prev = jm0 == 1 ? Sarr[0][m] : MIN_SCORE, Dm_prev = MIN_SCORE;
      int32_t Snm = Sn[m];
      const int32_t p = (int32_t)x[m - 1];
      int32_t rSup = MIN_SCORE, unusedI = MIN_SCORE;
      if (jm0 <= kc1) bnd_SI((int32_t)jm0 - 1, rSup, unusedI);
      for (int32_t j = (int32_t)jm0; j <= k1; ++j) {
        const int32_t q = (int32_t)y[j - 1];
        const int32_t xcs = xp + imax(yp, go + ge * (j - 1));
        int32_t rS, rI;
        bnd_SI(j, rS, rI);
        const uint32_t rsb = sbits_at(m - 1, (uint64_t)j);
        uint32_t ib, dbm, sbm;
        const int32_t m_sc = rSup + score((uint8_t)p, (uint8_t)q);
        int32_t bi;
        if (rI + ge > rS + go) {
          bi = rI + ge;
          ib = TB_INS;
        } else {
          bi = rS + go;
          ib = rsb;
        }
        int32_t bd;
        if (Dm_prev + ge > Sm_prev + go) {
          bd = Dm_prev + ge;
          dbm = TB_DEL;
        } else {
          bd = Sm_prev + go;
          dbm = ((uint32_t)rowm[j - 1] >> 8) & 15u;  // s-bits of (m, j-1) as stored so far
        }
        sbm = TB_XCLIP_SUFFIX;
        // the cell starts from the column tracker (645-653): the first interior band row with the highest S + xs, from
        // the boundary row's packed key; with a dead x-suffix clip it stays below every real candidate
        int32_t b = MIN_SCORE;
        if (xs_live && (int32_t)rng[2 * j] <= m1) {  // (row m in the band and the band's start above it: row m-1 is in it)
          const int32_t key = ks_bnd[4 * (j - k0 + 1) + 2];
          if (key != (int32_t)0x80000000) {
            b = (key >> 12) + xs;
            Lx[j] = (uint32_t)(mi - (4095 - (key & 4095)));
          }
        }
        if (m_sc > b) {
          b = m_sc;
          sbm = (p == q) ? TB_MATCH : TB_SUBST;
        }
        if (bi > b) {
          b = bi;
          sbm = TB_INS;
        }
        if (bd > b) {
          b = bd;
          sbm = TB_DEL;
        }
        if (xcs > b) {
          b = xcs;
          sbm = TB_XCLIP_PREFIX;
        }
        const int32_t ycs = yp + go + ge * (mi - 1);
        if (ycs > b) {
          b = ycs;
          sbm = TB_YCLIP_PREFIX;
        }
        if (b + ys > Snm) {  // 655-660 at i == m, then the cell's own put()
          Snm = b + ys;
          Sn[m] = Snm;
          Ly[m] = (uint32_t)(n - (uint64_t)j);  // (the eager mark on (m, n) is overwritten below: column n comes last)
        }
        rowm[j] = (uint16_t)(ib | (dbm << 4) | (sbm << 8));
        Sm_prev = b;
        Dm_prev = bd;
        rSup = rS;  // S(m-1, j) is the next column's diagonal input
      }
      if (coln_empty) {
        Sarr[n % 2][m] = MIN_SCORE;  // S[m] ends the loop reset (556-561) ...
        rowm[n] = (uint16_t)(TB_XCLIP_SUFFIX << 8);  // ... and its nibble, written last, replaces the eager marks (671-674)
      }  // (else column n's own pass below rewrites the s-bits of (m, n); its i / d bits are still untouched)
      // what column n reads of column n-1 in row m
      Sm_last = k1 == (int32_t)n - 1 && jm0 <= kc1 ? Sm_prev : MIN_SCORE;
      Dm_last = k1 == (int32_t)n - 1 && jm0 <= kc1 ? Dm_prev : MIN_SCORE;
    }
    C::sync();
    if (!coln_empty) {
      // Column n holds band cells: the literal loop runs it (its extra Sn terms, 590-596, are not the packed cell's),
      // reading column n-1 from the rolling arrays as the reference would have left them -- MIN_SCORE outside the
      // band, the strip fill's export inside, row 0's closed form and row m from the pass above.
      const int pc = (int)((n - 1) % 2);
      for (uint64_t i = (uint64_t)lane; i <= m; i += W) {
        Sarr[pc][i] = MIN_SCORE;
        Iarr[pc][i] = MIN_SCORE;
        Darr[pc][i] = MIN_SCORE;
      }
      C::sync();
      const uint64_t ps = rng[2 * (n - 1)], pe = rng[2 * (n - 1) + 1];
      const int32_t* lastcol = reinterpret_cast<const int32_t*>(ks_last);
      for (uint64_t i = umax64(1, ps) + (uint64_t)lane; i < umin64(pe, m); i += W) {
        const int32_t vs = lastcol[2 * i], vd = lastcol[2 * i + 1];
        Sarr[pc][i] = vs <= -(1 << 29) ? MIN_SCORE : vs >> 2;
        Darr[pc][i] = vd <= -(1 << 29) ? MIN_SCORE : vd >> 2;
      }
      if (lane == 0) {
        if (ps == 0 && pe > 0) Sarr[pc][0] = imax(row0_D(sc, (int32_t)n - 1), yp);
        Sarr[pc][m] = Sm_last;  // (lane 0 ran the row-m pass)
        Darr[pc][m] = Dm_last;
        const uint64_t en = rng[2 * n + 1];
        if (en < m) Sarr[n % 2][en] = MIN_SCORE;  // the row just below column n's band keeps its MIN_SCORE (689)
      }
      C::sync();
      lit_from = n;
    } else {
      lit_from = n + 1;
    }
  }
  if constexpr (FASTR <= 0) {  // the literal loop: every column, or (strip path) column n alone when it holds band cells
  uint32_t known_busy = 0;  // columns from here on already seen not to be of the plain kind
  for (uint64_t j = lit_from; j <= n; ++j) {  // banded.rs:511-681
    if (known_busy > 0) {
      known_busy -= 1;
    } else {
      // Columns without band cells (most of a long y) only store: S/I/D[i_start-1] = S[m] = MIN_SCORE, the
      // x-suffix-clip nibble of row m, and the MIN_SCORE reset ahead of the next column.  Nothing is read and
      // every array store writes the same constant, so a run of such columns is done one column per lane.
      // A column is taken here only if its successor is of the same kind (the reset then stays short).
      const uint64_t jc = j + (uint64_t)lane;
      bool plain = false;
      uint64_t c_start = 0, c_end = 0, c_to = 0;
      if (jc + 1 <= n) {
        c_start = rng[2 * jc];
        c_end = rng[2 * jc + 1];
        const uint64_t n_start = rng[2 * (jc + 1)], n_end = rng[2 * (jc + 1) + 1];
        plain = c_start >= 1 && c_start >= c_end && n_start >= 1 && n_start >= n_end;
        c_to = umin64(m + 1, n_end);
      }
      const uint32_t bal = C::ballot(plain);
      uint32_t run = 0;
      while (run < (uint32_t)W && ((bal >> run) & 1u)) ++run;
      if (run > 0) {
        if ((uint32_t)lane < run) {
          int32_t* S = Sarr[jc % 2];
          int32_t* I = Iarr[jc % 2];
          int32_t* D = Darr[jc % 2];
          S[c_start - 1] = MIN_SCORE;
          I[c_start - 1] = MIN_SCORE;
          D[c_start - 1] = MIN_SCORE;
          S[m] = MIN_SCORE;
          // S[m] + ys > Sn[m] cannot hold: S[m] is MIN_SCORE, ys <= 0 and Sn[m] never drops below MIN_SCORE
          if (c_end < m + 1) set_s(m, jc, TB_XCLIP_SUFFIX);
          for (uint64_t i = c_end; i < c_to; ++i) {
            S[i] = MIN_SCORE;
            I[i] = MIN_SCORE;
            D[i] = MIN_SCORE;
          }
        }
        C::sync();
        j += run - 1;
        continue;
      }
      // lanes 1.. looked at the columns after this one: skip the test while they were not plain either
      uint32_t ahead = 0;
      while (ahead + 1 < (uint32_t)W && !((bal >> (ahead + 1)) & 1u)) ++ahead;
      known_busy = ahead;
    }
    int32_t* S = Sarr[j % 2];
    int32_t* I = Iarr[j % 2];
    int32_t* D = Darr[j % 2];
    const int32_t* Sp = Sarr[1 - j % 2];
    const int32_t* Dp = Darr[1 - j % 2];
    const uint64_t i_start = rng[2 * j], i_end = rng[2 * j + 1];
    const bool last = j == n;
    if (lane == 0) {
      if (i_start == 0) {
        uint32_t db, sb;
        I[0] = MIN_SCORE;
        if (j == 1) {
          D[0] = go;
          db = TB_START;
        } else {
          const int32_t d_score = go + ge * ((int32_t)j - 1), c_score = yp + go;
          if (d_score > c_score) {
            D[0] = d_score;
            db = TB_DEL;
          } else {
            D[0] = c_score;
            db = TB_YCLIP_PREFIX;
          }
        }
        if (D[0] > yp) {
          S[0] = D[0];
          sb = TB_DEL;
        } else {
          S[0] = yp;
          sb = TB_YCLIP_PREFIX;
        }
        if (S[0] + ys > Sn[0]) {
          Sn[0] = S[0] + ys;
          Ly[0] = (uint32_t)(n - j);
          set_s(0, n, TB_YCLIP_SUFFIX);
        }
        put(0, j, (db << 4) | (sb << 8));
      }
      for (uint64_t i = sat_sub64(i_start, 1); i < i_start; ++i) {
        S[i] = MIN_SCORE;
        I[i] = MIN_SCORE;
        D[i] = MIN_SCORE;
      }
      S[m] = MIN_SCORE;
    }
    C::sync();
    const uint8_t q = y[j - 1];
    const int32_t xclip_score = xp + imax(last ? imax(yp, Sn[0]) : yp, go + ge * ((int32_t)j - 1));
    const uint64_t lo = umax64(1, i_start), hi = i_end, hi_main = umin64(hi, m);
    // values of row lo-1 in this column, handed from chunk to chunk (the same in every lane)
    int32_t cS = 0, cI = 0, cSn = 0;
    uint32_t csb = 0;
    int32_t trk_val = MIN_SCORE;  // the column tracker S[m] (banded.rs:645-649), rows < m
    uint64_t trk_i = 0;
    bool trk_hit = false;
    int32_t lane_trk_val = MIN_SCORE;  // this lane's best S + xs so far (updates only above MIN_SCORE matter)
    uint32_t lane_trk_i = 0;
    if (lo < hi) {
      cS = S[lo - 1];
      cI = I[lo - 1];
      cSn = Sn[lo - 1];
      csb = (rd(lo - 1, j) >> 8) & 15u;
      // geometry of column j-1 for the D-open lookups, and where this column's cells go, as base + 32-bit offset
      // (sequence lengths are below 2^24, so the row arithmetic of the chunk loop is 32-bit)
      const uint64_t jj = j - 1;
      const uint32_t ps = jj == 0 ? 0u : rng[2 * jj], pe = jj == 0 ? 0xFFFFFFFFu : rng[2 * jj + 1];
      const uint16_t* const pbase = jj == 0 ? col0 : cells;
      const uint32_t poff = (jj == 0 || STRIP || SCORES) ? 0u : colstart[jj] - ps;  // cell (i, j-1) = pbase[poff + i] for ps <= i < pe
      uint16_t* const wbase = last ? coln : cells;
      const uint32_t woff = (last || SCORES) ? 0u : colstart[j] - (uint32_t)i_start;  // cell (i, j) = wbase[woff + i]
      const uint32_t lo32 = (uint32_t)lo, hm32 = (uint32_t)hi_main;
      const int32_t ly_now = (int32_t)(n - j);
      for (uint32_t base = lo32; base < hm32; base += W) {
        const uint32_t i = base + (uint32_t)lane;
        const bool act = i < hm32;  // 1 <= i < m
        // lanes past the end of the column repeat its last row: every load stays in bounds, nothing is stored,
        // and nothing flows from a higher lane to a lower one
        const uint32_t ic = act ? i : hm32 - 1;
        const uint8_t p = x[ic - 1];
        const int32_t m_score = Sp[ic - 1] + score(p, q);
        const int32_t d_score = Dp[ic] + ge, s_open = Sp[ic] + go;
        const int32_t snold = Sn[ic];
        int32_t best_d;
        uint32_t db;
        if (d_score > s_open) {
          best_d = d_score;
          db = TB_DEL;
        } else {
          best_d = s_open;
          if ((STRIP || SCORES) && jj != 0) {  // (column n-1's interior cells live in the strip fill's 4-bit traceback)
            db = sbits_at(ic, jj);
          } else {
            const uint32_t pc = (ic >= ps && ic < pe) ? (uint32_t)pbase[poff + ic] : 0u;
            db = (pc >> 8) & 15u;
          }
        }
        const int32_t yclip_score = yp + go + ge * ((int32_t)ic - 1);
        const int32_t A = imax(imax(imax(MIN_SCORE, m_score), imax(best_d, xclip_score)), yclip_score);
        // prefix maximum of I(i) - gs*i over the chunk
        int32_t v;
        {
          const int32_t aprev = C::up(A, 1), snprev = C::up(snold, 1);
          if (lane == 0) {
            int32_t bi = imax(cI + ge, cS + go);
            if (last) bi = imax(bi, cSn + go);
            v = bi - gs * (int32_t)i;
          } else {
            v = (last ? imax(aprev, snprev) : aprev) + go - gs * (int32_t)i;
          }
          for (int d = 1; d < W; d <<= 1) {
            const int32_t t = C::up(v, d);
            if (lane >= d) v = imax(v, t);
          }
        }
        const int32_t best_i = v + gs * (int32_t)i;
        // S of the cell, literally (i < m: the running best starts at MIN_SCORE)
        int32_t best = MIN_SCORE;
        uint32_t sb = TB_START;
        if (m_score > best) {
          best = m_score;
          sb = (p == q) ? TB_MATCH : TB_SUBST;
        }
        if (best_i > best) {
          best = best_i;
          sb = TB_INS;
        }
        if (best_d > best) {
          best = best_d;
          sb = TB_DEL;
        }
        if (xclip_score > best) {
          best = xclip_score;
          sb = TB_XCLIP_PREFIX;
        }
        if (yclip_score > best) {
          best = yclip_score;
          sb = TB_YCLIP_PREFIX;
        }
        int32_t sncur = snold;
        if (act && best + ys > snold) {  // row tracker, banded.rs:650-654
          sncur = best + ys;
          Sn[i] = sncur;
          Ly[i] = (uint32_t)ly_now;
          if (!last) coln[i] = (uint16_t)((coln[i] & ~0x0F00u) | (TB_YCLIP_SUFFIX << 8));
        }
        // the I nibble needs the final values of row i-1
        int32_t pS = C::up(best, 1), pI = C::up(best_i, 1), pSn = C::up(sncur, 1);
        uint32_t psb = (uint32_t)C::up((int32_t)sb, 1);
        if (lane == 0) {
          pS = cS;
          pI = cI;
          pSn = cSn;
          psb = csb;
        }
        uint32_t ib;
        {
          const int32_t i_score = pI + ge, s_score = pS + go;
          int32_t bl;
          if (i_score > s_score) {
            bl = i_score;
            ib = TB_INS;
          } else {
            bl = s_score;
            ib = psb;
          }
          if (last && pSn + go > bl) ib = TB_YCLIP_SUFFIX;
        }
        if (act) {
          S[i] = best;
          I[i] = best_i;
          D[i] = best_d;
          if (!SCORES || last) wbase[woff + i] = (uint16_t)(ib | (db << 4) | (sb << 8));
          // column tracker, this lane's share: its rows come in ascending order, so a strict > keeps the first
          if (best + xs > lane_trk_val) {
            lane_trk_val = best + xs;
            lane_trk_i = i;
          }
        }
        const uint32_t left = hm32 - 1 - base;
        const int src = left < (uint32_t)(W - 1) ? (int)left : W - 1;
        cS = C::from(best, src);
        cI = C::from(best_i, src);
        cSn = C::from(sncur, src);
        csb = (uint32_t)C::from((int32_t)sb, src);
      }
    }
    if (lo < hi_main) {  // first row with the highest S + xs over all lanes (lowest row wins ties), once per column
      long long key = lane_trk_val > MIN_SCORE
                          ? (long long)((unsigned long long)(long long)lane_trk_val << 32) +
                                (long long)(0xFFFFFFFFu - lane_trk_i)
                          : (long long)0x8000000000000000ull;
      key = C::all_max(key);
      const int32_t bv = (int32_t)(key >> 32);
      if (key != (long long)0x8000000000000000ull && bv > trk_val) {
        trk_val = bv;
        trk_i = (uint64_t)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFll));
        trk_hit = true;
      }
    }
    if (lane == 0) {
      if (trk_hit) {
        S[m] = trk_val;
        Lx[j] = (uint32_t)(m - trk_i);
        set_s(m, j, TB_XCLIP_SUFFIX);
      }
      if (lo < hi && hi == m + 1) {  // the cell of row m: it starts from the column tracker
        const uint64_t i = m;
        const uint8_t p = x[i - 1];
        uint32_t ib, db, sb;
        const int32_t m_score = Sp[i - 1] + score(p, q);
        const int32_t i_score = cI + ge;
        int32_t s_score = cS + go;
        int32_t best_i;
        if (i_score > s_score) {
          best_i = i_score;
          ib = TB_INS;
        } else {
          best_i = s_score;
          ib = csb;
        }
        if (last) {
          const int32_t clip_score = cSn + go;
          if (clip_score > best_i) {
            best_i = clip_score;
            ib = TB_YCLIP_SUFFIX;
          }
        }
        const int32_t d_score = Dp[i] + ge;
        s_score = Sp[i] + go;
        int32_t best_d;
        if (d_score > s_score) {
          best_d = d_score;
          db = TB_DEL;
        } else {
          best_d = s_score;
          db = (rd(i, j - 1) >> 8) & 15u;
        }
        sb = TB_XCLIP_SUFFIX;
        int32_t best = S[i];
        if (m_score > best) {
          best = m_score;
          sb = (p == q) ? TB_MATCH : TB_SUBST;
        }
        if (best_i > best) {
          best = best_i;
          sb = TB_INS;
        }
        if (best_d > best) {
          best = best_d;
          sb = TB_DEL;
        }
        if (xclip_score > best) {
          best = xclip_score;
          sb = TB_XCLIP_PREFIX;
        }
        const int32_t yclip_score = yp + go + ge * ((int32_t)i - 1);
        if (yclip_score > best) {
          best = yclip_score;
          sb = TB_YCLIP_PREFIX;
        }
        S[i] = best;
        I[i] = best_i;
        D[i] = best_d;
        if (S[i] + xs > S[m]) {
          S[m] = S[i] + xs;
          Lx[j] = (uint32_t)(m - i);
          set_s(m, j, TB_XCLIP_SUFFIX);
        }
        if (S[i] + ys > Sn[i]) {
          Sn[i] = S[i] + ys;
          Ly[i] = (uint32_t)(n - j);
          set_s(i, n, TB_YCLIP_SUFFIX);
        }
        put(i, j, ib | (db << 4) | (sb << 8));
      }
      if (S[m] + ys > Sn[m]) {
        Sn[m] = S[m] + ys;
        Ly[m] = (uint32_t)(n - j);
        set_s(m, n, TB_YCLIP_SUFFIX);
      }
      if (i_end < m + 1) {
        set_s(m, j, TB_XCLIP_SUFFIX);
        S[m] = MIN_SCORE;
      }
    }
    C::sync();
    {
      const uint64_t to = umin64(m + 1, rng[2 * umin64(n, j + 1) + 1]);
      for (uint64_t i = i_end + (uint64_t)lane; i < to; i += W) {
        S[i] = MIN_SCORE;
        I[i] = MIN_SCORE;
        D[i] = MIN_SCORE;
      }
    }
    C::sync();
  }
  }  // literal column loop
  {
    // banded.rs:684-701.  Rows 0..m-1 are independent except for the running x-suffix-clip tracker S[m], which ends
    // as the first row (lowest index) holding the highest S[i] + xs, if that beats the value the loop started from;
    // row m comes last and sees the tracker's final value.
    int32_t* S = Sfin;
    const uint64_t bs = rng[2 * n], be = rng[2 * n + 1];
    int32_t bv = MIN_SCORE;
    uint32_t bi = 0;
    bool has = false;
    const int32_t Sm0 = S[m];
    C::sync();
    for (uint64_t i = (uint64_t)lane; i < m; i += W) {
      if (i < bs || i > be) S[i] = MIN_SCORE;
      if (Sn[i] > S[i]) {
        S[i] = Sn[i];
        set_s(i, n, TB_YCLIP_SUFFIX);
      }
      const int32_t v = S[i] + xs;
      if (v > Sm0 && (!has || v > bv)) {  // this lane's rows ascend: a strict > keeps its first maximum
        bv = v;
        bi = (uint32_t)i;
        has = true;
      }
    }
    long long key = has ? (long long)((unsigned long long)(long long)bv << 32) + (long long)(0xFFFFFFFFu - bi)
                        : (long long)0x8000000000000000ull;
    key = C::all_max(key);
    C::sync();
    if (lane == 0) {
      if (key != (long long)0x8000000000000000ull) {
        S[m] = (int32_t)(key >> 32);
        Lx[n] = (uint32_t)(m - (uint64_t)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFll)));
        set_s(m, n, TB_XCLIP_SUFFIX);
      }
      if (Sn[m] > S[m]) {  // i == m (S[m] + xs > S[m] cannot hold: xs <= 0)
        S[m] = Sn[m];
        set_s(m, n, TB_YCLIP_SUFFIX);
      }
    }
    C::sync();
  }
  if (lane == 0) {
    int32_t* S = Sfin;
    int32_t* I = Iarr[n % 2];
    const uint64_t bs = rng[2 * n], be = rng[2 * n + 1];
    for (uint64_t i = umax64(1, bs); i < be; ++i) {  // banded.rs:705-723
      const int32_t s_score = S[i - 1] + go;
      if (s_score > I[i]) {
        I[i] = s_score;
        set_i(i, n, (rd(i - 1, n) >> 8) & 15u);
      }
      if (s_score > S[i]) {
        S[i] = s_score;
        set_s(i, n, TB_INS);
        if (S[i] + xs > S[m]) {
          S[m] = S[i] + xs;
          Lx[n] = (uint32_t)(m - i);
          set_s(m, n, TB_XCLIP_SUFFIX);
        }
      }
    }
  }
  C::sync();
  // the two closed-form border passes (banded.rs:725-765) touch one traceback cell per index, except at
  // the far corner (j = n, i = m), which lane 0 does afterwards
  if (!STRIP)  // (the strip path's initialisation has written row 0's final cells)
    for (uint64_t j = 1 + (uint64_t)lane; j < n; j += W) {
      const int32_t d_score = go + ge * ((int32_t)j - 1);
      set_s(0, j, d_score > yp ? TB_DEL : TB_YCLIP_PREFIX);
    }
  for (uint64_t i = 1 + (uint64_t)lane; i < m; i += W) {
    const int32_t c_score = go + ge * ((int32_t)i - 1);
    set_s(i, 0, c_score > xp ? TB_INS : TB_XCLIP_PREFIX);
  }
  C::sync();
  if (lane == 0) {
    int32_t* S = Sfin;
    if (n >= 1) {  // banded.rs:725-744, j = n
      const uint64_t j = n;
      const int32_t d_score = go + ge * ((int32_t)j - 1);
      set_s(0, j, d_score > yp ? TB_DEL : TB_YCLIP_PREFIX);
      int32_t best_score = imax(d_score, yp);
      if (ys > best_score) {
        best_score = ys;
        set_s(0, j, TB_YCLIP_SUFFIX);
      }
      if (xs + best_score > S[m]) {
        S[m] = xs + best_score;
        Lx[n] = (uint32_t)m;
        set_s(m, n, TB_XCLIP_SUFFIX);
      }
    }
    if (m >= 1) {  // banded.rs:746-765, i = m
      const uint64_t i = m;
      const int32_t c_score = go + ge * ((int32_t)i - 1);
      set_s(i, 0, c_score > xp ? TB_INS : TB_XCLIP_PREFIX);
      int32_t best_score = imax(c_score, xp);
      if (xs > best_score) {
        best_score = xs;
        set_s(i, 0, TB_XCLIP_SUFFIX);
      }
      if (ys + best_score > S[m]) {
        S[m] = ys + best_score;
        Ly[m] = (uint32_t)n;
        set_s(m, n, TB_YCLIP_SUFFIX);
      }
    }
    out.score = S[m];
  }
  } else {
    out.score = Sfin[m];
  }
  if (lane != 0) return;
  if (STRIP && PHASE != 2 && out.score < -(1 << 27)) {  // not a real score: the sentinel arithmetic does not cover it -- literal kernel
    *redo = true;
    return;
  }
  if (PHASE == 1) return;
  // walk, banded.rs:767-855 (ops written backwards).  A legitimate walk emits at most m + n + 4 ops; the
  // reference can loop forever on some custom clip settings (an Xclip/Yclip of length 0): that is
  // reported as status 1 instead of hanging.
  uint64_t i = m, j = n;
  uint32_t xstart = 0, ystart = 0, xend = (uint32_t)m, yend = (uint32_t)n;
  uint32_t nops = 0, nclip = 0, clips[4] = {0, 0, 0, 0};
  const uint64_t ops_cap = m + n + 4;
  bool overflow = false;
  auto push = [&](uint32_t code) {  // (SCORES: counted, not stored -- an overflow is still the reference's panic)
    if (nops >= ops_cap) {
      overflow = true;
      return;
    }
    if (!SCORES) *(--ops_end) = (uint8_t)code;
    ++nops;
  };
  auto push_clip = [&](uint32_t code, uint32_t len) {
    if (!filter_clips) {
      push(code);
      if (nclip < 4) clips[nclip] = len;
      ++nclip;
    }
  };
  uint32_t layer = rd_part(i, j, 2);
  uint64_t guard = 4 * (m + n) + 64;
  // STRIP: runs of Match / Subst / Ins / Del moves between interior band cells -- nearly the whole path -- in 32-bit
  // arithmetic with the strip's table entry cached and ONE traceback load per move: the nibble of the cell moved to
  // also answers that cell's own "from extension" question on the next move.  Anything else (a border, a clip, a
  // cell outside the band, the op budget) leaves the run before the move is made; the general step below does it.
  uint32_t ks_cst = 0xFFFFFFFFu, ks_cja = 0, ks_coff = 0, ks_csteps = 0;
  // (the traceback word is requested before the band check is known -- its address does not depend on it -- so the
  //  two loads of a move overlap instead of following each other; the strip table's step count keeps it in bounds)
  auto nib32 = [&](int32_t ii, int32_t jj) -> uint32_t {
    const uint32_t st = (uint32_t)(ii - 1) >> KS_ROWS_LOG2, rem = (uint32_t)(ii - 1) & (uint32_t)(KS_ROWS - 1),
                   l = rem >> KS_R_LOG2, r = rem & (uint32_t)(KS_R - 1);
    if (st != ks_cst) {
      ks_cst = st;
      ks_cja = ks_tab[KS_TAB * st];
      ks_coff = ks_tab[KS_TAB * st + 1];
      ks_csteps = ks_tab[KS_TAB * st + 2];
    }
    const uint32_t t = (uint32_t)jj - ks_cja + l;
    const uint32_t tc = t < ks_csteps ? t : 0u;
    const uint32_t word = ks_tb[(ks_coff + ((tc >> 3) * (uint32_t)KS_TBW + (r >> 2)) * (uint32_t)KS_G + l) * 4u + (r & 3u)];
    const uint32_t bs = rng[2 * jj], be = rng[2 * jj + 1];
    if (!((uint32_t)ii >= bs && (uint32_t)ii < be)) return 16u;
    return (word >> (4u * (7u - (t & 7u)))) & 15u;
  };
  bool interior = false;  // SCORES: the walk stopped on a cell with i < m and j < n
  while (layer != TB_START) {
    if (SCORES && i < m && j < n) {
      interior = true;
      break;
    }
    if (guard-- == 0 || overflow) {
      out.status = 1;
      break;
    }
    if (!SCORES && STRIP && i >= 1 && i < m && j >= 1 && j < n &&
        (layer == TB_INS || layer == TB_DEL || layer == TB_MATCH || layer == TB_SUBST)) {
      int32_t fi = (int32_t)i, fj = (int32_t)j;
      uint32_t nbc = nib32(fi, fj);
      bool moved = false;
      while (nbc != 16u && nops < ops_cap && guard > 0) {
        uint32_t code, nl = 0;
        int32_t ti = fi, tj = fj;
        bool known = false;
        if (layer == TB_INS) {
          code = 3;
          ti = fi - 1;
          if (nbc & NB_IEXT) {
            nl = TB_INS;
            known = true;
          }
        } else if (layer == TB_DEL) {
          code = 2;
          tj = fj - 1;
          if (nbc & NB_DEXT) {
            nl = TB_DEL;
            known = true;
          }
        } else if (layer == TB_MATCH || layer == TB_SUBST) {
          code = layer == TB_MATCH ? 0u : 1u;
          ti = fi - 1;
          tj = fj - 1;
        } else {
          break;
        }
        if (ti < 1 || tj < 1) break;  // the move lands on row 0 / column 0
#if defined(__CUDA_ARCH__)
        // One pair per lane: a move's loads are 32 different lines per warp, and the traceback word changes line
        // every few moves, so without help nearly every move waits for some lane's miss.  The path mostly runs
        // down the diagonal: the lines of the cell a few moves ahead are requested now.
        {
          constexpr int32_t kAhead = 12;
          const int32_t pi = ti - kAhead, pj = tj - kAhead;
          if (pi >= 1 && pj >= 1) {
            const uint32_t pst = (uint32_t)(pi - 1) >> KS_ROWS_LOG2, prem = (uint32_t)(pi - 1) & (uint32_t)(KS_ROWS - 1),
                           pl = prem >> KS_R_LOG2, pr = prem & (uint32_t)(KS_R - 1);
            if (pst == ks_cst) {  // (a strip change ahead: its table entry is not at hand, skip)
              const uint32_t pt = (uint32_t)pj - ks_cja + pl;
              if (pt < ks_csteps)
                asm volatile("prefetch.global.L1 [%0];" ::"l"(
                    ks_tb + ((size_t)(ks_coff + ((pt >> 3) * (uint32_t)KS_TBW + (pr >> 2)) * (uint32_t)KS_G + pl) * 4u + (pr & 3u))));
            }
            asm volatile("prefetch.global.L1 [%0];" ::"l"(rng + 2 * (size_t)pj));
          }
        }
#endif
        const uint32_t nbn = nib32(ti, tj);
        if (nbn == 16u) break;        // ... or outside the band (reads as START there)
        if (!known) nl = ks_sbits((uint64_t)ti, (uint64_t)tj, nbn);
        *(--ops_end) = (uint8_t)code;
        ++nops;
        --guard;
        fi = ti;
        fj = tj;
        nbc = nbn;
        layer = nl;
        moved = true;
      }
      i = (uint64_t)fi;
      j = (uint64_t)fj;
      if (moved) {
        ++guard;  // the general loop's own decrement above stood for one of the moves
        continue;
      }
    }
    uint32_t next;
    if (layer == TB_INS) {
      push(3);
      next = rd_part(i, j, 0);
      if (i == 0) { out.status = 1; break; }
      i -= 1;
    } else if (layer == TB_DEL) {
      push(2);
      next = rd_part(i, j, 1);
      if (j == 0) { out.status = 1; break; }
      j -= 1;
    } else if (layer == TB_MATCH || layer == TB_SUBST) {
      push(layer == TB_MATCH ? 0 : 1);
      if (i == 0 || j == 0) { out.status = 1; break; }
      next = rd_part(i - 1, j - 1, 2);
      i -= 1;
      j -= 1;
    } else if (layer == TB_XCLIP_PREFIX) {
      push_clip(4, (uint32_t)i);
      xstart = (uint32_t)i;
      i = 0;
      next = rd_part(0, j, 2);
    } else if (layer == TB_XCLIP_SUFFIX) {
      push_clip(4, Lx[j]);
      if (Lx[j] > i) { out.status = 1; break; }
      i -= Lx[j];
      xend = (uint32_t)i;
      next = rd_part(i, j, 2);
    } else if (layer == TB_YCLIP_PREFIX) {
      push_clip(5, (uint32_t)j);
      ystart = (uint32_t)j;
      j = 0;
      next = rd_part(i, 0, 2);
    } else if (layer == TB_YCLIP_SUFFIX) {
      push_clip(5, Ly[i]);
      if (Ly[i] > j) { out.status = 1; break; }
      j -= Ly[i];
      yend = (uint32_t)j;
      next = rd_part(i, j, 2);
    } else {
      out.status = 1;
      break;
    }
    layer = next;
  }
  if (out.status == 0 && !interior) {
    if (i != 0) {  // banded.rs:834-844
      const int32_t i_score = go + ge * ((int32_t)i - 1);
      if (i_score > xp) {
        for (uint64_t t = 0; t < i; ++t) push(3);
        xstart = 0;
      } else {
        push_clip(4, (uint32_t)i);
        xstart = (uint32_t)i;
      }
    }
    if (j != 0) {  // banded.rs:845-855
      const int32_t d_score = go + ge * ((int32_t)j - 1);
      if (d_score > yp) {
        for (uint64_t t = 0; t < j; ++t) push(2);
        ystart = 0;
      } else {
        push_clip(5, (uint32_t)j);
        ystart = (uint32_t)j;
      }
    }
  }
  if (overflow) out.status = 1;
  if (nclip > 4) out.status = 1;
  out.xend = xend;
  out.yend = yend;
  out.xstart = SCORES ? 0u : xstart;
  out.ystart = SCORES ? 0u : ystart;
  if (SCORES) return;  // (ops and clip lengths stay 0)
  out.n_ops = nops;
  const uint32_t nc = nclip > 4 ? 4 : nclip;
  for (uint32_t q = 0; q < 4; ++q) out.clip[q] = q < nc ? clips[nc - 1 - q] : 0u;
}

#if defined(__CUDACC__) && !defined(B2A_BANDED_NO_KERNELS)  // (b2a_banded_strip_notb.cu: the device functions only)

// K4: one warp per pair
__global__ void __launch_bounds__(128) band_kernel(const BandedParams prm, uint32_t n_wave) {
  __shared__ uint32_t shared_u32[4][K4_SHARED_WORDS];
  const uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = (int)(threadIdx.x & 31u);
  if (t >= n_wave) return;
  const uint64_t p = (uint64_t)prm.pair_lo + t;
  const uint64_t m = prm.x_len[p], n = prm.y_len[p];
  uint64_t cells = 0;
  BandHintsD hint;
  if (prm.hint_match_off) {
    hint.mxy = prm.hint_match_xy + 2 * prm.hint_match_off[p];
    hint.n_matches = prm.hint_match_off[p + 1] - prm.hint_match_off[p];
  }
  if (prm.hint_path_off) {
    hint.pidx = prm.hint_path_idx + prm.hint_path_off[p];
    hint.n_path = prm.hint_path_off[p + 1] - prm.hint_path_off[p];
    hint.have_path = true;
  }
  hint.allowed_mismatches = prm.allowed_mismatches;
  hint.use_lcskpp_union = prm.use_lcskpp_union;
  uint32_t touched[2] = {0u, 0xFFFFFFFFu};  // (whole range, unless the band construction says less)
  const uint32_t st = band_create_d<32>(lane, prm.blob + prm.x_off[p], m, prm.blob + prm.y_off[p], n, prm.k, prm.w,
                                        prm.sc, prm.has_match_scores, prm.slab + (uint64_t)t * prm.slab_stride,
                                        prm.cap_matches, prm.ranges + prm.ranges_off[t] / 4, &cells,
                                        shared_u32[threadIdx.x >> 5], hint, touched);
  // pairs whose band suits the register-resident K3 loop are marked (bit 8) while the ranges are still hot
  const bool fast = st == 0 && cells <= BANDED_MAX_CELLS &&
                    banded_fast_ok<32, K3_FAST_ROWS>(lane, prm.ranges + prm.ranges_off[t] / 4, m, n, touched[0], touched[1]);
  uint32_t cols3[3] = {0, 0, 0};
  const bool strip = prm.strip_ok && st == 0 && cells <= BANDED_MAX_CELLS &&
                     banded_strip_ok<32>(lane, prm.ranges + prm.ranges_off[t] / 4, m, n, cols3, touched[0], touched[1],
                                         (prm.strip_ok & 2) != 0);
  if (lane != 0) return;
  prm.num_cells[p] = cells;
  prm.k4_status[p] = st | (fast ? 0x100u : 0u) | (strip ? 0x200u : 0u);
  if (prm.band_cols) {
    prm.band_cols[3 * p] = cols3[0];
    prm.band_cols[3 * p + 1] = cols3[1];
    prm.band_cols[3 * p + 2] = cols3[2];
  }
}

#ifndef B2A_K3_MINB
#define B2A_K3_MINB 8  // resident CTAs per SM asked of ptxas for K3 (latency-bound: more warps win)
#endif
// K3: one warp per pair.  FASTR == 0: the literal column loop, for every pair K4 did not mark; FASTR > 0: the
// register-resident loop, for the marked ones (each kernel skips the other's pairs).
// SCORES: a score-only call (banded_compute_d): score, xend, yend and status only; prm.ops_scratch may be null.
template <int FASTR, int PHASE = 0, int W = 32, bool SCORES = false>
__device__ __forceinline__ void banded_fill_body(const BandedParams& prm, uint32_t n_wave) {
  // W = 32: one warp per pair; W = 1 (the strip path's walk): one thread per pair
  const uint32_t t = W == 32 ? (blockIdx.x * blockDim.x + threadIdx.x) >> 5 : blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = W == 32 ? (int)(threadIdx.x & 31u) : 0;
  if (t >= n_wave) return;
  const uint64_t p = (uint64_t)prm.pair_lo + t;
  const uint64_t m = prm.x_len[p], n = prm.y_len[p];
  BandedOut o;
  const uint32_t k4raw = prm.k4_status[p];
  const uint32_t k4 = k4raw & 0xFFu;
  // bit 8: K4 marked the pair for the register-resident loop, bit 9: for the strip-wavefront fill, bit 10: the strip
  // path handed it back.  The strip kernels take 9 & !10; the column-loop kernels take the unmarked pairs (beside the
  // strip kernels, on a stream of their own) or, in a later pass, the pairs handed back.
  const bool strip_pair = (k4raw & 0x200u) && !(k4raw & 0x400u);
  if (FASTR < 0) {
    if (!strip_pair) return;
  } else {
    if (prm.redo_pass ? (k4raw & 0x600u) != 0x600u : (k4raw & 0x200u) != 0u) return;
    if (((k4raw >> 8) & 1u) != (FASTR > 0 ? 1u : 0u)) return;  // the other kernel's pair
  }
  bool redo = false;
  if (k4 != 0) {
    o = BandedOut{};
    o.status = 1 + k4;
  } else {
    const uint8_t* cm = prm.codemap;
    const int32_t* lut = prm.lut;
    const int32_t alpha = prm.sc.alpha;
    const DevScoring sc = prm.sc;
    uint32_t* err = prm.err_flag;
    auto score = [=](uint8_t a, uint8_t b) -> int32_t {
      if (alpha) {
        int32_t ca = cm[a], cb = cm[b];
        if (ca == 0xFF || cb == 0xFF) {  // byte outside the scoring alphabet: flag, stay in bounds
          atomicOr(err, 4u);
          ca = cb = 0;
        }
        return lut[ca * alpha + cb];
      }
      return a == b ? sc.match_score : sc.mismatch_score;
    };
    banded_compute_d<W, decltype(score), FASTR, PHASE, SCORES>(lane, prm.blob + prm.x_off[p], m, prm.blob + prm.y_off[p], n,
                                                       prm.sc, score, prm.ranges + prm.ranges_off[t] / 4, prm.num_cells[p],
                                                       prm.fill + prm.fill_off[t], prm.filter_clips != 0,
                                                       SCORES ? nullptr : prm.ops_scratch + prm.ops_off[p], o,
                                                       FASTR < 0 ? prm.strip + prm.strip_off[t] : nullptr,
                                                       FASTR < 0 ? prm.band_cols + 3 * p : nullptr, &redo);
  }
  if (lane != 0) return;
  if (FASTR < 0 && (redo || o.status)) {  // outside what the strip path covers: the column-loop kernels' later pass takes it
    prm.k4_status[p] = k4raw | 0x400u;
    return;
  }
  if (PHASE == 1) return;  // the walk (its own kernel) reports the pair
  if (o.status) {  // no alignment is reported for a pair the reference panics / hangs on (or that hit a capacity)
    o.score = MIN_SCORE;
    o.n_ops = 0;
    o.xstart = o.xend = o.ystart = o.yend = 0;
    o.clip[0] = o.clip[1] = o.clip[2] = o.clip[3] = 0;
  }
  prm.score[p] = o.score;
  if (!SCORES) prm.xstart[p] = o.xstart;
  prm.xend[p] = o.xend;
  if (!SCORES) prm.ystart[p] = o.ystart;
  prm.yend[p] = o.yend;
  if (!SCORES) {
    prm.n_ops[p] = o.n_ops;
    prm.ops_src[p] = prm.ops_off[p] - o.n_ops;
  }
  prm.status[p] = o.status;
  if (o.status) atomicOr(prm.err_flag, o.status == 2 ? 2u : (o.status == 4 ? 8u : 1u));
  if (!SCORES)
    for (int q = 0; q < 4; ++q) prm.clip_len[4 * p + q] = o.clip[q];
}

__global__ void __launch_bounds__(128, B2A_K3_MINB) banded_fill_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<0>(prm, n_wave);
}
__global__ void __launch_bounds__(128, 4) banded_fill_fast_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<K3_FAST_ROWS>(prm, n_wave);
}
__global__ void __launch_bounds__(128, 8) banded_strip_finish_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<-1, 1>(prm, n_wave);
}
__global__ void __launch_bounds__(128) banded_strip_walk_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<-1, 2, 1>(prm, n_wave);  // one pair per thread
}
// the score-only twins.  The strip path keeps its walk kernel (one pair per thread) after the finish pass: measured
// against a finish pass that walks on lane 0 itself, it took slightly less K3 time (DESIGN.md §4)
__global__ void __launch_bounds__(128, B2A_K3_MINB) banded_fill_scores_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<0, 0, 32, true>(prm, n_wave);
}
__global__ void __launch_bounds__(128, 4) banded_fill_fast_scores_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<K3_FAST_ROWS, 0, 32, true>(prm, n_wave);
}
__global__ void __launch_bounds__(128, 8) banded_strip_finish_scores_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<-1, 1, 32, true>(prm, n_wave);
}
__global__ void __launch_bounds__(128) banded_strip_walk_scores_kernel(const BandedParams prm, uint32_t n_wave) {
  banded_fill_body<-1, 2, 1, true>(prm, n_wave);  // one pair per thread
}

#endif

}  // namespace b2a
