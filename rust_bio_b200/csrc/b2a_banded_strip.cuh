// K3s: the banded DP fill as a row-strip wavefront with K1's packed cell (b2a_fill.cuh), for the pairs K4
// marks strip-eligible.
//
// Reference: rust-bio 4.0.1 src/alignment/pairwise/banded.rs, compute_alignment's hot loop 511-681 for the
// interior cells 1 <= i <= m-1, 1 <= j <= n-1 of the band.  What the literal / register-resident K3 loops
// (b2a_banded.cuh) pay per cell -- ~75 instructions of strict-comparison chains plus ~300 per column of uniform
// work -- this kernel does with the fill's ~20-instruction packed cell (DPX add-max chains, one 3-way max that
// yields the score and its source, 4-bit traceback) plus a band mask:
//   * lanes own FIXED rows: 8 lanes x KS_R rows (16: strips of 128 rows), four pairs to a warp; a strip sweeps only the
//     columns where the band meets its rows ([ja, jb], found by two binary searches: the band's starts and ends
//     do not decrease), lane l one column behind lane l-1, the vertical I chain handed down by warp shuffle;
//   * a cell outside the band is computed like any other and then its S is FORCED to the sentinel (NEG4),
//     which is what the reference reads there for an eligible band: every value outside the previous column's
//     band is MIN_SCORE (rows below were reset 676-680, the row above was set 556-561, the band never moves up or
//     shrinks, empty columns are Band::new sentinels).  The sentinel is not MIN_SCORE itself but it orders the same:
//     with every real score within +-2^26 (engine guard), a value derived from a sentinel stays below every real
//     one, so wherever a real candidate exists the same candidate wins with the same strict-comparison order, and
//     a walked cell only ever holds real values (a real S/I/D has a real winning predecessor, by induction from the
//     final score).  Cells whose value is sentinel-derived may pick a different source than the reference's
//     MIN_SCORE arithmetic would -- unobservable, unless the final score itself is not real: the finish pass
//     (banded_compute_d, STRIP mode) detects that and hands the pair to the literal kernel;
//   * the y-prefix clip term yclip_score(i) (636-642) is live in a band (row 0 need not be above a cell): it shares
//     priority code 0 with the x-prefix clip term; which of the two it was is re-derived at walk time (the
//     x clip wins ties: it is tested first, 631-642);
//   * row trackers Sn/Ly (655-660) as packed keys 4096*S + (4095 - column offset in the strip's window), first
//     column wins ties; the eager s-bit write of (i, n) becomes one store at the end of the strip;
//   * row 0, column 0, row m (which starts from the column tracker), column n (the literal loop, on the S / D of
//     column n-1 this kernel exports), the end-of-matrix passes and the walk stay in the finish pass; this kernel
//     leaves it the boundary row m-1 (S, I, column tracker per column), Sn/Ly, the (i, n) marks, the per-strip
//     windows and the 4-bit traceback.
//   * the column tracker S[m] / Lx (648-653, live with the x-suffix clip: local mode) as K1's packed key
//     4096*S + (4095 - row), handed down the lanes and through the boundary row; it needs x no longer than 4,095;
//   * substitution scores by MatchParams compare / select, or (F_LUT: a tabulated MatchFunc such as BLOSUM62) from
//     K1's scaled LUT in shared memory with the sequence bytes mapped to LUT codes as they are loaded;
// Not handled here (K4 / the host do not mark such pairs): trackers when the y-prefix clip is dead, scores exceed
// 2^17 or (column tracker) x is longer than 4,095, gaps inside the band's column range.
#pragma once
#include "b2a_banded.cuh"
#include "b2a_fill.cuh"

namespace b2a {

enum : int { F_CLIPY = 64 };  // y-prefix clip live (with F_CLIPX / F_TRACK_ROWS of b2a_common.cuh)

// per-pair strip area: [strip table: nstrips x {ja, traceback offset in uint4 units, steps stored, 0}][boundary row: (cols+2) x int4 {4S, 4I+2, column-tracker key, 0}][traceback]
struct KsLayout {
  uint64_t tab, bnd, last, tb, total;
};
B2A_HD uint32_t ks_nstrips(uint64_t m) { return m >= 2 ? (uint32_t)((m - 1 + KS_ROWS - 1) / KS_ROWS) : 0u; }
// score_only: the area of a score-only call (F_NOTB fill), without the traceback region
B2A_HD KsLayout ks_layout(uint64_t m, uint64_t band_cols, uint64_t strip_cols, bool score_only = false) {
  KsLayout L;
  const uint64_t ns = ks_nstrips(m);
  uint64_t b = 0;
  L.tab = b; b = al16(b + ns * KS_TAB * 4);
  L.bnd = b; b = al16(b + (band_cols + 2) * 16);
  L.last = b; b = al16(b + (m + 1) * 8);  // column n-1's {4S, D} per row, when column n holds band cells
  L.tb = b;
  // a strip of `len` columns stores ceil((len + 14) / 8) groups of 8 steps, KS_TBW x KS_G uint4 each
  if (!score_only) b += (strip_cols / 8 + 3 * ns) * (uint64_t)(KS_TBW * KS_G * 16);
  L.total = (b + 255) & ~255ull;
  return L;
}

struct StripParams {
  const uint8_t* blob;
  const uint64_t* x_off;
  const uint32_t* x_len;
  const uint64_t* y_off;
  const uint32_t* y_len;
  uint32_t pair_lo;            // first pair of the sub-wave
  const uint32_t* elig;        // [n_elig] sub-wave-local indices of the strip-eligible pairs
  uint32_t n_elig;
  uint32_t* task_counter;
  const uint32_t* ranges;
  const uint64_t* ranges_off;  // per sub-wave-local pair
  uint8_t* fill;               // K3 slabs (Sn / Ly / coln live there)
  const uint64_t* fill_off;
  uint8_t* strip;              // strip areas
  const uint64_t* strip_off;   // per sub-wave-local pair
  const uint64_t* num_cells;   // per pair (batch index)
  const uint32_t* band_cols;   // per pair (batch index): {first, last non-empty column, strip columns}
  uint32_t* k4_status;         // per pair (batch index): bit 10 = hand the pair to the literal kernel
  const int32_t* lut;          // tabulated MatchFunc (F_LUT): K1's scaled LUT 4*score + 3 - (4*gap_open + 1), sc.alpha^2 entries
  const uint8_t* codemap;      // byte -> LUT code, 0xFF = not in the scoring alphabet
  uint32_t* err_flag;          // bit 2: a sequence byte outside the scoring alphabet
  DevScoring sc;
  int32_t one, ge4;            // opaque 1 and 4 * gap_extend (see b2a_fill.cuh)
  int32_t flags;
};

#if defined(__CUDA_ARCH__)
#define KS_SHFL(v, src) __shfl_sync(0xffffffffu, (v), (src), KS_G)
#elif defined(B2A_HOST_WARP) && !defined(__CUDACC__)
inline int32_t host_shfl_group(int32_t v, int src, int G) {
  if (!host_warp) return v;
  const int me = host_lane;
  return (int32_t)host_warp_exchange(v, [&](const long long* x) { return x[(me / G) * G + (src % G)]; });
}
#define KS_SHFL(v, src) host_shfl_group((v), (src), KS_G)
#else
#define KS_SHFL(v, src) (v)
#endif

B2A_HD int32_t ks_warp_max(int32_t v) {
#if defined(__CUDA_ARCH__)
  return __reduce_max_sync(0xffffffffu, v);
#elif defined(B2A_HOST_WARP) && !defined(__CUDACC__)
  if (!host_warp) return v;
  return (int32_t)host_warp_exchange(v, [&](const long long* x) {
    long long t = x[0];
    for (int l = 1; l < 32; ++l) t = x[l] > t ? x[l] : t;
    return t;
  });
#else
  return v;
#endif
}

// what one lane group (8 lanes) knows about its pair
struct KsPair {
  const uint8_t* x;
  const uint8_t* y;
  const uint32_t* rng;
  int32_t m, n;       // m == 0: no pair in this slot
  int32_t c0, c1;     // first / last non-empty band column, clipped to [1, n-1]
  int32_t* Sn;
  uint32_t* Ly;
  uint16_t* coln;
  uint32_t* tab;      // strip table
  int4* bnd;          // boundary row, indexed by j - c0 + 1
  int2* last;         // column n-1's {4S, D} per row (written when the strip's window ends at column n-1)
  uint4* tb;
};

// scoring tables of a task (F_LUT): shared memory on the device, plain memory in the host build
struct KsLut {
  const int32_t* lut;     // host build: base of the scaled LUT
  uint32_t lut_base;      // device: shared-space byte address of the LUT (0 in the host build)
  const uint8_t* cmap;    // byte -> code
  uint32_t* err_flag;
};

template <int FLAGS, bool LASTSTRIP>
B2A_HD void ks_column_step(const DevScoring& sc, const KsLut& T, const int32_t one, const int32_t ge4, const int32_t j, const int32_t q,
                           const int32_t a_band, const uint32_t h_band, const int32_t cjkey, const int32_t y4_first,
                           int32_t (&Sp)[KS_R], int32_t (&Dp)[KS_R], int32_t (&SnR)[KS_R], uint32_t (&tbacc)[KS_R],
                           const int32_t (&xc)[KS_R], const int32_t sdiag, int32_t& sup, int32_t& iup, int32_t& Tv,
                           const int32_t rowbase, const int32_t cap_row, int32_t& cap_s, int32_t& cap_i) {
  constexpr bool TR = (FLAGS & F_TRACK_ROWS) != 0;
  constexpr bool TC = (FLAGS & F_TRACK_COLS) != 0;
  constexpr bool CX = (FLAGS & F_CLIPX) != 0;
  constexpr bool CY = (FLAGS & F_CLIPY) != 0;
  constexpr bool LUT = (FLAGS & F_LUT) != 0;
  constexpr bool NOTB = (FLAGS & F_NOTB) != 0;
  const int32_t go4i = 4 * sc.gap_open + 2, go4d = 4 * sc.gap_open + 1;
  const int32_t ma4 = 4 * sc.match_score + 3 - go4d, mi4 = 4 * sc.mismatch_score + 3 - go4d;
  const int32_t x4 = CX ? scale4(xclip_score(sc, j)) : NEG4;
  const int32_t k2 = one + one, k16 = k2 * 8, k1024 = k16 * 64;
  int32_t sdo = fmad(sdiag, one, go4d);
  int32_t iop = fmad(sup, one, go4i);
  int32_t s4 = sup;
  int32_t Tl = KEY_NONE;  // packed column tracker of this lane's band rows (local row index), as in K1
#pragma unroll
  for (int r = 0; r < KS_R; ++r) {
    // LUT: xc[r] is the byte address of the row symbol's LUT row, q the column symbol's byte offset inside a row
    const int32_t sub4 = LUT ? lut_at(T.lut, (uint32_t)fmad(q, one, xc[r])) : ((xc[r] == q) ? ma4 : mi4);
    const int32_t m4 = fmad(sdo, one, sub4);
    int32_t i4 = addmax(iup, ge4, iop);
    const int32_t dop = Sp[r];
    int32_t d4 = addmax(Dp[r], ge4, dop);
    int32_t sP = max3(m4, i4, d4);
    if (CX && CY) sP = max3(sP, x4, fmad(ge4, r, y4_first));
    else if (CY) sP = imax(sP, fmad(ge4, r, y4_first));
    else if (CX) sP = imax(sP, x4);
    s4 = sP & ~3;
    if (!NOTB) {
      const int32_t fi = addmin(i4, -iop, 4), fd = addmin(d4, -dop, 4);
      tbacc[r] = (uint32_t)(fmad((int32_t)tbacc[r], k16, fmad(fd, k2, fi)) + sP - s4);
    }
    // Outside the band S is forced to the sentinel (what the reference reads there is MIN_SCORE).  I and D need no
    // forcing: a column's band rows are one run and so are a row's band columns (starts and ends never decrease), so
    // neither chain re-enters the band once it has left it -- above the band I derives from the sentinel top and a
    // forced S only; below it D does; and what the other chain carries there (a real value decayed by extensions)
    // is never read by a band cell.
    const bool inb = (uint32_t)(a_band + r) < h_band;
    if (!inb) s4 = NEG4;
    if (TR) {
      if (inb) SnR[r] = imax(SnR[r], fmad(s4, k1024, cjkey));
    }
    if (TC) {  // banded.rs:648-653: the first band row with the highest S + xs
      if (inb) Tl = imax(Tl, fmad(s4, k1024, 4095 - r));
    }
    if (LASTSTRIP) {
      if (r == cap_row) {
        cap_s = s4;
        cap_i = i4;
      }
    }
    sdo = dop;
    Sp[r] = fmad(s4, one, go4d);
    iop = fmad(s4, one, go4i);
    Dp[r] = d4;
    iup = i4;
  }
  sup = s4;
  if (TC) {
    if (Tl != KEY_NONE) Tv = imax(Tv, Tl - (rowbase + 1));  // local row index -> 4095 - i
  }
}

// S(0, j) of the banded aligner for 1 <= j < n (banded.rs:523-545), scaled; row 0 has to be in the band there
B2A_HD int32_t ks_row0_S4(const DevScoring& sc, int32_t j) { return 4 * imax(row0_D(sc, j), sc.yclip_prefix); }

// first column in [lo, hi] whose band END exceeds `row` (ends do not decrease over the band's columns); hi + 1 if none
B2A_HD int32_t ks_first_col_end_above(const uint32_t* rng, int32_t lo, int32_t hi, int32_t row) {
  int32_t a = lo, b = hi + 1;
  while (a < b) {
    const int32_t mid = (a + b) >> 1;
    if ((int32_t)rng[2 * mid + 1] > row) b = mid;
    else a = mid + 1;
  }
  return a;
}
// last column in [lo, hi] whose band START is <= `row`; lo - 1 if none
B2A_HD int32_t ks_last_col_start_upto(const uint32_t* rng, int32_t lo, int32_t hi, int32_t row) {
  int32_t a = lo - 1, b = hi;
  while (a < b) {
    const int32_t mid = (a + b + 1) >> 1;
    if ((int32_t)rng[2 * mid] <= row) a = mid;
    else b = mid - 1;
  }
  return a;
}

// One strip of one task (four pairs, 8 lanes each).  `s` is the strip index, the same for the four pairs; a pair
// with fewer strips idles.  Returns, per lane group, the uint4 units its strip used (for the strip table).
template <int FLAGS, bool LASTSTRIP>
B2A_HD void ks_run_strip(const KsPair& P, const DevScoring& sc, const KsLut& T, const int32_t one, const int32_t ge4, const int32_t lane,
                         const int32_t s, int32_t& prev_ja, int32_t& prev_jb, uint32_t& tb_used, bool& redo) {
  constexpr bool TR = (FLAGS & F_TRACK_ROWS) != 0;
  constexpr bool TC = (FLAGS & F_TRACK_COLS) != 0;
  constexpr bool LUT = (FLAGS & F_LUT) != 0;
  constexpr bool NOTB = (FLAGS & F_NOTB) != 0;  // score-only: no traceback (the strip table still records the windows)
  auto code_of = [&](uint8_t byte) -> int32_t {  // LUT code of a sequence byte; a byte outside the alphabet is flagged
    int32_t c = (int32_t)T.cmap[byte];
    if (c == 0xFF) {
#if defined(__CUDA_ARCH__)
      atomicOr(T.err_flag, 4u);
#else
      *T.err_flag |= 4u;
#endif
      c = 0;
    }
    return c;
  };
  const int32_t l = lane % KS_G;
  const int32_t m = P.m, n = P.n;
  const bool have = m >= 2 && s < (int32_t)ks_nstrips((uint64_t)m);
  const int32_t rowbase = s * KS_ROWS + l * KS_R;  // the row above this lane's first row
  const int32_t strip_lo = s * KS_ROWS + 1, strip_hi = imin(strip_lo + KS_ROWS - 1, m - 1);
  // the strip's column window: the band's columns that hold a row of [strip_lo, strip_hi]
  int32_t ja = 1, jb = 0;
  if (have && l == 0 && P.c0 <= P.c1) {
    ja = ks_first_col_end_above(P.rng, P.c0, P.c1, strip_lo);  // end > strip_lo  <=>  some row >= strip_lo is in the band
    jb = ks_last_col_start_upto(P.rng, P.c0, P.c1, strip_hi);
  }
  ja = KS_SHFL(ja, 0);
  jb = KS_SHFL(jb, 0);
  const int32_t len = (have && jb >= ja) ? jb - ja + 1 : 0;
  if (TR && len > 4095) redo = true;  // the packed row-tracker key holds a 12-bit column offset
  // (NOTB: no groups of 8 steps to fill and store)
  const int32_t nsteps = NOTB ? ks_warp_max(len > 0 ? len + KS_G - 1 : 0) : (ks_warp_max(len > 0 ? len + KS_G - 1 : 0) + 7) & ~7;
  const uint32_t K = (len > 0 && !NOTB) ? (uint32_t)((len + KS_G - 1 + 7) >> 3) : 0u;
  uint4* tbs = P.tb + tb_used;
  if (have && l == 0) {
    P.tab[KS_TAB * s] = (uint32_t)ja;
    P.tab[KS_TAB * s + 1] = tb_used;
    P.tab[KS_TAB * s + 2] = K * 8u;
    P.tab[KS_TAB * s + 3] = 0u;
  }
  // lane state
  int32_t Sp[KS_R], Dp[KS_R], SnR[KS_R], xc[KS_R];
  uint32_t tbacc[KS_R];
  const uint32_t s0 = have ? P.rng[0] : 1u, e0 = have ? P.rng[1] : 0u;  // column 0's band
#pragma unroll
  for (int r = 0; r < KS_R; ++r) {
    const int32_t i = rowbase + 1 + r;
    xc[r] = (have && i <= m) ? (int32_t)P.x[i - 1] : 0;
    if (LUT) xc[r] = (int32_t)(T.lut_base + (uint32_t)(((have && i <= m) ? code_of((uint8_t)xc[r]) : 0) * sc.alpha * 4));
    // the column before the window: outside the band, except column 0 when the window starts at column 1
    const bool in0 = have && ja == 1 && i < m && (uint32_t)i >= s0 && (uint32_t)i < e0;
    Sp[r] = (in0 ? 4 * col0_S(sc, i) : NEG4) + (4 * sc.gap_open + 1);
    Dp[r] = NEG4 + 1;
    SnR[r] = KEY_NONE;
    tbacc[r] = 0;
  }
  // the boundary row this strip leaves: its bottom row for the strip below, or row m-1 (the pair's last strip; another
  // pair of the warp may be in its last strip while this one is not) for the finish pass's row m
  const bool my_last = LASTSTRIP && have && s == (int32_t)ks_nstrips((uint64_t)m) - 1;
  int32_t cap_row = -1;
  if (my_last && m - 1 > rowbase && m - 1 <= rowbase + KS_R) cap_row = m - 2 - rowbase;  // row m-1 is mine
  const bool writer = have && (my_last ? cap_row >= 0 : l == KS_G - 1);
  // S(i0, ja-1) for the first row's diagonal: row 0 (strip 0) or the boundary row of the strip above
  int32_t sup_prev = NEG4;
  int32_t in_s = NEG4, in_i = NEG4 + 2, in_tv = KEY_NONE;
  const bool top_row0 = have && l == 0 && s == 0, top_mem = have && l == 0 && s > 0;
  if (len > 0 && top_row0) {
    const int32_t jp = ja - 1;
    if (jp == 0) sup_prev = (s0 == 0 && e0 > 0) ? 0 : NEG4;
    else sup_prev = P.rng[2 * jp] == 0 ? ks_row0_S4(sc, jp) : NEG4;
  }
  auto bnd_at = [&](int32_t j) -> int4 {  // the boundary row the strip above left (its window: [prev_ja, prev_jb])
    if (j >= prev_ja && j <= prev_jb) return P.bnd[j - P.c0 + 1];
    return make_int4(NEG4, NEG4 + 2, KEY_NONE, 0);
  };
  int4 pre = make_int4(NEG4, NEG4 + 2, KEY_NONE, 0);
  if (len > 0 && top_mem) {
    sup_prev = bnd_at(ja - 1).x;
    pre = bnd_at(ja);
  }
  int32_t cap_s = NEG4, cap_i = NEG4 + 2;
  const int32_t y4_row0 = 4 * (sc.yclip_prefix + sc.gap_open) + ge4 * rowbase;  // 4 * yclip_score(rowbase + 1)
  // the column's band range and y symbol are requested one step ahead (the loads are L1 hits, but with three warps
  // per scheduler their latency showed up as a quarter of the stall samples when they were issued where they are used)
  int32_t nsj = 0, nej = 0, nq = 0;
  auto fetch_col = [&](int32_t jr) {
    if (jr >= 0 && jr < len) {
      const int32_t j = ja + jr;
      nsj = (int32_t)P.rng[2 * j];
      nej = (int32_t)P.rng[2 * j + 1];
      nq = (int32_t)P.y[j - 1];
      if (LUT) nq = code_of((uint8_t)nq) * 4;
    }
  };
  fetch_col(-l);
  for (int32_t t = 0; t < nsteps; ++t) {
    const int32_t jr = t - l;  // column offset inside the window
    const bool active = jr >= 0 && jr < len;
    const int32_t sj = nsj, ej = nej, q = nq;
    fetch_col(jr + 1);
    if (active) {
      const int32_t j = ja + jr;
      const int32_t top = imin(ej, m) - sj;  // rows [sj, min(ej, m)) are cells of this kernel (row m is the finish pass's)
      const uint32_t h_band = top > 0 ? (uint32_t)top : 0u;
      if (top_row0) {
        in_s = (sj == 0 && ej > 0) ? ks_row0_S4(sc, j) : NEG4;
        in_i = NEG4 + 2;
        in_tv = KEY_NONE;
      } else if (top_mem) {
        in_s = pre.x;
        in_i = pre.y;
        in_tv = pre.z;
        if (jr + 1 < len) pre = bnd_at(j + 1);
      }
      int32_t sup = in_s, iup = in_i, Tv = in_tv;
      ks_column_step<FLAGS, LASTSTRIP>(sc, T, one, ge4, j, q, rowbase + 1 - sj, h_band, 4095 - jr, y4_row0, Sp, Dp, SnR,
                                       tbacc, xc, sup_prev, sup, iup, Tv, rowbase, cap_row, cap_s, cap_i);
      sup_prev = in_s;
      if (writer) {
        int4 o;
        o.x = (my_last && cap_row != KS_R - 1) ? cap_s : sup;
        o.y = (my_last && cap_row != KS_R - 1) ? cap_i : iup;
        o.z = TC ? Tv : KEY_NONE;  // (the rows below row m-1 are outside the band: the capture lane's tracker is complete)
        o.w = 0;
        P.bnd[j - P.c0 + 1] = o;
      }
      in_s = sup;
      in_i = iup;
      in_tv = Tv;
    } else if (!NOTB) {
#pragma unroll
      for (int r = 0; r < KS_R; ++r) tbacc[r] <<= 4;
    }
    in_s = B2A_SHFL_UP(in_s, KS_G);
    in_i = B2A_SHFL_UP(in_i, KS_G);
    if (TC) in_tv = B2A_SHFL_UP(in_tv, KS_G);
    if (!NOTB && (t & 7) == 7 && (uint32_t)(t >> 3) < K) {
      uint4* dst = tbs + (size_t)(t >> 3) * KS_TBW * KS_G + l;
#pragma unroll
      for (int qd = 0; qd < KS_TBW; ++qd) {
        uint4 v;
        v.x = tbacc[qd * 4 + 0];
        v.y = tbacc[qd * 4 + 1];
        v.z = tbacc[qd * 4 + 2];
        v.w = tbacc[qd * 4 + 3];
        dst[qd * KS_G] = v;
      }
    }
  }
  // Column n's literal pass (finish kernel) reads S and D of column n-1, rows of its band only.  A window that ends
  // at column n-1 leaves exactly that column in every lane's registers (idle steps touch neither Sp nor Dp), so the
  // export happens here, outside the column loop.
  if (len > 0 && jb == n - 1) {
    const int32_t sj = (int32_t)P.rng[2 * jb], ej = (int32_t)P.rng[2 * jb + 1];
    const int32_t top = imin(ej, m) - sj;
    const uint32_t h_band = top > 0 ? (uint32_t)top : 0u;
#pragma unroll
    for (int r = 0; r < KS_R; ++r) {
      if ((uint32_t)(rowbase + 1 - sj + r) < h_band) {
        int2 v;
        v.x = Sp[r] - (4 * sc.gap_open + 1);  // S travels open-biased
        v.y = Dp[r];
        P.last[rowbase + 1 + r] = v;
      }
    }
  }
  // the rows of this strip: Sn / Ly and the eager s-bit write of (i, n) (banded.rs:655-660), or their initial values
  if (have) {
#pragma unroll
    for (int r = 0; r < KS_R; ++r) {
      const int32_t i = rowbase + 1 + r;
      if (i <= m - 1) {
        int32_t sn = MIN_SCORE;
        uint32_t ly = 0;
        uint16_t mark = 0;
        if (TR && SnR[r] != KEY_NONE) {
          sn = (SnR[r] >> 12) + sc.yclip_suffix;
          ly = (uint32_t)(n - (ja + (4095 - (SnR[r] & 4095))));
          mark = (uint16_t)(TB_YCLIP_SUFFIX << 8);
        }
        P.Sn[i] = sn;
        P.Ly[i] = ly;
        P.coln[i] = mark;
      }
    }
  }
  if (have) {
    prev_ja = ja;
    prev_jb = len > 0 ? jb : ja - 1;
    tb_used += K * (uint32_t)(KS_TBW * KS_G);
  }
}

template <int FLAGS>
B2A_HD void ks_run_task(const StripParams& prm, const KsLut& T, const uint32_t task, const int lane) {
  const int32_t g = lane / KS_G;
  const uint32_t slot = task * 4 + (uint32_t)g;
  KsPair P{};
  uint64_t pair = 0;
  if (slot < prm.n_elig) {
    const uint32_t t = prm.elig[slot];
    pair = (uint64_t)prm.pair_lo + t;
    P.m = (int32_t)prm.x_len[pair];
    P.n = (int32_t)prm.y_len[pair];
    P.x = prm.blob + prm.x_off[pair];
    P.y = prm.blob + prm.y_off[pair];
    P.rng = prm.ranges + prm.ranges_off[t] / 4;
    const K3Layout L = k3_layout((uint64_t)P.m, (uint64_t)P.n, prm.num_cells[pair]);
    uint8_t* slab = prm.fill + prm.fill_off[t];
    P.Sn = reinterpret_cast<int32_t*>(slab + L.Sn);
    P.Ly = reinterpret_cast<uint32_t*>(slab + L.Ly);
    P.coln = reinterpret_cast<uint16_t*>(slab + L.coln);
    const int32_t bc0 = (int32_t)prm.band_cols[3 * pair], bc1 = (int32_t)prm.band_cols[3 * pair + 1];
    P.c0 = imax(bc0, 1);
    P.c1 = imin(bc1, P.n - 1);
    const KsLayout S = ks_layout((uint64_t)P.m, (uint64_t)(P.c1 >= P.c0 ? P.c1 - P.c0 + 1 : 0), prm.band_cols[3 * pair + 2],
                                 (FLAGS & F_NOTB) != 0);
    uint8_t* area = prm.strip + prm.strip_off[t];
    P.tab = reinterpret_cast<uint32_t*>(area + S.tab);
    P.bnd = reinterpret_cast<int4*>(area + S.bnd);
    P.last = reinterpret_cast<int2*>(area + S.last);
    P.tb = reinterpret_cast<uint4*>(area + S.tb);
  }
  const int32_t ns = (int32_t)ks_nstrips((uint64_t)P.m);
  const int32_t ns_max = ks_warp_max(ns);
  int32_t prev_ja = 1, prev_jb = 0;
  uint32_t tb_used = 0;
  bool redo = false;
  // F_NOTB twins with exactly three of the four trackers / prefix clips live and no LUT run the capturing form for every
  // strip: one inlined copy of the strip loop instead of two.  Chosen by -Xptxas -v: with two copies three of these
  // twins spill a few words more than their full kernels; with one copy for every twin, two others do, and the
  // capture's three instructions per cell slow the common twins (semiglobal's K3 by 10 %).  Split this way no twin
  // spills more than its full kernel (DESIGN.md §4).
  constexpr int kLive = ((FLAGS & F_TRACK_ROWS) != 0) + ((FLAGS & F_TRACK_COLS) != 0) + ((FLAGS & F_CLIPX) != 0) +
                        ((FLAGS & F_CLIPY) != 0);
  constexpr bool kOneCopy = (FLAGS & F_NOTB) != 0 && (FLAGS & F_LUT) == 0 && kLive == 3;
  for (int32_t s = 0; s < ns_max; ++s) {
    // the capture of row m-1 costs three instructions per cell: only the warp's passes that hold a pair's last strip pay it
    const bool any_last = kOneCopy || ks_warp_max((P.m >= 2 && s == ns - 1) ? 1 : 0) != 0;
    if (any_last) ks_run_strip<FLAGS, true>(P, prm.sc, T, prm.one, prm.ge4, lane, s, prev_ja, prev_jb, tb_used, redo);
    else ks_run_strip<FLAGS, false>(P, prm.sc, T, prm.one, prm.ge4, lane, s, prev_ja, prev_jb, tb_used, redo);
  }
  if (redo && P.m >= 2 && lane % KS_G == 0) prm.k4_status[pair] |= 0x400u;
}

#if defined(__CUDACC__)

#ifndef B2A_KS_MINB
#define B2A_KS_MINB 3
#endif
constexpr int KS_WARPS = 4;

// dynamic shared memory of a CTA (F_LUT only): the scaled LUT, then the 256-byte code map
B2A_HD uint32_t ks_smem_bytes(int flags, int alpha) { return (flags & F_LUT) ? lut_smem_bytes(alpha) + 256u : 0u; }

template <int FLAGS>
__global__ void __launch_bounds__(KS_WARPS * 32, B2A_KS_MINB) banded_strip_fill_kernel(const StripParams prm) {
  extern __shared__ __align__(128) uint8_t ks_smem[];
  const int lane = threadIdx.x & 31;
  KsLut T{};
  if (FLAGS & F_LUT) {
    int32_t* lut_s = reinterpret_cast<int32_t*>(ks_smem);
    uint8_t* cmap_s = ks_smem + lut_smem_bytes(prm.sc.alpha);
    for (int k = threadIdx.x; k < prm.sc.alpha * prm.sc.alpha; k += blockDim.x) lut_s[k] = prm.lut[k];
    for (int k = threadIdx.x; k < 256; k += blockDim.x) cmap_s[k] = prm.codemap[k];
    __syncthreads();
    T.lut = lut_s;
    T.lut_base = (uint32_t)__cvta_generic_to_shared(lut_s);
    T.cmap = cmap_s;
    T.err_flag = prm.err_flag;
  }
  const uint32_t ntasks = (prm.n_elig + 3) / 4;
  for (;;) {
    uint32_t task = 0;
    if (lane == 0) task = atomicAdd(prm.task_counter, 1u);
    task = __shfl_sync(0xffffffffu, task, 0);
    if (task >= ntasks) break;
    ks_run_task<FLAGS>(prm, T, task, lane);
    __syncwarp();
  }
}

// Launches the F_NOTB twin for `flags` (which include F_NOTB) on `st`.  The twins are instantiated in
// b2a_banded_strip_notb.cu, a translation unit of their own, so that they compile beside b2a_engine.cu.
// Returns cudaErrorInvalidValue for a flag set without a twin.
cudaError_t launch_banded_strip_fill_notb(int flags, unsigned grid, size_t smem, cudaStream_t st, const StripParams& sp);

#endif

}  // namespace b2a
