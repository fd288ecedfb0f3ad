// Host-side batch plan: sort pairs by shape, cut them into blocks of up to 32, size
// the HBM arenas and the traceback waves.  Pure C++ (used by the engine and by
// the CPU simulation harness in tests/sim/).
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

#include "b2a_common.cuh"

namespace b2a {

struct Wave {
  uint32_t block_lo, block_hi;  // [lo, hi)
  uint64_t bnd_bytes, rows_bytes, rowm_bytes, tb_bytes;
  uint64_t strip_tasks;  // sum over the wave's blocks of 32 * nstrips
};

struct Plan {
  int G = 1, R = 16;
  uint64_t n_pairs = 0;
  std::vector<uint32_t> order;  // sorted index -> caller index
  std::vector<uint32_t> pm, pn; // sorted
  std::vector<Block> blocks;
  std::vector<Wave> waves;
  uint64_t seq_bytes = 0, ops_bytes = 0;
  uint64_t max_bnd = 0, max_rows = 0, max_rowm = 0, max_tb = 0;  // per-wave maxima
  uint64_t max_strip_tasks = 0;
  uint64_t max_fin = 0;    // F_FINISH: bytes of the finish region of the wave with the most blocks (else 0)
  uint64_t total_tb = 0;   // traceback bytes the fill stores over the whole batch
  uint64_t cells = 0;
  uint32_t smem_seq_bytes = 0;  // per-warp staging
  uint32_t maxm = 0, maxn = 0;
};

inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

// `flags`: the fill's kernel flags (F_BND8 halves the boundary record; F_NOTB, a score-only batch, stores no
// traceback, and its waves close on the rest of the per-wave scratch -- boundary rows, rows arena, row-m cells --
// against the same budget; F_FINISH adds the finish region, max_fin, and changes nothing else).
// Blocks hold 32 pairs (the last one the rest), except in the warp-per-pair shape (G == 32) with a traceback: there a
// block's traceback is sized by its real pairs, and a block closes early when its next pair would take it past
// `tb_budget`, so that waves can close between long pairs.  A single pair above the budget still gets a block (and a
// wave) of its own: the engine refuses such a batch (max_tb > tb_budget) before it allocates anything.
inline void build_plan(Plan& p, const uint32_t* x_len, const uint32_t* y_len, uint64_t n_pairs, int G,
                       int R, uint64_t tb_budget, int flags = 0) {
  const uint64_t bnd_rec = (flags & F_BND8) ? 8 : 16;
  const bool notb = (flags & F_NOTB) != 0;
  p.G = G;
  p.R = R;
  p.n_pairs = n_pairs;
  p.order.resize(n_pairs);
  std::iota(p.order.begin(), p.order.end(), 0u);
  bool uniform_all = true;
  for (uint64_t i = 1; i < n_pairs && uniform_all; ++i)
    uniform_all = (x_len[i] == x_len[0]) && (y_len[i] == y_len[0]);
  if (!uniform_all) {
    std::stable_sort(p.order.begin(), p.order.end(), [&](uint32_t a, uint32_t b) {
      if (x_len[a] != x_len[b]) return x_len[a] > x_len[b];
      return y_len[a] > y_len[b];
    });
  }
  p.pm.resize(n_pairs);
  p.pn.resize(n_pairs);
  p.cells = 0;
  for (uint64_t i = 0; i < n_pairs; ++i) {
    p.pm[i] = x_len[p.order[i]];
    p.pn[i] = y_len[p.order[i]];
    p.cells += (uint64_t)p.pm[i] * p.pn[i];
  }
  const int P = 32 / G, TBW = tbw_of(R);
  // traceback bytes of one warp-task (32/G pairs) over every strip of a block with these maxima
  auto task_tb = [&](uint32_t maxm, uint32_t maxn) -> uint64_t {
    const uint64_t nstrips = maxm >= 2 ? (maxm - 1 + G * R - 1) / (G * R) : 0;
    const uint64_t K = maxn ? (maxn + G - 1 + 7) / 8 : 0;
    return nstrips * K * TBW * 512;
  };
  const bool per_pair = G == 32 && !notb;  // the warp-per-pair shape's tasks are its pairs
  p.blocks.clear();
  for (uint64_t first = 0; first < n_pairs;) {
    uint32_t q = 0, mm = 0, mn = 0;
    while (q < 32 && first + q < n_pairs) {
      const uint32_t m2 = std::max(mm, p.pm[first + q]), n2 = std::max(mn, p.pn[first + q]);
      if (per_pair && q > 0 && (uint64_t)(q + 1) * task_tb(m2, n2) > tb_budget) break;
      mm = m2;
      mn = n2;
      ++q;
    }
    Block k{};
    k.first = (uint32_t)first;
    k.npairs = q;
    p.blocks.push_back(k);
    first += q;
  }
  const uint32_t nblocks = (uint32_t)p.blocks.size();
  p.waves.clear();
  p.seq_bytes = p.ops_bytes = 0;
  p.max_bnd = p.max_rows = p.max_rowm = p.max_tb = 0;
  p.max_strip_tasks = 0;
  p.max_fin = 0;
  p.total_tb = 0;
  p.smem_seq_bytes = 0;
  p.maxm = p.maxn = 0;
  Wave w{0, 0, 0, 0, 0, 0, 0};
  for (uint32_t b = 0; b < nblocks; ++b) {
    Block& k = p.blocks[b];
    k.maxm = k.maxn = 0;
    for (uint32_t q = 0; q < k.npairs; ++q) {
      k.maxm = std::max(k.maxm, p.pm[k.first + q]);
      k.maxn = std::max(k.maxn, p.pn[k.first + q]);
    }
    k.uniform = 1;
    for (uint32_t q = 0; q < k.npairs; ++q)
      if (p.pm[k.first + q] != k.maxm || p.pn[k.first + q] != k.maxn) k.uniform = 0;
    k.nstrips = k.maxm >= 2 ? (k.maxm - 1 + G * R - 1) / (G * R) : 0;
    const uint32_t xw = std::max<uint32_t>((k.maxm + 3) / 4, k.nstrips * G * R / 4);
    k.xwords = (uint32_t)align_up(std::max<uint32_t>(xw, 4), 4);
    k.ywords = (uint32_t)align_up(std::max<uint32_t>((k.maxn + 3) / 4, 4), 4);
    k.K = k.maxn ? (k.maxn + G - 1 + 7) / 8 : 0;
    k.rows_pad = k.nstrips * G * R + 2;
    p.maxm = std::max(p.maxm, k.maxm);
    p.maxn = std::max(p.maxn, k.maxn);
    // the warp-per-pair shape runs (pair, strip) tasks that stage one strip of x (b2a_fill.cuh), and y unless the
    // engine picks F_YSTREAM (y read from the arena: G * R bytes of staging)
    const uint32_t stage_x = G == 32 ? (uint32_t)(G * R) : k.xwords * P * 4;
    p.smem_seq_bytes = std::max<uint32_t>(p.smem_seq_bytes, stage_x + k.ywords * P * 4);
    const uint64_t bnd = align_up((uint64_t)(k.maxn + 1) * 32 * bnd_rec, 256);
    const uint64_t rows = align_up((uint64_t)ROWS_ARRAYS * k.rows_pad * 32 * 4, 256);
    const uint64_t rowm = align_up((uint64_t)(k.maxn + 1) * 32 * 2, 256);
    const uint32_t tasks = G == 32 ? k.npairs : (uint32_t)G;  // warp-tasks that store a traceback
    const uint64_t tb = notb ? 0 : align_up((uint64_t)tasks * k.nstrips * k.K * TBW * 512, 256);
    const bool full = notb ? w.bnd_bytes + w.rows_bytes + w.rowm_bytes + bnd + rows + rowm > tb_budget
                           : w.tb_bytes + tb > tb_budget;
    if (b > w.block_lo && full) {  // close the wave
      w.block_hi = b;
      p.waves.push_back(w);
      w = Wave{b, b, 0, 0, 0, 0, 0};
    }
    k.seq_off = p.seq_bytes;
    p.seq_bytes += align_up((uint64_t)32 * (k.xwords + k.ywords) * 4, 256);
    k.ops_off = p.ops_bytes;
    p.ops_bytes += align_up((uint64_t)32 * (k.maxm + k.maxn + 4), 256);
    k.strip_task_base = w.strip_tasks;
    w.strip_tasks += (uint64_t)(G == 32 ? k.npairs : 32) * k.nstrips;
    k.bnd_off = w.bnd_bytes;
    k.rows_off = w.rows_bytes;
    k.rowm_off = w.rowm_bytes;
    k.tb_off = w.tb_bytes;
    w.bnd_bytes += bnd;
    w.rows_bytes += rows;
    w.rowm_bytes += rowm;
    w.tb_bytes += tb;
    if (!notb) p.total_tb += (uint64_t)tasks * k.nstrips * k.K * TBW * 512;
  }
  if (nblocks) {
    w.block_hi = nblocks;
    p.waves.push_back(w);
  }
  for (const Wave& v : p.waves) {
    p.max_bnd = std::max(p.max_bnd, v.bnd_bytes);
    p.max_rows = std::max(p.max_rows, v.rows_bytes);
    p.max_rowm = std::max(p.max_rowm, v.rowm_bytes);
    p.max_tb = std::max(p.max_tb, v.tb_bytes);
    p.max_strip_tasks = std::max(p.max_strip_tasks, v.strip_tasks);
    if (flags & F_FINISH)  // FIN_FIELDS words per pair of every block of the wave
      p.max_fin = std::max<uint64_t>(p.max_fin, (uint64_t)(v.block_hi - v.block_lo) * FIN_FIELDS * 32 * 4);
  }
}

// Kernel flags for a scoring (SURVEY 3.2 "derived mode specialisations").
// `score_bound` = (maxm+maxn+2)*max|score, go, ge| + |go|: every real S/I/D lies within +-score_bound.
inline int scoring_flags(const DevScoring& sc, int64_t score_bound = (1ll << 40), uint32_t maxm = ~0u,
                         uint32_t maxn = ~0u) {
  const bool xp = sc.xclip_prefix > DEAD_CLIP, xs = sc.xclip_suffix > DEAD_CLIP;
  const bool yp = sc.yclip_prefix > DEAD_CLIP, ys = sc.yclip_suffix > DEAD_CLIP;
  int f = 0;
  if (xs || (xp && yp)) {
    f = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;  // general variant
  } else if (ys) {
    f = F_TRACK_ROWS;
  }
  if (sc.alpha) f |= F_LUT;
  // local-style clips: xclip_score(j) = xp + max(yp, go + ge (j-1)) == 0 for every j (go, ge <= 0)
  if ((f & F_CLIPX) && sc.xclip_prefix == 0 && sc.yclip_prefix == 0) f |= F_RELU;
  if ((f & (F_TRACK_ROWS | F_TRACK_COLS)) && score_bound < (1ll << 17) && maxm <= 4095 && maxn <= 4095)
    f |= F_PACKTRK;
  else if ((f & (F_TRACK_ROWS | F_TRACK_COLS)) && score_bound < (1ll << 18))
    f |= F_PACKREL;  // longer sequences: the packed keys with chunk- / strip-relative indices
  return f;
}

// Whether the fill may use the 8-byte strip boundary record (F_BND8) on top of `flags` = scoring_flags(...):
// the packed-tracker form only (its record carries no row index), and every S4 / I4 of the record within a signed
// 16-bit half.  Fills without trackers (global), the long-sequence form (F_PACKREL) and the explicit (value, row)
// trackers keep the 16-byte record.
inline bool boundary8_ok(int flags, int64_t score_bound) {
  return (flags & F_PACKTRK) != 0 && 4 * score_bound + 3 < (1ll << 15);
}

// Whether the banded strip-wavefront fill (b2a_banded_strip.cuh) may take pairs of a batch; `sc` carries the mode's
// clip preset.  Its sentinel arithmetic covers every real score within +-2^26.  Row / column trackers exist there
// only as packed keys: every band cell's S has to be real (a live y-prefix clip guarantees it: S >= yclip_score(i))
// and below 2^17, and the column tracker's key also holds the row (x no longer than 4,095).  Otherwise the pairs run
// the K3 column loops.
inline bool banded_strip_gate(const DevScoring& sc, int64_t score_bound, uint32_t maxm) {
  const bool xs_dead = sc.xclip_suffix <= DEAD_CLIP, ys_dead = sc.yclip_suffix <= DEAD_CLIP;
  const bool yp_live = sc.yclip_prefix > DEAD_CLIP;
  const bool trackers_ok = (xs_dead && ys_dead) || (yp_live && score_bound < (1ll << 17) && (xs_dead || maxm <= 4095));
  return score_bound < (1ll << 26) && trackers_ok;
}

}  // namespace b2a
