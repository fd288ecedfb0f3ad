// CPU simulation of the warp-per-pair fill on long pairs (tests/test_long_pairs.py): the 32x8 and 32x16
// strip-pipelined fill, full and score-only (F_NOTB), with the flags b2a_engine.cu's stage_front picks plus
// F_YSTREAM: y read from the staged-sequence arena as the kernel streams it.  Every y word the fill loads goes through the
// B2A_HOST_YREAD hook, which counts loads outside the pair's own words; the arena's bytes around each pair's y can be
// poisoned.  Also: the plan (blocks, waves, traceback bytes) and the rows-arena index helper.  Builds on the harness of
// b2a_sim.cpp.  Test tool only.
#include <cstdint>

namespace {
uint64_t siml_y_oob = 0;    // y words loaded outside [0, ceil(n / 4)) of the pair
uint64_t siml_y_loads = 0;  // y words loaded
inline void siml_yread(int32_t n, int32_t w) {
  ++siml_y_loads;
  if (w < 0 || w >= (n + 3) / 4) ++siml_y_oob;
}
}  // namespace
#define B2A_HOST_YREAD(c, w) siml_yread((c).n, (w))

#include "b2a_sim.cpp"

namespace {

template <int R, bool NOTB>
void fill_dispatch_long(int flags, const Plan& p, const Block& blk, const DevScoring& sc, const int32_t* lut,
                        std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                        std::vector<uint8_t>& tb) {
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
  constexpr int NB = NOTB ? F_NOTB : 0;
#define SIML_CASE(F) \
  case (NB | F_YSTREAM | (F)): fill_block_piped<R, NB | F_YSTREAM | (F)>(p, blk, sc, lut, seq, bnd, rows, tb); break;
  switch (flags) {  // the flag cases of b2a_fill_inst.cu with a LUT (every batch here has at most 64 symbols)
    SIML_CASE(F_LUT)
    SIML_CASE(F_LUT | F_TRACK_ROWS)
    SIML_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK)
    SIML_CASE(F_LUT | ALL)
    SIML_CASE(F_LUT | ALL | F_PACKTRK)
    SIML_CASE(F_LUT | ALL | F_RELU)
    SIML_CASE(F_LUT | ALL | F_PACKTRK | F_RELU)
    SIML_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIML_CASE(F_LUT | ALL | F_PACKTRK | F_BND8)
    SIML_CASE(F_LUT | ALL | F_PACKTRK | F_RELU | F_BND8)
    SIML_CASE(F_LUT | F_TRACK_ROWS | F_PACKREL)
    SIML_CASE(F_LUT | ALL | F_PACKREL)
    SIML_CASE(F_LUT | ALL | F_PACKREL | F_RELU)
    default: std::abort();
  }
#undef SIML_CASE
}

int siml_last_flags = 0;

}  // namespace

extern "C" {

// One batch through K0's staging, the 32xR strip-pipelined fill and K2 (walk_pair, or walk_pair_coop<32> on 32
// emulated lanes), in caller order.  score_only: the F_NOTB fill, no traceback arena, and the score-only walk (then
// only score, xend, yend and status are written).  poison >= 0: every byte of the staged y area that is not one of a
// pair's n symbols (the tail of the pair's last word, the words after it, the slots of padding pairs) holds that byte.
// *y_oob: y words the fill loaded outside the pair's own ceil(n / 4) words.
int siml_align(int mode, const sim_scoring* s, const uint8_t* blob, const uint64_t* x_off, const uint32_t* x_len,
               const uint64_t* y_off, const uint32_t* y_len, uint64_t n_pairs, int R, int score_only, int warp_walk,
               int garbage, int poison, int32_t* score, uint32_t* xstart, uint32_t* xend, uint32_t* ystart,
               uint32_t* yend, uint32_t* n_ops, uint32_t* clip_len, uint32_t* status, uint8_t* ops,
               const uint64_t* ops_off, uint64_t* y_oob, uint64_t* y_loads) {
  constexpr int G = 32, P = 1;
  if (R != 8 && R != 16) return -1;
  DevScoring sc{};
  sc.gap_open = s->gap_open;
  sc.gap_extend = s->gap_extend;
  sc.xclip_prefix = s->xclip_prefix;
  sc.xclip_suffix = s->xclip_suffix;
  sc.yclip_prefix = s->yclip_prefix;
  sc.yclip_suffix = s->yclip_suffix;
  if (mode == 1) sc.xclip_prefix = sc.xclip_suffix = sc.yclip_prefix = sc.yclip_suffix = MIN_SCORE;
  if (mode == 2) { sc.xclip_prefix = sc.xclip_suffix = MIN_SCORE; sc.yclip_prefix = sc.yclip_suffix = 0; }
  if (mode == 3) sc.xclip_prefix = sc.xclip_suffix = sc.yclip_prefix = sc.yclip_suffix = 0;
  sc.match_score = s->match_score;
  sc.mismatch_score = s->mismatch_score;
  uint8_t codemap[256];
  for (int k = 0; k < 256; ++k) codemap[k] = (uint8_t)k;
  std::vector<int32_t> lut;
  int64_t maxabs = std::max<int64_t>(std::llabs((long long)s->match_score), std::llabs((long long)s->mismatch_score));
  {
    bool present[256] = {false};
    for (uint64_t p = 0; p < n_pairs; ++p) {
      for (uint32_t k = 0; k < x_len[p]; ++k) present[blob[x_off[p] + k]] = true;
      for (uint32_t k = 0; k < y_len[p]; ++k) present[blob[y_off[p] + k]] = true;
    }
    std::vector<int> syms;
    for (int k = 0; k < 256; ++k)
      if (present[k]) syms.push_back(k);
    if (syms.empty()) syms.push_back(0);
    if ((int)syms.size() > (s->table ? 128 : 64)) return -2;
    for (size_t a = 0; a < syms.size(); ++a) codemap[syms[a]] = (uint8_t)a;
    sc.alpha = (int32_t)syms.size();
    const size_t aa = (size_t)sc.alpha * sc.alpha;
    lut.resize(aa + (size_t)lut_entries(sc.alpha));
    if (s->table) maxabs = 0;
    for (int a = 0; a < sc.alpha; ++a)
      for (int b = 0; b < sc.alpha; ++b) {
        const int32_t v = s->table ? s->table[syms[a] * 256 + syms[b]] : (a == b ? s->match_score : s->mismatch_score);
        lut[(size_t)a * sc.alpha + b] = v;
        maxabs = std::max<int64_t>(maxabs, std::llabs((long long)v));
      }
    for (size_t k = 0; k < aa; ++k) lut[aa + k] = 4 * lut[k] + 3 - (4 * sc.gap_open + 1);
    for (size_t k = aa; k < (size_t)lut_entries(sc.alpha); ++k) lut[aa + k] = LUT_POISON;
  }
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull);  // (for maxm / maxn)
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t bound = ((int64_t)p.maxm + p.maxn + 2) * unit - (int64_t)sc.gap_open;
  int flags = scoring_flags(sc, bound, p.maxm, p.maxn);
  if (boundary8_ok(flags, bound)) flags |= F_BND8;
  if (score_only) flags |= F_NOTB;
  flags |= F_YSTREAM;  // the form the engine runs when y does not fit the staging
  siml_last_flags = flags;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull, flags);
  const int32_t* lut_plain = lut.data();
  const int32_t* lut_scaled = lut.data() + (size_t)sc.alpha * sc.alpha;
  const uint8_t gb = (uint8_t)garbage;
  std::vector<uint8_t> seq(p.seq_bytes, 0), bnd(p.max_bnd, gb), rows(p.max_rows, gb), rowm(p.max_rowm, gb), tb,
      opsb(p.ops_bytes, 0);
  if (!score_only) tb.assign(p.max_tb, gb);
  for (const Block& blk : p.blocks) {  // K0: [pair][word] x, then [pair][word] y
    uint32_t* seqw = reinterpret_cast<uint32_t*>(seq.data() + blk.seq_off);
    if (poison >= 0)
      std::memset(seqw + (size_t)G * blk.xwords, poison, (size_t)G * blk.ywords * 4);
    for (uint32_t q = 0; q < blk.npairs; ++q) {
      const uint32_t orig = p.order[blk.first + q];
      uint8_t* xb = reinterpret_cast<uint8_t*>(seqw + (size_t)q * blk.xwords);
      for (uint32_t k = 0; k < x_len[orig]; ++k) xb[k] = codemap[blob[x_off[orig] + k]];
      uint8_t* yb = reinterpret_cast<uint8_t*>(seqw + (size_t)G * blk.xwords + (size_t)q * blk.ywords);
      for (uint32_t k = 0; k < y_len[orig]; ++k) yb[k] = codemap[blob[y_off[orig] + k]];
    }
  }
  siml_y_oob = siml_y_loads = 0;
  for (const Block& blk : p.blocks) {
    if (R == 8) {
      if (score_only) fill_dispatch_long<8, true>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb);
      else fill_dispatch_long<8, false>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb);
    } else {
      if (score_only) fill_dispatch_long<16, true>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb);
      else fill_dispatch_long<16, false>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb);
    }
    for (uint32_t lane = 0; lane < blk.npairs; ++lane) {
      const uint32_t sp = blk.first + lane;
      PairView v;
      v.sc = sc;
      v.lut = lut_plain;
      v.P = P;
      v.m = (int32_t)p.pm[sp];
      v.n = (int32_t)p.pn[sp];
      v.pi = (int32_t)lane;
      v.set_shape(G, R);
      v.nstrips = (int32_t)blk.nstrips;
      v.K = (int32_t)blk.K;
      v.sub = (int32_t)lane;
      v.g = 0;
      v.packtrk = (flags & F_PACKTRK) ? 1 : 0;
      v.bnd8 = (flags & F_BND8) ? 1 : 0;
      v.maxn = (int32_t)blk.maxn;
      v.bnd_base = bnd_index(G, 0, (int32_t)lane, v.maxn);
      v.bnd_stride = (int32_t)(bnd_index(G, 1, (int32_t)lane, v.maxn) - v.bnd_base);
      const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
      v.xw = seqw + (size_t)lane * blk.xwords;
      v.yw = seqw + (size_t)G * blk.xwords + (size_t)lane * blk.ywords;
      v.bnd = reinterpret_cast<const int4*>(bnd.data() + blk.bnd_off);
      v.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
      v.rows_pad = (int32_t)blk.rows_pad;
      v.rowm = reinterpret_cast<uint16_t*>(rowm.data() + blk.rowm_off);
      v.tb = score_only ? nullptr : reinterpret_cast<const uint32_t*>(tb.data() + blk.tb_off);
      const uint32_t cap = blk.maxm + blk.maxn + 4;
      uint8_t* ops_end = score_only ? nullptr : opsb.data() + blk.ops_off + (size_t)(lane + 1) * cap;
      WalkOut o;
      if (warp_walk) {
        LaneFibers::run([&](int l) {
          WalkOut mine;
          if (score_only) walk_pair_coop<32, true>(l, v, mode == 2 || mode == 3, nullptr, mine);
          else walk_pair_coop<32>(l, v, mode == 2 || mode == 3, ops_end, mine);
          if (l == 0) o = mine;
        });
      } else if (score_only) {
        walk_pair<true>(v, mode == 2 || mode == 3, nullptr, o);
      } else {
        walk_pair(v, mode == 2 || mode == 3, ops_end, o);
      }
      const uint32_t dst = p.order[sp];
      status[dst] = o.status;
      if (score_only) {  // as walk_store<true>
        score[dst] = o.status ? MIN_SCORE : o.score;
        xend[dst] = o.status ? 0u : o.xend;
        yend[dst] = o.status ? 0u : o.yend;
        continue;
      }
      score[dst] = o.score;
      xstart[dst] = o.xstart;
      xend[dst] = o.xend;
      ystart[dst] = o.ystart;
      yend[dst] = o.yend;
      n_ops[dst] = o.n_ops;
      for (int k = 0; k < 4; ++k) clip_len[4 * (size_t)dst + k] = o.clip[k];
      std::memcpy(ops + ops_off[dst], ops_end - o.n_ops, o.n_ops);
    }
  }
  *y_oob = siml_y_oob;
  *y_loads = siml_y_loads;
  return 0;
}

int siml_fill_flags() { return siml_last_flags; }

// The plan of a batch: per block (first, npairs, maxm, maxn, nstrips, K, tb_off, strip_task_base) into blocks_out
// (8 x uint64 per block, up to max_blocks), per wave (block_lo, block_hi, tb_bytes) into waves_out (up to max_waves);
// scalars[0..3] = number of blocks, number of waves, total_tb, max_tb.
void siml_plan(const uint32_t* x_len, const uint32_t* y_len, uint64_t n_pairs, int G, int R, uint64_t budget, int flags,
               uint64_t* blocks_out, uint64_t max_blocks, uint64_t* waves_out, uint64_t max_waves, uint64_t* scalars) {
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, budget, flags);
  for (size_t b = 0; b < p.blocks.size() && b < max_blocks; ++b) {
    const Block& k = p.blocks[b];
    const uint64_t v[8] = {k.first, k.npairs, k.maxm, k.maxn, k.nstrips, k.K, k.tb_off, k.strip_task_base};
    std::memcpy(blocks_out + 8 * b, v, sizeof v);
  }
  for (size_t w = 0; w < p.waves.size() && w < max_waves; ++w) {
    waves_out[3 * w + 0] = p.waves[w].block_lo;
    waves_out[3 * w + 1] = p.waves[w].block_hi;
    waves_out[3 * w + 2] = p.waves[w].tb_bytes;
  }
  scalars[0] = p.blocks.size();
  scalars[1] = p.waves.size();
  scalars[2] = p.total_tb;
  scalars[3] = p.max_tb;
}

// Every field of a plan, serialised in a fixed order (tests/golden/plan_digests.json holds their SHA-256 for plans
// with fewer than 32 lanes per pair, which this change leaves as they were).  Returns the byte count; writes at most
// cap bytes.
uint64_t siml_plan_bytes(const uint32_t* x_len, const uint32_t* y_len, uint64_t n_pairs, int G, int R, uint64_t budget,
                         int flags, uint8_t* out, uint64_t cap) {
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, budget, flags);
  std::vector<uint64_t> v;
  v.push_back(p.n_pairs);
  for (uint32_t o : p.order) v.push_back(o);
  for (uint32_t o : p.pm) v.push_back(o);
  for (uint32_t o : p.pn) v.push_back(o);
  for (const Block& k : p.blocks) {
    const uint64_t f[18] = {k.first, k.npairs, k.maxm, k.maxn, k.uniform, k.nstrips, k.xwords, k.ywords, k.K,
                            k.rows_pad, k.seq_off, k.bnd_off, k.rows_off, k.rowm_off, k.tb_off, k.ops_off,
                            k.strip_task_base, 0};
    v.insert(v.end(), f, f + 18);
  }
  for (const Wave& w : p.waves) {
    const uint64_t f[7] = {w.block_lo, w.block_hi, w.bnd_bytes, w.rows_bytes, w.rowm_bytes, w.tb_bytes, w.strip_tasks};
    v.insert(v.end(), f, f + 7);
  }
  const uint64_t sc[12] = {p.seq_bytes, p.ops_bytes, p.max_bnd, p.max_rows, p.max_rowm, p.max_tb,
                           p.max_strip_tasks, p.total_tb, p.cells, p.smem_seq_bytes, p.maxm, p.maxn};
  v.insert(v.end(), sc, sc + 12);
  const uint64_t bytes = v.size() * 8;
  if (out) std::memcpy(out, v.data(), std::min<uint64_t>(bytes, cap));
  return bytes;
}

// the rows-arena element index the fill and K2 use (rows_index in b2a_common.cuh)
uint64_t siml_rows_index(int arr, int32_t rows_pad, int32_t row, int32_t pi) {
  return (uint64_t)rows_index(arr, rows_pad, row * 32 + pi);
}

}  // extern "C"
