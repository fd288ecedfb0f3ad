// CPU simulation of a score-only batch (b2a_batch_stage_scores): the F_NOTB fill and the score-only K2
// (walk_pair<true> / walk_pair_coop<32, true>) with the flags picked as b2a_engine.cu's stage_front picks them --
// scoring_flags(), F_BND8 when boundary8_ok() -- plus F_NOTB, and the plan sized for them.  Builds on the harness of
// b2a_sim.cpp (lane / warp emulation, fill_block, fill_block_piped).  Test tool only (tests/test_score_only.py).
#include "b2a_sim.cpp"

namespace {

int sims_last_flags = 0;  // the flags the last sims_align_scores ran its fill with

template <int G, int R, bool PIPED>
void fill_dispatch_notb(int flags, const Plan& p, const Block& blk, const DevScoring& sc, const int32_t* lut,
                        std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                        std::vector<uint8_t>& tb) {
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
#define SIMS_CASE(F)                                                                                   \
  case (F_NOTB | (F)):                                                                                 \
    if constexpr (PIPED) fill_block_piped<R, F_NOTB | (F)>(p, blk, sc, lut, seq, bnd, rows, tb);       \
    else fill_block<G, R, F_NOTB | (F)>(p, blk, sc, lut, seq, bnd, rows, tb);                          \
    break;
  switch (flags) {  // the F_NOTB instantiations of b2a_fill_inst.cu (-DB2A_NOTB)
    SIMS_CASE(0)
    SIMS_CASE(F_TRACK_ROWS)
    SIMS_CASE(F_TRACK_ROWS | F_PACKTRK)
    SIMS_CASE(ALL)
    SIMS_CASE(ALL | F_PACKTRK)
    SIMS_CASE(ALL | F_RELU)
    SIMS_CASE(ALL | F_PACKTRK | F_RELU)
    SIMS_CASE(F_LUT)
    SIMS_CASE(F_LUT | F_TRACK_ROWS)
    SIMS_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK)
    SIMS_CASE(F_LUT | ALL)
    SIMS_CASE(F_LUT | ALL | F_PACKTRK)
    SIMS_CASE(F_LUT | ALL | F_RELU)
    SIMS_CASE(F_LUT | ALL | F_PACKTRK | F_RELU)
    SIMS_CASE(F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIMS_CASE(ALL | F_PACKTRK | F_BND8)
    SIMS_CASE(ALL | F_PACKTRK | F_RELU | F_BND8)
    SIMS_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIMS_CASE(F_LUT | ALL | F_PACKTRK | F_BND8)
    SIMS_CASE(F_LUT | ALL | F_PACKTRK | F_RELU | F_BND8)
    SIMS_CASE(F_TRACK_ROWS | F_PACKREL)
    SIMS_CASE(ALL | F_PACKREL)
    SIMS_CASE(ALL | F_PACKREL | F_RELU)
    SIMS_CASE(F_LUT | F_TRACK_ROWS | F_PACKREL)
    SIMS_CASE(F_LUT | ALL | F_PACKREL)
    SIMS_CASE(F_LUT | ALL | F_PACKREL | F_RELU)
    default: std::abort();
  }
#undef SIMS_CASE
}

}  // namespace

extern "C" {

// Outputs: score, xend, yend, status per pair (caller order).  Shapes 1x16, 8x20 and 132 (= 32x8 with
// strip-pipelined tasks); warp_walk: K2 as walk_pair_coop<32, true> on 32 emulated lanes (else walk_pair<true>).
// poison < 0: the fill and the walk get tb = nullptr.  poison = 0..255: they get a traceback arena of the size the
// full path would use, filled with that byte; returns -3 if a single byte of it changed.
int sims_align_scores(int mode, const sim_scoring* s, const uint8_t* blob, const uint64_t* x_off, const uint32_t* x_len,
                      const uint64_t* y_off, const uint32_t* y_len, uint64_t n_pairs, int Gsel, int R, int warp_walk,
                      int garbage, int poison, int32_t* score, uint32_t* xend, uint32_t* yend, uint32_t* status) {
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
  // alphabet + LUT as the engine builds them (b2a_engine.cu stage_front)
  uint8_t codemap[256];
  for (int k = 0; k < 256; ++k) codemap[k] = (uint8_t)k;
  std::vector<int32_t> lut;  // [plain | 4*v+3 - (4*go+1) | poison row]
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
    if ((int)syms.size() <= (s->table ? 128 : 64)) {
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
    } else if (s->table) {
      return -2;
    }
  }
  const bool piped = Gsel == 132;
  const int G = piped ? 32 : Gsel;
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull);  // (for maxm / maxn)
  const int P = 32 / G;
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t bound = ((int64_t)p.maxm + p.maxn + 2) * unit - (int64_t)sc.gap_open;
  int flags = scoring_flags(sc, bound, p.maxm, p.maxn);
  if (boundary8_ok(flags, bound)) flags |= F_BND8;
  const uint64_t full_tb = [&] {  // what the full path's plan would give the arena
    Plan q;
    build_plan(q, x_len, y_len, n_pairs, G, R, ~0ull, flags);
    return q.max_tb;
  }();
  flags |= F_NOTB;
  sims_last_flags = flags;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull, flags);
  if (p.max_tb != 0 || p.total_tb != 0) return -4;
  const int32_t* lut_plain = lut.data();
  const int32_t* lut_scaled = lut.data() + (size_t)sc.alpha * sc.alpha;
  const uint8_t gb = (uint8_t)garbage;
  std::vector<uint8_t> seq(p.seq_bytes, 0), bnd(p.max_bnd, gb), rows(p.max_rows, gb), rowm(p.max_rowm, gb);
  std::vector<uint8_t> tb;  // empty: data() is null
  if (poison >= 0) tb.assign(full_tb + 64, (uint8_t)poison);
  const std::vector<uint8_t> tb_before = tb;
  for (const Block& blk : p.blocks) {  // K0: [task][word][pair slot]
    uint32_t* seqw = reinterpret_cast<uint32_t*>(seq.data() + blk.seq_off);
    for (uint32_t q = 0; q < blk.npairs; ++q) {
      const uint32_t orig = p.order[blk.first + q];
      const uint32_t sub = q / P, slot = q % P;
      uint32_t* xw = seqw + (size_t)sub * blk.xwords * P;
      for (uint32_t k = 0; k < x_len[orig]; ++k)
        reinterpret_cast<uint8_t*>(&xw[(k >> 2) * P + slot])[k & 3] = codemap[blob[x_off[orig] + k]];
      uint32_t* yw = seqw + (size_t)G * blk.xwords * P + (size_t)sub * blk.ywords * P;
      for (uint32_t k = 0; k < y_len[orig]; ++k)
        reinterpret_cast<uint8_t*>(&yw[(k >> 2) * P + slot])[k & 3] = codemap[blob[y_off[orig] + k]];
    }
  }
  for (const Block& blk : p.blocks) {
    switch ((piped ? 10000 : 0) + G * 100 + R) {
      case 116: fill_dispatch_notb<1, 16, false>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 820: fill_dispatch_notb<8, 20, false>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 13208: fill_dispatch_notb<32, 8, true>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      default: return -1;
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
      v.sub = (int32_t)lane / P;
      v.g = (int32_t)lane % P;
      v.packtrk = (flags & F_PACKTRK) ? 1 : 0;
      v.bnd8 = (flags & F_BND8) ? 1 : 0;
      v.maxn = (int32_t)blk.maxn;
      v.bnd_base = bnd_index(G, 0, (int32_t)lane, v.maxn);
      v.bnd_stride = (int32_t)(bnd_index(G, 1, (int32_t)lane, v.maxn) - v.bnd_base);
      const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
      v.xw = seqw + (size_t)v.sub * blk.xwords * P + v.g;
      v.yw = seqw + (size_t)G * blk.xwords * P + (size_t)v.sub * blk.ywords * P + v.g;
      v.bnd = reinterpret_cast<const int4*>(bnd.data() + blk.bnd_off);
      v.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
      v.rows_pad = (int32_t)blk.rows_pad;
      v.rowm = reinterpret_cast<uint16_t*>(rowm.data() + blk.rowm_off);
      v.tb = tb.empty() ? nullptr : reinterpret_cast<const uint32_t*>(tb.data() + blk.tb_off);
      WalkOut o;
      if (warp_walk) {
        LaneFibers::run([&](int l) {
          WalkOut mine;
          walk_pair_coop<32, true>(l, v, mode == 2 || mode == 3, nullptr, mine);
          if (l == 0) o = mine;
        });
      } else {
        walk_pair<true>(v, mode == 2 || mode == 3, nullptr, o);
      }
      const uint32_t dst = p.order[sp];
      // as walk_store<true>: a panicking pair reports MIN_SCORE and no coordinates
      score[dst] = o.status ? MIN_SCORE : o.score;
      xend[dst] = o.status ? 0u : o.xend;
      yend[dst] = o.status ? 0u : o.yend;
      status[dst] = o.status;
    }
  }
  if (tb != tb_before) return -3;
  return 0;
}

int sims_fill_flags() { return sims_last_flags; }

// the plan of a batch for `flags` (F_NOTB: a score-only plan): its waves, and the traceback bytes in *total_tb
int sims_plan_waves(const uint32_t* x_len, const uint32_t* y_len, uint64_t n_pairs, int G, int R, uint64_t budget,
                    int flags, uint64_t* total_tb) {
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, budget, flags);
  *total_tb = p.total_tb;
  return (int)p.waves.size();
}

}  // extern "C"
