// CPU simulation of the fill + walk with the engine's boundary-record choice (F_BND8, b2a_plan.h boundary8_ok).
// Builds on the harness of b2a_sim.cpp (lane / warp emulation, fill_block, fill_block_piped, fill_dispatch) and adds
// one entry point that stages a batch like sim_align_batch_g does, but picks the flags as b2a_engine.cu's
// stage_front does -- scoring_flags(), then F_BND8 when boundary8_ok() -- sizes the plan for that record and runs the
// F_BND8 kernel variants where they apply.  Test tool only (tests/test_boundary_record.py).
#include "b2a_sim.cpp"

namespace {

int sim8_last_flags = 0;  // the flags the last sim8_align_batch ran its fill with (sim8_fill_flags)

template <int G, int R, bool PIPED = false>
void fill_dispatch8(int flags, const Plan& p, const Block& blk, const DevScoring& sc, const int32_t* lut,
                    std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                    std::vector<uint8_t>& tb) {
  if (!(flags & F_BND8)) {
    fill_dispatch<G, R, PIPED>(flags, p, blk, sc, lut, seq, bnd, rows, tb);
    return;
  }
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
#define SIM8_CASE(F)                                                                        \
  case (F):                                                                                 \
    if constexpr (PIPED) fill_block_piped<R, (F)>(p, blk, sc, lut, seq, bnd, rows, tb);     \
    else fill_block<G, R, (F)>(p, blk, sc, lut, seq, bnd, rows, tb);                        \
    break;
  switch (flags) {  // the F_BND8 instantiations of b2a_fill_inst.cu
    SIM8_CASE(F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIM8_CASE(ALL | F_PACKTRK | F_BND8)
    SIM8_CASE(ALL | F_PACKTRK | F_RELU | F_BND8)
    SIM8_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIM8_CASE(F_LUT | ALL | F_PACKTRK | F_BND8)
    SIM8_CASE(F_LUT | ALL | F_PACKTRK | F_RELU | F_BND8)
    default: std::abort();
  }
#undef SIM8_CASE
}

}  // namespace

extern "C" {

// Outputs as sim_align_batch_g; shapes 1x16, 8x20 and 132 (= 32x8 with strip-pipelined tasks); LUT scoring;
// warp_walk: K2 as walk_pair_coop<32> on 32 emulated lanes (else the one-lane walk_pair).
int sim8_align_batch(int mode, const sim_scoring* s, const uint8_t* blob, const uint64_t* x_off, const uint32_t* x_len,
                     const uint64_t* y_off, const uint32_t* y_len, uint64_t n_pairs, int Gsel, int R, int warp_walk,
                     int garbage, int32_t* score, uint32_t* xstart, uint32_t* xend, uint32_t* ystart,
                     uint32_t* yend, uint32_t* n_ops, uint32_t* clip_len, uint32_t* status, uint8_t* ops, const uint64_t* ops_off) {
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
  if (s->table) return -2;  // MatchParams only
  // alphabet + LUT as the engine builds them (b2a_engine.cu)
  uint8_t codemap[256];
  for (int k = 0; k < 256; ++k) codemap[k] = (uint8_t)k;
  bool present[256] = {false};
  for (uint64_t p = 0; p < n_pairs; ++p) {
    for (uint32_t k = 0; k < x_len[p]; ++k) present[blob[x_off[p] + k]] = true;
    for (uint32_t k = 0; k < y_len[p]; ++k) present[blob[y_off[p] + k]] = true;
  }
  std::vector<int> syms;
  for (int k = 0; k < 256; ++k)
    if (present[k]) syms.push_back(k);
  if (syms.empty()) syms.push_back(0);
  if (syms.size() > 64) return -2;  // LUT alphabets only
  for (size_t a = 0; a < syms.size(); ++a) codemap[syms[a]] = (uint8_t)a;
  sc.alpha = (int32_t)syms.size();
  const size_t aa = (size_t)sc.alpha * sc.alpha;
  std::vector<int32_t> lut(aa + (size_t)lut_entries(sc.alpha));  // [plain | 4*v+3]
  for (int a = 0; a < sc.alpha; ++a)
    for (int b = 0; b < sc.alpha; ++b) lut[(size_t)a * sc.alpha + b] = a == b ? s->match_score : s->mismatch_score;
  for (size_t k = 0; k < aa; ++k) lut[aa + k] = 4 * lut[k] + 3 - (4 * sc.gap_open + 1);
  for (size_t k = aa; k < (size_t)lut_entries(sc.alpha); ++k) lut[aa + k] = LUT_POISON;
  const int64_t maxabs = std::max<int64_t>(std::llabs((long long)s->match_score), std::llabs((long long)s->mismatch_score));

  const bool piped = Gsel == 132;
  const int G = piped ? 32 : Gsel;
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull);  // (for maxm / maxn)
  const int P = 32 / G;
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t bound = ((int64_t)p.maxm + p.maxn + 2) * unit - (int64_t)sc.gap_open;
  int flags = scoring_flags(sc, bound, p.maxm, p.maxn);
  if (boundary8_ok(flags, bound)) flags |= F_BND8;  // as stage_front
  sim8_last_flags = flags;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull, flags);  // the boundary arena sized for the record
  const int32_t* lut_plain = lut.data();
  const int32_t* lut_scaled = lut.data() + aa;
  // scratch starts as caller-chosen garbage: nothing may depend on its initial contents
  const uint8_t gb = (uint8_t)garbage;
  std::vector<uint8_t> seq(p.seq_bytes, 0), bnd(p.max_bnd, gb), rows(p.max_rows, gb), rowm(p.max_rowm, gb),
      tb(p.max_tb, gb), opsb(p.ops_bytes, 0);
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
      case 116: fill_dispatch8<1, 16>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 820: fill_dispatch8<8, 20>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 13208: fill_dispatch8<32, 8, true>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
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
      v.tb = reinterpret_cast<const uint32_t*>(tb.data() + blk.tb_off);
      const uint32_t cap = blk.maxm + blk.maxn + 4;
      uint8_t* ops_end = opsb.data() + blk.ops_off + (size_t)(lane + 1) * cap;
      WalkOut o;
      if (warp_walk) {
        LaneFibers::run([&](int l) {
          WalkOut mine;
          walk_pair_coop<32>(l, v, mode == 2 || mode == 3, ops_end, mine);
          if (l == 0) o = mine;
        });
      } else {
        walk_pair(v, mode == 2 || mode == 3, ops_end, o);
      }
      const uint32_t dst = p.order[sp];
      score[dst] = o.score;
      xstart[dst] = o.xstart;
      xend[dst] = o.xend;
      ystart[dst] = o.ystart;
      yend[dst] = o.yend;
      n_ops[dst] = o.n_ops;
      status[dst] = o.status;
      for (int k = 0; k < 4; ++k) clip_len[4 * (size_t)dst + k] = o.clip[k];
      std::memcpy(ops + ops_off[dst], ops_end - o.n_ops, o.n_ops);
    }
  }
  return 0;
}

// the 8-byte record choice (b2a_plan.h boundary8_ok), and the flags the last sim8_align_batch's fill ran with
int sim8_boundary8_ok(int flags, int64_t score_bound) { return boundary8_ok(flags, score_bound) ? 1 : 0; }
int sim8_fill_flags() { return sim8_last_flags; }

}  // extern "C"
