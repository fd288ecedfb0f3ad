// CPU simulation of the thread-per-pair fill that finishes each pair's matrix itself (F_FINISH, b2a_fill.cuh) and of
// K2 on top of it.  Builds on the harness of b2a_sim.cpp (lane emulation, LaneFibers) and adds one entry point that
// stages a batch like sim8_align_batch does, picks the flags as b2a_engine.cu's stage_front / batch_stage_impl do --
// scoring_flags(), F_BND8 when boundary8_ok(), F_FINISH for G = 1 without F_PACKREL, F_NOTB for score-only batches --
// and runs the fill with those flags (or without F_FINISH, for the comparison) and K2 as one lane or 32 emulated lanes
// per pair.  Test tool only (tests/test_fused_finish.py).
#include "b2a_sim.cpp"

namespace {

int simf_last_flags = 0;

// fill_kernel's per-lane setup for G = 1, with the row-m arena and the finish region of F_FINISH
template <int R, int FLAGS>
void fill_block_fin(const Plan& p, const Block& blk, uint32_t b, const DevScoring& sc, const int32_t* lut,
                    std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                    std::vector<uint8_t>& rowm, std::vector<int32_t>& fin, std::vector<uint8_t>& tb) {
  constexpr int G = 1, P = 32, TBW = tbw_of(R);
  for (int lane = 0; lane < 32; ++lane) {
    LaneCtx<G> c;
    c.sc = sc;
    c.lut = lut;
    c.ge4 = 4 * sc.gap_extend;
    c.lut_base = 0;
    c.one = 1;
    c.only_strip = -1;
    c.prog_mine = nullptr;
    c.prog_prev = nullptr;
    const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
    c.xs = seqw;
    c.ys = seqw + (size_t)G * blk.xwords * P;
    c.g = lane;
    c.l = 0;
    c.lane = lane;
    c.pi = lane;
    const bool valid = (uint32_t)c.pi < blk.npairs;
    c.m = valid ? (int32_t)p.pm[blk.first + c.pi] : 0;
    c.n = valid ? (int32_t)p.pn[blk.first + c.pi] : 0;
    c.maxn = (int32_t)blk.maxn;
    c.maxm = (int32_t)blk.maxm;
    c.nstrips = (int32_t)blk.nstrips;
    c.K = (int32_t)blk.K;
    c.rows_pad = (int32_t)blk.rows_pad;
    c.uniform = blk.uniform != 0;
    c.bnd = reinterpret_cast<int4*>(bnd.data() + blk.bnd_off);
    c.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
    c.tb = (FLAGS & F_NOTB) ? nullptr : reinterpret_cast<uint4*>(tb.data() + blk.tb_off);
    if (FLAGS & F_FINISH) {
      c.rowm = reinterpret_cast<uint16_t*>(rowm.data() + blk.rowm_off);
      c.fin = fin.data() + (size_t)b * FIN_FIELDS * 32;
    }
    (void)TBW;
    fill_lane<G, R, FLAGS>(c);
  }
}

template <int R>
bool fill_dispatch_fin(int flags, const Plan& p, const Block& blk, uint32_t b, const DevScoring& sc, const int32_t* lut,
                       std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                       std::vector<uint8_t>& rowm, std::vector<int32_t>& fin, std::vector<uint8_t>& tb) {
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
#define SIMF_ONE(F) \
  case (F): fill_block_fin<R, (F)>(p, blk, b, sc, lut, seq, bnd, rows, rowm, fin, tb); return true;
#define SIMF_CASE(F) SIMF_ONE(F) SIMF_ONE((F) | F_FINISH) SIMF_ONE((F) | F_NOTB) SIMF_ONE((F) | F_NOTB | F_FINISH)
  switch (flags) {  // the non-F_PACKREL cases of b2a_fill_inst.cu, with and without F_FINISH / F_NOTB
    SIMF_CASE(0)
    SIMF_CASE(F_TRACK_ROWS)
    SIMF_CASE(F_TRACK_ROWS | F_PACKTRK)
    SIMF_CASE(ALL)
    SIMF_CASE(ALL | F_PACKTRK)
    SIMF_CASE(ALL | F_RELU)
    SIMF_CASE(ALL | F_PACKTRK | F_RELU)
    SIMF_CASE(F_LUT)
    SIMF_CASE(F_LUT | F_TRACK_ROWS)
    SIMF_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK)
    SIMF_CASE(F_LUT | ALL)
    SIMF_CASE(F_LUT | ALL | F_PACKTRK)
    SIMF_CASE(F_LUT | ALL | F_RELU)
    SIMF_CASE(F_LUT | ALL | F_PACKTRK | F_RELU)
    SIMF_CASE(F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIMF_CASE(ALL | F_PACKTRK | F_BND8)
    SIMF_CASE(ALL | F_PACKTRK | F_RELU | F_BND8)
    SIMF_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK | F_BND8)
    SIMF_CASE(F_LUT | ALL | F_PACKTRK | F_BND8)
    SIMF_CASE(F_LUT | ALL | F_PACKTRK | F_RELU | F_BND8)
    default: return false;
  }
#undef SIMF_CASE
#undef SIMF_ONE
}

}  // namespace

extern "C" {

// Outputs as sim_align_batch_g (score-only: score, xend, yend and status; the rest stay 0), G = 1, R = 8 or 16.
// bits: 2 explicit (value, index) trackers (no F_PACKTRK / F_BND8), 4 MatchParams compare path (no LUT), 8 K2 as
// walk_pair_coop<32> on 32 emulated lanes, 32 score-only (F_NOTB fill, the score-only K2), 64 no F_FINISH (K2's own
// finish, the comparison), 128 check the rows arena's S, I and Sn arrays of every finished pair: none of their words
// may differ from the garbage byte afterwards (untouched[0] = 1 when none does).
int simf_align_batch(int mode, const sim_scoring* s, const uint8_t* blob, const uint64_t* x_off, const uint32_t* x_len,
                     const uint64_t* y_off, const uint32_t* y_len, uint64_t n_pairs, int R, int bits, int garbage,
                     int32_t* score, uint32_t* xstart, uint32_t* xend, uint32_t* ystart, uint32_t* yend,
                     uint32_t* n_ops, uint32_t* clip_len, uint32_t* status, uint8_t* ops, const uint64_t* ops_off,
                     int32_t* untouched) {
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
  // alphabet + LUT as the engine builds them (b2a_engine.cu)
  uint8_t codemap[256];
  for (int k = 0; k < 256; ++k) codemap[k] = (uint8_t)k;
  std::vector<int32_t> lut;  // [plain | 4*v+3]
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
    const bool use_lut = s->table || !(bits & 4);
    if (use_lut) {
      if (syms.size() > 64) return -2;
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
  }
  const int G = 1, P = 32;
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull);  // (for maxm / maxn)
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t bound = ((int64_t)p.maxm + p.maxn + 2) * unit - (int64_t)sc.gap_open;
  int flags = scoring_flags(sc, bound, p.maxm, p.maxn);
  if (bits & 2) flags &= ~(F_PACKTRK | F_PACKREL);
  if (boundary8_ok(flags, bound)) flags |= F_BND8;  // as stage_front
  const bool scores = (bits & 32) != 0;
  if (scores) flags |= F_NOTB;
  if (!(flags & F_PACKREL) && !(bits & 64)) flags |= F_FINISH;  // as batch_stage_impl for G = 1
  if (flags & F_PACKREL) return -3;                                // (the long-sequence form is out of scope here)
  simf_last_flags = flags;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull, flags);
  const int32_t* lut_plain = lut.data();
  const int32_t* lut_scaled = lut.data() + (size_t)sc.alpha * sc.alpha;
  // scratch starts as caller-chosen garbage: nothing may depend on its initial contents
  const uint8_t gb = (uint8_t)garbage;
  std::vector<uint8_t> seq(p.seq_bytes, 0), bnd(p.max_bnd, gb), rows(p.max_rows, gb), rowm(p.max_rowm, gb),
      tb(p.max_tb, gb), opsb(p.ops_bytes, 0);
  std::vector<int32_t> fin(p.max_fin / 4 + 1);
  std::memset(fin.data(), gb, fin.size() * 4);
  for (const Block& blk : p.blocks) {  // K0: [task][word][pair slot]
    uint32_t* seqw = reinterpret_cast<uint32_t*>(seq.data() + blk.seq_off);
    for (uint32_t q = 0; q < blk.npairs; ++q) {
      const uint32_t orig = p.order[blk.first + q];
      for (uint32_t k = 0; k < x_len[orig]; ++k)
        reinterpret_cast<uint8_t*>(&seqw[(k >> 2) * P + q])[k & 3] = codemap[blob[x_off[orig] + k]];
      uint32_t* yw = seqw + (size_t)blk.xwords * P;
      for (uint32_t k = 0; k < y_len[orig]; ++k)
        reinterpret_cast<uint8_t*>(&yw[(k >> 2) * P + q])[k & 3] = codemap[blob[y_off[orig] + k]];
    }
  }
  int32_t all_untouched = 1;
  for (uint32_t b = 0; b < (uint32_t)p.blocks.size(); ++b) {
    const Block& blk = p.blocks[b];
    const bool ok = R == 16 ? fill_dispatch_fin<16>(flags, p, blk, b, sc, lut_scaled, seq, bnd, rows, rowm, fin, tb)
                  : R == 8  ? fill_dispatch_fin<8>(flags, p, blk, b, sc, lut_scaled, seq, bnd, rows, rowm, fin, tb)
                            : false;
    if (!ok) return -1;
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
      v.sub = 0;
      v.g = (int32_t)lane;
      v.packtrk = (flags & F_PACKTRK) ? 1 : 0;
      v.bnd8 = (flags & F_BND8) ? 1 : 0;
      v.fin = (flags & F_FINISH) ? fin.data() + (size_t)b * FIN_FIELDS * 32 : nullptr;
      v.maxn = (int32_t)blk.maxn;
      v.bnd_base = bnd_index(G, 0, (int32_t)lane, v.maxn);
      v.bnd_stride = (int32_t)(bnd_index(G, 1, (int32_t)lane, v.maxn) - v.bnd_base);
      const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
      v.xw = seqw + v.g;
      v.yw = seqw + (size_t)blk.xwords * P + v.g;
      v.bnd = reinterpret_cast<const int4*>(bnd.data() + blk.bnd_off);
      v.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
      v.rows_pad = (int32_t)blk.rows_pad;
      v.rowm = reinterpret_cast<uint16_t*>(rowm.data() + blk.rowm_off);
      v.tb = reinterpret_cast<const uint32_t*>(tb.data() + blk.tb_off);
      const uint32_t cap = blk.maxm + blk.maxn + 4;
      uint8_t* ops_end = scores ? nullptr : opsb.data() + blk.ops_off + (size_t)(lane + 1) * cap;
      const bool filter = mode == 2 || mode == 3;
      WalkOut o;
      if (bits & 8) {
        LaneFibers::run([&](int l) {
          WalkOut mine;
          if (scores) walk_pair_coop<32, true>(l, v, filter, ops_end, mine);
          else walk_pair_coop<32>(l, v, filter, ops_end, mine);
          if (l == 0) o = mine;
        });
      } else if (scores) {
        walk_pair<true>(v, filter, ops_end, o);
      } else {
        walk_pair(v, filter, ops_end, o);
      }
      if ((bits & 128) && v.finished()) {  // S, I and Sn of every row slot of this pair: still the garbage
        for (int arr : {(int)ROWS_SL, (int)ROWS_IL, (int)ROWS_SN})
          for (int32_t i = 0; i < v.rows_pad; ++i) {
            const uint8_t* w = reinterpret_cast<const uint8_t*>(&v.row(arr, i));
            for (int k = 0; k < 4; ++k)
              if (w[k] != gb) all_untouched = 0;
          }
      }
      const uint32_t dst = p.order[sp];
      score[dst] = o.score;
      xend[dst] = o.xend;
      yend[dst] = o.yend;
      status[dst] = o.status;
      if (!scores) {
        xstart[dst] = o.xstart;
        ystart[dst] = o.ystart;
        n_ops[dst] = o.n_ops;
        for (int k = 0; k < 4; ++k) clip_len[4 * (size_t)dst + k] = o.clip[k];
        std::memcpy(ops + ops_off[dst], ops_end - o.n_ops, o.n_ops);
      }
    }
  }
  if (untouched) *untouched = all_untouched;
  return 0;
}

// the flags the last simf_align_batch ran its fill with
int simf_fill_flags() { return simf_last_flags; }

}  // extern "C"
