// CPU simulation harness for the kernel LOGIC (test tool, not a product path and
// not a fallback: nothing in rust_bio_b200/ loads it).  It compiles the very same
// per-lane code the GPU runs -- fill_lane<G,R,FLAGS> (b2a_fill.cuh), walk_pair (b2a_walk.cuh) and
// the banded K4/K3 functions (b2a_banded.cuh) -- for the host, stages a batch exactly as K0 does, and
// lets the not-gpu tests diff the result against the oracle without a GPU.  The thread-per-pair fill
// shape (G = 1) needs no warp primitives and runs lane after lane; the shapes whose lanes exchange
// values (G > 1 fill wavefront, the W = 32 banded kernels) run on 32 cooperatively scheduled contexts
// that stand in for the lanes of one warp (B2A_HOST_WARP hooks in b2a_common.cuh).
#define B2A_HOST_WARP 1
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <functional>
#include <vector>

#include <ucontext.h>

#include "../../rust_bio_b200/csrc/b2a_fill.cuh"
#include "../../rust_bio_b200/csrc/b2a_plan.h"
#include "../../rust_bio_b200/csrc/b2a_walk.cuh"

using namespace b2a;

// 32 cooperatively scheduled contexts of this thread stand in for the lanes of one warp (see HostWarp in
// b2a_common.cuh): a barrier switches to the next unfinished lane, round robin.
struct LaneFibers {
  static constexpr int W = 32;
  static constexpr size_t kStack = 512 * 1024;
  ucontext_t main_ctx;
  ucontext_t ctx[W];
  std::vector<char> stacks;
  bool done[W];
  int cur = 0;
  std::function<void(int)> body;
  HostWarp hw;
  static LaneFibers* self;

  static void entry() {
    LaneFibers* f = self;
    f->body(f->cur);
    f->done[f->cur] = true;
    next_lane(f);
  }
  static void next_lane(void* p) {
    LaneFibers* f = static_cast<LaneFibers*>(p);
    const int from = f->cur;
    int to = -1;
    for (int d = 1; d <= W; ++d) {
      const int cand = (from + d) % W;
      if (!f->done[cand]) {
        to = cand;
        break;
      }
    }
    if (to == from) return;  // the only lane left: its barrier is a no-op
    if (to < 0) {            // every lane finished
      swapcontext(&f->ctx[from], &f->main_ctx);
      return;
    }
    f->cur = to;
    host_lane = to;
    swapcontext(&f->ctx[from], &f->ctx[to]);
  }
  static void run(std::function<void(int)> body) {
    LaneFibers f;
    f.body = std::move(body);
    f.stacks.resize(kStack * W);
    f.hw.next_lane = &LaneFibers::next_lane;
    f.hw.other_warp = nullptr;
    f.hw.harness = &f;
    self = &f;
    host_warp = &f.hw;
    for (int l = 0; l < W; ++l) {
      f.done[l] = false;
      getcontext(&f.ctx[l]);
      f.ctx[l].uc_stack.ss_sp = f.stacks.data() + kStack * l;
      f.ctx[l].uc_stack.ss_size = kStack;
      f.ctx[l].uc_link = nullptr;
      makecontext(&f.ctx[l], &LaneFibers::entry, 0);
    }
    f.cur = 0;
    host_lane = 0;
    swapcontext(&f.main_ctx, &f.ctx[0]);
    host_warp = nullptr;
    self = nullptr;
  }
};
LaneFibers* LaneFibers::self = nullptr;

// Several emulated warps at once, for the strip-pipelined fill: the lanes of a warp rotate at its barriers as in
// LaneFibers; a lane that polls another warp's progress word lets the next warp run (other_warp hook), so a
// consumer strip and the producer strip above it advance side by side like two resident warps.
struct WarpSet {
  static constexpr int W = 32;
  static constexpr size_t kStack = 256 * 1024;
  struct Warp {
    ucontext_t ctx[W];
    bool done[W];
    int cur = 0, ndone = 0;
    HostWarp hw;
    std::function<void(int)> body;
    std::vector<char> stacks;
  };
  std::vector<Warp*> warps;
  int curw = 0;
  ucontext_t main_ctx;
  uint64_t idle_spins = 0;
  static WarpSet* self;

  static void entry() {
    WarpSet* s = self;
    Warp* w = s->warps[s->curw];
    const int lane = w->cur;
    w->body(lane);
    w->done[lane] = true;
    w->ndone += 1;
    next_lane(s);
  }
  void enter(int nw) {  // continue warp nw at its current lane (never returns to a finished context)
    curw = nw;
    host_warp = &warps[nw]->hw;
    host_lane = warps[nw]->cur;
  }
  // leave the running context for another warp that still has work; false if there is none
  bool to_other_warp(ucontext_t* from) {
    const int n = (int)warps.size();
    for (int d = 1; d < n; ++d) {
      const int cand = (curw + d) % n;
      if (warps[cand]->ndone < W) {
        enter(cand);
        swapcontext(from, &warps[cand]->ctx[warps[cand]->cur]);
        return true;
      }
    }
    return false;
  }
  static void next_lane(void* p) {
    WarpSet* s = static_cast<WarpSet*>(p);
    Warp* w = s->warps[s->curw];
    const int from = w->cur;
    if (w->ndone == W) {  // this warp is finished: hand over for good
      if (!s->to_other_warp(&w->ctx[from])) swapcontext(&w->ctx[from], &s->main_ctx);
      return;
    }
    int to = -1;
    for (int d = 1; d <= W; ++d) {
      const int cand = (from + d) % W;
      if (!w->done[cand]) {
        to = cand;
        break;
      }
    }
    if (to == from) return;
    w->cur = to;
    host_lane = to;
    swapcontext(&w->ctx[from], &w->ctx[to]);
  }
  static void other_warp(void* p) {
    WarpSet* s = static_cast<WarpSet*>(p);
    Warp* w = s->warps[s->curw];
    if (!s->to_other_warp(&w->ctx[w->cur])) {
      if (++s->idle_spins > (1ull << 26)) std::abort();  // polling with nobody left to publish: a deadlock
    } else {
      s->idle_spins = 0;
    }
  }
  static void run(std::vector<std::function<void(int)>> bodies) {
    WarpSet s;
    for (auto& b : bodies) {
      Warp* w = new Warp();
      w->body = std::move(b);
      w->stacks.resize(kStack * W);
      w->hw.next_lane = &WarpSet::next_lane;
      w->hw.other_warp = &WarpSet::other_warp;
      w->hw.harness = &s;
      for (int l = 0; l < W; ++l) {
        w->done[l] = false;
        getcontext(&w->ctx[l]);
        w->ctx[l].uc_stack.ss_sp = w->stacks.data() + kStack * l;
        w->ctx[l].uc_stack.ss_size = kStack;
        w->ctx[l].uc_link = nullptr;
        makecontext(&w->ctx[l], &WarpSet::entry, 0);
      }
      s.warps.push_back(w);
    }
    if (!s.warps.empty()) {
      self = &s;
      s.enter(0);
      swapcontext(&s.main_ctx, &s.warps[0]->ctx[0]);
      self = nullptr;
      host_warp = nullptr;
    }
    for (Warp* w : s.warps) delete w;
  }
};
WarpSet* WarpSet::self = nullptr;


namespace {

template <int G, int R, int FLAGS>
void fill_block(const Plan& p, const Block& blk, const DevScoring& sc, const int32_t* lut,
                std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                std::vector<uint8_t>& tb) {
  constexpr int P = 32 / G, TBW = tbw_of(R);
  // one warp-task per `sub` (32/G pairs), set up like fill_kernel does
  for (int sub = 0; sub < G; ++sub) {
    auto lane_body = [&](int lane) {
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
      c.xs = seqw + (size_t)sub * blk.xwords * P;
      c.ys = seqw + (size_t)G * blk.xwords * P + (size_t)sub * blk.ywords * P;
      c.g = lane / G;
      c.l = lane % G;
      c.lane = lane;
      c.pi = sub * P + c.g;
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
      c.tb = reinterpret_cast<uint4*>(tb.data() + blk.tb_off) + (size_t)sub * blk.nstrips * blk.K * TBW * 32;
      fill_lane<G, R, FLAGS>(c);
    };
    if (G == 1) {
      for (int lane = 0; lane < 32; ++lane) lane_body(lane);  // no lane talks to another one
    } else {
      LaneFibers::run(lane_body);  // the wavefront hands rows from lane to lane: lock-step
    }
  }
}

// The warp-per-pair shape as the engine runs it: every (pair, strip) of the block is a task of its own warp, the
// strips of a pair run side by side and hand the boundary row over through a progress word per task
// (fill_kernel's strip tasks: only_strip, the staged x slice with its biased pointer, prog_mine / prog_prev).
template <int R, int FLAGS>
void fill_block_piped(const Plan& p, const Block& blk, const DevScoring& sc, const int32_t* lut,
                      std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd, std::vector<uint8_t>& rows,
                      std::vector<uint8_t>& tb) {
  constexpr int G = 32, P = 1, TBW = tbw_of(R);
  if (blk.nstrips == 0) return;
  std::vector<uint32_t> progress((size_t)32 * blk.nstrips, 0u);
  for (uint32_t sub = 0; sub < blk.npairs; ++sub) {  // padding pairs of the block have no tasks
    std::vector<std::function<void(int)>> bodies;
    std::vector<std::vector<uint32_t>> slices(blk.nstrips);
    for (uint32_t strip = 0; strip < blk.nstrips; ++strip) {
      const uint32_t task = sub * blk.nstrips + strip;
      const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
      // what the kernel stages: G*R symbols of x for this strip, all of y
      const uint32_t xoff_words = strip * G * R / 4;
      slices[strip].assign(seqw + (size_t)sub * blk.xwords * P + xoff_words,
                           seqw + (size_t)sub * blk.xwords * P + xoff_words + G * R / 4);
      const uint32_t* xs_biased = slices[strip].data() - xoff_words;  // indexed by absolute row word
      uint32_t* prog = progress.data();
      bodies.push_back([&, task, strip, sub, xs_biased, prog, seqw](int lane) {
        LaneCtx<G> c;
        c.sc = sc;
        c.lut = lut;
        c.ge4 = 4 * sc.gap_extend;
        c.lut_base = 0;
        c.one = 1;
        c.only_strip = (int32_t)strip;
        c.prog_mine = prog + task;
        c.prog_prev = strip > 0 ? prog + task - 1 : nullptr;
        c.xs = xs_biased;
        c.ys = seqw + (size_t)G * blk.xwords * P + (size_t)sub * blk.ywords * P;
        c.g = 0;
        c.l = lane;
        c.lane = lane;
        c.pi = (int32_t)sub;
        c.m = (int32_t)p.pm[blk.first + sub];
        c.n = (int32_t)p.pn[blk.first + sub];
        c.maxn = (int32_t)blk.maxn;
        c.maxm = (int32_t)blk.maxm;
        c.nstrips = (int32_t)blk.nstrips;
        c.K = (int32_t)blk.K;
        c.rows_pad = (int32_t)blk.rows_pad;
        c.uniform = blk.uniform != 0;
        c.bnd = reinterpret_cast<int4*>(bnd.data() + blk.bnd_off);
        c.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
        c.tb = reinterpret_cast<uint4*>(tb.data() + blk.tb_off) + (size_t)sub * blk.nstrips * blk.K * TBW * 32;
        fill_lane<G, R, FLAGS>(c);
      });
    }
    // consumers first on odd pairs: they poll before their producer has run at all; producers yield at every
    // publish, so the strips advance 16 columns at a time, side by side
    if (sub & 1) std::reverse(bodies.begin(), bodies.end());
    WarpSet::run(std::move(bodies));
  }
}

template <int G, int R, bool PIPED = false>
void fill_dispatch(int flags, const Plan& p, const Block& blk, const DevScoring& sc,
                   const int32_t* lut, std::vector<uint8_t>& seq, std::vector<uint8_t>& bnd,
                   std::vector<uint8_t>& rows, std::vector<uint8_t>& tb) {
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
#define SIM_CASE(F)                                                                         \
  case (F):                                                                                 \
    if constexpr (PIPED) fill_block_piped<R, (F)>(p, blk, sc, lut, seq, bnd, rows, tb);     \
    else fill_block<G, R, (F)>(p, blk, sc, lut, seq, bnd, rows, tb);                        \
    break;
  switch (flags) {
    SIM_CASE(0)
    SIM_CASE(F_TRACK_ROWS)
    SIM_CASE(F_TRACK_ROWS | F_PACKTRK)
    SIM_CASE(ALL)
    SIM_CASE(ALL | F_PACKTRK)
    SIM_CASE(F_LUT)
    SIM_CASE(F_LUT | F_TRACK_ROWS)
    SIM_CASE(F_LUT | F_TRACK_ROWS | F_PACKTRK)
    SIM_CASE(F_LUT | ALL)
    SIM_CASE(F_LUT | ALL | F_PACKTRK)
    SIM_CASE(ALL | F_RELU)
    SIM_CASE(ALL | F_PACKTRK | F_RELU)
    SIM_CASE(F_LUT | ALL | F_RELU)
    SIM_CASE(F_LUT | ALL | F_PACKTRK | F_RELU)
    SIM_CASE(F_TRACK_ROWS | F_PACKREL)
    SIM_CASE(ALL | F_PACKREL)
    SIM_CASE(ALL | F_PACKREL | F_RELU)
    SIM_CASE(F_LUT | F_TRACK_ROWS | F_PACKREL)
    SIM_CASE(F_LUT | ALL | F_PACKREL)
    SIM_CASE(F_LUT | ALL | F_PACKREL | F_RELU)
    default: std::abort();
  }
}

}  // namespace

extern "C" {

struct sim_scoring {
  int32_t gap_open, gap_extend, xclip_prefix, xclip_suffix, yclip_prefix, yclip_suffix;
  int32_t match_score, mismatch_score, has_match_scores;
  const int32_t* table;
  const uint8_t* alphabet;
  uint32_t alphabet_len;
};

// Same outputs as the engine: per pair score/xstart/xend/ystart/yend/n_ops/clip_len[4]/status and
// ops (m+n+4 bytes per pair at ops + ops_off[p], alignment order).
int sim_align_batch_g(int mode, const sim_scoring* s, const uint8_t* blob, const uint64_t* x_off,
                    const uint32_t* x_len, const uint64_t* y_off, const uint32_t* y_len,
                    uint64_t n_pairs, int Gsel /* lanes per pair; 132 = 32 with strip-pipelined tasks */, int R, int modebits /*1 general variant, 2 no packed trackers, 4 no LUT for MatchParams*/, int garbage, int32_t* score, uint32_t* xstart,
                    uint32_t* xend, uint32_t* ystart, uint32_t* yend, uint32_t* n_ops,
                    uint32_t* clip_len, uint32_t* status, uint8_t* ops, const uint64_t* ops_off) {
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
  // alphabet + LUT exactly as the engine builds them (b2a_engine.cu): LUT whenever <= 64 symbols
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
    const bool use_lut = s->table || !(modebits & 4);  // modebits & 4: force MatchParams compare path
    if (use_lut && syms.size() <= 64) {
      for (size_t a = 0; a < syms.size(); ++a) codemap[syms[a]] = (uint8_t)a;
      sc.alpha = (int32_t)syms.size();
      const size_t aa = (size_t)sc.alpha * sc.alpha;
      lut.resize(aa + (size_t)lut_entries(sc.alpha));
      if (s->table) maxabs = 0;
      for (int a = 0; a < sc.alpha; ++a)
        for (int b = 0; b < sc.alpha; ++b) {
          const int32_t v = s->table ? s->table[syms[a] * 256 + syms[b]]
                                     : (a == b ? s->match_score : s->mismatch_score);
          lut[(size_t)a * sc.alpha + b] = v;
          maxabs = std::max<int64_t>(maxabs, std::llabs((long long)v));
        }
      for (size_t k = 0; k < aa; ++k) lut[aa + k] = 4 * lut[k] + 3 - (4 * sc.gap_open + 1);
      for (size_t k = aa; k < (size_t)lut_entries(sc.alpha); ++k) lut[aa + k] = LUT_POISON;
    }
  }
  const bool piped = Gsel == 132;
  const int G = piped ? 32 : Gsel;
  Plan p;
  build_plan(p, x_len, y_len, n_pairs, G, R, ~0ull);
  const int P = 32 / G;
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t bound = ((int64_t)p.maxm + p.maxn + 2) * unit - (int64_t)sc.gap_open;
  int flags = scoring_flags(sc, bound, p.maxm, p.maxn);
  if (modebits & 1) {
    flags |= F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
    if (bound < (1ll << 17) && p.maxm <= 4095 && p.maxn <= 4095) flags |= F_PACKTRK;
  }
  if (modebits & 2) flags &= ~(F_PACKTRK | F_PACKREL);
  if ((modebits & 16) && (flags & (F_TRACK_ROWS | F_TRACK_COLS))) {  // the long-sequence form of the packed trackers
    flags &= ~F_PACKTRK;
    flags |= F_PACKREL;
  }
  const int32_t* lut_plain = lut.data();
  const int32_t* lut_scaled = lut.data() + (size_t)sc.alpha * sc.alpha;
  // scratch starts as caller-chosen garbage: nothing may depend on its initial contents
  const uint8_t gb = (uint8_t)garbage;
  std::vector<uint8_t> seq(p.seq_bytes, 0), bnd(p.max_bnd, gb), rows(p.max_rows, gb),
      rowm(p.max_rowm, gb), tb(p.max_tb, gb), opsb(p.ops_bytes, 0);
  // K0 equivalent: stage sequences as [task][word][pair slot] (b2a_kernels.cuh pack_kernel)
  for (const Block& blk : p.blocks) {
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
      case 104: fill_dispatch<1, 4>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 108: fill_dispatch<1, 8>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 116: fill_dispatch<1, 16>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 416: fill_dispatch<4, 16>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 808: fill_dispatch<8, 8>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 820: fill_dispatch<8, 20>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 3208: fill_dispatch<32, 8>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
      case 13208: fill_dispatch<32, 8, true>(flags, p, blk, sc, lut_scaled, seq, bnd, rows, tb); break;
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
      if (modebits & 8) {  // the warp-per-pair K2: 32 emulated lanes on this pair
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

int sim_align_batch(int mode, const sim_scoring* s, const uint8_t* blob, const uint64_t* x_off,
                    const uint32_t* x_len, const uint64_t* y_off, const uint32_t* y_len, uint64_t n_pairs, int R,
                    int modebits, int garbage, int32_t* score, uint32_t* xstart, uint32_t* xend, uint32_t* ystart,
                    uint32_t* yend, uint32_t* n_ops, uint32_t* clip_len, uint32_t* status, uint8_t* ops,
                    const uint64_t* ops_off) {
  return sim_align_batch_g(mode, s, blob, x_off, x_len, y_off, y_len, n_pairs, 1, R, modebits, garbage, score, xstart,
                           xend, ystart, yend, n_ops, clip_len, status, ops, ops_off);
}
}

// ---------------------------------------------------------------------------------------------
// Banded path: the device functions of b2a_banded.cuh (K4 band construction + K3 banded fill/walk)
// compiled for the host, one pair at a time.
#include "../../rust_bio_b200/csrc/b2a_banded.cuh"

extern "C" int sim_banded_batch(int mode, const sim_scoring* s, uint32_t k, uint32_t w, const uint8_t* blob,
                                const uint64_t* x_off, const uint32_t* x_len, const uint64_t* y_off,
                                const uint32_t* y_len, uint64_t n_pairs, uint32_t cap_matches, int garbage,
                                int32_t* score, uint32_t* xstart, uint32_t* xend, uint32_t* ystart,
                                uint32_t* yend, uint32_t* n_ops, uint32_t* clip_len, uint32_t* status,
                                uint64_t* num_cells, uint64_t* ranges_out /*optional: 2*(n+1) per pair, flat*/,
                                uint8_t* ops, const uint64_t* ops_off) {
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
  const int32_t* table = s->table;
  uint64_t rpos = 0;
  for (uint64_t p = 0; p < n_pairs; ++p) {
    const uint64_t m = x_len[p], n = y_len[p];
    const uint8_t* x = blob + x_off[p];
    const uint8_t* y = blob + y_off[p];
    std::vector<uint8_t> slab(k4_slab_bytes(cap_matches, (uint32_t)std::min(m, n)), (uint8_t)garbage);
    std::vector<uint32_t> rng(2 * (n + 1), 0xCDCDCDCDu);
    uint64_t cells = 0;
    std::vector<uint32_t> shared_vec(K4_SHARED_WORDS, 0u);
    uint32_t* shared_u32 = shared_vec.data();
    const uint32_t st = band_create_d<1>(0, x, m, y, n, k, w, sc, s->has_match_scores, slab.data(), cap_matches,
                                         rng.data(), &cells, shared_u32);
    num_cells[p] = cells;
    if (ranges_out) {
      for (uint64_t j = 0; j <= n; ++j) {
        ranges_out[rpos + 2 * j] = rng[2 * j];
        ranges_out[rpos + 2 * j + 1] = rng[2 * j + 1];
      }
      rpos += 2 * (n + 1);
    }
    BandedOut o{};
    std::vector<uint8_t> opsbuf(m + n + 16, 0);
    if (st != 0) {
      o.status = 1 + st;
    } else {
      std::vector<uint8_t> fill(k3_slab_bytes(m, n, cells), (uint8_t)garbage);
      auto scoref = [&](uint8_t a, uint8_t b) -> int32_t {
        if (table) return table[(size_t)a * 256 + b];
        return a == b ? sc.match_score : sc.mismatch_score;
      };
      banded_compute_d<1>(0, x, m, y, n, sc, scoref, rng.data(), cells, fill.data(), mode == 2 || mode == 3,
                       opsbuf.data() + opsbuf.size(), o);
    }
    score[p] = o.score;
    xstart[p] = o.xstart;
    xend[p] = o.xend;
    ystart[p] = o.ystart;
    yend[p] = o.yend;
    n_ops[p] = o.n_ops;
    status[p] = o.status;
    for (int q = 0; q < 4; ++q) clip_len[4 * p + q] = o.clip[q];
    std::memcpy(ops + ops_off[p], opsbuf.data() + opsbuf.size() - o.n_ops, o.n_ops);
  }
  return 0;
}

// One pair through K4 with caller-supplied band inputs (banded.rs:313-401) + K3; custom mode (clips kept).
extern "C" int sim_banded_hinted_one(const sim_scoring* s, uint32_t k, uint32_t w, const uint8_t* x, uint32_t m32,
                                     const uint8_t* y, uint32_t n32, const uint32_t* match_xy, uint64_t n_matches,
                                     const uint32_t* path_idx, uint64_t n_path, int have_path,
                                     int allowed_mismatches, int use_lcskpp_union, uint32_t cap_matches, int garbage,
                                     int32_t* score, uint32_t* coords /*xstart,xend,ystart,yend*/, uint32_t* n_ops,
                                     uint32_t* clip_len, uint32_t* status, uint64_t* num_cells, uint8_t* ops) {
  DevScoring sc{};
  sc.gap_open = s->gap_open;
  sc.gap_extend = s->gap_extend;
  sc.xclip_prefix = s->xclip_prefix;
  sc.xclip_suffix = s->xclip_suffix;
  sc.yclip_prefix = s->yclip_prefix;
  sc.yclip_suffix = s->yclip_suffix;
  sc.match_score = s->match_score;
  sc.mismatch_score = s->mismatch_score;
  const int32_t* table = s->table;
  const uint64_t m = m32, n = n32;
  std::vector<uint8_t> slab(k4_slab_bytes(cap_matches, (uint32_t)std::min(m, n)), (uint8_t)garbage);
  std::vector<uint32_t> rng(2 * (n + 1), 0xCDCDCDCDu);
  BandHintsD hint;
  hint.mxy = match_xy;
  hint.n_matches = n_matches;
  hint.pidx = path_idx;
  hint.n_path = n_path;
  hint.have_path = have_path != 0;
  hint.allowed_mismatches = allowed_mismatches;
  hint.use_lcskpp_union = use_lcskpp_union;
  uint64_t cells = 0;
  std::vector<uint32_t> shared_vec(K4_SHARED_WORDS, 0u);
    uint32_t* shared_u32 = shared_vec.data();
  const uint32_t st = band_create_d<1>(0, x, m, y, n, k, w, sc, s->has_match_scores, slab.data(), cap_matches,
                                       rng.data(), &cells, shared_u32, hint);
  *num_cells = cells;
  BandedOut o{};
  std::vector<uint8_t> opsbuf(m + n + 16, 0);
  if (st != 0) {
    o.status = 1 + st;
  } else {
    std::vector<uint8_t> fill(k3_slab_bytes(m, n, cells), (uint8_t)garbage);
    auto scoref = [&](uint8_t a, uint8_t b) -> int32_t {
      if (table) return table[(size_t)a * 256 + b];
      return a == b ? sc.match_score : sc.mismatch_score;
    };
    banded_compute_d<1>(0, x, m, y, n, sc, scoref, rng.data(), cells, fill.data(), false,
                        opsbuf.data() + opsbuf.size(), o);
  }
  *score = o.score;
  coords[0] = o.xstart;
  coords[1] = o.xend;
  coords[2] = o.ystart;
  coords[3] = o.yend;
  *n_ops = o.n_ops;
  *status = o.status;
  for (int q = 0; q < 4; ++q) clip_len[q] = o.clip[q];
  std::memcpy(ops, opsbuf.data() + opsbuf.size() - o.n_ops, o.n_ops);
  return 0;
}


static int g_last_banded_fast = 0;
extern "C" int sim_last_banded_fast() { return g_last_banded_fast; }

// The W = 32 instantiations of K4 and K3 (what the GPU runs) with 32 host contexts as the lanes of one warp.
// Same interface and outputs as sim_banded_hinted_one; have_matches = 0 lets K4 find the matches itself.
extern "C" int sim_banded_warp32_one(int mode, const sim_scoring* s, uint32_t k, uint32_t w, const uint8_t* x,
                                     uint32_t m32, const uint8_t* y, uint32_t n32, int have_matches,
                                     const uint32_t* match_xy, uint64_t n_matches, const uint32_t* path_idx,
                                     uint64_t n_path, int have_path, int allowed_mismatches, int use_lcskpp_union,
                                     uint32_t cap_matches, int garbage, int32_t* score, uint32_t* coords,
                                     uint32_t* n_ops, uint32_t* clip_len, uint32_t* status, uint64_t* num_cells,
                                     uint64_t* ranges_out /*2*(n+1) or null*/, uint8_t* ops) {
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
  const int32_t* table = s->table;
  const uint64_t m = m32, n = n32;
  std::vector<uint8_t> slab(k4_slab_bytes(cap_matches, (uint32_t)std::min(m, n)), (uint8_t)garbage);
  std::vector<uint32_t> rng(2 * (n + 1), 0xCDCDCDCDu);
  BandHintsD hint;
  if (have_matches) {
    hint.mxy = match_xy;
    hint.n_matches = n_matches;
  }
  hint.pidx = path_idx;
  hint.n_path = n_path;
  hint.have_path = have_path != 0;
  hint.allowed_mismatches = allowed_mismatches;
  hint.use_lcskpp_union = use_lcskpp_union;
  std::vector<uint32_t> shared_vec(K4_SHARED_WORDS, 0u);
    uint32_t* shared_u32 = shared_vec.data();
  uint32_t st_lane[32];
  uint64_t cells_lane[32];
  auto run32 = [&](std::function<void(int)> body) { LaneFibers::run(body); };
  run32([&](int l) {
    uint64_t c = 0;
    st_lane[l] = band_create_d<32>(l, x, m, y, n, k, w, sc, s->has_match_scores, slab.data(), cap_matches, rng.data(),
                                   &c, shared_u32, hint);
    cells_lane[l] = c;
  });
  for (int l = 1; l < 32; ++l)
    if (st_lane[l] != st_lane[0] || cells_lane[l] != cells_lane[0]) return -1;  // lanes must agree
  const uint32_t st = st_lane[0];
  const uint64_t cells = cells_lane[0];
  *num_cells = cells;
  if (ranges_out)
    for (uint64_t j = 0; j <= n; ++j) {
      ranges_out[2 * j] = rng[2 * j];
      ranges_out[2 * j + 1] = rng[2 * j + 1];
    }
  BandedOut o{};
  std::vector<uint8_t> opsbuf(m + n + 16, 0);
  if (st != 0) {
    o.status = 1 + st;
  } else {
    std::vector<uint8_t> fill(k3_slab_bytes(m, n, cells), (uint8_t)garbage);
    auto scoref = [&](uint8_t a, uint8_t b) -> int32_t {
      if (table) return table[(size_t)a * 256 + b];
      return a == b ? sc.match_score : sc.mismatch_score;
    };
    // as on the device: the register-resident column loop for the pairs whose band suits it (unless the test
    // asks for the literal loop), the literal loop otherwise
    bool fast_lane[32];
    run32([&](int l) { fast_lane[l] = cells <= BANDED_MAX_CELLS && banded_fast_ok<32, K3_FAST_ROWS>(l, rng.data(), m, n); });
    const bool fast = fast_lane[0] && !getenv("B2A_SIM_BANDED_LITERAL");
    g_last_banded_fast = fast ? 1 : 0;
    run32([&](int l) {
      BandedOut mine{};
      if (fast)
        banded_compute_d<32, decltype(scoref), K3_FAST_ROWS>(l, x, m, y, n, sc, scoref, rng.data(), cells, fill.data(),
                                                             mode == 2 || mode == 3, opsbuf.data() + opsbuf.size(), mine);
      else
        banded_compute_d<32>(l, x, m, y, n, sc, scoref, rng.data(), cells, fill.data(), mode == 2 || mode == 3,
                             opsbuf.data() + opsbuf.size(), mine);
      if (l == 0) o = mine;
    });
  }
  *score = o.score;
  coords[0] = o.xstart;
  coords[1] = o.xend;
  coords[2] = o.ystart;
  coords[3] = o.yend;
  *n_ops = o.n_ops;
  *status = o.status;
  for (int q = 0; q < 4; ++q) clip_len[q] = o.clip[q];
  std::memcpy(ops, opsbuf.data() + opsbuf.size() - o.n_ops, o.n_ops);
  return 0;
}


// ---------------------------------------------------------------------------------------------
// The strip-wavefront banded fill (b2a_banded_strip.cuh) as the GPU runs it: K4 per pair on an emulated warp, then ONE
// warp-task of up to four pairs (8 emulated lanes each) through ks_run_task, then the finish pass per pair.
// path[p]: 1 = the strip path produced the result, 0 = not eligible / handed back (no result reported).
#include "../../rust_bio_b200/csrc/b2a_banded_strip.cuh"

extern "C" int sim_banded_strip_task(int mode, const sim_scoring* s, uint32_t k, uint32_t w, const uint8_t* blob,
                                     uint64_t blob_bytes, const uint64_t* x_off, const uint32_t* x_len, const uint64_t* y_off,
                                     const uint32_t* y_len, uint32_t n_pairs, uint32_t cap_matches, int garbage,
                                     int32_t* score, uint32_t* coords /*4 per pair*/, uint32_t* n_ops,
                                     uint32_t* clip_len, uint32_t* status, uint32_t* path, uint8_t* ops,
                                     const uint64_t* ops_off) {
  if (n_pairs > 4) return -2;
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
  const int32_t* table = s->table;
  auto run32 = [&](std::function<void(int)> body) { LaneFibers::run(body); };
  // the alphabet as the engine's stage_front finds it: the caller's, else every byte value of the blob in one flat pass
  // (the padding between sequences included)
  std::vector<int> syms;
  {
    std::vector<bool> present(256, false);
    if (s->alphabet && s->alphabet_len) {
      for (uint32_t q = 0; q < s->alphabet_len; ++q) present[s->alphabet[q]] = true;
    } else {
      for (uint64_t t = 0; t < blob_bytes; ++t) present[blob[t]] = true;
    }
    for (int b = 0; b < 256; ++b)
      if (present[b]) syms.push_back(b);
    if (syms.empty()) syms.push_back(0);
  }
  // tabulated MatchFunc: codes over that alphabet and K1's scaled LUT, as stage_front builds them
  std::vector<uint8_t> cmap(256, 0xFF);
  std::vector<int32_t> lut_scaled;
  if (table) {
    if (syms.size() > 128) return -3;
    sc.alpha = (int32_t)syms.size();
    for (int a = 0; a < sc.alpha; ++a) cmap[syms[a]] = (uint8_t)a;
    lut_scaled.resize((size_t)sc.alpha * sc.alpha);
    for (int a = 0; a < sc.alpha; ++a)
      for (int b = 0; b < sc.alpha; ++b)
        lut_scaled[(size_t)a * sc.alpha + b] = 4 * table[(size_t)syms[a] * 256 + syms[b]] + 3 - (4 * sc.gap_open + 1);
  }
  // the host's part of the decision (b2a_engine.cu banded_impl): score_bound as stage_front computes it (the largest
  // |score| over that alphabet), then the gate of b2a_plan.h
  uint32_t maxm = 0, maxn = 0;
  for (uint32_t p = 0; p < n_pairs; ++p) {
    maxm = std::max(maxm, x_len[p]);
    maxn = std::max(maxn, y_len[p]);
  }
  int64_t maxabs = std::max<int64_t>(std::llabs((long long)s->match_score), std::llabs((long long)s->mismatch_score));
  if (table) {
    maxabs = 0;
    for (int a : syms)
      for (int b : syms) maxabs = std::max<int64_t>(maxabs, std::llabs((long long)table[(size_t)a * 256 + b]));
  }
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t score_bound = ((int64_t)maxm + maxn + 2) * unit - (int64_t)sc.gap_open;
  const bool batch_ok = banded_strip_gate(sc, score_bound, maxm);
  std::vector<std::vector<uint32_t>> rngs(n_pairs);
  std::vector<uint64_t> cells(n_pairs, 0);
  std::vector<uint32_t> cols(3 * (size_t)n_pairs + 3, 0), k4(n_pairs, 0), elig;
  std::vector<uint64_t> roff(n_pairs, 0), foff(n_pairs, 0), soff(n_pairs, 0);
  std::vector<uint32_t> rng_all;
  std::vector<uint8_t> fill_all, strip_all;
  for (uint32_t p = 0; p < n_pairs; ++p) {
    const uint64_t m = x_len[p], n = y_len[p];
    const uint8_t* x = blob + x_off[p];
    const uint8_t* y = blob + y_off[p];
    std::vector<uint8_t> slab(k4_slab_bytes(cap_matches, (uint32_t)std::min(m, n)), (uint8_t)garbage);
    rngs[p].assign(2 * (n + 1), 0xCDCDCDCDu);
    BandHintsD hint;
    std::vector<uint32_t> shared_vec(K4_SHARED_WORDS, 0u);
    uint32_t* shared_u32 = shared_vec.data();
    uint32_t st_lane[32];
    uint64_t c_lane[32];
    run32([&](int l) {
      uint64_t c = 0;
      st_lane[l] = band_create_d<32>(l, x, m, y, n, k, w, sc, s->has_match_scores, slab.data(), cap_matches,
                                     rngs[p].data(), &c, shared_u32, hint);
      c_lane[l] = c;
    });
    cells[p] = c_lane[0];
    path[p] = 0;
    status[p] = 0;
    if (st_lane[0] != 0 || !batch_ok || cells[p] > BANDED_MAX_CELLS) continue;
    bool ok_lane[32];
    uint32_t c3[32][3];
    run32([&](int l) { ok_lane[l] = banded_strip_ok<32>(l, rngs[p].data(), m, n, c3[l], 0, ~0ull, !getenv("B2A_SIM_STRIP_NO_LASTCOL")); });
    if (!ok_lane[0]) continue;
    for (int q = 0; q < 3; ++q) cols[3 * p + q] = c3[0][q];
    k4[p] = 0x200u;
  }
  // arenas as the engine lays them out
  uint64_t rb = 0, fb = 0, sb = 0;
  for (uint32_t p = 0; p < n_pairs; ++p) {
    const uint64_t m = x_len[p], n = y_len[p];
    roff[p] = rb;
    rb += ((n + 1) * 8 + 15) & ~15ull;
    foff[p] = fb;
    fb += k3_slab_bytes(m, n, cells[p]);
    soff[p] = sb;
    if (k4[p]) {
      const uint64_t c0 = std::max<uint64_t>(cols[3 * p], 1), c1 = std::min<uint64_t>(cols[3 * p + 1], n - 1);
      sb += ks_layout(m, c1 >= c0 ? c1 - c0 + 1 : 0, cols[3 * p + 2]).total;
      elig.push_back(p);
    }
  }
  if (elig.empty()) return 0;
  rng_all.assign(rb / 4 + 4, 0);
  for (uint32_t p = 0; p < n_pairs; ++p) std::memcpy(rng_all.data() + roff[p] / 4, rngs[p].data(), rngs[p].size() * 4);
  fill_all.assign(fb + 16, (uint8_t)garbage);
  strip_all.assign(sb + 16, (uint8_t)garbage);
  uint32_t counter = 0;
  StripParams sp{};
  sp.blob = blob;
  sp.x_off = x_off;
  sp.x_len = x_len;
  sp.y_off = y_off;
  sp.y_len = y_len;
  sp.pair_lo = 0;
  sp.elig = elig.data();
  sp.n_elig = (uint32_t)elig.size();
  sp.task_counter = &counter;
  sp.ranges = rng_all.data();
  sp.ranges_off = roff.data();
  sp.fill = fill_all.data();
  sp.fill_off = foff.data();
  sp.strip = strip_all.data();
  sp.strip_off = soff.data();
  sp.num_cells = cells.data();
  sp.band_cols = cols.data();
  sp.k4_status = k4.data();
  sp.sc = sc;
  sp.one = 1;
  sp.ge4 = 4 * sc.gap_extend;
  const int fl = (sc.yclip_suffix > DEAD_CLIP ? (int)F_TRACK_ROWS : 0) | (sc.xclip_suffix > DEAD_CLIP ? (int)F_TRACK_COLS : 0) |
                 (sc.xclip_prefix > DEAD_CLIP ? (int)F_CLIPX : 0) | (sc.yclip_prefix > DEAD_CLIP ? (int)F_CLIPY : 0) |
                 (table ? (int)F_LUT : 0);
  uint32_t err_flag = 0;
  KsLut T{};
  T.lut = lut_scaled.data();
  T.lut_base = 0;
  T.cmap = cmap.data();
  T.err_flag = &err_flag;
  sp.sc = sc;
  run32([&](int l) {
    switch (fl) {
#define SIM_KS_CASE1(F) \
  case (F): ks_run_task<(F)>(sp, T, 0, l); break;
#define SIM_KS_CASE(F) SIM_KS_CASE1(F) SIM_KS_CASE1((F) | F_LUT)
      SIM_KS_CASE(0)
      SIM_KS_CASE(F_TRACK_ROWS)
      SIM_KS_CASE(F_CLIPX)
      SIM_KS_CASE(F_CLIPY)
      SIM_KS_CASE(F_TRACK_ROWS | F_CLIPX)
      SIM_KS_CASE(F_TRACK_ROWS | F_CLIPY)
      SIM_KS_CASE(F_CLIPX | F_CLIPY)
      SIM_KS_CASE(F_TRACK_ROWS | F_CLIPX | F_CLIPY)
      SIM_KS_CASE(F_TRACK_COLS)
      SIM_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS)
      SIM_KS_CASE(F_TRACK_COLS | F_CLIPX)
      SIM_KS_CASE(F_TRACK_COLS | F_CLIPY)
      SIM_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPX)
      SIM_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPY)
      SIM_KS_CASE(F_TRACK_COLS | F_CLIPX | F_CLIPY)
      SIM_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPX | F_CLIPY)
#undef SIM_KS_CASE
#undef SIM_KS_CASE1
    }
  });
  for (uint32_t p : elig) {
    if (k4[p] & 0x400u) continue;  // the fill handed the pair back
    const uint64_t m = x_len[p], n = y_len[p];
    const uint8_t* x = blob + x_off[p];
    const uint8_t* y = blob + y_off[p];
    auto scoref = [&](uint8_t a, uint8_t b) -> int32_t {
      if (table) return table[(size_t)a * 256 + b];
      return a == b ? sc.match_score : sc.mismatch_score;
    };
    std::vector<uint8_t> opsbuf(m + n + 16, 0);
    BandedOut o{};
    bool redo = false;
    // as on the device: phase 1 (everything up to the final score) by the 32 lanes of a warp, then the walk by ONE
    // thread (the strip path's walk kernel gives a pair to each lane)
    run32([&](int l) {
      BandedOut mine{};
      bool r2 = false;
      banded_compute_d<32, decltype(scoref), -1, 1>(l, x, m, y, n, sc, scoref, rng_all.data() + roff[p] / 4, cells[p],
                                                    fill_all.data() + foff[p], mode == 2 || mode == 3,
                                                    opsbuf.data() + opsbuf.size(), mine, strip_all.data() + soff[p],
                                                    cols.data() + 3 * p, &r2);
      if (l == 0) redo = r2;
    });
    if (!redo) {
      bool r2 = false;
      banded_compute_d<1, decltype(scoref), -1, 2>(0, x, m, y, n, sc, scoref, rng_all.data() + roff[p] / 4, cells[p],
                                                   fill_all.data() + foff[p], mode == 2 || mode == 3,
                                                   opsbuf.data() + opsbuf.size(), o, strip_all.data() + soff[p],
                                                   cols.data() + 3 * p, &r2);
    }
    if (redo || o.status) continue;
    path[p] = 1;
    score[p] = o.score;
    coords[4 * p + 0] = o.xstart;
    coords[4 * p + 1] = o.xend;
    coords[4 * p + 2] = o.ystart;
    coords[4 * p + 3] = o.yend;
    n_ops[p] = o.n_ops;
    for (int q = 0; q < 4; ++q) clip_len[4 * p + q] = o.clip[q];
    std::memcpy(ops + ops_off[p], opsbuf.data() + opsbuf.size() - o.n_ops, o.n_ops);
  }
  return 0;
}


// the kernel-variant choice of the engine (b2a_plan.h scoring_flags), for the host-logic tests
extern "C" int sim_scoring_flags(int32_t xclip_prefix, int32_t xclip_suffix, int32_t yclip_prefix, int32_t yclip_suffix,
                                 int32_t alpha, int64_t score_bound, uint32_t maxm, uint32_t maxn) {
  DevScoring sc{};
  sc.gap_open = -5;
  sc.gap_extend = -1;
  sc.xclip_prefix = xclip_prefix;
  sc.xclip_suffix = xclip_suffix;
  sc.yclip_prefix = yclip_prefix;
  sc.yclip_suffix = yclip_suffix;
  sc.alpha = alpha;
  return scoring_flags(sc, score_bound, maxm, maxn);
}

// whether the engine lets a banded batch run the strip-wavefront fill (b2a_plan.h banded_strip_gate); clips with the
// mode's preset applied
extern "C" int sim_banded_strip_gate(int32_t xclip_prefix, int32_t xclip_suffix, int32_t yclip_prefix,
                                     int32_t yclip_suffix, int64_t score_bound, uint32_t maxm) {
  DevScoring sc{};
  sc.xclip_prefix = xclip_prefix;
  sc.xclip_suffix = xclip_suffix;
  sc.yclip_prefix = yclip_prefix;
  sc.yclip_suffix = yclip_suffix;
  return banded_strip_gate(sc, score_bound, maxm) ? 1 : 0;
}
