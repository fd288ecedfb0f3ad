// CPU simulation of the recomputed traceback (tests/test_traceback_recompute.py): one warp-per-pair pair through the
// engine's recompute path (b2a_engine.cu plan_recompute / recompute_wave) -- the F_NOTB | F_CKPT pass over every strip,
// K2's finish (finish_matrix_coop on 32 emulated lanes) and the windowed walk, refilling with F_REFILL the window that
// holds the row the walk waits for.  Windows of any W are forced by the caller.  Around every refill the rows arena,
// the row-m cells and the boundary row are compared byte for byte.  Builds on the harness of b2a_sim_long.cpp.  Test
// tool only.
#include "b2a_sim_long.cpp"

namespace {

// The strips [lo, hi) of the one pair of `blk` as strip-pipelined tasks (fill_kernel's F_REFILL / F_CKPT setup):
// F_CKPT stores checkpoint rows into `ckpt`; F_REFILL reads strip lo's top boundary from `bnd` (the scratch row) and
// stores the traceback of the window's strips at window-relative offsets into `tb`.
template <int R, int FLAGS>
void fill_window(const Block& blk, int32_t m, int32_t n, const DevScoring& sc, const int32_t* lut,
                 std::vector<uint8_t>& seq, uint8_t* bnd, std::vector<uint8_t>& rows, uint8_t* tb, int4* ckpt,
                 int32_t win, int32_t lo, int32_t hi) {
  constexpr int G = 32, TBW = tbw_of(R);
  constexpr bool REFILL = (FLAGS & F_REFILL) != 0;
  std::vector<uint32_t> progress((size_t)(hi - lo), 0u);
  std::vector<std::function<void(int)>> bodies;
  std::vector<std::vector<uint32_t>> slices(hi - lo);
  const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
  for (int32_t strip = lo; strip < hi; ++strip) {
    const uint32_t xoff_words = (uint32_t)strip * G * R / 4;
    slices[strip - lo].assign(seqw + xoff_words, seqw + xoff_words + G * R / 4);
    const uint32_t* xs_biased = slices[strip - lo].data() - xoff_words;
    uint32_t* prog = progress.data() + (strip - lo);
    bodies.push_back([&, strip, xs_biased, prog](int lane) {
      LaneCtx<G> c;
      c.sc = sc;
      c.lut = lut;
      c.ge4 = 4 * sc.gap_extend;
      c.lut_base = 0;
      c.one = 1;
      c.only_strip = strip;
      c.prog_mine = prog;
      c.prog_prev = strip > lo ? prog - 1 : nullptr;
      c.xs = xs_biased;
      c.ys = seqw + (size_t)G * blk.xwords;
      c.g = 0;
      c.l = lane;
      c.lane = lane;
      c.pi = 0;
      c.m = m;
      c.n = n;
      c.maxn = (int32_t)blk.maxn;
      c.maxm = (int32_t)blk.maxm;
      c.nstrips = (int32_t)blk.nstrips;
      c.K = (int32_t)blk.K;
      c.rows_pad = (int32_t)blk.rows_pad;
      c.uniform = blk.uniform != 0;
      c.bnd = reinterpret_cast<int4*>(bnd);
      c.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
      c.ckpt = ckpt;
      c.win = win;
      c.strip_lo = REFILL ? lo : 0;
      c.tb = reinterpret_cast<uint4*>(tb);
      (void)TBW;
      fill_lane<G, R, FLAGS>(c);
    });
  }
  WarpSet::run(std::move(bodies));
}

// the flag cases of launch_fill_recompute_32_R with a LUT (every batch here has at most 64 symbols)
template <int R>
void fill_window_dispatch(int flags, const Block& blk, int32_t m, int32_t n, const DevScoring& sc, const int32_t* lut,
                          std::vector<uint8_t>& seq, uint8_t* bnd, std::vector<uint8_t>& rows, uint8_t* tb,
                          int4* ckpt, int32_t win, int32_t lo, int32_t hi) {
  constexpr int ALL = F_TRACK_ROWS | F_TRACK_COLS | F_CLIPX;
  constexpr int P1 = F_NOTB | F_CKPT | F_YSTREAM | F_LUT, RF = F_REFILL | F_YSTREAM | F_LUT;
#define SIMR_CASE(F) \
  case (F): fill_window<R, (F)>(blk, m, n, sc, lut, seq, bnd, rows, tb, ckpt, win, lo, hi); break;
  switch (flags) {
    SIMR_CASE(P1)
    SIMR_CASE(P1 | F_TRACK_ROWS)
    SIMR_CASE(P1 | F_TRACK_ROWS | F_PACKREL)
    SIMR_CASE(P1 | ALL)
    SIMR_CASE(P1 | ALL | F_PACKREL)
    SIMR_CASE(P1 | ALL | F_RELU)
    SIMR_CASE(P1 | ALL | F_PACKREL | F_RELU)
    SIMR_CASE(RF)
    SIMR_CASE(RF | F_CLIPX)
    SIMR_CASE(RF | F_CLIPX | F_RELU)
    default: std::abort();
  }
#undef SIMR_CASE
}

}  // namespace

extern "C" {

// One pair (x, y) through the recomputed traceback with W = `win` strips per window, on the 32xR shape.  Outputs as
// siml_align for its one pair (ops: n_ops bytes in alignment order), plus counts[0..3] = windows, windows refilled,
// bytes of the rows arena / row-m cells / boundary row that a refill changed, and the fill flags of pass 1.
// Returns 0, or -1 for a bad shape, -2 for too many symbols, -3 when the walk asked for windows out of order.
int simr_align(int mode, const sim_scoring* s, const uint8_t* x, uint32_t m, const uint8_t* y, uint32_t n, int R,
               int win, int32_t* score, uint32_t* xstart, uint32_t* xend, uint32_t* ystart, uint32_t* yend,
               uint32_t* n_ops, uint32_t* clip_len, uint32_t* status, uint8_t* ops, uint64_t* counts) {
  constexpr int G = 32;
  if ((R != 8 && R != 16) || win < 1 || m < 2 || n < 1) return -1;
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
  // alphabet + LUT as siml_align (and the engine) build them
  uint8_t codemap[256];
  for (int k = 0; k < 256; ++k) codemap[k] = (uint8_t)k;
  std::vector<int32_t> lut;
  int64_t maxabs = std::max<int64_t>(std::llabs((long long)s->match_score), std::llabs((long long)s->mismatch_score));
  {
    bool present[256] = {false};
    for (uint32_t k = 0; k < m; ++k) present[x[k]] = true;
    for (uint32_t k = 0; k < n; ++k) present[y[k]] = true;
    std::vector<int> syms;
    for (int k = 0; k < 256; ++k)
      if (present[k]) syms.push_back(k);
    if ((int)syms.size() > 64) return -2;
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
  const int64_t unit = std::max<int64_t>(maxabs, std::max<int64_t>(-(int64_t)sc.gap_open, -(int64_t)sc.gap_extend));
  const int64_t bound = ((int64_t)m + n + 2) * unit - (int64_t)sc.gap_open;
  // the flags of a recomputing batch (b2a_engine.cu plan_recompute)
  int flags = scoring_flags(sc, bound, m, n);
  const bool trackers = (flags & (F_TRACK_ROWS | F_TRACK_COLS)) != 0;
  flags &= ~(F_PACKTRK | F_BND8);
  if (trackers && bound < (1ll << 18)) flags |= F_PACKREL;
  flags |= F_YSTREAM;
  Plan p;
  build_plan(p, &m, &n, 1, G, R, ~0ull, flags);
  const Block& blk = p.blocks[0];
  const int32_t ns = (int32_t)blk.nstrips, GR = G * R;
  const int32_t W = std::min<int32_t>(win, ns), nw = (ns + W - 1) / W;
  const uint64_t strip_tb = (uint64_t)blk.K * tbw_of(R) * 512;
  const uint8_t gb = 0x3C;
  std::vector<uint8_t> seq(p.seq_bytes, 0), bnd(p.max_bnd, gb), rows(p.max_rows, gb), rowm(p.max_rowm, gb),
      scratch((size_t)(blk.maxn + 1) * 16, gb), tb((size_t)W * strip_tb, gb), opsb((size_t)m + n + 4, 0);
  std::vector<int4> ckpt((size_t)std::max(nw - 1, 1) * (blk.maxn + 1), int4{0x3C3C3C3C, 0x3C3C3C3C, 0x3C3C3C3C, 0x3C3C3C3C});
  {  // K0
    uint32_t* seqw = reinterpret_cast<uint32_t*>(seq.data() + blk.seq_off);
    uint8_t* xb = reinterpret_cast<uint8_t*>(seqw);
    for (uint32_t k = 0; k < m; ++k) xb[k] = codemap[x[k]];
    uint8_t* yb = reinterpret_cast<uint8_t*>(seqw + (size_t)G * blk.xwords);
    for (uint32_t k = 0; k < n; ++k) yb[k] = codemap[y[k]];
  }
  const int32_t* lut_plain = lut.data();
  const int32_t* lut_scaled = lut.data() + (size_t)sc.alpha * sc.alpha;
  auto fill = [&](int f, uint8_t* b, uint8_t* t, int32_t lo, int32_t hi) {
    if (R == 8) fill_window_dispatch<8>(f, blk, (int32_t)m, (int32_t)n, sc, lut_scaled, seq, b, rows, t, ckpt.data(), W, lo, hi);
    else fill_window_dispatch<16>(f, blk, (int32_t)m, (int32_t)n, sc, lut_scaled, seq, b, rows, t, ckpt.data(), W, lo, hi);
  };
  // pass 1
  fill(flags | F_NOTB | F_CKPT, bnd.data() + blk.bnd_off, nullptr, 0, ns);
  // K2
  PairView v;
  v.sc = sc;
  v.lut = lut_plain;
  v.P = 1;
  v.m = (int32_t)m;
  v.n = (int32_t)n;
  v.pi = 0;
  v.set_shape(G, R);
  v.nstrips = ns;
  v.K = (int32_t)blk.K;
  v.sub = 0;
  v.g = 0;
  v.packtrk = 0;
  v.bnd8 = 0;
  v.maxn = (int32_t)blk.maxn;
  v.bnd_base = bnd_index(G, 0, 0, v.maxn);
  v.bnd_stride = (int32_t)(bnd_index(G, 1, 0, v.maxn) - v.bnd_base);
  const uint32_t* seqw = reinterpret_cast<const uint32_t*>(seq.data() + blk.seq_off);
  v.xw = seqw;
  v.yw = seqw + (size_t)G * blk.xwords;
  v.bnd = reinterpret_cast<const int4*>(bnd.data() + blk.bnd_off);
  v.rows = reinterpret_cast<int32_t*>(rows.data() + blk.rows_off);
  v.rows_pad = (int32_t)blk.rows_pad;
  v.rowm = reinterpret_cast<uint16_t*>(rowm.data() + blk.rowm_off);
  v.tb = reinterpret_cast<const uint32_t*>(tb.data());
  v.row_lo = 1;
  v.row_hi = 0;  // no window yet
  EndState es;
  LaneFibers::run([&](int l) {
    EndState mine;
    finish_matrix_coop<32>(l, v, mine);
    if (l == 0) es = mine;
  });
  uint8_t* ops_end = opsb.data() + opsb.size();
  WalkState w;
  walk_begin(v, es, ops_end, w);
  const bool filter = mode == 2 || mode == 3;
  uint64_t filled = 0, clobbered = 0;
  int32_t above = nw;
  while (!walk_run<false, true>(v, es, filter, w, 0x7fffffff)) {
    if (!walk_waits(v, w.i, w.j, w.layer)) return -3;
    const int32_t k = (w.i >= 1 && w.i < (int32_t)m) ? ((w.i - 1) / GR) / W : nw;
    if (k >= above) return -3;
    above = k;
    const int32_t lo = k * W, hi = std::min(lo + W, ns);
    const std::vector<uint8_t> rows0 = rows, rowm0 = rowm, bnd0 = bnd;
    if (k > 0) std::memcpy(scratch.data(), ckpt.data() + (size_t)(k - 1) * (blk.maxn + 1), scratch.size());
    else std::memset(scratch.data(), gb, scratch.size());  // (strip 0 reads row 0's closed forms, not the row)
    std::memset(tb.data(), gb, tb.size());
    fill((flags & (F_LUT | F_CLIPX | F_RELU)) | F_YSTREAM | F_REFILL, scratch.data(), tb.data(), lo, hi);
    for (size_t q = 0; q < rows.size(); ++q) clobbered += rows[q] != rows0[q];
    for (size_t q = 0; q < rowm.size(); ++q) clobbered += rowm[q] != rowm0[q];
    for (size_t q = 0; q < bnd.size(); ++q) clobbered += bnd[q] != bnd0[q];
    ++filled;
    v.s0 = lo;
    v.row_lo = lo * GR + 1;
    v.row_hi = std::min(hi * GR, (int32_t)m - 1);
  }
  WalkOut o;
  walk_finish(es, w, o);
  *score = o.score;
  *xstart = o.xstart;
  *xend = o.xend;
  *ystart = o.ystart;
  *yend = o.yend;
  *n_ops = o.n_ops;
  *status = o.status;
  for (int k = 0; k < 4; ++k) clip_len[k] = o.clip[k];
  std::memcpy(ops, ops_end - o.n_ops, o.n_ops);
  counts[0] = (uint64_t)nw;
  counts[1] = filled;
  counts[2] = clobbered;
  counts[3] = (uint64_t)flags;
  return 0;
}

}  // extern "C"
