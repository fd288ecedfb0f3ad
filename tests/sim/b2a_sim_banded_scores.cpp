// CPU simulation of the banded aligner's score-only call (b2a_align_batch_banded_scores): K4 as the full call runs it,
// then banded_compute_d<..., SCORES = true> -- the literal column loop (W = 1 or 32), the register-resident loop, or the
// strip-wavefront fill's F_NOTB twin (ks_run_task), its finish pass and the walk.  Each call can give the K3
// slab its full size with the interior-cell region poisoned, and the strip area its full size with the traceback
// region poisoned; both must come back unchanged.  Builds on the harness of b2a_sim.cpp.  Test tool only
// (tests/test_banded_score_only.py).
#include "b2a_sim.cpp"

namespace {

DevScoring simb_scoring(int mode, const sim_scoring* s) {
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
  return sc;
}

// a slab of the score-only size (poison < 0), or of the full call's size whose bytes past the score-only layout's
// `cells` offset hold `poison`
struct PoisonedSlab {
  std::vector<uint8_t> buf;
  uint64_t from = 0;
  std::vector<uint8_t> tail;
  void init(uint64_t so_bytes, uint64_t full_bytes, uint64_t poison_from, int poison, uint8_t garbage) {
    buf.assign(poison >= 0 ? std::max(so_bytes, full_bytes) : so_bytes, garbage);
    from = poison >= 0 ? poison_from : buf.size();
    for (uint64_t t = from; t < buf.size(); ++t) buf[t] = (uint8_t)poison;
    tail.assign(buf.begin() + (ptrdiff_t)from, buf.end());
  }
  bool intact() const { return std::equal(tail.begin(), tail.end(), buf.begin() + (ptrdiff_t)from); }
};

}  // namespace

extern "C" {

// One pair: K4 (W = 32; caller matches / path when have_matches), then score-only K3 on the path `loop` asks for:
// 0 = as on the device (the register-resident loop when banded_fast_ok, else the literal loop), 1 = literal W = 32,
// 2 = literal W = 1.  *fast = 1 when the register-resident loop ran.  Returns -1 if the 32 lanes disagree on K4, -3 if
// the poisoned interior-cell region changed.
int simb_warp32_one(int mode, const sim_scoring* s, uint32_t k, uint32_t w, const uint8_t* x, uint32_t m32,
                    const uint8_t* y, uint32_t n32, int have_matches, const uint32_t* match_xy, uint64_t n_matches,
                    const uint32_t* path_idx, uint64_t n_path, int have_path, int allowed_mismatches,
                    int use_lcskpp_union, uint32_t cap_matches, int loop, int poison, int32_t* score, uint32_t* xend,
                    uint32_t* yend, uint32_t* status, uint64_t* num_cells, int* fast_out) {
  const DevScoring sc = simb_scoring(mode, s);
  const int32_t* table = s->table;
  const uint64_t m = m32, n = n32;
  std::vector<uint8_t> slab(k4_slab_bytes(cap_matches, (uint32_t)std::min(m, n)), 0x3C);
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
  uint32_t st_lane[32];
  uint64_t cells_lane[32];
  LaneFibers::run([&](int l) {
    uint64_t c = 0;
    st_lane[l] = band_create_d<32>(l, x, m, y, n, k, w, sc, s->has_match_scores, slab.data(), cap_matches, rng.data(),
                                   &c, shared_vec.data(), hint);
    cells_lane[l] = c;
  });
  for (int l = 1; l < 32; ++l)
    if (st_lane[l] != st_lane[0] || cells_lane[l] != cells_lane[0]) return -1;
  const uint32_t st = st_lane[0];
  const uint64_t cells = cells_lane[0];
  *num_cells = cells;
  *fast_out = 0;
  BandedOut o{};
  bool intact = true;
  if (st != 0) {
    o = BandedOut{};
    o.status = 1 + st;
  } else {
    PoisonedSlab fill;
    if (cells > BANDED_MAX_CELLS)  // (a refused band: no state at all)
      fill.init(256, 256, 256, poison, 0x3C);
    else
      fill.init(k3_slab_bytes(m, n, cells, true), k3_slab_bytes(m, n, cells), k3_layout(m, n, 0).cells, poison, 0x3C);
    auto scoref = [&](uint8_t a, uint8_t b) -> int32_t {
      if (table) return table[(size_t)a * 256 + b];
      return a == b ? sc.match_score : sc.mismatch_score;
    };
    const bool filter = mode == 2 || mode == 3;
    if (loop == 2) {
      banded_compute_d<1, decltype(scoref), 0, 0, true>(0, x, m, y, n, sc, scoref, rng.data(), cells, fill.buf.data(),
                                                         filter, nullptr, o);
    } else {
      bool fast_lane[32];
      LaneFibers::run([&](int l) {
        fast_lane[l] = cells <= BANDED_MAX_CELLS && banded_fast_ok<32, K3_FAST_ROWS>(l, rng.data(), m, n);
      });
      const bool fast = loop == 0 && fast_lane[0];
      *fast_out = fast ? 1 : 0;
      LaneFibers::run([&](int l) {
        BandedOut mine{};
        if (fast)
          banded_compute_d<32, decltype(scoref), K3_FAST_ROWS, 0, true>(l, x, m, y, n, sc, scoref, rng.data(), cells,
                                                                        fill.buf.data(), filter, nullptr, mine);
        else
          banded_compute_d<32, decltype(scoref), 0, 0, true>(l, x, m, y, n, sc, scoref, rng.data(), cells,
                                                             fill.buf.data(), filter, nullptr, mine);
        if (l == 0) o = mine;
      });
    }
    intact = fill.intact();
  }
  // as banded_fill_body: a pair with a status reports MIN_SCORE and no coordinates
  *score = o.status ? MIN_SCORE : o.score;
  *xend = o.status ? 0u : o.xend;
  *yend = o.status ? 0u : o.yend;
  *status = o.status;
  return intact ? 0 : -3;
}

// Up to four pairs as sim_banded_strip_task runs them, in score-only form: K4 per pair (W = 32), ONE warp-task of the
// F_NOTB strip fill, then the score-only finish pass per pair on 32 emulated lanes and the walk on one.
// path[p] = 1: the strip path produced the pair's result; 2: K4 marked the pair but the strip path handed it back to the
// column loops (bit 10, from the fill or the finish pass); 0: not marked.  Returns -3 if a poisoned
// region (interior cells of a slab, traceback of a strip area) changed.
int simb_strip_task(int mode, const sim_scoring* s, uint32_t k, uint32_t w, const uint8_t* blob, uint64_t blob_bytes,
                    const uint64_t* x_off, const uint32_t* x_len, const uint64_t* y_off, const uint32_t* y_len,
                    uint32_t n_pairs, uint32_t cap_matches, int poison, int32_t* score, uint32_t* xend, uint32_t* yend,
                    uint32_t* status, uint32_t* path) {
  if (n_pairs > 4) return -2;
  const DevScoring sc0 = simb_scoring(mode, s);
  DevScoring sc = sc0;
  const int32_t* table = s->table;
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
  std::vector<uint8_t> cmap(256, 0xFF);
  std::vector<int32_t> lut_scaled;
  if (table) {
    if (syms.size() > 128) return -4;
    sc.alpha = (int32_t)syms.size();
    for (int a = 0; a < sc.alpha; ++a) cmap[syms[a]] = (uint8_t)a;
    lut_scaled.resize((size_t)sc.alpha * sc.alpha);
    for (int a = 0; a < sc.alpha; ++a)
      for (int b = 0; b < sc.alpha; ++b)
        lut_scaled[(size_t)a * sc.alpha + b] = 4 * table[(size_t)syms[a] * 256 + syms[b]] + 3 - (4 * sc.gap_open + 1);
  }
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
  for (uint32_t p = 0; p < n_pairs; ++p) {
    const uint64_t m = x_len[p], n = y_len[p];
    std::vector<uint8_t> slab(k4_slab_bytes(cap_matches, (uint32_t)std::min(m, n)), 0x3C);
    rngs[p].assign(2 * (n + 1), 0xCDCDCDCDu);
    BandHintsD hint;
    std::vector<uint32_t> shared_vec(K4_SHARED_WORDS, 0u);
    uint32_t st_lane[32];
    uint64_t c_lane[32];
    LaneFibers::run([&](int l) {
      uint64_t c = 0;
      st_lane[l] = band_create_d<32>(l, blob + x_off[p], m, blob + y_off[p], n, k, w, sc, s->has_match_scores,
                                     slab.data(), cap_matches, rngs[p].data(), &c, shared_vec.data(), hint);
      c_lane[l] = c;
    });
    cells[p] = c_lane[0];
    path[p] = 0;
    status[p] = 0;
    if (st_lane[0] != 0 || !batch_ok || cells[p] > BANDED_MAX_CELLS) continue;
    bool ok_lane[32];
    uint32_t c3[32][3];
    LaneFibers::run([&](int l) { ok_lane[l] = banded_strip_ok<32>(l, rngs[p].data(), m, n, c3[l], 0, ~0ull, true); });
    if (!ok_lane[0]) continue;
    for (int q = 0; q < 3; ++q) cols[3 * p + q] = c3[0][q];
    k4[p] = 0x200u;
  }
  // arenas as the engine lays them out in a score-only call; with poison >= 0 every slab and strip area gets the full
  // call's size and the bytes past the score-only layout hold `poison`
  uint64_t rb = 0, fb = 0, sb = 0;
  std::vector<std::pair<uint64_t, uint64_t>> fill_poison, strip_poison;  // [from, to) in the arenas
  for (uint32_t p = 0; p < n_pairs; ++p) {
    const uint64_t m = x_len[p], n = y_len[p];
    roff[p] = rb;
    rb += ((n + 1) * 8 + 15) & ~15ull;
    foff[p] = fb;
    const uint64_t so_f = k3_slab_bytes(m, n, cells[p], true), full_f = k3_slab_bytes(m, n, cells[p]);
    if (poison >= 0 && cells[p] <= BANDED_MAX_CELLS) fill_poison.push_back({fb + k3_layout(m, n, 0).cells, fb + full_f});
    fb += poison >= 0 ? full_f : so_f;
    soff[p] = sb;
    if (k4[p]) {
      const uint64_t c0 = std::max<uint64_t>(cols[3 * p], 1), c1 = std::min<uint64_t>(cols[3 * p + 1], n - 1);
      const KsLayout so = ks_layout(m, c1 >= c0 ? c1 - c0 + 1 : 0, cols[3 * p + 2], true);
      const KsLayout full = ks_layout(m, c1 >= c0 ? c1 - c0 + 1 : 0, cols[3 * p + 2]);
      if (poison >= 0) strip_poison.push_back({sb + so.tb, sb + full.total});
      sb += poison >= 0 ? full.total : so.total;
      elig.push_back(p);
    }
  }
  if (elig.empty()) return 0;
  std::vector<uint32_t> rng_all(rb / 4 + 4, 0);
  for (uint32_t p = 0; p < n_pairs; ++p) std::memcpy(rng_all.data() + roff[p] / 4, rngs[p].data(), rngs[p].size() * 4);
  std::vector<uint8_t> fill_all(fb + 16, 0x3C), strip_all(sb + 16, 0x3C);
  for (auto& r : fill_poison) std::fill(fill_all.begin() + (ptrdiff_t)r.first, fill_all.begin() + (ptrdiff_t)r.second, (uint8_t)poison);
  for (auto& r : strip_poison) std::fill(strip_all.begin() + (ptrdiff_t)r.first, strip_all.begin() + (ptrdiff_t)r.second, (uint8_t)poison);
  const std::vector<uint8_t> fill_before = fill_all, strip_before = strip_all;
  uint32_t counter = 0;
  StripParams sp{};
  sp.blob = blob;
  sp.x_off = x_off;
  sp.x_len = x_len;
  sp.y_off = y_off;
  sp.y_len = y_len;
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
                 (table ? (int)F_LUT : 0) | (int)F_NOTB;
  uint32_t err_flag = 0;
  KsLut T{};
  T.lut = lut_scaled.data();
  T.cmap = cmap.data();
  T.err_flag = &err_flag;
  LaneFibers::run([&](int l) {
    switch (fl) {
#define SIMB_KS_CASE1(F) \
  case (F): ks_run_task<(F)>(sp, T, 0, l); break;
#define SIMB_KS_CASE(F) SIMB_KS_CASE1((F) | F_NOTB) SIMB_KS_CASE1((F) | F_LUT | F_NOTB)
      SIMB_KS_CASE(0)
      SIMB_KS_CASE(F_TRACK_ROWS)
      SIMB_KS_CASE(F_CLIPX)
      SIMB_KS_CASE(F_CLIPY)
      SIMB_KS_CASE(F_TRACK_ROWS | F_CLIPX)
      SIMB_KS_CASE(F_TRACK_ROWS | F_CLIPY)
      SIMB_KS_CASE(F_CLIPX | F_CLIPY)
      SIMB_KS_CASE(F_TRACK_ROWS | F_CLIPX | F_CLIPY)
      SIMB_KS_CASE(F_TRACK_COLS)
      SIMB_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS)
      SIMB_KS_CASE(F_TRACK_COLS | F_CLIPX)
      SIMB_KS_CASE(F_TRACK_COLS | F_CLIPY)
      SIMB_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPX)
      SIMB_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPY)
      SIMB_KS_CASE(F_TRACK_COLS | F_CLIPX | F_CLIPY)
      SIMB_KS_CASE(F_TRACK_COLS | F_TRACK_ROWS | F_CLIPX | F_CLIPY)
#undef SIMB_KS_CASE
#undef SIMB_KS_CASE1
    }
  });
  for (uint32_t p : elig) {
    if (k4[p] & 0x400u) {  // the fill handed the pair back
      path[p] = 2;
      continue;
    }
    const uint64_t m = x_len[p], n = y_len[p];
    auto scoref = [&](uint8_t a, uint8_t b) -> int32_t {
      if (table) return table[(size_t)a * 256 + b];
      return a == b ? sc.match_score : sc.mismatch_score;
    };
    BandedOut o{};
    bool redo = false;
    // as on the device: the finish pass (up to the final score) on 32 lanes, then the walk by ONE thread
    LaneFibers::run([&](int l) {
      BandedOut mine{};
      bool r2 = false;
      banded_compute_d<32, decltype(scoref), -1, 1, true>(l, blob + x_off[p], m, blob + y_off[p], n, sc0, scoref,
                                                          rng_all.data() + roff[p] / 4, cells[p],
                                                          fill_all.data() + foff[p], mode == 2 || mode == 3, nullptr,
                                                          mine, strip_all.data() + soff[p], cols.data() + 3 * p, &r2);
      if (l == 0) redo = r2;
    });
    if (!redo) {
      bool r2 = false;
      banded_compute_d<1, decltype(scoref), -1, 2, true>(0, blob + x_off[p], m, blob + y_off[p], n, sc0, scoref,
                                                         rng_all.data() + roff[p] / 4, cells[p], fill_all.data() + foff[p],
                                                         mode == 2 || mode == 3, nullptr, o, strip_all.data() + soff[p],
                                                         cols.data() + 3 * p, &r2);
    }
    if (redo || o.status) {  // handed back to the column loops, as banded_fill_body does
      path[p] = 2;
      continue;
    }
    path[p] = 1;
    score[p] = o.score;
    xend[p] = o.xend;
    yend[p] = o.yend;
  }
  for (auto& r : fill_poison)
    if (!std::equal(fill_all.begin() + (ptrdiff_t)r.first, fill_all.begin() + (ptrdiff_t)r.second,
                    fill_before.begin() + (ptrdiff_t)r.first))
      return -3;
  for (auto& r : strip_poison)
    if (!std::equal(strip_all.begin() + (ptrdiff_t)r.first, strip_all.begin() + (ptrdiff_t)r.second,
                    strip_before.begin() + (ptrdiff_t)r.first))
      return -3;
  return 0;
}

// bytes of one pair's K3 slab and strip area, full and score-only: {k3 full, k3 score-only, ks full, ks score-only}
void simb_sizes(uint64_t m, uint64_t n, uint64_t cells, uint64_t band_cols, uint64_t strip_cols, uint64_t* out) {
  out[0] = k3_slab_bytes(m, n, cells);
  out[1] = k3_slab_bytes(m, n, cells, true);
  out[2] = ks_layout(m, band_cols, strip_cols).total;
  out[3] = ks_layout(m, band_cols, strip_cols, true).total;
}

}  // extern "C"
