// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// CPU restatement ("oracle") of rust-bio 4.0.1 `bio::alignment::pairwise::Aligner`
// (reference src/alignment/pairwise/mod.rs).  The build does not compile rust-bio
// (it needs no Rust toolchain), so this file restates the algorithm statement by
// statement: same loop order (y outer, x inner), same strict comparisons, same
// write order of every traceback store, same u16 row-major (m+1)x(n+1) traceback
// matrix that is re-initialised on every call, same rolling two-column i32
// S/I/D arrays.  Each function cites the reference lines it follows.
//
// Parity is PINNED: tests/test_oracle_golden.py checks this oracle against every
// known-answer vector in the reference's own tests and doctests for this path
// (mod.rs:21-160, 1203-1769; see tests/golden/pairwise_vectors.json).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
// reference legs may load this library.  Built with -fwrapv so that i32
// arithmetic wraps like Rust release builds.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <pthread.h>
#include <sched.h>
#include <thread>
#include <vector>

namespace {

constexpr int32_t MIN_SCORE = -858993459;  // mod.rs:174

// Traceback moves, mod.rs:1036-1045
constexpr uint16_t TB_START = 0, TB_INS = 1, TB_DEL = 2, TB_SUBST = 3, TB_MATCH = 4,
                   TB_XCLIP_PREFIX = 5, TB_XCLIP_SUFFIX = 6, TB_YCLIP_PREFIX = 7,
                   TB_YCLIP_SUFFIX = 8;

// TracebackCell, mod.rs:1026-1114: bits 0-3 I, 4-7 D, 8-11 S.
struct Cell {
  uint16_t v = 0;
  void set_i(uint16_t x) { v = (uint16_t)((v & ~0x000F) | x); }
  void set_d(uint16_t x) { v = (uint16_t)((v & ~0x00F0) | (x << 4)); }
  void set_s(uint16_t x) { v = (uint16_t)((v & ~0x0F00) | (x << 8)); }
  void set_all(uint16_t x) { set_i(x); set_d(x); set_s(x); }
  uint16_t i() const { return v & 15; }
  uint16_t d() const { return (v >> 4) & 15; }
  uint16_t s() const { return (v >> 8) & 15; }
};

}  // namespace

extern "C" {

// Same layout as b2a_scoring in include/b200align.h (Scoring<F>, mod.rs:238-247).
struct orc_scoring {
  int32_t gap_open, gap_extend;
  int32_t xclip_prefix, xclip_suffix, yclip_prefix, yclip_suffix;
  int32_t match_score, mismatch_score;
  int32_t has_match_scores;
  const int32_t* table;  // 256x256 tabulated MatchFunc or NULL (MatchParams)
  const uint8_t* alphabet;  // unused by the oracle (layout parity with b2a_scoring)
  uint32_t alphabet_len;
};

// bio_types::alignment::Alignment (fields built at mod.rs:911-921)
struct orc_alignment {
  int32_t score;
  uint32_t ystart, xstart, yend, xend, ylen, xlen;
  uint32_t mode;   // 0 Custom, 1 Global, 2 Semiglobal, 3 Local
  uint32_t n_ops;  // ops[k] = code | (clip_len << 3); codes 0 Match 1 Subst 2 Del 3 Ins 4 Xclip 5 Yclip
};

}  // extern "C"

namespace {

struct Op {
  uint32_t code, len;
};

// Aligner<F>, mod.rs:472-481
struct FullAligner {
  std::vector<int32_t> I[2], D[2], S[2];
  std::vector<size_t> Lx, Ly;
  std::vector<int32_t> Sn;
  std::vector<Cell> tb;  // Traceback, mod.rs:1118-1168
  size_t rows = 0, cols = 0;
  orc_scoring sc{};

  inline int32_t score(uint8_t a, uint8_t b) const {
    if (sc.table) return sc.table[(size_t)a * 256 + b];  // closure MatchFunc, mod.rs:221-228
    return a == b ? sc.match_score : sc.mismatch_score;  // MatchParams, mod.rs:208-217
  }
  Cell& at(size_t i, size_t j) { return tb[i * cols + j]; }  // mod.rs:1144-1161

  // Aligner::custom, mod.rs:591-922
  void custom(const uint8_t* x, size_t m, const uint8_t* y, size_t n, orc_alignment* out,
              std::vector<Op>& operations) {
    // traceback.init(m, n): mod.rs:593, 1135-1141, 1163-1167
    rows = m + 1;
    cols = n + 1;
    tb.clear();
    tb.resize(rows * cols, Cell{});

    // initial conditions, mod.rs:597-672
    for (int k = 0; k < 2; ++k) {
      I[k].assign(m + 1, MIN_SCORE);
      D[k].assign(m + 1, MIN_SCORE);
      S[k].assign(m + 1, MIN_SCORE);
      S[k][0] = 0;
      if (k == 0) {
        Cell c;
        c.set_all(TB_START);
        at(0, 0) = c;
        Lx.assign(n + 1, 0);
        Ly.assign(m + 1, 0);
        Sn.assign(m + 1, MIN_SCORE);
        Sn[0] = sc.yclip_suffix;
        Ly[0] = n;
      }
      for (size_t i = 1; i <= m; ++i) {
        Cell c;
        c.set_all(TB_START);
        if (i == 1) {
          I[k][i] = sc.gap_open;
          c.set_i(TB_START);
        } else {
          int32_t i_score = sc.gap_open + sc.gap_extend * ((int32_t)i - 1);
          int32_t c_score = sc.xclip_prefix + sc.gap_open;
          if (i_score > c_score) {
            I[k][i] = i_score;
            c.set_i(TB_INS);
          } else {
            I[k][i] = c_score;
            c.set_i(TB_XCLIP_PREFIX);
          }
        }
        if (i == m) {
          c.set_s(TB_XCLIP_SUFFIX);
        } else {
          S[k][i] = MIN_SCORE;
        }
        if (I[k][i] > S[k][i]) {
          S[k][i] = I[k][i];
          c.set_s(TB_INS);
        }
        if (sc.xclip_prefix > S[k][i]) {
          S[k][i] = sc.xclip_prefix;
          c.set_s(TB_XCLIP_PREFIX);
        }
        if (i != m && S[k][i] + sc.xclip_suffix > S[k][m]) {
          S[k][m] = S[k][i] + sc.xclip_suffix;
          Lx[0] = m - i;
        }
        if (k == 0) at(i, 0) = c;
        if (S[k][i] + sc.yclip_suffix > Sn[i]) {
          Sn[i] = S[k][i] + sc.yclip_suffix;
          Ly[i] = n;
        }
      }
    }

    // the fill, mod.rs:674-806
    for (size_t j = 1; j <= n; ++j) {
      const size_t curr = j % 2, prev = 1 - curr;
      {  // i = 0, mod.rs:678-717
        Cell c;
        I[curr][0] = MIN_SCORE;
        if (j == 1) {
          D[curr][0] = sc.gap_open;
          c.set_d(TB_START);
        } else {
          int32_t d_score = sc.gap_open + sc.gap_extend * ((int32_t)j - 1);
          int32_t c_score = sc.yclip_prefix + sc.gap_open;
          if (d_score > c_score) {
            D[curr][0] = d_score;
            c.set_d(TB_DEL);
          } else {
            D[curr][0] = c_score;
            c.set_d(TB_YCLIP_PREFIX);
          }
        }
        if (D[curr][0] > sc.yclip_prefix) {
          S[curr][0] = D[curr][0];
          c.set_s(TB_DEL);
        } else {
          S[curr][0] = sc.yclip_prefix;
          c.set_s(TB_YCLIP_PREFIX);
        }
        if (j == n && Sn[0] > S[curr][0]) {
          S[curr][0] = Sn[0];
          c.set_s(TB_YCLIP_SUFFIX);
        } else if (S[curr][0] + sc.yclip_suffix > Sn[0]) {
          Sn[0] = S[curr][0] + sc.yclip_suffix;
          Ly[0] = n - j;
        }
        at(0, j) = c;
      }
      for (size_t i = 1; i <= m; ++i) S[curr][i] = MIN_SCORE;  // mod.rs:719-721

      const uint8_t q = y[j - 1];
      const int32_t xclip_score =
          sc.xclip_prefix +
          std::max(sc.yclip_prefix, sc.gap_open + sc.gap_extend * ((int32_t)j - 1));  // mod.rs:724-728
      for (size_t i = 1; i < m + 1; ++i) {  // mod.rs:729-805
        const uint8_t p = x[i - 1];
        Cell c;
        const int32_t m_score = S[prev][i - 1] + score(p, q);

        const int32_t i_score = I[curr][i - 1] + sc.gap_extend;
        int32_t s_score = S[curr][i - 1] + sc.gap_open;
        int32_t best_i_score;
        if (i_score > s_score) {
          best_i_score = i_score;
          c.set_i(TB_INS);
        } else {
          best_i_score = s_score;
          c.set_i(at(i - 1, j).s());
        }

        const int32_t d_score = D[prev][i] + sc.gap_extend;
        s_score = S[prev][i] + sc.gap_open;
        int32_t best_d_score;
        if (d_score > s_score) {
          best_d_score = d_score;
          c.set_d(TB_DEL);
        } else {
          best_d_score = s_score;
          c.set_d(at(i, j - 1).s());
        }

        c.set_s(TB_XCLIP_SUFFIX);
        int32_t best_s_score = S[curr][i];
        if (m_score > best_s_score) {
          best_s_score = m_score;
          c.set_s(p == q ? TB_MATCH : TB_SUBST);
        }
        if (best_i_score > best_s_score) {
          best_s_score = best_i_score;
          c.set_s(TB_INS);
        }
        if (best_d_score > best_s_score) {
          best_s_score = best_d_score;
          c.set_s(TB_DEL);
        }
        if (xclip_score > best_s_score) {
          best_s_score = xclip_score;
          c.set_s(TB_XCLIP_PREFIX);
        }
        const int32_t yclip_score =
            sc.yclip_prefix + sc.gap_open + sc.gap_extend * ((int32_t)i - 1);
        if (yclip_score > best_s_score) {
          best_s_score = yclip_score;
          c.set_s(TB_YCLIP_PREFIX);
        }

        S[curr][i] = best_s_score;
        I[curr][i] = best_i_score;
        D[curr][i] = best_d_score;

        if (S[curr][i] + sc.xclip_suffix > S[curr][m]) {  // mod.rs:793-796
          S[curr][m] = S[curr][i] + sc.xclip_suffix;
          Lx[j] = m - i;
        }
        if (S[curr][i] + sc.yclip_suffix > Sn[i]) {  // mod.rs:799-802
          Sn[i] = S[curr][i] + sc.yclip_suffix;
          Ly[i] = n - j;
        }
        at(i, j) = c;
      }
    }

    // suffix clipping in the j = n column, mod.rs:809-821
    for (size_t i = 0; i <= m; ++i) {
      const size_t j = n, curr = j % 2;
      if (Sn[i] > S[curr][i]) {
        S[curr][i] = Sn[i];
        at(i, j).set_s(TB_YCLIP_SUFFIX);
      }
      if (S[curr][i] + sc.xclip_suffix > S[curr][m]) {
        S[curr][m] = S[curr][i] + sc.xclip_suffix;
        Lx[j] = m - i;
        at(m, j).set_s(TB_XCLIP_SUFFIX);
      }
    }
    // recompute the last column of I, mod.rs:825-843
    for (size_t i = 1; i <= m; ++i) {
      const size_t j = n, curr = j % 2;
      const int32_t s_score = S[curr][i - 1] + sc.gap_open;
      if (s_score > I[curr][i]) {
        I[curr][i] = s_score;
        const uint16_t s_bit = at(i - 1, j).s();
        at(i, j).set_i(s_bit);
      }
      if (s_score > S[curr][i]) {
        S[curr][i] = s_score;
        at(i, j).set_s(TB_INS);
        if (S[curr][i] + sc.xclip_suffix > S[curr][m]) {
          S[curr][m] = S[curr][i] + sc.xclip_suffix;
          Lx[j] = m - i;
          at(m, j).set_s(TB_XCLIP_SUFFIX);
        }
      }
    }

    // traceback walk, mod.rs:845-908
    size_t i = m, j = n;
    operations.clear();
    size_t xstart = 0, ystart = 0, xend = m, yend = n;
    uint16_t last_layer = at(i, j).s();
    for (;;) {
      uint16_t next_layer;
      if (last_layer == TB_START) break;
      switch (last_layer) {
        case TB_INS:
          operations.push_back({3, 0});
          next_layer = at(i, j).i();
          i -= 1;
          break;
        case TB_DEL:
          operations.push_back({2, 0});
          next_layer = at(i, j).d();
          j -= 1;
          break;
        case TB_MATCH:
          operations.push_back({0, 0});
          next_layer = at(i - 1, j - 1).s();
          i -= 1;
          j -= 1;
          break;
        case TB_SUBST:
          operations.push_back({1, 0});
          next_layer = at(i - 1, j - 1).s();
          i -= 1;
          j -= 1;
          break;
        case TB_XCLIP_PREFIX:
          operations.push_back({4, (uint32_t)i});
          xstart = i;
          i = 0;
          next_layer = at(0, j).s();
          break;
        case TB_XCLIP_SUFFIX:
          operations.push_back({4, (uint32_t)Lx[j]});
          i -= Lx[j];
          xend = i;
          next_layer = at(i, j).s();
          break;
        case TB_YCLIP_PREFIX:
          operations.push_back({5, (uint32_t)j});
          ystart = j;
          j = 0;
          next_layer = at(i, 0).s();
          break;
        case TB_YCLIP_SUFFIX:
          operations.push_back({5, (uint32_t)Ly[i]});
          j -= Ly[i];
          yend = j;
          next_layer = at(i, j).s();
          break;
        default:
          // panic!("Dint expect this!") mod.rs:905
          out->score = MIN_SCORE;
          out->n_ops = 0xFFFFFFFFu;
          return;
      }
      last_layer = next_layer;
    }
    std::reverse(operations.begin(), operations.end());  // mod.rs:910
    out->score = S[n % 2][m];
    out->ystart = (uint32_t)ystart;
    out->xstart = (uint32_t)xstart;
    out->yend = (uint32_t)yend;
    out->xend = (uint32_t)xend;
    out->ylen = (uint32_t)n;
    out->xlen = (uint32_t)m;
    out->mode = 0;
    out->n_ops = (uint32_t)operations.size();
  }

  // Alignment::filter_clip_operations (bio-types; call sites mod.rs:974,1006)
  static void filter_clips(std::vector<Op>& ops) {
    ops.erase(std::remove_if(ops.begin(), ops.end(), [](const Op& o) { return o.code >= 4; }),
              ops.end());
  }

  // global / semiglobal / local, mod.rs:925-1015
  void align(int mode, const uint8_t* x, size_t m, const uint8_t* y, size_t n,
             orc_alignment* out, std::vector<Op>& ops) {
    const int32_t saved[4] = {sc.xclip_prefix, sc.xclip_suffix, sc.yclip_prefix, sc.yclip_suffix};
    if (mode == 1) {  // global, mod.rs:935-938
      sc.xclip_prefix = sc.xclip_suffix = sc.yclip_prefix = sc.yclip_suffix = MIN_SCORE;
    } else if (mode == 2) {  // semiglobal, mod.rs:964-967
      sc.xclip_prefix = sc.xclip_suffix = MIN_SCORE;
      sc.yclip_prefix = sc.yclip_suffix = 0;
    } else if (mode == 3) {  // local, mod.rs:996-999
      sc.xclip_prefix = sc.xclip_suffix = sc.yclip_prefix = sc.yclip_suffix = 0;
    }
    custom(x, m, y, n, out, ops);
    out->mode = (uint32_t)mode;
    if (mode == 2 || mode == 3) {
      filter_clips(ops);
      out->n_ops = (uint32_t)ops.size();
    }
    sc.xclip_prefix = saved[0];
    sc.xclip_suffix = saved[1];
    sc.yclip_prefix = saved[2];
    sc.yclip_suffix = saved[3];
  }
};

}  // namespace

// CPUs in this process's affinity mask (what nproc reports), in ascending order
static std::vector<int> orc_allowed_cpus() {
  std::vector<int> out;
  cpu_set_t set;
  CPU_ZERO(&set);
  if (sched_getaffinity(0, sizeof(set), &set) == 0)
    for (int c = 0; c < CPU_SETSIZE; ++c)
      if (CPU_ISSET(c, &set)) out.push_back(c);
  return out;
}

extern "C" {

// One pair. ops must hold m+n+4 entries. Returns 0, or -1 on the reference's panic path.
int orc_align(int mode, const orc_scoring* scoring, const uint8_t* x, uint32_t m, const uint8_t* y,
              uint32_t n, orc_alignment* out, uint32_t* ops) {
  FullAligner a;
  a.sc = *scoring;
  std::vector<Op> v;
  a.align(mode, x, m, y, n, out, v);
  if (out->n_ops == 0xFFFFFFFFu) return -1;
  for (size_t k = 0; k < v.size(); ++k) ops[k] = v[k].code | (v[k].len << 3);
  return 0;
}

// A batch, statically partitioned over `threads` host threads, one reusable
// FullAligner (scratch) per thread as mod.rs:505-506 intends.  ops may be NULL
// (timing only); otherwise ops_off[p] is where pair p's ops go (capacity
// x_len+y_len+4 each).  Returns wall seconds of the align loop.
double orc_align_batch(int mode, const orc_scoring* scoring, const uint8_t* blob,
                       const uint64_t* x_off, const uint32_t* x_len, const uint64_t* y_off,
                       const uint32_t* y_len, uint64_t n_pairs, orc_alignment* out, uint32_t* ops,
                       const uint64_t* ops_off, int threads) {
  if (threads < 1) threads = 1;
  auto t0 = std::chrono::steady_clock::now();
  // the CPUs this process may run on (cgroup / taskset aware); thread t is pinned to one of them so that the
  // baseline does not depend on how the scheduler happens to migrate 128 threads (1.2 vs 6.5 GCUPS
  // between two boxes with the same thread count)
  std::vector<int> cpus = orc_allowed_cpus();
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) {
    pool.emplace_back([=]() {
      if (!cpus.empty() && threads > 1) {
        cpu_set_t set;
        CPU_ZERO(&set);
        CPU_SET(cpus[(size_t)t % cpus.size()], &set);
        pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
      }
      FullAligner a;
      a.sc = *scoring;
      std::vector<Op> v;
      const uint64_t lo = n_pairs * (uint64_t)t / (uint64_t)threads;
      const uint64_t hi = n_pairs * (uint64_t)(t + 1) / (uint64_t)threads;
      for (uint64_t p = lo; p < hi; ++p) {
        a.align(mode, blob + x_off[p], x_len[p], blob + y_off[p], y_len[p], &out[p], v);
        if (ops && out[p].n_ops != 0xFFFFFFFFu)
          for (size_t k = 0; k < v.size(); ++k) ops[ops_off[p] + k] = v[k].code | (v[k].len << 3);
      }
    });
  }
  for (auto& th : pool) th.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

int orc_hardware_threads() {
  const std::vector<int> cpus = orc_allowed_cpus();
  return cpus.empty() ? (int)std::thread::hardware_concurrency() : (int)cpus.size();
}

}  // extern "C"
