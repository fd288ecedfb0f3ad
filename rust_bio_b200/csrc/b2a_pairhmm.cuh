// Batched pair-HMM likelihoods (bio::stats::pairhmm::PairHMM::prob_related): the probability that x and y are
// related, summed over every alignment, in f64 log space.  A three-state forward recursion (match, gap in y "fx",
// gap in x "fy") over rows i of x and columns j of y, restated from the reference's literal loop so that its results
// come out bit for bit on the host (pairhmm.rs:104-280), with per-base emission classes standing for the
// reference's EmissionParameters trait object.
//
// Warp per pair, lanes over y: lane l owns C consecutive columns of a strip of 32 * C and runs row i = t - l at step
// t.  The reference keeps two rolling rows and resets only fm between rows, so a skipped (banded) cell keeps fx, fy
// and min_edit_dist from two rows earlier; here that buffer is the lane's registers: P (row i - 1, as it stands)
// and Q (row i - 2's fx, fy, min_edit_dist).  The left neighbour's last column comes by a shuffle, lane 0 of a later
// strip reads it from the previous strip's per-row record.  The lane logic is B2A_HD so that tests/sim compiles the
// very code the GPU runs; the kernels are in b2a_pairhmm.cu.
#pragma once
#include <math.h>
#include <string.h>

#include "b2a_common.cuh"

namespace b2a {

// Tiers, picked per pair by the host from len_y (pairhmm_tier): columns per lane, one strip for the first five;
// PT_STRIP runs strips of 32 * 8 columns.
enum : int {
  PT_DONE = 0,  // an empty side: answered on the host from the closed form
  PT_C1 = 1,    // len_y <= 32
  PT_C2 = 2,    // <= 64
  PT_C4 = 3,    // <= 128
  PT_C5 = 4,    // <= 160
  PT_C8 = 5,    // <= 256
  PT_STRIP = 6, // > 256: strips of 256 columns, C = 8
  PT_COUNT
};
constexpr uint32_t kPhmmMedNone = 0xFFFFFFFFu;  // min_edit_dist == usize::MAX

inline int pairhmm_tier(uint32_t m, uint32_t n) {
  if (m == 0 || n == 0) return PT_DONE;
  if (n <= 32) return PT_C1;
  if (n <= 64) return PT_C2;
  if (n <= 128) return PT_C4;
  if (n <= 160) return PT_C5;
  if (n <= 256) return PT_C8;
  return PT_STRIP;
}

// The gap-parameter cache of PairHMM::new (pairhmm.rs:69-95) plus the mode and band of the call.
struct PairHmmGap {
  double no_gap, no_gap_x_ext, no_gap_y_ext;
  double gap_x, gap_y, gap_x_ext, gap_y_ext;
  double col0_first;  // fm(row above, 0) at row 0: ln_one (+) prob_start_gap_x(0)
  double col0_rest;   // ... at every later row: ln_zero (+) prob_start_gap_x(i)
  uint32_t max_ed;    // band: a cell is skipped when its three min_edit_dist neighbours all exceed it
  int banded, do_x_ext, do_y_ext, free_start, free_end;
};

// One record per row of a strip's last column, as it stands in the reference's buffer (stale or not).
struct PairHmmRec {
  double fm, fx, fy;
  uint32_t med, pad;
};

// ---- LogProb arithmetic, statement for statement (probs/mod.rs:36-43, 213-271; fastexp.rs:33-58) ----

constexpr double kLnZero = -__builtin_inf();

// Every product and sum of FastExp rounds on its own: no contraction into a DFMA on the device.
B2A_HD double ph_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
B2A_HD double ph_add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// FastExp::fastexp.  The argument is <= 0 on every path here (a difference to a maximum, or ln_1m_exp's p <
// -0.693), so the truncating cast stays in range.
B2A_HD double ph_fastexp(double v) {
  if (!(v > -500.0)) return 0.0;
  double x = ph_mul(1.442695041, v);
  long long bits = (long long)x;
  x = ph_add(x, -(double)bits);
  double f2 = x, x_tmp = x;
  bits += 1023;
  bits <<= 52;
  f2 = ph_mul(f2, 0.006935931);
  x_tmp = ph_add(x_tmp, 4.831794110);
  f2 = ph_add(f2, 0.019890581);
  x_tmp = ph_mul(x_tmp, x);
  f2 = ph_mul(f2, x);
  f2 = ph_add(f2, 0.143440676);
  f2 = ph_mul(f2, x_tmp);
  f2 = ph_add(f2, 1.0);
#if defined(__CUDA_ARCH__)
  const double scale = __longlong_as_double(bits);
#else
  double scale;
  memcpy(&scale, &bits, 8);
#endif
  return ph_mul(scale, f2);
}

B2A_HD double ph_log1p(double v) { return log1p(v); }

// LogProb::ln_add_exp
B2A_HD double ph_add_exp(double self, double other) {
  if (other == kLnZero) return self;
  double p0 = self, p1 = other;
  if (p1 > p0) {
    const double t = p0;
    p0 = p1;
    p1 = t;
  }
  if (p0 == kLnZero) return kLnZero;
  if (p0 == __builtin_inf()) return __builtin_inf();
  return p0 + ph_log1p(ph_fastexp(p1 - p0));
}

// LogProb::ln_sum_exp over three values: the first maximum, then the others in order (a zero-term sum is -0.0)
B2A_HD double ph_sum_exp3(double a, double b, double c) {
  double pmax = a;
  int imax = 0;
  if (b > pmax) pmax = b, imax = 1;
  if (c > pmax) pmax = c, imax = 2;
  if (pmax == kLnZero) return kLnZero;
  if (pmax == __builtin_inf()) return __builtin_inf();
  double s = -0.0;
  if (imax != 0 && a != kLnZero) s += ph_fastexp(a - pmax);
  if (imax != 1 && b != kLnZero) s += ph_fastexp(b - pmax);
  if (imax != 2 && c != kLnZero) s += ph_fastexp(c - pmax);
  return pmax + ph_log1p(s);
}

// LogProb::ln_sum_exp over v[0 .. n)
B2A_HD double ph_sum_exp(const double* v, uint64_t n) {
  if (n == 0) return kLnZero;
  double pmax = v[0];
  uint64_t imax = 0;
  for (uint64_t i = 1; i < n; ++i)
    if (v[i] > pmax) pmax = v[i], imax = i;
  if (pmax == kLnZero) return kLnZero;
  if (pmax == __builtin_inf()) return __builtin_inf();
  double s = -0.0;
  for (uint64_t i = 0; i < n; ++i)
    if (i != imax && v[i] != kLnZero) s += ph_fastexp(v[i] - pmax);
  return pmax + ph_log1p(s);
}

// ln_sum3_exp_approx (pairhmm.rs:26-40): two swaps only, so p1 need not be the second largest
B2A_HD double ph_sum3_approx(double p0, double p1, double p2) {
  if (p1 < p2) {
    const double t = p1;
    p1 = p2;
    p2 = t;
  }
  if (p1 > p0) {
    const double t = p1;
    p1 = p0;
    p0 = t;
  }
  if (p0 - p1 > 10.0) return p0;
  return ph_sum_exp3(p0, p1, p2);
}

// the final cap at ln_one (pairhmm.rs:275-279); a NaN passes through (the reference's assert: a per-pair panic)
B2A_HD double ph_cap(double p) { return p > 0.0 ? 0.0 : p; }

B2A_HD uint32_t ph_sat1(uint32_t v) { return v == kPhmmMedNone ? v : v + 1; }

// ---- warp exchange of the lane code (one warp on the device, 32 emulated lanes in tests/sim) ----

B2A_HD double ph_up(double v) {  // lane - 1's value (lane 0 keeps its own)
#if defined(__CUDA_ARCH__)
  return __shfl_up_sync(0xffffffffu, v, 1);
#elif defined(B2A_HOST_WARP)
  long long b;
  memcpy(&b, &v, 8);
  const int me = host_lane;
  b = host_warp_exchange(b, [&](const long long* x) { return me >= 1 ? x[me - 1] : x[me]; });
  double r;
  memcpy(&r, &b, 8);
  return r;
#else
  return v;
#endif
}
B2A_HD uint32_t ph_up_u32(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return __shfl_up_sync(0xffffffffu, v, 1);
#elif defined(B2A_HOST_WARP)
  const int me = host_lane;
  return (uint32_t)host_warp_exchange((long long)v, [&](const long long* x) { return me >= 1 ? x[me - 1] : x[me]; });
#else
  return v;
#endif
}
B2A_HD double ph_from(double v, int src) {
#if defined(__CUDA_ARCH__)
  return __shfl_sync(0xffffffffu, v, src);
#elif defined(B2A_HOST_WARP)
  long long b;
  memcpy(&b, &v, 8);
  b = host_warp_exchange(b, [&](const long long* x) { return x[src & 31]; });
  double r;
  memcpy(&r, &b, 8);
  return r;
#else
  (void)src;
  return v;
#endif
}

// ---- one pair ----

struct PairHmmSeq {
  const uint8_t *x, *cx, *y, *cy;  // cx / cy: the class bytes beside x / y, or nullptr (every class 0)
  uint32_t m, n;
};

// emit: [4 * n_classes] = emit_match, emit_mismatch, emit_x, emit_y, each indexed by class.  rec: the pair's m
// strip-boundary records (used when n > 32 * C).  cols: 3 * m doubles for the semiglobal end (free_end only).  The
// result, capped at ln_one (NaN: the reference's assert), is valid in every lane.
template <int C>
B2A_HD double pairhmm_warp(const PairHmmGap& g, const double* emit, uint32_t ncls, const PairHmmSeq& s,
                           PairHmmRec* rec, double* cols, int lane) {
  const uint32_t m = s.m, n = s.n;
  const uint32_t strip_cols = 32u * C;
  const uint32_t nstrips = (n + strip_cols - 1) / strip_cols;
  const uint32_t owner_col = (n - 1) % strip_cols;  // 0-based column of j_ = n within the last strip
  const int owner = (int)(owner_col / C), owner_k = (int)(owner_col % C);
  const double* e_match = emit;
  const double* e_mismatch = emit + ncls;
  const double* e_x = emit + 2 * ncls;
  const double* e_y = emit + 3 * ncls;
  double fin_fm = kLnZero, fin_fx = kLnZero, fin_fy = kLnZero;  // the owner's last-row values (global end)
  for (uint32_t st = 0; st < nstrips; ++st) {
    const bool first = st == 0, last = st + 1 == nstrips;
    const uint32_t c0 = st * strip_cols + (uint32_t)lane * C;  // j_ - 1 of the lane's first column
    uint8_t yc[C], ycls[C];
    double pfm[C], pfx[C], pfy[C], qfx[C], qfy[C];
    uint32_t pmed[C], qmed[C];
#pragma unroll
    for (int k = 0; k < C; ++k) {
      const uint32_t j = c0 + k;
      yc[k] = j < n ? s.y[j] : 0;
      ycls[k] = j < n && s.cy ? s.cy[j] : 0;
      pfm[k] = pfx[k] = pfy[k] = qfx[k] = qfy[k] = kLnZero;
      pmed[k] = qmed[k] = kPhmmMedNone;
    }
    // the left neighbour column: row i (lc_*) and row i - 1 (lp_*), as they stand in the buffer
    double lc_fm = kLnZero, lc_fx = kLnZero, lc_fy = kLnZero, lp_fm, lp_fx, lp_fy;
    uint32_t lc_med = kPhmmMedNone, lp_med;
    for (uint32_t t = 0; t < m + 31; ++t) {
      const int64_t i = (int64_t)t - lane;
      const bool row = i >= 0 && i < (int64_t)m;
      lp_fm = lc_fm, lp_fx = lc_fx, lp_fy = lc_fy, lp_med = lc_med;
      // what lane - 1 computed at step t - 1: its row i
      const double r_fm = ph_up(pfm[C - 1]), r_fx = ph_up(pfx[C - 1]), r_fy = ph_up(pfy[C - 1]);
      const uint32_t r_med = ph_up_u32(pmed[C - 1]);
      lc_fm = r_fm, lc_fx = r_fx, lc_fy = r_fy, lc_med = r_med;
      if (lane == 0 && row) {
        if (first) {  // column 0 (pairhmm.rs:134-142): fx, fy stay ln_zero
          lp_fm = i == 0 ? g.col0_first : g.col0_rest;
          lp_fx = lp_fy = kLnZero;
          lp_med = g.free_start ? 0u : kPhmmMedNone;
          lc_fm = lc_fx = lc_fy = kLnZero;
          lc_med = i > 0 && g.free_start ? 0u : kPhmmMedNone;
        } else {
          const PairHmmRec r = rec[i];
          lc_fm = r.fm, lc_fx = r.fx, lc_fy = r.fy, lc_med = r.med;
          if (i == 0) lp_fm = lp_fx = lp_fy = kLnZero, lp_med = kPhmmMedNone;
        }
      }
      if (!row) continue;
      const uint8_t xc = s.x[i];
      const uint32_t xcls = s.cx ? s.cx[i] : 0;
      const double emit_x = e_x[xcls];
      // tl: row i - 1, column to the left; lf: row i, column to the left
      double tl_fm = lp_fm, tl_fx = lp_fx, tl_fy = lp_fy, lf_fm = lc_fm, lf_fy = lc_fy;
      uint32_t tl_med = lp_med, lf_med = lc_med;
#pragma unroll
      for (int k = 0; k < C; ++k) {
        if (c0 + k >= n) break;
        const double o_fm = pfm[k], o_fx = pfx[k], o_fy = pfy[k];
        const uint32_t o_med = pmed[k];
        double n_fm, n_fx, n_fy;
        uint32_t n_med;
        // (reference names: topleft = tl_med, top = lf_med, left = o_med)
        const uint32_t near = lf_med < o_med ? lf_med : o_med;
        const bool skip = g.banded && (tl_med < near ? tl_med : near) > g.max_ed;
        if (skip) {  // fm was reset; fx, fy and min_edit_dist keep row i - 2's values
          n_fm = kLnZero, n_fx = qfx[k], n_fy = qfy[k], n_med = qmed[k];
        } else {
          const bool is_match = xc == yc[k];
          const double exy = is_match ? e_match[ycls[k]] : e_mismatch[ycls[k]];
          n_fm = exy + ph_sum3_approx(g.no_gap + tl_fm, g.no_gap_x_ext + tl_fx, g.no_gap_y_ext + tl_fy);
          n_fx = emit_x + (g.gap_y + o_fm);
          if (g.do_y_ext) n_fx = ph_add_exp(n_fx, g.gap_y_ext + o_fx);
          n_fy = e_y[ycls[k]] + (g.gap_x + lf_fm);
          if (g.do_x_ext) n_fy = ph_add_exp(n_fy, g.gap_x_ext + lf_fy);
          if (g.banded) {
            const uint32_t a = is_match ? tl_med : ph_sat1(tl_med), b = ph_sat1(o_med), c = ph_sat1(lf_med);
            const uint32_t bc = b < c ? b : c;
            n_med = a < bc ? a : bc;
          } else {
            n_med = o_med;  // (not written without a band: stays usize::MAX)
          }
        }
        qfx[k] = o_fx, qfy[k] = o_fy, qmed[k] = o_med;
        pfm[k] = n_fm, pfx[k] = n_fx, pfy[k] = n_fy, pmed[k] = n_med;
        tl_fm = o_fm, tl_fx = o_fx, tl_fy = o_fy, tl_med = o_med;
        lf_fm = n_fm, lf_fy = n_fy, lf_med = n_med;
      }
      if (!last && lane == 31) rec[i] = PairHmmRec{pfm[C - 1], pfx[C - 1], pfy[C - 1], pmed[C - 1], 0};
      if (last && lane == owner) {
        double o_fm = kLnZero, o_fx = kLnZero, o_fy = kLnZero;
#pragma unroll
        for (int k = 0; k < C; ++k)
          if (k == owner_k) o_fm = pfm[k], o_fx = pfx[k], o_fy = pfy[k];
        if (g.free_end) {
          cols[3 * (uint64_t)i] = o_fm, cols[3 * (uint64_t)i + 1] = o_fx, cols[3 * (uint64_t)i + 2] = o_fy;
        } else if (i + 1 == (int64_t)m) {
          fin_fm = o_fm, fin_fx = o_fx, fin_fy = o_fy;
        }
      }
    }
#if defined(__CUDA_ARCH__)
    __syncwarp();  // lane 31's records are visible to lane 0 of the next strip
#endif
  }
  double p = 0.0;
  if (lane == owner) p = ph_cap(g.free_end ? ph_sum_exp(cols, 3 * (uint64_t)m) : ph_sum_exp3(fin_fm, fin_fx, fin_fy));
  return ph_from(p, owner);
}

// The result of a pair with an empty side (the literal loop's closed forms): both empty and a global end give
// ln_one (the untouched fm(0, 0)), anything else ln_zero.
inline double pairhmm_empty(uint32_t m, uint32_t n, bool free_end) {
  return m == 0 && n == 0 && !free_end ? 0.0 : kLnZero;
}

}  // namespace b2a

#include <cmath>
namespace b2a {

// ---- host only ----

// ln_1m_exp (probs/mod.rs:36-43) with the host libm; false where the reference's assert!(p <= 0.0) fires
inline bool pairhmm_ln_1m_exp(double p, double* out) {
  if (!(p <= 0.0)) return false;
  *out = p < -0.693 ? std::log1p(-ph_fastexp(p)) : std::log(-std::expm1(p));
  return true;
}

// PairHMM::new's cache and the call's mode and band.  Returns 0, or 1 / 2 / 3 for the ln_one_minus_exp that asserts
// (its argument: kPairHmmAssertArg[rc - 1]).
constexpr const char* kPairHmmAssertArg[3] = {"prob_gap_x (+) prob_gap_y", "prob_gap_x_extend", "prob_gap_y_extend"};
inline int pairhmm_gap_cache(double gx, double gy, double gxe, double gye, bool free_start, bool free_end,
                                     uint64_t max_edit_dist, PairHmmGap* g) {
  *g = PairHmmGap{};
  if (!pairhmm_ln_1m_exp(ph_add_exp(gx, gy), &g->no_gap)) return 1;
  if (!pairhmm_ln_1m_exp(gxe, &g->no_gap_x_ext)) return 2;
  if (!pairhmm_ln_1m_exp(gye, &g->no_gap_y_ext)) return 3;
  g->gap_x = gx, g->gap_y = gy, g->gap_x_ext = gxe, g->gap_y_ext = gye;
  g->do_x_ext = gxe != kLnZero, g->do_y_ext = gye != kLnZero;
  const double start = free_start ? 0.0 : kLnZero;  // StartEndGapParameters::prob_start_gap_x
  g->col0_first = ph_add_exp(0.0, start);
  g->col0_rest = ph_add_exp(kLnZero, start);
  g->free_start = free_start, g->free_end = free_end;
  // None is UINT64_MAX; Some(usize::MAX) skips nothing either.  A finite min_edit_dist never exceeds len_y < 2^31,
  // so any other bound of 2^32 - 1 or more behaves like 2^32 - 2 on u32 values with 0xFFFFFFFF for usize::MAX.
  g->banded = max_edit_dist != ~0ull;
  g->max_ed = max_edit_dist >= 0xFFFFFFFEull ? 0xFFFFFFFEu : (uint32_t)max_edit_dist;
  return 0;
}

}  // namespace b2a

#if defined(__CUDACC__)
#include <cuda_runtime.h>
namespace b2a {

// Launch of b2a_pairhmm.cu: persistent warps take the tier's tasks from *ctr; each warp owns rec_stride records and
// cols_stride doubles of scratch.  prob[p] is pair p's capped result, in caller order.
struct PairHmmArgs {
  const uint8_t* seq;
  const uint8_t* cls;  // or nullptr
  const uint64_t* x_off;
  const uint32_t* x_len;
  const uint64_t* y_off;
  const uint32_t* y_len;
  const uint32_t* tasks;
  uint32_t n_tasks;
  uint32_t n_classes;
  const double* emit;  // [4 * n_classes]
  PairHmmGap g;
  double* prob;
  PairHmmRec* rec;
  uint64_t rec_stride;
  double* cols;
  uint64_t cols_stride;
};
cudaError_t pairhmm_grid(int tier, int num_sms, uint32_t n_tasks, int* ctas, int* warps_per_cta);
cudaError_t launch_pairhmm(int tier, const PairHmmArgs& a, int ctas, int warps_per_cta, uint32_t* ctr,
                           cudaStream_t st);

}  // namespace b2a
#endif
