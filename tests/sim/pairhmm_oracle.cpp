// CPU oracle of bio::stats::pairhmm::PairHMM::prob_related (test infrastructure): a statement-by-statement C++
// restatement of the reference's PairHMM::new and prob_related (src/stats/pairhmm/pairhmm.rs:26-40, 69-95, 104-280),
// LogProb::{ln_add_exp, ln_sum_exp, ln_one_minus_exp} and ln_1m_exp (src/stats/probs/mod.rs:36-43, 213-271) and
// FastExp (src/utils/fastexp.rs:33-58), with the emission trait object in its tabulated per-class form.  It uses the
// host libm (log1p, expm1, log), as Rust's f64 methods do on Linux, and is built without FP contraction.  It shares
// no code with the kernels.  Threaded batch form for the benchmark and the GPU tests.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <thread>
#include <utility>
#include <vector>

namespace {

const double LN_ZERO = -std::numeric_limits<double>::infinity();
const double LN_ONE = 0.0;
const uint64_t USIZE_MAX = ~0ull;

double fastexp(double self) {
  const double MIN_VAL = -500.0;
  if (self > MIN_VAL) {
    double x = 1.442695041 * self;
    int64_t bits = (int64_t)x;
    x -= (double)bits;
    double f2 = x;
    double x_tmp = x;
    bits += 1023;
    bits <<= 52;
    f2 *= 0.006935931;
    x_tmp += 4.831794110;
    f2 += 0.019890581;
    x_tmp *= x;
    f2 *= x;
    f2 += 0.143440676;
    f2 *= x_tmp;
    f2 += 1.0;
    double b;
    std::memcpy(&b, &bits, 8);
    return b * f2;
  }
  return 0.0;
}

// false: assert!(p <= 0.0) panics
bool ln_1m_exp(double p, double* out) {
  if (!(p <= 0.0)) return false;
  if (p < -0.693)
    *out = std::log1p(-fastexp(p));
  else
    *out = std::log(-std::expm1(p));
  return true;
}

double ln_sum_exp(const double* probs, size_t n) {
  if (n == 0) return LN_ZERO;
  double pmax = probs[0];
  size_t imax = 0;
  for (size_t i = 1; i < n; ++i) {
    if (probs[i] > pmax) {
      pmax = probs[i];
      imax = i;
    }
  }
  if (pmax == LN_ZERO) return LN_ZERO;
  if (pmax == std::numeric_limits<double>::infinity()) return std::numeric_limits<double>::infinity();
  double sum = -0.0;  // <f64 as Sum>: a fold from -0.0
  for (size_t i = 0; i < n; ++i) {
    if (i == imax || probs[i] == LN_ZERO) continue;
    sum += fastexp(probs[i] - pmax);
  }
  return pmax + std::log1p(sum);
}

double ln_add_exp(double self, double other) {
  if (other == LN_ZERO) return self;
  double p0 = self, p1 = other;
  if (p1 > p0) std::swap(p0, p1);
  if (p0 == LN_ZERO) return LN_ZERO;
  if (p0 == std::numeric_limits<double>::infinity()) return std::numeric_limits<double>::infinity();
  return p0 + std::log1p(fastexp(p1 - p0));
}

double ln_sum3_exp_approx(double p0, double p1, double p2) {
  if (p1 < p2) std::swap(p1, p2);
  if (p1 > p0) std::swap(p1, p0);
  if (p0 - p1 > 10.0) return p0;
  const double v[3] = {p0, p1, p2};
  return ln_sum_exp(v, 3);
}

uint64_t sat_add1(uint64_t v) { return v == USIZE_MAX ? v : v + 1; }

struct Gap {
  double prob_no_gap, prob_no_gap_x_extend, prob_no_gap_y_extend, prob_gap_x, prob_gap_y, prob_gap_x_extend,
      prob_gap_y_extend;
  bool do_gap_x_extend, do_gap_y_extend;
};

// PairHMM::new: 0, or 1 / 2 / 3 for the ln_one_minus_exp that asserts
int pairhmm_new(double gx, double gy, double gxe, double gye, Gap* g) {
  if (!ln_1m_exp(ln_add_exp(gx, gy), &g->prob_no_gap)) return 1;
  if (!ln_1m_exp(gxe, &g->prob_no_gap_x_extend)) return 2;
  if (!ln_1m_exp(gye, &g->prob_no_gap_y_extend)) return 3;
  g->prob_gap_x = gx;
  g->prob_gap_y = gy;
  g->prob_gap_x_extend = gxe;
  g->prob_gap_y_extend = gye;
  g->do_gap_y_extend = gye != LN_ZERO;
  g->do_gap_x_extend = gxe != LN_ZERO;
  return 0;
}

struct Emission {
  const uint8_t *x, *cx, *y, *cy;
  size_t len_x, len_y;
  const double *emit_match, *emit_mismatch, *emit_x, *emit_y;
  int cls_x(size_t i) const { return cx ? cx[i] : 0; }
  int cls_y(size_t j) const { return cy ? cy[j] : 0; }
  // (is_match, prob)
  std::pair<bool, double> prob_emit_xy(size_t i, size_t j) const {
    if (x[i] == y[j]) return {true, emit_match[cls_y(j)]};
    return {false, emit_mismatch[cls_y(j)]};
  }
  double prob_emit_x(size_t i) const { return emit_x[cls_x(i)]; }
  double prob_emit_y(size_t j) const { return emit_y[cls_y(j)]; }
};

// prob_related; the result before the NaN assert (a NaN is the reference's panic)
double prob_related(const Gap& gp, const Emission& ep, bool free_start_gap_x, bool free_end_gap_x, bool has_max,
                    uint64_t max_edit_dist) {
  std::vector<double> fm[2], fx[2], fy[2];
  std::vector<uint64_t> min_edit_dist[2];
  std::vector<double> prob_cols;
  for (int k = 0; k < 2; ++k) {
    fm[k].assign(ep.len_y + 1, LN_ZERO);
    fx[k].assign(ep.len_y + 1, LN_ZERO);
    fy[k].assign(ep.len_y + 1, LN_ZERO);
    min_edit_dist[k].assign(ep.len_y + 1, USIZE_MAX);
  }
  if (free_end_gap_x) prob_cols.reserve(ep.len_x * 3);
  int prev = 0, curr = 1;
  fm[prev][0] = LN_ONE;
  auto prob_start_gap_x = [&](size_t) { return free_start_gap_x ? LN_ONE : LN_ZERO; };
  for (size_t i = 0; i < ep.len_x; ++i) {
    fm[prev][0] = ln_add_exp(fm[prev][0], prob_start_gap_x(i));
    if (free_start_gap_x) min_edit_dist[prev][0] = 0;
    const double prob_emit_x = ep.prob_emit_x(i);
    for (size_t j = 0; j < ep.len_y; ++j) {
      const size_t j_ = j + 1;
      const size_t j_minus_one = j_ - 1;
      const uint64_t min_edit_dist_topleft = min_edit_dist[prev][j_minus_one];
      const uint64_t min_edit_dist_top = min_edit_dist[curr][j_minus_one];
      const uint64_t min_edit_dist_left = min_edit_dist[prev][j_];
      if (has_max) {
        if (std::min(min_edit_dist_topleft, std::min(min_edit_dist_top, min_edit_dist_left)) > max_edit_dist) continue;
      }
      const std::pair<bool, double> emit_xy = ep.prob_emit_xy(i, j);
      const double prob_match_mismatch =
          emit_xy.second + ln_sum3_exp_approx(gp.prob_no_gap + fm[prev][j_minus_one],
                                              gp.prob_no_gap_x_extend + fx[prev][j_minus_one],
                                              gp.prob_no_gap_y_extend + fy[prev][j_minus_one]);
      double prob_gap_y = prob_emit_x + (gp.prob_gap_y + fm[prev][j_]);
      if (gp.do_gap_y_extend) prob_gap_y = ln_add_exp(prob_gap_y, gp.prob_gap_y_extend + fx[prev][j_]);
      double prob_gap_x = ep.prob_emit_y(j) + (gp.prob_gap_x + fm[curr][j_minus_one]);
      if (gp.do_gap_x_extend) prob_gap_x = ln_add_exp(prob_gap_x, gp.prob_gap_x_extend + fy[curr][j_minus_one]);
      uint64_t med = 0;
      if (has_max)
        med = std::min(emit_xy.first ? min_edit_dist_topleft : sat_add1(min_edit_dist_topleft),
                       std::min(sat_add1(min_edit_dist_left), sat_add1(min_edit_dist_top)));
      fm[curr][j_] = prob_match_mismatch;
      fx[curr][j_] = prob_gap_y;
      fy[curr][j_] = prob_gap_x;
      if (has_max) min_edit_dist[curr][j_] = med;
    }
    if (free_end_gap_x) {
      prob_cols.push_back(fm[curr].back());
      prob_cols.push_back(fx[curr].back());
      prob_cols.push_back(fy[curr].back());
    }
    std::swap(curr, prev);
    for (double& v : fm[curr]) v = LN_ZERO;
  }
  double p;
  if (free_end_gap_x) {
    p = ln_sum_exp(prob_cols.data(), prob_cols.size());
  } else {
    const double v[3] = {fm[prev].back(), fx[prev].back(), fy[prev].back()};
    p = ln_sum_exp(v, 3);
  }
  if (std::isnan(p)) return p;
  return p > LN_ONE ? LN_ONE : p;
}

}  // namespace

extern "C" {

double orc_fastexp(double v) { return fastexp(v); }
double orc_ln_add_exp(double a, double b) { return ln_add_exp(a, b); }
double orc_ln_sum_exp(const double* v, uint64_t n) { return ln_sum_exp(v, n); }
int orc_ln_one_minus_exp(double p, double* out) { return ln_1m_exp(p, out) ? 0 : 1; }
double orc_ln_sum3_exp_approx(double a, double b, double c) { return ln_sum3_exp_approx(a, b, c); }

// gap[4]: prob_gap_x, prob_gap_y, prob_gap_x_extend, prob_gap_y_extend.  has_max = 0: None.  emit: [4][n_classes]
// (match, mismatch, x, y).  Returns 0, or 1 / 2 / 3 when PairHMM::new asserts (no result written).
int orc_pairhmm_batch(const double* gap, int free_start, int free_end, int has_max, uint64_t max_edit_dist,
                      const double* emit, uint32_t n_classes, const uint8_t* blob, const uint8_t* cls,
                      const uint64_t* xo, const uint32_t* xl, const uint64_t* yo, const uint32_t* yl, uint64_t n,
                      int threads, double* out) {
  Gap g;
  const int rc = pairhmm_new(gap[0], gap[1], gap[2], gap[3], &g);
  if (rc) return rc;
  auto one = [&](uint64_t p) {
    Emission e{blob + xo[p], cls ? cls + xo[p] : nullptr, blob + yo[p], cls ? cls + yo[p] : nullptr, xl[p], yl[p],
               emit, emit + n_classes, emit + 2 * n_classes, emit + 3 * n_classes};
    out[p] = prob_related(g, e, free_start != 0, free_end != 0, has_max != 0, max_edit_dist);
  };
  if (threads <= 1 || n < 2) {
    for (uint64_t p = 0; p < n; ++p) one(p);
    return 0;
  }
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&, t]() {
      for (uint64_t p = (uint64_t)t; p < n; p += (uint64_t)threads) one(p);
    });
  for (auto& th : pool) th.join();
  return 0;
}

}  // extern "C"
