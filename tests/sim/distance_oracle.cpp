// CPU oracle of bio::alignment::distance (test infrastructure).  The reference computes levenshtein and
// bounded_levenshtein with the editdistancek and triple_accel crates and hamming with a loop (distance.rs:25-172);
// the crates are not in its tree, so this file restates the DEFINITIONS instead: a textbook O(mn) two-row dynamic
// program for the unit-cost edit distance, a loop for Hamming, and bounded_levenshtein's rule
// (Some(d) iff d <= min(k, max(|x|, |y|))).  Nothing here shares code with the kernels.
#include <algorithm>
#include <cstdint>
#include <vector>

extern "C" {

uint32_t orc_levenshtein(const uint8_t* x, uint32_t m, const uint8_t* y, uint32_t n) {
  std::vector<uint32_t> prev(n + 1), cur(n + 1);
  for (uint32_t j = 0; j <= n; ++j) prev[j] = j;
  for (uint32_t i = 1; i <= m; ++i) {
    cur[0] = i;
    for (uint32_t j = 1; j <= n; ++j)
      cur[j] = std::min({prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (x[i - 1] == y[j - 1] ? 0u : 1u)});
    std::swap(prev, cur);
  }
  return prev[n];
}

// 0xFFFFFFFF: None
uint32_t orc_bounded_levenshtein(const uint8_t* x, uint32_t m, const uint8_t* y, uint32_t n, uint32_t k) {
  const uint32_t d = orc_levenshtein(x, m, y, n);
  return d <= std::min(k, std::max(m, n)) ? d : 0xFFFFFFFFu;
}

// -1: the lengths differ (the reference panics)
int64_t orc_hamming(const uint8_t* x, uint32_t m, const uint8_t* y, uint32_t n) {
  if (m != n) return -1;
  int64_t d = 0;
  for (uint32_t i = 0; i < m; ++i) d += x[i] != y[i];
  return d;
}

}  // extern "C"
