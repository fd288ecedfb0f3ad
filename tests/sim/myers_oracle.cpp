// CPU oracle of bio::pattern_matching::myers (test infrastructure): the textbook semi-global dynamic program of
// Sellers (1980) under unit costs, D[0][j] = 0, D[i][0] = i, read off row m at every column, with the match relation
// of MyersBuilder (pattern byte p matches text byte t when t == p, when t is one of p's ambiguity equivalents, or
// when t is a text wildcard).  It restates the definitions and shares no code with the kernels; the definition
// oracle of the edit distance it is tied to (orc_levenshtein) comes along.
#include "distance_oracle.cpp"

extern "C" {

// row[j - 1] = D[m][j] for j = 1..n.  ambig: NULL or 256 rows x 32 bytes (bit t of row p); wildcards: NULL or 32
// bytes.
void orc_myers_row(const uint8_t* x, uint32_t m, const uint8_t* y, uint32_t n, const uint8_t* ambig,
                   const uint8_t* wildcards, uint32_t* row) {
  auto bit = [](const uint8_t* r, uint32_t t) { return ((r[t >> 3] >> (t & 7)) & 1) != 0; };
  auto match = [&](uint8_t p, uint8_t t) {
    return t == p || (ambig && bit(ambig + 32 * p, t)) || (wildcards && bit(wildcards, t));
  };
  std::vector<uint32_t> prev(n + 1, 0), cur(n + 1);  // row 0: D[0][j] = 0
  for (uint32_t i = 1; i <= m; ++i) {
    cur[0] = i;
    for (uint32_t j = 1; j <= n; ++j)
      cur[j] = std::min({prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (match(x[i - 1], y[j - 1]) ? 0u : 1u)});
    std::swap(prev, cur);
  }
  for (uint32_t j = 1; j <= n; ++j) row[j - 1] = prev[j];
}

}  // extern "C"
