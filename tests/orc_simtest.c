/* Serial C reference of the similar tests of docs/SPEC.md section 23.  TEST INFRASTRUCTURE ONLY.  Brute force over every pair of
 * compared tests; only the size filter is applied before the LCS, because it is exact arithmetic. */
#include <stdint.h>
#include <stdlib.h>

/* seq[beg[t] .. beg[t] + k[t]) is the sequence of test t (blind hashes of its kept lines).  The pairs go to pa / pb / plcs in
 * ascending (a, b) order; *n is always set; returns -3 when cap is short, -1 on no memory. */
static uint32_t lcs_of(const uint64_t* x, uint32_t ka, const uint64_t* y, uint32_t kb, uint32_t* row) {
  for (uint32_t j = 0; j <= kb; ++j) row[j] = 0;
  for (uint32_t i = 0; i < ka; ++i) {
    uint32_t diag = 0;
    for (uint32_t j = 0; j < kb; ++j) {
      const uint32_t up = row[j + 1];
      row[j + 1] = x[i] == y[j] ? diag + 1 : (up > row[j] ? up : row[j]);
      diag = up;
    }
  }
  return row[kb];
}

int orc_similar(const uint64_t* seq, const int64_t* beg, const uint32_t* k, int32_t nt, int32_t min_lines, int32_t P, int32_t* pa,
                int32_t* pb, uint32_t* plcs, int64_t cap, int64_t* n) {
  uint32_t kmax = 0;
  for (int32_t t = 0; t < nt; ++t) if (k[t] > kmax) kmax = k[t];
  uint32_t* row = malloc(sizeof(uint32_t) * ((size_t)kmax + 1));
  if (!row) return -1;
  int64_t m = 0;
  for (int32_t a = 0; a < nt; ++a) {
    const uint32_t ka = k[a];
    if (ka < (uint32_t)min_lines) continue;
    const uint64_t* x = seq + beg[a];
    for (int32_t b = a + 1; b < nt; ++b) {
      const uint32_t kb = k[b];
      if (kb < (uint32_t)min_lines) continue;
      const uint32_t lo = ka < kb ? ka : kb;
      if (200ull * lo < (uint64_t)P * (ka + kb)) continue;
      const uint32_t l = lcs_of(x, ka, seq + beg[b], kb, row);
      if (200ull * l >= (uint64_t)P * (ka + kb)) {
        if (m < cap) { pa[m] = a; pb[m] = b; plcs[m] = l; }
        ++m;
      }
    }
  }
  free(row);
  *n = m;
  return m > cap ? -3 : 0;
}

/* The partners of one test a over the whole corpus: every compared b != a that pairs with a, by brute force, into other[] (cap
 * entries, ascending); returns how many there are, or -1 on no memory. */
int64_t orc_similar_row(const uint64_t* seq, const int64_t* beg, const uint32_t* k, int32_t nt, int32_t a, int32_t min_lines, int32_t P,
                        int32_t* other, int64_t cap) {
  if (k[a] < (uint32_t)min_lines) return 0;
  uint32_t kmax = 0;
  for (int32_t t = 0; t < nt; ++t) if (k[t] > kmax) kmax = k[t];
  uint32_t* row = malloc(sizeof(uint32_t) * ((size_t)kmax + 1));
  if (!row) return -1;
  int64_t m = 0;
  for (int32_t b = 0; b < nt; ++b) {
    const uint32_t ka = k[a], kb = k[b];
    if (b == a || kb < (uint32_t)min_lines) continue;
    const uint32_t lo = ka < kb ? ka : kb;
    if (200ull * lo < (uint64_t)P * (ka + kb)) continue;
    const uint32_t l = lcs_of(seq + beg[a], ka, seq + beg[b], kb, row);
    if (200ull * l >= (uint64_t)P * (ka + kb)) { if (m < cap) other[m] = b; ++m; }
  }
  free(row);
  return m;
}

/* The LCS of n pairs: out[i] = lcs(seq of a[i], seq of b[i]).  Returns -1 on no memory. */
int orc_lcs_pairs(const uint64_t* seq, const int64_t* beg, const uint32_t* k, const int32_t* a, const int32_t* b, int64_t n, uint32_t* out) {
  uint32_t kmax = 0;
  for (int64_t i = 0; i < n; ++i) if (k[b[i]] > kmax) kmax = k[b[i]];
  uint32_t* row = malloc(sizeof(uint32_t) * ((size_t)kmax + 1));
  if (!row) return -1;
  for (int64_t i = 0; i < n; ++i) out[i] = lcs_of(seq + beg[a[i]], k[a[i]], seq + beg[b[i]], k[b[i]], row);
  free(row);
  return 0;
}
