/* tests/orc_diff_marks.c - CPU reference of the edit marks of a revision pair (docs/SPEC.md section 14).
 * TEST INFRASTRUCTURE ONLY, compiled by tests/orc_marks.py.  Plain C99, one thread.
 *
 * The serial canonical edit script of SPEC section 8 (the script orc_diff_script traces: common prefix / suffix trimmed,
 * Myers' greedy search with the rows of V kept, backtrack from the last edit to the first), written out per line:
 * del[i] = 1 for every line i of `a` it deletes, ins[j] = 1 for every line j of `b` it inserts (both zeroed first).
 * A remainder empty on one side is one pure hunk: every line of the other remainder is marked.  Returns the edit
 * distance, or -1 when memory runs out. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int64_t orc_diff_marks(const uint64_t* a, int64_t n, const uint64_t* b, int64_t m, uint8_t* del, uint8_t* ins) {
  memset(del, 0, (size_t)n);
  memset(ins, 0, (size_t)m);
  int64_t pre = 0;
  while (pre < n && pre < m && a[pre] == b[pre]) ++pre;
  int64_t suf = 0;
  while (suf < n - pre && suf < m - pre && a[n - 1 - suf] == b[m - 1 - suf]) ++suf;
  a += pre; b += pre; del += pre; ins += pre;
  n -= pre + suf; m -= pre + suf;
  if (n == 0 || m == 0) {
    memset(del, 1, (size_t)n);
    memset(ins, 1, (size_t)m);
    return n + m;
  }
  const int64_t off = n + m + 1;
  int64_t* V = (int64_t*)calloc((size_t)(2 * (n + m) + 3), sizeof(int64_t));
  int64_t** rows = (int64_t**)calloc((size_t)(n + m + 1), sizeof(int64_t*));   /* rows[d][k + d] */
  if (!V || !rows) { free(V); free(rows); return -1; }
  int found = 0;
  int64_t D;
  V[off + 1] = 0;
  for (D = 0; D <= n + m && !found; ++D) {
    for (int64_t k = -D; k <= D; k += 2) {
      int64_t x = (k == -D || (k != D && V[off + k - 1] < V[off + k + 1])) ? V[off + k + 1] : V[off + k - 1] + 1;
      int64_t y = x - k;
      while (x < n && y < m && a[x] == b[y]) { ++x; ++y; }
      V[off + k] = x;
      if (x >= n && y >= m) found = 1;
    }
    rows[D] = (int64_t*)malloc(sizeof(int64_t) * (size_t)(2 * D + 1));
    if (!rows[D]) { found = -1; break; }
    memcpy(rows[D], V + off - D, sizeof(int64_t) * (size_t)(2 * D + 1));
  }
  if (found == 1) {
    --D;
    int64_t x = n, y = m;
    for (int64_t d = D; d >= 1; --d) {
      const int64_t k = x - y;
      const int64_t* P = rows[d - 1];                     /* P[kk + d - 1] */
      const int down = (k == -d || (k != d && P[k - 1 + d - 1] < P[k + 1 + d - 1]));
      const int64_t pk = down ? k + 1 : k - 1;
      const int64_t px = P[pk + d - 1], py = px - pk;
      if (down) ins[py] = 1; else del[px] = 1;
      x = px; y = py;
    }
  }
  for (int64_t i = 0; i <= n + m; ++i) free(rows[i]);
  free(rows); free(V);
  return found == 1 ? D : -1;
}
