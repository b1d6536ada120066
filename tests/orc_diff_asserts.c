/* tests/orc_diff_asserts.c - CPU reference of the changed assertion lines of revision pairs (docs/SPEC.md section 8).
 * TEST INFRASTRUCTURE ONLY, compiled together with oracle/orc.c by tests/orc_asserts.py.  Plain C99, one thread.
 *
 * Per pair: the serial canonical edit script of orc_diff_script (common prefix / suffix trimmed, Myers' greedy search with
 * the rows of V kept, backtrack from the last edit to the first), and for every line it deletes from `old` or inserts into
 * `new` the event orc_scan gives that line when it scans the side's file: the event exists exactly for the assertion lines,
 * and its statement, category, identifier and hash are the scan's.  A pair whose remainder is empty on one side lists every
 * line of the other.  A pair with both remainders non-empty and an edit distance above 23 168 lines is not traced (the
 * device keeps no rows for it: include/tosemscan.h) and contributes nothing. */
#include "orc.h"
#include <stdlib.h>
#include <string.h>

#define TRACE_MAX_D 23168

typedef struct {                    /* one side of one pair, as orc_scan sees the file */
  int64_t n;                        /* lines */
  uint64_t* hash;                   /* [n] */
  orc_assert_event** ev;            /* [n] event of the line, or NULL */
  orc_assert_event* evs; int64_t n_ev;
} Side;

static void side_free(Side* s) { free(s->hash); free(s->ev); free(s->evs); memset(s, 0, sizeof *s); }

static int side_load(const uint8_t* arena, const int32_t* off, const int32_t* len, const uint8_t* ext, Side* s) {
  orc_file_stat st;
  int64_t na = 0, nh = 0, base[2];
  memset(s, 0, sizeof *s);
  if (orc_scan(arena, off, len, ext, NULL, 1, 1, &st, NULL, NULL, NULL, 0, &na, NULL, 0, &nh, NULL, NULL)) return -1;
  s->n = st.n_lines;
  s->hash = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(s->n + 1));
  s->ev = (orc_assert_event**)calloc((size_t)(s->n + 1), sizeof(orc_assert_event*));
  s->evs = (orc_assert_event*)malloc(sizeof(orc_assert_event) * (size_t)(na + 1));
  if (!s->hash || !s->ev || !s->evs) return -1;
  if (orc_scan(arena, off, len, ext, NULL, 1, 1, &st, NULL, NULL, s->evs, na, &s->n_ev, NULL, 0, &nh, s->hash, base)) return -1;
  /* line starts of the file, in order; the events come in line order too */
  const uint8_t* p = arena + off[0];
  uint32_t pos = 0;
  int64_t e = 0;
  for (int64_t i = 0; i < s->n; ++i) {
    if (e < s->n_ev && s->evs[e].line_off == pos) s->ev[i] = &s->evs[e++];
    const uint8_t* nl = memchr(p + pos, '\n', (size_t)((uint32_t)len[0] - pos));
    pos = nl ? (uint32_t)(nl - p) + 1 : (uint32_t)len[0];
  }
  return e == s->n_ev ? 0 : -1;
}

/* Edit script of a[0..n) -> b[0..m) (both non-empty): del[] / ins[] get the deleted / inserted indices, ascending. */
static int64_t script(const uint64_t* a, int64_t n, const uint64_t* b, int64_t m, int64_t* del, int64_t* nd, int64_t* ins, int64_t* ni) {
  const int64_t off = n + m + 1;
  int32_t* V = (int32_t*)calloc((size_t)(2 * (n + m) + 3), sizeof(int32_t));
  int32_t** rows = (int32_t**)calloc((size_t)(n + m + 1), sizeof(int32_t*));
  int64_t D = 0;
  int found = 0;
  if (!V || !rows) { free(V); free(rows); return -1; }
  V[off + 1] = 0;
  for (D = 0; D <= n + m && !found; ++D) {
    for (int64_t k = -D; k <= D; k += 2) {
      int64_t x = (k == -D || (k != D && V[off + k - 1] < V[off + k + 1])) ? V[off + k + 1] : V[off + k - 1] + 1;
      int64_t y = x - k;
      while (x < n && y < m && a[x] == b[y]) { ++x; ++y; }
      V[off + k] = (int32_t)x;
      if (x >= n && y >= m) found = 1;
    }
    rows[D] = (int32_t*)malloc(sizeof(int32_t) * (size_t)(2 * D + 1));
    if (!rows[D]) { found = -1; break; }
    memcpy(rows[D], V + off - D, sizeof(int32_t) * (size_t)(2 * D + 1));
  }
  *nd = *ni = 0;
  if (found == 1) {
    --D;
    int64_t x = n, y = m;
    for (int64_t dd = D; dd >= 1; --dd) {
      const int64_t k = x - y;
      const int32_t* P = rows[dd - 1];
      const int down = (k == -dd || (k != dd && P[k - 1 + dd - 1] < P[k + 1 + dd - 1]));
      const int64_t pk = down ? k + 1 : k - 1;
      const int64_t px = P[pk + dd - 1], py = px - pk;
      if (down) ins[(*ni)++] = py; else del[(*nd)++] = px;
      x = px; y = py;
    }
    for (int64_t i = 0; i < *nd / 2; ++i) { int64_t t = del[i]; del[i] = del[*nd - 1 - i]; del[*nd - 1 - i] = t; }
    for (int64_t i = 0; i < *ni / 2; ++i) { int64_t t = ins[i]; ins[i] = ins[*ni - 1 - i]; ins[*ni - 1 - i] = t; }
  }
  for (int64_t i = 0; i <= n + m; ++i) free(rows[i]);
  free(rows); free(V);
  return found == 1 ? D : -1;
}

static void put(const Side* s, int64_t line, uint32_t pair, uint16_t g, int64_t* counts, orc_assert_event* out, int64_t cap, int64_t* k) {
  const orc_assert_event* e = s->ev[line];
  if (!e) return;                                          /* not an assertion line */
  if (counts) counts[(size_t)g * ORC_K + e->cat]++;
  if (out && *k < cap) { out[*k] = *e; out[*k].file = pair; }
  ++*k;
}

int orc_diff_pairs_asserts(const uint8_t* arena_old, const int32_t* off_old, const int32_t* len_old, const uint8_t* ext_old,
                           const uint16_t* grp_old, const uint8_t* arena_new, const int32_t* off_new, const int32_t* len_new,
                           const uint8_t* ext_new, const uint16_t* grp_new, int32_t n_pairs, int32_t n_groups,
                           int64_t* added_counts, int64_t* removed_counts, orc_assert_event* aev, int64_t aev_cap, int64_t* n_aev,
                           orc_assert_event* rev, int64_t rev_cap, int64_t* n_rev) {
  if (added_counts) memset(added_counts, 0, sizeof(int64_t) * (size_t)n_groups * ORC_K);
  if (removed_counts) memset(removed_counts, 0, sizeof(int64_t) * (size_t)n_groups * ORC_K);
  int64_t ka = 0, kr = 0;
  for (int32_t i = 0; i < n_pairs; ++i) {
    Side A, B;
    if (side_load(arena_old, off_old + i, len_old + i, ext_old + i, &A) || side_load(arena_new, off_new + i, len_new + i, ext_new + i, &B)) {
      side_free(&A); side_free(&B); return -1;
    }
    const uint16_t ga = grp_old ? grp_old[i] : 0, gb = grp_new ? grp_new[i] : 0;
    if (ga >= n_groups || gb >= n_groups) { side_free(&A); side_free(&B); return -1; }
    int64_t n = A.n, m = B.n, pre = 0, suf = 0;
    while (pre < n && pre < m && A.hash[pre] == B.hash[pre]) ++pre;
    while (suf < n - pre && suf < m - pre && A.hash[n - 1 - suf] == B.hash[m - 1 - suf]) ++suf;
    n -= pre + suf; m -= pre + suf;
    int rc = 0;
    if (n == 0 || m == 0) {
      for (int64_t x = 0; x < n; ++x) put(&A, pre + x, (uint32_t)i, ga, removed_counts, rev, rev_cap, &kr);
      for (int64_t y = 0; y < m; ++y) put(&B, pre + y, (uint32_t)i, gb, added_counts, aev, aev_cap, &ka);
    } else if (n + m - 2 * orc_lcs(A.hash + pre, n, B.hash + pre, m) <= TRACE_MAX_D) {
      int64_t* del = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
      int64_t* ins = (int64_t*)malloc(sizeof(int64_t) * (size_t)m);
      int64_t nd = 0, ni = 0;
      if (!del || !ins || script(A.hash + pre, n, B.hash + pre, m, del, &nd, ins, &ni) < 0) rc = -1;
      for (int64_t j = 0; rc == 0 && j < nd; ++j) put(&A, pre + del[j], (uint32_t)i, ga, removed_counts, rev, rev_cap, &kr);
      for (int64_t j = 0; rc == 0 && j < ni; ++j) put(&B, pre + ins[j], (uint32_t)i, gb, added_counts, aev, aev_cap, &ka);
      free(del); free(ins);
    }
    side_free(&A); side_free(&B);
    if (rc) return -1;
  }
  if (n_aev) *n_aev = ka;
  if (n_rev) *n_rev = kr;
  return 0;
}
