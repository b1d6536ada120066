/* CPU reference of the scores and the pairing of docs/SPEC.md section 17 (TEST INFRASTRUCTURE ONLY, tests/orc_assert_edits.py).
 * Serial and plain: the LCS by the O(nm) table of one row, every candidate of a hunk scored, then qsort and the greedy pass.
 * Entries of each side come sorted by key (hunk); a line is bytes[off[i], off[i] + len[i]). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int64_t lcs(const uint8_t* a, int64_t n, const uint8_t* b, int64_t m, int32_t* row) {
  memset(row, 0, sizeof(int32_t) * (size_t)(m + 1));
  for (int64_t i = 0; i < n; ++i) {
    int32_t diag = 0;                                      /* row[j] of the previous row, before it is overwritten */
    for (int64_t j = 1; j <= m; ++j) {
      const int32_t up = row[j];
      row[j] = a[i] == b[j - 1] ? diag + 1 : (up > row[j - 1] ? up : row[j - 1]);
      diag = up;
    }
  }
  return row[m];
}

typedef struct { int64_t score, i, j; } cand_t;

static int cmp(const void* x, const void* y) {
  const cand_t *p = (const cand_t*)x, *q = (const cand_t*)y;
  if (p->score != q->score) return p->score > q->score ? -1 : 1;
  if (p->i != q->i) return p->i < q->i ? -1 : 1;
  return (p->j > q->j) - (p->j < q->j);
}

/* Edits (rev, aev, score) of the entries; returns their number, or -1 when out of memory / more than cap. */
int64_t orc_assert_edits(int64_t n_old, const uint64_t* ko, const int64_t* oo, const int64_t* lo, const uint8_t* bo,
                         int64_t n_new, const uint64_t* kn, const int64_t* on, const int64_t* ln, const uint8_t* bn,
                         int64_t* rev, int64_t* aev, int64_t* score, int64_t cap) {
  int64_t maxlen = 1, nc = 0, cc = 1024, ne = 0;
  for (int64_t j = 0; j < n_new; ++j) if (ln[j] > maxlen) maxlen = ln[j];
  int32_t* row = (int32_t*)malloc(sizeof(int32_t) * (size_t)(maxlen + 1));
  cand_t* c = (cand_t*)malloc(sizeof(cand_t) * (size_t)cc);
  char *uo = (char*)calloc((size_t)n_old + 1, 1), *un = (char*)calloc((size_t)n_new + 1, 1);
  if (!row || !c || !uo || !un) return -1;
  int64_t j0 = 0;
  for (int64_t i = 0; i < n_old; ++i) {
    while (j0 < n_new && kn[j0] < ko[i]) ++j0;
    for (int64_t j = j0; j < n_new && kn[j] == ko[i]; ++j) {
      const int64_t l = lcs(bo + oo[i], lo[i], bn + on[j], ln[j], row);
      const int64_t s = lo[i] + ln[j] ? 120000 * l / (lo[i] + ln[j]) : 0;
      if (s < 30000) continue;
      if (nc == cc) {
        cc *= 2;
        c = (cand_t*)realloc(c, sizeof(cand_t) * (size_t)cc);
        if (!c) return -1;
      }
      c[nc].score = s; c[nc].i = i; c[nc].j = j; ++nc;
    }
  }
  qsort(c, (size_t)nc, sizeof(cand_t), cmp);
  for (int64_t k = 0; k < nc; ++k) {
    if (uo[c[k].i] || un[c[k].j]) continue;
    uo[c[k].i] = un[c[k].j] = 1;
    if (ne == cap) { ne = -1; break; }
    rev[ne] = c[k].i; aev[ne] = c[k].j; score[ne] = c[k].score; ++ne;
  }
  free(row); free(c); free(uo); free(un);
  return ne;
}
