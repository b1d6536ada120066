/* orc_similarity.c - serial CPU reference of the rename similarity of docs/SPEC.md section 13.  TEST INFRASTRUCTURE ONLY.
 *
 * Works from the raw bytes: it splits every file at LF itself (section 2), hashes each line with orc_line_hash
 * (section 3) and weighs it (its bytes, plus 1 for the LF, minus 1 for the CR of a CRLF), so it shares no line records
 * with the device path.  Per file the (hash, weight) pairs are sorted and equal hashes merged; per candidate the two
 * sorted lists are walked together and min(w, w') summed. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "orc.h"

typedef struct { uint64_t h; int64_t w; } HW;
typedef struct { HW* e; int64_t n; } List;

static int cmp_hw(const void* x, const void* y) {
  const uint64_t a = ((const HW*)x)->h, b = ((const HW*)y)->h;
  return a < b ? -1 : a > b;
}

static int file_list(const uint8_t* p, int64_t len, List* out) {
  int64_t lines = 0;
  for (int64_t i = 0; i < len; ++i) lines += p[i] == 0x0A;
  lines += len > 0 && p[len - 1] != 0x0A;
  out->e = (HW*)malloc(sizeof(HW) * (size_t)(lines ? lines : 1));
  out->n = 0;
  if (!out->e) return -1;
  int64_t pos = 0, k = 0;
  while (pos < len) {
    const uint8_t* lf = (const uint8_t*)memchr(p + pos, 0x0A, (size_t)(len - pos));
    const int64_t end = lf ? (int64_t)(lf - p) : len;
    int64_t w = end - pos;
    if (lf) w += (end > pos && p[end - 1] == 0x0D) ? 0 : 1;
    out->e[k].h = orc_line_hash(p + pos, (uint64_t)(end - pos));
    out->e[k].w = w;
    ++k;
    pos = end + 1;
  }
  qsort(out->e, (size_t)k, sizeof(HW), cmp_hw);
  int64_t m = 0;
  for (int64_t i = 0; i < k; ++i) {
    if (m && out->e[m - 1].h == out->e[i].h) out->e[m - 1].w += out->e[i].w;
    else out->e[m++] = out->e[i];
  }
  out->n = m;
  return 0;
}

static void free_lists(List* l, int32_t n) {
  if (!l) return;
  for (int32_t i = 0; i < n; ++i) free(l[i].e);
  free(l);
}

/* common[c] of file cand_old[c] of side a and file cand_new[c] of side b; 0 on success, -1 on a bad index or no memory. */
int orc_similarity(const uint8_t* arena_a, const int32_t* off_a, const int32_t* len_a, int32_t n_a,
                   const uint8_t* arena_b, const int32_t* off_b, const int32_t* len_b, int32_t n_b,
                   const int32_t* cand_old, const int32_t* cand_new, int64_t n_cand, int64_t* common) {
  List* la = (List*)calloc((size_t)(n_a > 0 ? n_a : 1), sizeof(List));
  List* lb = (List*)calloc((size_t)(n_b > 0 ? n_b : 1), sizeof(List));
  int rc = (la && lb) ? 0 : -1;
  for (int32_t i = 0; rc == 0 && i < n_a; ++i) rc = file_list(arena_a + off_a[i], len_a[i], &la[i]);
  for (int32_t i = 0; rc == 0 && i < n_b; ++i) rc = file_list(arena_b + off_b[i], len_b[i], &lb[i]);
  for (int64_t c = 0; rc == 0 && c < n_cand; ++c) {
    if (cand_old[c] < 0 || cand_old[c] >= n_a || cand_new[c] < 0 || cand_new[c] >= n_b) { rc = -1; break; }
    const List* x = &la[cand_old[c]];
    const List* y = &lb[cand_new[c]];
    int64_t i = 0, j = 0, s = 0;
    while (i < x->n && j < y->n) {
      if (x->e[i].h < y->e[j].h) ++i;
      else if (x->e[i].h > y->e[j].h) ++j;
      else { s += x->e[i].w < y->e[j].w ? x->e[i].w : y->e[j].w; ++i; ++j; }
    }
    common[c] = s;
  }
  free_lists(la, n_a);
  free_lists(lb, n_b);
  return rc;
}
