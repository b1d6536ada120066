/* orc_clones.c - serial CPU reference of the clone classes of docs/SPEC.md section 15.  TEST INFRASTRUCTURE ONLY.
 *
 * States section 15 literally from the raw bytes: it splits every file at LF itself (section 2), hashes each line with
 * orc_line_hash and keys each window with orc_ngram_hashes (section 3), flags assertion lines with orc_is_assert_line
 * (section 4), groups the windows by a qsort of (key, position), and walks the classes serially in position order. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "orc.h"

typedef struct { uint64_t k; int64_t p; } KP;

static int cmp_kp(const void* x, const void* y) {
  const KP* a = (const KP*)x; const KP* b = (const KP*)y;
  if (a->k != b->k) return a->k < b->k ? -1 : 1;
  return a->p < b->p ? -1 : a->p > b->p;
}

/* Returns 0, -1 (bad argument / no memory) or -3 (class_cap < classes or member_cap < fragments; the counts are set). */
int orc_clones(const uint8_t* arena, const int32_t* off, const int32_t* len, const uint8_t* ext, int32_t n_files, int32_t n,
               int64_t* line_base, uint32_t* file_dup, uint32_t* file_dup_assert, int64_t* class_base, uint32_t* class_len,
               int64_t class_cap, int64_t* n_classes, int64_t* member, int64_t member_cap, int64_t* n_members) {
  if (n < 1 || n > 1024 || n_files < 0) return -1;
  int64_t T = 0;
  line_base[0] = 0;
  for (int32_t f = 0; f < n_files; ++f) {
    const uint8_t* p = arena + off[f];
    int64_t lines = 0;
    for (int32_t i = 0; i < len[f]; ++i) lines += p[i] == 0x0A;
    lines += len[f] > 0 && p[len[f] - 1] != 0x0A;
    T += lines;
    line_base[f + 1] = T;
  }
  const size_t m = (size_t)(T ? T : 1);
  uint64_t* hash = (uint64_t*)malloc(8 * m); uint64_t* key = (uint64_t*)malloc(8 * m);
  uint8_t* empty = (uint8_t*)malloc(m); uint8_t* flag = (uint8_t*)malloc(m); uint8_t* covered = (uint8_t*)calloc(m, 1);
  int32_t* file = (int32_t*)malloc(4 * m); int64_t* gid = (int64_t*)malloc(8 * m);
  KP* w = (KP*)malloc(sizeof(KP) * m);
  int64_t *gstart = (int64_t*)malloc(8 * m), *gcount = (int64_t*)malloc(8 * m);
  uint8_t* gext = (uint8_t*)malloc(m);
  int rc = (hash && key && empty && flag && covered && file && gid && w && gstart && gcount && gext) ? 0 : -1;
  int64_t nw = 0, ng = 0, nc = 0, nm = 0;
  if (rc == 0) {
    int64_t l = 0;
    for (int32_t f = 0; f < n_files; ++f) {                /* section 2: lines; section 3: hashes; section 4: flags */
      const uint8_t* p = arena + off[f];
      int64_t pos = 0;
      while (pos < len[f]) {
        const uint8_t* lf = (const uint8_t*)memchr(p + pos, 0x0A, (size_t)(len[f] - pos));
        const int64_t end = lf ? (int64_t)(lf - p) : len[f];
        const int64_t ll = end - pos;
        hash[l] = orc_line_hash(p + pos, (uint64_t)ll);
        empty[l] = ll == 0 || (ll == 1 && p[pos] == 0x0D);
        flag[l] = ext[f] != 0 && orc_is_assert_line(p + pos, (uint32_t)ll);
        file[l] = f;
        ++l;
        pos = end + 1;
      }
    }
    orc_ngram_hashes(hash, line_base, n_files, n, key);
    for (int64_t p = 0; p < T; ++p) {                     /* 1. windows: n lines of one file, not all empty */
      gid[p] = -1;
      if (p + n > line_base[file[p] + 1]) continue;
      int all_empty = 1;
      for (int32_t k = 0; k < n && all_empty; ++k) all_empty = empty[p + k];
      if (all_empty) continue;
      w[nw].k = key[p]; w[nw].p = p; ++nw;
    }
    qsort(w, (size_t)nw, sizeof(KP), cmp_kp);              /* 2. groups: runs of equal keys, positions ascending */
    for (int64_t i = 0; i < nw; ++i) {
      if (i == 0 || w[i].k != w[i - 1].k) { gstart[ng] = i; gcount[ng] = 0; ++ng; }
      gcount[ng - 1]++;
      gid[w[i].p] = ng - 1;
    }
    for (int64_t g = 0; g < ng; ++g) {                     /* 3. left-extendable */
      gext[g] = 0;
      if (gcount[g] < 2) continue;
      int64_t prev = -1;
      int ok = 1;
      for (int64_t i = gstart[g]; i < gstart[g] + gcount[g] && ok; ++i) {
        const int64_t q = w[i].p;
        if (q == line_base[file[q]] || gid[q - 1] < 0) ok = 0;
        else if (prev < 0) prev = gid[q - 1];
        else if (gid[q - 1] != prev) ok = 0;
      }
      gext[g] = (uint8_t)(ok && gcount[prev] == gcount[g]);
    }
    for (int64_t p = 0; p < T; ++p) {                      /* 4. classes in representative order; 5. coverage */
      const int64_t g = gid[p];
      if (g < 0 || gcount[g] < 2) continue;
      for (int32_t k = 0; k < n; ++k) covered[p + k] = 1;
      if (gext[g] || w[gstart[g]].p != p) continue;
      int64_t r = 0;
      while (p + r + 1 < T && file[p + r + 1] == file[p] && gid[p + r + 1] >= 0 && gcount[gid[p + r + 1]] >= 2 && gext[gid[p + r + 1]]) ++r;
      if (nc < class_cap && class_len) class_len[nc] = (uint32_t)(n + r);
      if (nc < class_cap && class_base) class_base[nc] = nm;
      for (int64_t i = gstart[g]; i < gstart[g] + gcount[g]; ++i, ++nm)
        if (nm < member_cap && member) member[nm] = w[i].p;
      ++nc;
    }
    if (nc <= class_cap && class_base) class_base[nc] = nm;
    for (int32_t f = 0; f < n_files; ++f) {
      uint32_t d = 0, a = 0;
      for (int64_t x = line_base[f]; x < line_base[f + 1]; ++x) { d += covered[x]; a += covered[x] && flag[x]; }
      if (file_dup) file_dup[f] = d;
      if (file_dup_assert) file_dup_assert[f] = a;
    }
    *n_classes = nc; *n_members = nm;
    if (nc > class_cap || nm > member_cap) rc = -3;
  }
  free(hash); free(key); free(empty); free(flag); free(covered); free(file); free(gid); free(w); free(gstart); free(gcount); free(gext);
  return rc;
}
