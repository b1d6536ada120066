/* orc_blind.c - serial CPU reference of the blind clones of docs/SPEC.md section 21.  TEST INFRASTRUCTURE ONLY.
 *
 * orc_blind_lines states the lexer of section 21 literally from the raw bytes: it splits every file at LF itself (section 2),
 * lexes its lines in order from the code state, writes each line's blind form into a buffer and hashes it with orc_bytes_hash
 * (section 3), and flags assertion lines with orc_is_assert_line (section 4).  orc_clone_walk is section 15 over a
 * caller-supplied line sequence (hashes, assertion flags and per-file bases; no line is empty): n-gram keys with
 * orc_ngram_hashes, groups by a qsort of (key, position), and the serial class walk in position order. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "orc.h"

static const char* const kPy[] = {"and", "as", "assert", "async", "await", "break", "class", "continue", "def", "del", "elif", "else",
  "except", "finally", "for", "from", "global", "if", "import", "in", "is", "lambda", "nonlocal", "not", "or", "pass", "raise", "return",
  "try", "while", "with", "yield", 0};
static const char* const kCj[] = {"_", "_Alignas", "_Alignof", "_Atomic", "_Bool", "_Complex", "_Generic", "_Imaginary", "_Noreturn",
  "_Static_assert", "_Thread_local", "abstract", "alignas", "alignof", "and", "and_eq", "asm", "assert", "auto", "bitand", "bitor",
  "bool", "boolean", "break", "byte", "case", "catch", "char", "char16_t", "char32_t", "char8_t", "class", "co_await", "co_return",
  "co_yield", "compl", "concept", "const", "const_cast", "consteval", "constexpr", "constinit", "continue", "decltype", "default",
  "delete", "do", "double", "dynamic_cast", "else", "enum", "explicit", "export", "extends", "extern", "final", "finally", "float",
  "for", "friend", "goto", "if", "implements", "import", "inline", "instanceof", "int", "interface", "long", "mutable", "namespace",
  "native", "new", "noexcept", "not", "not_eq", "operator", "or", "or_eq", "package", "private", "protected", "public", "register",
  "reinterpret_cast", "requires", "restrict", "return", "short", "signed", "sizeof", "static", "static_assert", "static_cast",
  "strictfp", "struct", "super", "switch", "synchronized", "template", "this", "thread_local", "throw", "throws", "transient", "try",
  "typedef", "typeid", "typename", "union", "unsigned", "using", "virtual", "void", "volatile", "wchar_t", "while", "xor", "xor_eq", 0};
static const char* const kPyLit[] = {"True", "False", "None", 0};
static const char* const kCjLit[] = {"true", "false", "null", "nullptr", 0};
static const char* const kCjPre[] = {"L", "u", "U", "u8", "R", "LR", "uR", "UR", "u8R", 0};

enum { FAM_NONE = 0, FAM_PY = 1, FAM_CJ = 2 };

static int is_w(int c) { return c == 0x20 || c == 0x09 || c == 0x0D || c == 0x0B || c == 0x0C; }
static int is_digit(int c) { return c >= '0' && c <= '9'; }
static int is_alnum_(int c) { return is_digit(c) || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_'; }
static int is_ident(int c) { return is_alnum_(c) || c == '$' || c >= 0x80; }

static int in_list(const char* const* list, const uint8_t* p, int64_t n) {
  for (; *list; ++list)
    if ((int64_t)strlen(*list) == n && memcmp(*list, p, (size_t)n) == 0) return 1;
  return 0;
}

/* Index behind the delimiter that closes state st (PY 1: three double quotes, 2: three single quotes; CJ 1: star slash),
 * searched from i; -1 when none. */
static int64_t close_at(const uint8_t* l, int64_t n, int64_t i, int fam, int st) {
  if (fam == FAM_CJ) {
    for (; i + 1 < n; ++i)
      if (l[i] == '*' && l[i + 1] == '/') return i + 2;
    return -1;
  }
  const uint8_t q = st == 1 ? '"' : '\'';
  while (i < n) {
    if (l[i] == '\\') i += 2;
    else if (i + 2 < n && l[i] == q && l[i + 1] == q && l[i + 2] == q) return i + 3;
    else ++i;
  }
  return -1;
}

/* The literal whose quote is at i: returns the index behind it, *st = the state after it. */
static int64_t string_end(const uint8_t* l, int64_t n, int64_t i, int fam, int* st) {
  const uint8_t q = l[i];
  *st = 0;
  if (fam == FAM_PY && i + 2 < n && l[i + 1] == q && l[i + 2] == q) {
    const int s = q == '"' ? 1 : 2;
    const int64_t j = close_at(l, n, i + 3, fam, s);
    if (j < 0) { *st = s; return n; }
    return j;
  }
  for (int64_t j = i + 1; j < n;) {
    if (l[j] == '\\') j += 2;
    else if (l[j] == q) return j + 1;
    else ++j;
  }
  return n;
}

static void put(uint8_t* out, int64_t* m, const uint8_t* tok, int64_t k) {
  if (*m) out[(*m)++] = ' ';
  memcpy(out + *m, tok, (size_t)k);
  *m += k;
}

/* The blind form of line l[0, n) of family fam that starts in state *st into out (at most 2n + 16 bytes); *st = the state after it. */
static int64_t lex_line(const uint8_t* l, int64_t n, int fam, int* st, uint8_t* out) {
  int64_t m = 0, i = 0;
  if (*st) {
    i = close_at(l, n, 0, fam, *st);
    if (i < 0) return 0;
    *st = 0;
  }
  const char* const* kw = fam == FAM_PY ? kPy : kCj;
  const char* const* lit = fam == FAM_PY ? kPyLit : kCjLit;
  while (i < n) {
    const int c = l[i], nx = i + 1 < n ? l[i + 1] : -1;
    if (is_w(c)) { ++i; continue; }
    if (fam == FAM_PY && c == '#') break;
    if (fam == FAM_CJ && c == '/' && nx == '/') break;
    if (fam == FAM_CJ && c == '/' && nx == '*') {
      i = close_at(l, n, i + 2, fam, 1);
      if (i < 0) { *st = 1; return m; }
      continue;
    }
    if (is_digit(c) || (c == '.' && nx >= 0 && is_digit(nx))) {
      int64_t j = i + 1;
      while (j < n) {
        const int d = l[j];
        if (is_alnum_(d) || d == '.' || ((d == '+' || d == '-') && (l[j - 1] == 'e' || l[j - 1] == 'E' || l[j - 1] == 'p' || l[j - 1] == 'P'))) ++j;
        else if (fam == FAM_CJ && d == '\'' && j + 1 < n && is_alnum_(l[j + 1])) ++j;
        else break;
      }
      put(out, &m, (const uint8_t*)"N", 1);
      i = j;
      continue;
    }
    if (is_ident(c)) {
      int64_t j = i;
      while (j < n && is_ident(l[j])) ++j;
      const int64_t k = j - i;
      int prefix = 0;
      if (j < n && (l[j] == '"' || l[j] == '\'')) {
        if (fam == FAM_PY) {
          prefix = k <= 2;
          for (int64_t x = i; x < j && prefix; ++x) prefix = strchr("rRbBuUfF", l[x]) != NULL;
        } else {
          prefix = in_list(kCjPre, l + i, k);
        }
      }
      if (prefix) {
        int s;
        i = string_end(l, n, j, fam, &s);
        put(out, &m, (const uint8_t*)"S", 1);
        if (s) { *st = s; return m; }
        continue;
      }
      if (in_list(kw, l + i, k)) put(out, &m, l + i, k);
      else put(out, &m, (const uint8_t*)(in_list(lit, l + i, k) ? "N" : "I"), 1);
      i = j;
      continue;
    }
    if (c == '"' || c == '\'') {
      int s;
      i = string_end(l, n, i, fam, &s);
      put(out, &m, (const uint8_t*)"S", 1);
      if (s) { *st = s; return m; }
      continue;
    }
    put(out, &m, l + i, 1);
    ++i;
  }
  return m;
}

/* Per line of the corpus (files in order, lines of section 2): kept[l] (its blind form is not empty), bhash[l] = bytes_hash of
 * the blind form (0 when not kept) and flag[l] (assertion line of section 4).  line_base[n_files + 1].  Returns 0 or -1. */
int orc_blind_lines(const uint8_t* arena, const int32_t* off, const int32_t* len, const uint8_t* ext, int32_t n_files,
                    int64_t* line_base, uint8_t* kept, uint64_t* bhash, uint8_t* flag) {
  int64_t maxlen = 0, l = 0;
  for (int32_t f = 0; f < n_files; ++f) if (len[f] > maxlen) maxlen = len[f];
  uint8_t* buf = (uint8_t*)malloc((size_t)(2 * maxlen + 16));
  if (!buf) return -1;
  line_base[0] = 0;
  for (int32_t f = 0; f < n_files; ++f) {
    const uint8_t* p = arena + off[f];
    const int fam = ext[f] == 1 ? FAM_PY : (ext[f] >= 2 && ext[f] <= 6) ? FAM_CJ : FAM_NONE;
    int st = 0;
    int64_t pos = 0;
    while (pos < len[f]) {
      const uint8_t* lf = (const uint8_t*)memchr(p + pos, 0x0A, (size_t)(len[f] - pos));
      const int64_t end = lf ? (int64_t)(lf - p) : len[f];
      int64_t m = 0;
      if (fam == FAM_NONE) {
        for (int64_t i = pos; i < end; ++i) if (!is_w(p[i])) buf[m++] = p[i];
      } else {
        m = lex_line(p + pos, end - pos, fam, &st, buf);
      }
      kept[l] = m > 0;
      bhash[l] = m > 0 ? orc_bytes_hash(buf, (uint64_t)m) : 0;
      flag[l] = ext[f] != 0 && orc_is_assert_line(p + pos, (uint32_t)(end - pos));
      ++l;
      pos = end + 1;
    }
    line_base[f + 1] = l;
  }
  free(buf);
  return 0;
}

typedef struct { uint64_t k; int64_t p; } KP;

static int cmp_kp(const void* x, const void* y) {
  const KP* a = (const KP*)x; const KP* b = (const KP*)y;
  if (a->k != b->k) return a->k < b->k ? -1 : 1;
  return a->p < b->p ? -1 : a->p > b->p;
}

/* Section 15 over the line sequence hash[T], flag[T] with T = base[n_files] (files [base[f], base[f+1])).  Returns 0, -1 (bad
 * argument / no memory) or -3 (class_cap < classes or member_cap < fragments; the counts are set). */
int orc_clone_walk(const uint64_t* hash, const uint8_t* flag, const int64_t* base, int32_t n_files, int32_t n, uint32_t* file_dup,
                   uint32_t* file_dup_assert, int64_t* class_base, uint32_t* class_len, int64_t class_cap, int64_t* n_classes,
                   int64_t* member, int64_t member_cap, int64_t* n_members) {
  if (n < 1 || n > 1024 || n_files < 0) return -1;
  const int64_t T = n_files ? base[n_files] : 0;
  const size_t m = (size_t)(T ? T : 1);
  uint64_t* key = (uint64_t*)malloc(8 * m);
  uint8_t* covered = (uint8_t*)calloc(m, 1);
  int32_t* file = (int32_t*)malloc(4 * m); int64_t* gid = (int64_t*)malloc(8 * m);
  KP* w = (KP*)malloc(sizeof(KP) * m);
  int64_t *gstart = (int64_t*)malloc(8 * m), *gcount = (int64_t*)malloc(8 * m);
  uint8_t* gext = (uint8_t*)malloc(m);
  int rc = (key && covered && file && gid && w && gstart && gcount && gext) ? 0 : -1;
  int64_t nw = 0, ng = 0, nc = 0, nm = 0;
  if (rc == 0) {
    for (int32_t f = 0; f < n_files; ++f)
      for (int64_t p = base[f]; p < base[f + 1]; ++p) file[p] = f;
    if (T) orc_ngram_hashes(hash, base, n_files, n, key);
    for (int64_t p = 0; p < T; ++p) {                     /* 1. windows: n lines of one file */
      gid[p] = -1;
      if (p + n > base[file[p] + 1]) continue;
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
        if (q == base[file[q]] || gid[q - 1] < 0) ok = 0;
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
      for (int64_t x = base[f]; x < base[f + 1]; ++x) { d += covered[x]; a += covered[x] && flag[x]; }
      if (file_dup) file_dup[f] = d;
      if (file_dup_assert) file_dup_assert[f] = a;
    }
    *n_classes = nc; *n_members = nm;
    if (nc > class_cap || nm > member_cap) rc = -3;
  }
  free(key); free(covered); free(file); free(gid); free(w); free(gstart); free(gcount); free(gext);
  return rc;
}
