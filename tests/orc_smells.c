/* orc_smells.c - serial CPU reference of the test smells of docs/SPEC.md section 18.  TEST INFRASTRUCTURE ONLY.
 *
 * Built on the oracle: every file is split at LF (section 2), header lines are those orc_header_kind reports (the rule behind
 * the scan's header events, section 5), assertion lines are orc_is_assert_line (section 4, Rev A) and the duplicate key is
 * orc_bytes_hash of the stripped line (section 3).  Everything else - kinds, test headers, bodies, line kinds and the nine
 * smells - is section 18 stated one file, one test and one line at a time. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "orc.h"

enum { S_EMPTY = 1, S_FREE = 2, S_DUP = 4, S_REDUNDANT = 8, S_COND = 16, S_EXC = 32, S_SLEEP = 64, S_PRINT = 128, S_IGNORED = 256 };

typedef struct { const uint8_t* p; uint32_t n; } Str;    /* a line without its LF */

static int is_w(uint8_t c) { return c == 0x20 || c == 0x09 || c == 0x0D || c == 0x0B || c == 0x0C; }
static int is_id(uint8_t c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_'; }

static Str strip(Str s) {
  while (s.n && is_w(s.p[0])) { ++s.p; --s.n; }
  while (s.n && is_w(s.p[s.n - 1])) --s.n;
  return s;
}
static int starts(Str s, const char* lit) { size_t k = strlen(lit); return s.n >= k && memcmp(s.p, lit, k) == 0; }
static int equals(Str s, const char* lit) { return s.n == strlen(lit) && memcmp(s.p, lit, s.n) == 0; }
static int find_from(Str s, uint32_t from, const char* lit) {   /* first occurrence at or after `from`, or -1 */
  const uint32_t k = (uint32_t)strlen(lit);
  for (uint32_t i = from; i + k <= s.n; ++i)
    if (memcmp(s.p + i, lit, k) == 0) return (int)i;
  return -1;
}
static int has(Str s, const char* lit) { return find_from(s, 0, lit) >= 0; }
static uint32_t count_byte(Str s, uint8_t c) { uint32_t n = 0; for (uint32_t i = 0; i < s.n; ++i) n += s.p[i] == c; return n; }
static uint32_t count_tq(Str s, const char* q) {          /* non-overlapping occurrences, left to right */
  uint32_t n = 0;
  for (int i = find_from(s, 0, q); i >= 0; i = find_from(s, (uint32_t)i + 3, q)) ++n;
  return n;
}

static int family(int ext) { return ext == 1 ? 1 : ext == 4 ? 3 : (ext == 2 || ext == 3 || ext == 5 || ext == 6) ? 2 : 0; }

static int test_header(Str line, int fam) {
  Str s = strip(line);
  if (fam == 1) {
    uint32_t i = 0;
    if (starts(s, "async")) {
      i = 5;
      while (i < s.n && is_w(s.p[i])) ++i;
      if (i == 5) return 0;
    }
    Str t = {s.p + i, s.n - i};
    if (!starts(t, "def")) return 0;
    uint32_t j = 3;
    while (j < t.n && is_w(t.p[j])) ++j;
    return j > 3 && t.n - j >= 4 && memcmp(t.p + j, "test", 4) == 0;
  }
  if (fam == 2) {
    static const char* const pre[] = {"TEST(", "TEST_F(", "TEST_P(", "TYPED_TEST(", "TYPED_TEST_P(", "BOOST_AUTO_TEST_CASE(",
                                      "BOOST_FIXTURE_TEST_CASE(", "BOOST_DATA_TEST_CASE("};
    for (int k = 0; k < 8; ++k) if (starts(s, pre[k])) return 1;
    return 0;
  }
  return fam == 3 && has(line, "void") && has(line, "(");
}

static uint32_t indent_of(Str l) { uint32_t n = 0; while (n < l.n && (l.p[n] == 0x20 || l.p[n] == 0x09)) ++n; return n; }
static int comment(Str s, int fam) { return fam == 1 ? starts(s, "#") : (starts(s, "//") || starts(s, "/*") || starts(s, "*")); }

static int constant(Str x) {
  static const char* const k[] = {"True", "False", "true", "false", "None", "nullptr", "NULL", "0", "1"};
  for (int i = 0; i < 9; ++i) if (equals(x, k[i])) return 1;
  return 0;
}

static int redundant(Str s) {                             /* s: the stripped assertion line */
  if (s.n > 6 && starts(s, "assert") && is_w(s.p[6])) {
    Str x = strip((Str){s.p + 6, s.n - 6});
    if (constant(x)) return 1;
  }
  int a = -1, b = -1;
  for (uint32_t i = 0; i < s.n; ++i) { if (s.p[i] == '(' && a < 0) a = (int)i; if (s.p[i] == ')') b = (int)i; }
  if (a < 0 || b <= a) return 0;
  Str x = strip((Str){s.p + a + 1, (uint32_t)(b - a - 1)});
  if (constant(x)) return 1;
  int depth = 0, commas = 0;
  uint32_t at = 0;
  for (uint32_t i = 0; i < x.n; ++i) {
    const uint8_t c = x.p[i];
    if (c == '(' || c == '[' || c == '{') ++depth;
    else if (c == ')' || c == ']' || c == '}') --depth;
    else if (c == ',' && depth == 0) { ++commas; at = i; }
  }
  if (commas != 1) return 0;
  Str l = strip((Str){x.p, at}), r = strip((Str){x.p + at + 1, x.n - at - 1});
  return l.n > 0 && l.n == r.n && memcmp(l.p, r.p, l.n) == 0;
}

static int first_token_in(Str s, const char* const* words, int n) {
  uint32_t i = 0;
  while (i < s.n && (is_w(s.p[i]) || s.p[i] == '}')) ++i;
  uint32_t j = i;
  while (j < s.n && is_id(s.p[j])) ++j;
  Str t = {s.p + i, j - i};
  for (int k = 0; k < n; ++k) if (equals(t, words[k])) return 1;
  return 0;
}

static int prints(Str s) {
  if (has(s, "System.out.print") || has(s, "System.err.print")) return 1;
  static const char* const pats[] = {"print(", "pprint(", "printf(", "puts(", "cout", "cerr"};
  for (int k = 0; k < 6; ++k)
    for (int i = find_from(s, 0, pats[k]); i >= 0; i = find_from(s, (uint32_t)i + 1, pats[k]))
      if (i == 0 || !is_id(s.p[i - 1])) return 1;
  return 0;
}

static int empty_ok(Str l) {
  if (equals(strip(l), "pass")) return 1;
  for (uint32_t i = 0; i < l.n; ++i) {
    const uint8_t c = l.p[i];
    if (!is_w(c) && c != '{' && c != '}' && c != '(' && c != ')' && c != ';' && c != ':') return 0;
  }
  return 1;
}

/* One file: appends its tests to tests[*nt ...] (while *nt < test_cap; *nt counts all) and sets smell[0 .. n_lines). */
static void file_smells(const Str* L, int64_t n, int ext, int32_t f, uint16_t* smell, int32_t* tests, int64_t test_cap, int64_t* nt,
                        uint8_t* kind, uint8_t* head, uint8_t* code, uint64_t* hash) {
  const int fam = family(ext);
  if (!fam) return;
  int64_t d = 0;                                          /* section 10 kinds */
  for (int64_t i = 0; i < n; ++i) {
    if (strip(L[i]).n == 0) { kind[i] = 0; continue; }
    kind[i] = d == 0 ? 1 : 2;
    d += (int64_t)count_byte(L[i], '(') - (int64_t)count_byte(L[i], ')');
    if (d < 0) d = 0;
  }
  for (int64_t i = 0; i < n; ++i) head[i] = orc_header_kind(ext, L[i].p, L[i].n) != 0;
  for (int64_t b = 0; b < n; ++b) {
    if (!head[b] || !test_header(L[b], fam)) continue;
    int64_t e = b + 1;
    while (e < n && !head[e]) ++e;
    int64_t hs = b + 1;
    while (hs < e && kind[hs] == 2) ++hs;
    int64_t bend = e;
    if (fam == 1) {
      const uint32_t ind = indent_of(L[b]);
      for (int64_t l = hs; l < e; ++l)
        if (kind[l] == 1 && !comment(strip(L[l]), fam) && indent_of(L[l]) <= ind) { bend = l; break; }
    } else {
      int64_t run = 0; int opened = 0;
      for (int64_t l = b; l < e; ++l) {
        run += (int64_t)count_byte(L[l], '{') - (int64_t)count_byte(L[l], '}');
        opened |= count_byte(L[l], '{') > 0;
        if (opened && run <= 0) { bend = l + 1; break; }
      }
    }
    const int64_t hend = hs < bend ? hs : bend;
    uint32_t dq = 0, sq = 0;
    int all_empty_ok = 1;
    for (int64_t l = hend; l < bend; ++l) {
      const Str s = strip(L[l]);
      int doc = 0;
      if (fam == 1) {
        doc = (dq & 1) || (sq & 1) || starts(s, "\"\"\"") || starts(s, "'''");
        dq += count_tq(L[l], "\"\"\"");
        sq += count_tq(L[l], "'''");
      }
      code[l] = s.n > 0 && !comment(s, fam) && !doc;
      if (code[l] && !empty_ok(L[l])) all_empty_ok = 0;
    }
    uint32_t na = 0, bits = 0, inst = 0;
    for (int64_t l = b; l < bend; ++l) {
      const int in_code = l >= hend && code[l];
      const Str s = strip(L[l]);
      uint16_t m = 0;
      if ((l < hend || in_code) && orc_is_assert_line(L[l].p, L[l].n)) {
        hash[na] = orc_bytes_hash(s.p, s.n);
        for (uint32_t k = 0; k < na; ++k) if (hash[k] == hash[na]) { m |= S_DUP; break; }
        ++na;
        if (redundant(s)) m |= S_REDUNDANT;
      }
      if (in_code) {
        static const char* const cond[] = {"if", "elif", "for", "while", "switch"};
        static const char* const exc[] = {"try", "except", "catch", "raise", "throw"};
        if (first_token_in(s, cond, 5)) m |= S_COND;
        if (first_token_in(s, exc, 5)) m |= S_EXC;
        if (has(s, "sleep(") || has(s, "sleep_for(") || has(s, "sleep_until(")) m |= S_SLEEP;
        if (prints(s)) m |= S_PRINT;
        if (fam == 1 && (starts(s, "self.skipTest(") || starts(s, "pytest.skip("))) m |= S_IGNORED;
      }
      smell[l] = m;
    }
    int ign = 0;
    for (int64_t a = b - 1; a >= 0 && !head[a] && starts(strip(L[a]), "@"); --a) {
      if (fam == 1 && has(L[a], "skip")) ign = 1;
      if (fam == 3 && (has(L[a], "@Ignore") || has(L[a], "@Disabled"))) ign = 1;
    }
    if (fam == 3 && (has(L[b], "@Ignore") || has(L[b], "@Disabled"))) ign = 1;
    if (fam == 2 && has(L[b], "DISABLED_")) ign = 1;
    uint16_t hb = ign ? S_IGNORED : 0;
    if (na == 0) hb |= S_FREE | (all_empty_ok ? S_EMPTY : 0);
    smell[b] |= hb;
    for (int64_t l = b; l < bend; ++l) {
      bits |= smell[l];
      for (uint16_t m = smell[l]; m; m &= (uint16_t)(m - 1)) ++inst;
    }
    if (*nt < test_cap) {
      int32_t* t = tests + 6 * *nt;
      t[0] = f; t[1] = (int32_t)b; t[2] = (int32_t)(bend - b); t[3] = (int32_t)na; t[4] = (int32_t)bits; t[5] = (int32_t)inst;
    }
    ++*nt;
  }
}

/* tests: 6 int32 per test (tsm_smell_test).  Returns 0, -1 (bad argument / no memory) or -3 (line_cap < lines or test_cap < tests;
 * both counts are set). */
int orc_smells(const uint8_t* arena, const int32_t* off, const int32_t* len, const uint8_t* ext, int32_t n_files, int64_t* line_base,
               uint16_t* line_smell, int64_t line_cap, int64_t* n_lines, int32_t* tests, int64_t test_cap, int64_t* n_tests) {
  if (n_files < 0) return -1;
  int64_t T = 0, maxl = 1;
  line_base[0] = 0;
  for (int32_t f = 0; f < n_files; ++f) {
    const uint8_t* p = arena + off[f];
    int64_t lines = 0;
    for (int32_t i = 0; i < len[f]; ++i) lines += p[i] == 0x0A;
    lines += len[f] > 0 && p[len[f] - 1] != 0x0A;
    T += lines;
    line_base[f + 1] = T;
    if (lines > maxl) maxl = lines;
  }
  *n_lines = T;
  *n_tests = 0;
  const size_t m = (size_t)maxl;
  Str* L = (Str*)malloc(sizeof(Str) * m);
  uint8_t *kind = (uint8_t*)malloc(m), *head = (uint8_t*)malloc(m), *code = (uint8_t*)calloc(m, 1);
  uint64_t* hash = (uint64_t*)malloc(8 * m);
  uint16_t* smell = (uint16_t*)malloc(2 * m);
  if (!L || !kind || !head || !code || !hash || !smell) { free(L); free(kind); free(head); free(code); free(hash); free(smell); return -1; }
  const int fits = line_cap >= T;
  for (int32_t f = 0; f < n_files; ++f) {
    const uint8_t* p = arena + off[f];
    int64_t n = 0;
    uint32_t s = 0;
    for (int32_t i = 0; i <= len[f]; ++i)
      if (i == len[f] ? (uint32_t)i > s : p[i] == 0x0A) { L[n].p = p + s; L[n].n = (uint32_t)i - s; ++n; s = (uint32_t)i + 1; }
    memset(smell, 0, 2 * (size_t)(n ? n : 1));
    file_smells(L, n, ext[f], f, smell, tests, test_cap, n_tests, kind, head, code, hash);
    if (fits && line_smell) memcpy(line_smell + line_base[f], smell, 2 * (size_t)n);
  }
  free(L); free(kind); free(head); free(code); free(hash); free(smell);
  return (!fits && line_smell) || *n_tests > test_cap ? -3 : 0;
}
