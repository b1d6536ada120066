/* orc_lexsmells.c - serial CPU reference of the lexical test smells of docs/SPEC.md section 25.  TEST INFRASTRUCTURE ONLY.
 *
 * It reuses the section-21 lexer helpers of orc_blind.c (literal and comment ends, keyword lists) and the section-18 helpers of
 * orc_smells.c (stripping, test headers, comment lines, triple quotes), both compiled into this unit, and the oracle's header rule,
 * assertion rule and bytes_hash (orc.h).  One file at a time: every line is lexed into seen tokens (kind and bytes) stored
 * contiguously, so that an argument list over several lines is one slice of the file's tokens; each statement is then parsed
 * from that slice as a whole - the matching bracket, the arguments, the operands - rather than token by token as the kernels do. */
#define is_w blind_is_w
#define is_digit blind_is_digit
#include "orc_blind.c"
#undef is_w
#undef is_digit
#include "orc_smells.c"

enum { T_I = 'I', T_K = 'K', T_L = 'L', T_N = 'N', T_S = 'S', T_P = 'P' };
typedef struct { int kind; const uint8_t* p; uint32_t n; } Tok;

#define LEX_STMT_LINES 64
#define OBSCURE_LOCALS 10

static int tok_is(const Tok* t, int kind, const char* s) {
  return t->kind == kind && t->n == strlen(s) && memcmp(t->p, s, t->n) == 0;
}
static int punct(const Tok* t, char c) { return t->kind == T_P && t->p[0] == (uint8_t)c; }
static int tok_pre(const Tok* t, const char* s) { size_t k = strlen(s); return t->n >= k && memcmp(t->p, s, k) == 0; }
static int in_names(const Tok* t, const char* const* list) {
  for (; *list; ++list) if (tok_is(t, T_I, *list)) return 1;
  return 0;
}

/* The seen tokens of line l[0, n) of family fam from state *st, appended at out[*m]; *st = the state after it. */
static void lex_tokens(const uint8_t* l, int64_t n, int fam, int* st, Tok* out, int64_t* m) {
  int64_t i = 0;
  if (*st) {
    i = close_at(l, n, 0, fam, *st);
    if (i < 0) return;
    *st = 0;
  }
  const char* const* kw = fam == FAM_PY ? kPy : kCj;
  const char* const* lit = fam == FAM_PY ? kPyLit : kCjLit;
  while (i < n) {
    const int c = l[i], nx = i + 1 < n ? l[i + 1] : -1;
    if (blind_is_w(c)) { ++i; continue; }
    if (fam == FAM_PY && c == '#') break;
    if (fam == FAM_CJ && c == '/' && nx == '/') break;
    if (fam == FAM_CJ && c == '/' && nx == '*') {
      i = close_at(l, n, i + 2, fam, 1);
      if (i < 0) { *st = 1; return; }
      continue;
    }
    Tok t = {T_P, l + i, 1};
    if (blind_is_digit(c) || (c == '.' && nx >= 0 && blind_is_digit(nx))) {
      int64_t j = i + 1;
      while (j < n) {
        const int d = l[j];
        if (is_alnum_(d) || d == '.' || ((d == '+' || d == '-') && strchr("eEpP", l[j - 1]) && l[j - 1])) ++j;
        else if (fam == FAM_CJ && d == '\'' && j + 1 < n && is_alnum_(l[j + 1])) ++j;
        else break;
      }
      t.kind = T_N; t.n = (uint32_t)(j - i);
      out[(*m)++] = t;
      i = j;
      continue;
    }
    if (c == '"' || c == '\'' || is_ident(c)) {
      int64_t j = i;
      while (j < n && is_ident(l[j])) ++j;
      const int64_t k = j - i;
      int prefix = k == 0;                                 /* a bare quote opens a literal */
      if (k && j < n && (l[j] == '"' || l[j] == '\'')) {
        if (fam == FAM_PY) {
          prefix = k <= 2;
          for (int64_t x = i; x < j && prefix; ++x) prefix = strchr("rRbBuUfF", l[x]) != NULL;
        } else {
          prefix = in_list(kCjPre, l + i, k);
        }
      }
      if (prefix) {
        int s;
        const int64_t e = string_end(l, n, j, fam, &s);
        t.kind = T_S; t.n = (uint32_t)(e - i);
        out[(*m)++] = t;
        if (s) { *st = s; return; }
        i = e;
        continue;
      }
      t.kind = in_list(kw, l + i, k) ? T_K : in_list(lit, l + i, k) ? T_L : T_I;
      t.n = (uint32_t)k;
      out[(*m)++] = t;
      i = j;
      continue;
    }
    out[(*m)++] = t;
    ++i;
  }
}

static int depth_step(const Tok* t, int d) {
  if (t->kind != T_P) return d;
  const uint8_t c = t->p[0];
  return c == '(' || c == '[' || c == '{' ? d + 1 : c == ')' || c == ']' || c == '}' ? d - 1 : d;
}
/* index of the token that closes the bracket opened at t[i] (i < n), or -1 */
static int64_t close_of(const Tok* t, int64_t i, int64_t n) {
  int d = 0;
  for (int64_t k = i; k < n; ++k) { d = depth_step(t + k, d); if (d == 0) return k; }
  return -1;
}

/* the operand separators of section 25 at t[i] inside [a, b) */
static int cmp_sep(const Tok* t, int64_t i, int64_t a, int64_t b, int py) {
  if (punct(t + i, '<') || punct(t + i, '>') || punct(t + i, '=')) return 1;
  if (punct(t + i, '!') && i + 1 < b && punct(t + i + 1, '=')) return 1;
  if (py && (tok_is(t + i, T_K, "is") || tok_is(t + i, T_K, "in"))) return 1;
  if (py && tok_is(t + i, T_K, "not") && ((i > a && tok_is(t + i - 1, T_K, "is")) || (i + 1 < b && tok_is(t + i + 1, T_K, "in")))) return 1;
  return 0;
}
static int magic_operand(const Tok* t, int64_t a, int64_t b) {
  if (b - a == 1) return t[a].kind == T_N;
  return b - a == 2 && (punct(t + a, '-') || punct(t + a, '+')) && t[a + 1].kind == T_N;
}
static int has_magic(const Tok* t, int64_t a, int64_t b, int py) {
  int d = 0;
  int64_t s = a;
  for (int64_t i = a; i < b; ++i) {
    if (d == 0 && cmp_sep(t, i, a, b, py)) {
      if (magic_operand(t, s, i)) return 1;
      s = i + 1;
    }
    d = depth_step(t + i, d);
  }
  return magic_operand(t, s, b);
}
static int is_kwarg(const Tok* t, int64_t a, int64_t b) {
  return b - a >= 2 && t[a].kind == T_I && punct(t + a + 1, '=') && (b - a < 3 || !punct(t + a + 2, '='));
}
static int bool_suboptimal(const Tok* t, int64_t a, int64_t b, int ext) {
  const int py = ext == 1;
  int d = 0;
  for (int64_t i = a; i < b; ++i) {
    if (d == 0) {
      if (punct(t + i, '=') && i > a && (punct(t + i - 1, '=') || punct(t + i - 1, '!') || punct(t + i - 1, '<') || punct(t + i - 1, '>')))
        return 1;
      if (py && (punct(t + i, '<') || punct(t + i, '>') || tok_is(t + i, T_K, "is") || tok_is(t + i, T_K, "in"))) return 1;
    }
    d = depth_step(t + i, d);
  }
  if (py && b - a >= 3 && tok_is(t + a, T_I, "isinstance") && punct(t + a + 1, '(') && close_of(t, a + 1, b) == b - 1) return 1;
  if (ext == 4 && b > a && punct(t + b - 1, ')'))
    for (int64_t o = a; o < b - 1; ++o)
      if (punct(t + o, '(') && close_of(t, o, b) == b - 1)
        return o - a >= 2 && tok_is(t + o - 1, T_I, "equals") && punct(t + o - 2, '.');
  return 0;
}

enum { K_NONE, K_UNITTEST, K_NUMPY, K_GTEST, K_CASSERT, K_STATIC, K_JCALL };
static const char* const kArity1[] = {"assertTrue", "assertFalse", "assertIsNone", "assertIsNotNone", "assert_", 0};
static const char* const kArity3[] = {"assertAlmostEqual", "assertNotAlmostEqual", "assertAlmostEquals", "assertNotAlmostEquals", 0};
static const char* const kJArity1[] = {"assertTrue", "assertFalse", "assertNull", "assertNotNull", 0};
static const char* const kSubBool[] = {"assertTrue", "assertFalse", "assert_", "EXPECT_TRUE", "EXPECT_FALSE", "ASSERT_TRUE", "ASSERT_FALSE", 0};
static const char* const kSubEq[] = {"assertEqual", "assertEquals", "assertNotEqual", "assertNotEquals", "assertIs", "assertIsNot",
                                     "EXPECT_EQ", "EXPECT_NE", "ASSERT_EQ", "ASSERT_NE", 0};
static const char* const kPyGuest[] = {"open", "urlopen", "connect", "read_csv", "read_excel", "read_json", "read_parquet", "loadtxt",
                                       "genfromtxt", "imread", "listdir", 0};
static const char* const kCjGuestCall[] = {"fopen", "freopen", "open", "getConnection", 0};
static const char* const kCjGuestName[] = {"ifstream", "ofstream", "fstream", "File", "FileReader", "FileWriter", "FileInputStream",
                                           "FileOutputStream", "RandomAccessFile", "Files", 0};

static int has_assert(const Tok* t, int cj) {
  for (uint32_t q = 0; q + 6 <= t->n; ++q) {
    int a = 1;
    for (uint32_t j = 0; j < 6 && a; ++j) a = (t->p[q + j] | 0x20) == (uint8_t)"assert"[j];
    if (a) return 1;
    if (cj && q + 7 <= t->n && memcmp(t->p + q, "EXPECT_", 7) == 0) return 1;
  }
  return 0;
}

/* The LX_* facts (1 statement, 2 counted and unexplained, 4 magic, 8 suboptimal) of the statement of the line whose tokens are
 * t[lb, le); the walk may use the tokens up to t[wend) and the line ends ends[0 .. nends) (token index behind each line). */
static int statement(const Tok* t, int64_t lb, int64_t le, int64_t wend, const int64_t* ends, int64_t nends, int ext, int64_t* piece) {
  const int py = ext == 1;
  int64_t j = -1;
  int form = 0;                                            /* 1 PY assert, 2 Java assert, 3 call */
  for (int64_t i = lb; i < le && j < 0; ++i) {
    const int paren = i + 1 < le && punct(t + i + 1, '(');
    if (tok_is(t + i, T_K, "assert")) {
      if (py) { j = i; form = 1; }
      else if (ext == 4) { j = i; form = 2; }
      else if (paren) { j = i; form = 3; }
    } else if (!py && tok_is(t + i, T_K, "static_assert") && paren) { j = i; form = 3; }
    else if (t[i].kind == T_I && paren && has_assert(t + i, !py)) { j = i; form = 3; }
  }
  if (j < 0) return 0;
  const int64_t s = j + 1;
  if (form != 3) {
    int64_t cut = wend;
    int d = 0;
    if (form == 1) {
      int64_t pos = s;
      for (int64_t m = 0; m < nends; ++m) {
        for (; pos < ends[m]; ++pos) d = depth_step(t + pos, d);
        const int64_t first = m == 0 ? lb : ends[m - 1];
        if (d == 0 && !(ends[m] > first && punct(t + ends[m] - 1, '\\'))) { cut = ends[m]; break; }
      }
    } else {
      for (int64_t i = s; i < wend; ++i) {
        if (d == 0 && punct(t + i, ';')) { cut = i; break; }
        d = depth_step(t + i, d);
      }
    }
    int64_t msg = -1;
    d = 0;
    for (int64_t i = s; i < cut && msg < 0; ++i) {
      if (d == 0 && punct(t + i, form == 1 ? ',' : ':')) msg = i;
      d = depth_step(t + i, d);
    }
    return 1 | (msg < 0 ? 2 : 0) | (has_magic(t, s, msg < 0 ? cut : msg, py) ? 4 : 0);
  }
  /* the kind of the call */
  const Tok* name = t + j;
  int kind = K_NONE, arity = 0;
  if (name->kind == T_K) kind = tok_is(name, T_K, "static_assert") ? K_STATIC : K_CASSERT;
  else if (py) {
    if (tok_pre(name, "assert_") && name->n > 7) {
      kind = tok_pre(name, "assert_called") || tok_pre(name, "assert_awaited") || tok_is(name, T_I, "assert_any_call") ||
             tok_is(name, T_I, "assert_has_calls") || tok_is(name, T_I, "assert_not_called") ? K_NONE : K_NUMPY;
    } else if (j > lb && punct(t + j - 1, '.') && tok_pre(name, "assert")) {
      if (!(tok_pre(name, "assertRaises") || tok_pre(name, "assertWarns") || tok_is(name, T_I, "assertLogs") ||
            tok_is(name, T_I, "assertNoLogs"))) {
        kind = K_UNITTEST;
        arity = in_names(name, kArity1) ? 1 : in_names(name, kArity3) ? 3 : 2;
      }
    }
  } else if (tok_pre(name, "EXPECT_") || tok_pre(name, "ASSERT_")) kind = K_GTEST;
  else if (ext == 4 && tok_pre(name, "assert")) { kind = K_JCALL; arity = in_names(name, kJArity1) ? 1 : 2; }
  /* the list and its arguments: piece[2k], piece[2k + 1] */
  const int64_t close = close_of(t, s, wend);
  const int64_t la = s + 1, lz = close >= 0 ? close : wend;
  int64_t np = 0, a = la;
  int d = 0;
  for (int64_t i = la; i <= lz; ++i) {
    if (i == lz || (d == 0 && punct(t + i, ','))) {
      if (i > a) { piece[2 * np] = a; piece[2 * np + 1] = i; ++np; }
      a = i + 1;
    }
    if (i < lz) d = depth_step(t + i, d);
  }
  int magic = 0, sub = 0, any_lit = 0, kw_msg = 0, kw_err = 0;
  int64_t npos = 0;
  for (int64_t k = 0; k < np; ++k) {
    const int64_t pa = piece[2 * k], pz = piece[2 * k + 1];
    if (py && is_kwarg(t, pa, pz)) {
      kw_msg |= tok_is(t + pa, T_I, "msg");
      kw_err |= tok_is(t + pa, T_I, "err_msg");
      continue;
    }
    ++npos;
    magic |= has_magic(t, pa, pz, py);
    any_lit |= pz - pa == 1 && t[pa].kind == T_L;
  }
  if (in_names(name, kSubBool) && np) sub = bool_suboptimal(t, piece[0], piece[1], ext);
  if (in_names(name, kSubEq)) sub |= any_lit;
  const int flags = 1 | (magic ? 4 : 0) | (sub ? 8 : 0);
  int expl = 0;
  switch (kind) {
    case K_NONE: return flags;
    case K_UNITTEST: expl = npos > arity || kw_msg; break;
    case K_NUMPY: expl = kw_msg || kw_err; break;
    case K_GTEST: expl = close >= 0 && close + 2 < wend && punct(t + close + 1, '<') && punct(t + close + 2, '<'); break;
    case K_CASSERT: expl = 0; break;
    case K_STATIC: expl = np >= 2; break;
    default: {
      const int first = np && piece[1] - piece[0] == 1 && t[piece[0]].kind == T_S;
      const int last = np && piece[2 * np - 1] - piece[2 * np - 2] == 1 && t[piece[2 * np - 2]].kind == T_S;
      expl = np > arity && (first || last);
    }
  }
  return flags | (expl ? 0 : 2);
}

/* Mystery Guest of a code line's tokens t[a, b) */
static int mystery(const Tok* t, int64_t a, int64_t b, int ext) {
  for (int64_t i = a; i < b; ++i) {
    if (t[i].kind != T_I) continue;
    const int paren = i + 1 < b && punct(t + i + 1, '(');
    if (ext == 1 ? paren && in_names(t + i, kPyGuest) : ((paren && in_names(t + i, kCjGuestCall)) || in_names(t + i, kCjGuestName))) return 1;
  }
  return 0;
}

/* the local names of a code line's tokens t[a, b): their hashes appended at out[*m] */
static void local_names(const Tok* t, int64_t a, int64_t b, int ext, uint64_t* out, int64_t* m) {
  if (ext == 1) {
    int64_t i = a, k = 0;
    while (i < b && t[i].kind == T_I) {
      ++k;
      if (i + 1 < b && punct(t + i + 1, ',')) { i += 2; continue; }
      if (i + 1 < b && punct(t + i + 1, '=') && !(i + 2 < b && punct(t + i + 2, '='))) {
        for (int64_t x = 0; x < k; ++x) out[(*m)++] = orc_bytes_hash(t[a + 2 * x].p, t[a + 2 * x].n);
      }
      return;
    }
    return;
  }
  int d = 0;
  for (int64_t i = a; i < b; ++i) {
    if (d == 0 && punct(t + i, '=') && !(i > a && t[i - 1].kind == T_P && strchr("=!<>+-*/%&|^", t[i - 1].p[0])) &&
        !(i + 1 < b && punct(t + i + 1, '='))) {
      if (i - a >= 2 && t[i - 1].kind == T_I) {
        for (int64_t x = a; x < i; ++x)
          if (punct(t + x, '(') || punct(t + x, '.') || punct(t + x, '[')) return;
        out[(*m)++] = orc_bytes_hash(t[i - 1].p, t[i - 1].n);
      }
      return;
    }
    d = depth_step(t + i, d);
  }
}

static int cmp_u64(const void* x, const void* y) {
  const uint64_t a = *(const uint64_t*)x, b = *(const uint64_t*)y;
  return a < b ? -1 : a > b;
}

/* lex: 6 int32 per test (tsm_lex_test), in the order of orc_smells' tests.  Returns 0, -1 (bad argument / no memory) or -3
 * (line_cap < lines or test_cap < tests; both counts are set). */
int orc_lexsmells(const uint8_t* arena, const int32_t* off, const int32_t* len, const uint8_t* ext, int32_t n_files, int64_t* line_base,
                  uint8_t* line_lsmell, int64_t line_cap, int64_t* n_lines, int32_t* lex, int64_t test_cap, int64_t* n_tests) {
  if (n_files < 0) return -1;
  int64_t T = 0, maxl = 1, maxb = 1;
  line_base[0] = 0;
  for (int32_t f = 0; f < n_files; ++f) {
    const uint8_t* p = arena + off[f];
    int64_t lines = 0;
    for (int32_t i = 0; i < len[f]; ++i) lines += p[i] == 0x0A;
    lines += len[f] > 0 && p[len[f] - 1] != 0x0A;
    T += lines;
    line_base[f + 1] = T;
    if (lines > maxl) maxl = lines;
    if (len[f] > maxb) maxb = len[f];
  }
  *n_lines = T;
  *n_tests = 0;
  const size_t m = (size_t)maxl;
  Str* L = (Str*)malloc(sizeof(Str) * m);
  uint8_t *kind = (uint8_t*)malloc(m), *head = (uint8_t*)malloc(m), *cnt = (uint8_t*)malloc(m), *lsm = (uint8_t*)malloc(m);
  int64_t* tb = (int64_t*)malloc(8 * (m + 1));
  Tok* toks = (Tok*)malloc(sizeof(Tok) * (size_t)(maxb + 1));
  int64_t* piece = (int64_t*)malloc(16 * (size_t)(maxb + 1));
  uint64_t* names = (uint64_t*)malloc(8 * (size_t)(maxb + 1));
  if (!L || !kind || !head || !cnt || !lsm || !tb || !toks || !piece || !names) {
    free(L); free(kind); free(head); free(cnt); free(lsm); free(tb); free(toks); free(piece); free(names);
    return -1;
  }
  const int fits = line_cap >= T;
  for (int32_t f = 0; f < n_files; ++f) {
    const uint8_t* p = arena + off[f];
    int64_t n = 0;
    uint32_t s0 = 0;
    for (int32_t i = 0; i <= len[f]; ++i)
      if (i == len[f] ? (uint32_t)i > s0 : p[i] == 0x0A) { L[n].p = p + s0; L[n].n = (uint32_t)i - s0; ++n; s0 = (uint32_t)i + 1; }
    memset(lsm, 0, (size_t)(n ? n : 1));
    const int fam = family(ext[f]), lfam = ext[f] == 1 ? FAM_PY : FAM_CJ;
    if (fam) {
      int64_t nt = 0;
      int st = 0;
      for (int64_t l = 0; l < n; ++l) { tb[l] = nt; lex_tokens(L[l].p, L[l].n, lfam, &st, toks, &nt); }
      tb[n] = nt;
      int64_t d = 0;                                       /* section 10 kinds, section 5 headers */
      for (int64_t i = 0; i < n; ++i) {
        if (strip(L[i]).n == 0) { kind[i] = 0; continue; }
        kind[i] = d == 0 ? 1 : 2;
        d += (int64_t)count_byte(L[i], '(') - (int64_t)count_byte(L[i], ')');
        if (d < 0) d = 0;
      }
      for (int64_t i = 0; i < n; ++i) head[i] = orc_header_kind(ext[f], L[i].p, L[i].n) != 0;
      for (int64_t b = 0; b < n; ++b) {
        if (!head[b] || !test_header(L[b], fam)) continue;
        int64_t e = b + 1;                                 /* section 18 body, header statement and counted lines */
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
        for (int64_t l = b; l < bend; ++l) {
          const Str s = strip(L[l]);
          int doc = 0;
          if (l >= hend && fam == 1) {
            doc = (dq & 1) || (sq & 1) || starts(s, "\"\"\"") || starts(s, "'''");
            dq += count_tq(L[l], "\"\"\"");
            sq += count_tq(L[l], "'''");
          }
          cnt[l] = l < hend ? 1 : (s.n > 0 && !comment(s, fam) && !doc) ? 3 : 0;   /* 1 counted, 2 code */
        }
        int32_t n_st = 0, n_un = 0, n_mg = 0;
        int64_t nn = 0;
        for (int64_t l = b; l < bend; ++l) {
          if ((cnt[l] & 1) && orc_is_assert_line(L[l].p, L[l].n)) {
            const int64_t lim = l + LEX_STMT_LINES < bend ? l + LEX_STMT_LINES : bend;
            const int x = statement(toks, tb[l], tb[l + 1], tb[lim], tb + l + 1, lim - l, ext[f], piece);
            if (x) {
              ++n_st;
              if (x & 2) { ++n_un; lsm[l] |= 1; }
              if (x & 4) { ++n_mg; lsm[l] |= 2; }
              if (x & 8) lsm[l] |= 4;
            }
          }
          if (cnt[l] & 2) {
            if (mystery(toks, tb[l], tb[l + 1], ext[f])) lsm[l] |= 8;
            local_names(toks, tb[l], tb[l + 1], ext[f], names, &nn);
          }
        }
        qsort(names, (size_t)nn, 8, cmp_u64);
        int32_t nloc = 0;
        for (int64_t k = 0; k < nn; ++k) nloc += k == 0 || names[k] != names[k - 1];
        uint32_t bits = 0;
        int32_t inst = 0;
        for (int64_t l = b; l < bend; ++l) {
          if (n_un < 2) lsm[l] &= (uint8_t)~1u;            /* the roulette bit marks unexplained lines until it is decided */
          if (l == b && nloc > OBSCURE_LOCALS) lsm[l] |= 16;
          bits |= lsm[l];
          for (uint8_t q = lsm[l]; q; q &= (uint8_t)(q - 1)) ++inst;
        }
        if (*n_tests < test_cap) {
          int32_t* r = lex + 6 * *n_tests;
          r[0] = n_st; r[1] = n_un; r[2] = n_mg; r[3] = nloc; r[4] = (int32_t)bits; r[5] = inst;
        }
        ++*n_tests;
      }
    }
    if (fits && line_lsmell) memcpy(line_lsmell + line_base[f], lsm, (size_t)n);
  }
  free(L); free(kind); free(head); free(cnt); free(lsm); free(tb); free(toks); free(piece); free(names);
  return (!fits && line_lsmell) || *n_tests > test_cap ? -3 : 0;
}
