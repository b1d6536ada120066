// tsm_lexsmell_kernels.cuh - the lexical test smells (docs/SPEC.md section 25) from the section-18 tests of the smell stage
// (tsm_smell_kernels.cuh) and the lexer states of the blind front (tsm_blind_kernels.cuh).  Lines are global indices (< 2^32).
//
//   k_lex_body    one warp per test, 32 lines per round: the section-18 line kinds of its body again (header statement by the
//                 section-10 kinds, docstrings by a parity scan of ballots), as lx_flag (LB_COUNTED: header statement or code
//                 line, LB_CODE: code line) and lx_end (the body end) of every body line.
//   k_lex_lines   one thread per line, lexing with blind_lex and a token sink: on a code line the Mystery Guest calls and the
//                 local names it assigns (LineSink); on a counted assertion line the assertion call and its argument list,
//                 walked token by token over at most LEX_STMT_LINES lines of the body in registers (StmtSink).  Count-then-write:
//                 the first pass counts the names of every line, an xscan places them, the second pass (WRITE) hashes them.
//   k_lex_tests   persistent warps, one test at a time, 32 lines per round: the counts, the distinct local names by inserting
//                 their hashes into a hash set (open addressing, atomicCAS, half full at most): the warp's own LEX_SET_SLOTS
//                 slots of shared memory, or for a test of more than LEX_SET_SLOTS / 2 names its own 2 n slots of a global
//                 scratch table; then Assertion Roulette, the instance bits of every body line and the record.
#pragma once
#include "tsm_device.cuh"
#include "tsm_blind_kernels.cuh"
#include "tsm_smell_kernels.cuh"

namespace tsm {

constexpr uint32_t LEX_STMT_LINES = 64, LEX_OBSCURE_LOCALS = 10, LEX_SET_SLOTS = 512;
constexpr unsigned long long LEX_EMPTY = ~0ull;                                   // an empty slot of the name sets
constexpr uint8_t LB_COUNTED = 1, LB_CODE = 2;                                    // lx_flag
constexpr uint8_t LX_STMT = 1, LX_UNEXPL = 2, LX_MAGIC = 4, LX_SUB = 8, LX_GUEST = 16;   // per-line statement / code-line facts
constexpr uint32_t LS_ROULETTE = 1, LS_MAGIC = 2, LS_SUB = 4, LS_GUEST = 8, LS_OBSCURE = 16;   // TSM_LSMELL_* bits

// An identifier of k bytes: the first 16 in (lo, hi), little-endian.
struct LxName { unsigned long long lo, hi; uint32_t k; };
__host__ __device__ constexpr LxName lx_name(const char* s) {
  LxName r{0, 0, 0};
  for (; s[r.k]; ++r.k) {
    if (r.k < 8) r.lo |= (unsigned long long)(uint8_t)s[r.k] << (8 * r.k);
    else if (r.k < 16) r.hi |= (unsigned long long)(uint8_t)s[r.k] << (8 * (r.k - 8));
  }
  return r;
}
__device__ __forceinline__ unsigned long long lx_mask(uint32_t n) { return n >= 8 ? ~0ull : (1ull << (8 * n)) - 1; }
// exact name (names of up to 16 bytes)
__device__ __forceinline__ bool lx_is(const LxName& a, const LxName& b) { return a.k == b.k && a.lo == b.lo && a.hi == b.hi; }
// prefix of up to 16 bytes
__device__ __forceinline__ bool lx_pre(const LxName& a, const LxName& p) {
  return a.k >= p.k && (a.lo & lx_mask(p.k)) == p.lo && (p.k <= 8 || (a.hi & lx_mask(p.k - 8)) == p.hi);
}
// exact name of any length, the bytes past 16 read from the line
__device__ __forceinline__ bool lx_is_long(LineBytes& B, uint32_t i0, const LxName& a, const char* s) {
  const LxName p = lx_name(s);
  if (a.k != p.k || a.lo != p.lo || a.hi != p.hi) return false;
  for (uint32_t j = 16; j < p.k; ++j)
    if (B.at(i0 + j) != (uint8_t)s[j]) return false;
  return true;
}
// the identifier holds `assert` (ASCII case-insensitive), or (cj) `EXPECT_`
__device__ __forceinline__ bool lx_has_assert(LineBytes& B, uint32_t i0, uint32_t k, bool cj) {
  for (uint32_t q = 0; q + 6 <= k; ++q) {
    bool a = true;
    for (uint32_t j = 0; j < 6 && a; ++j) a = (B.at(i0 + q + j) | 0x20u) == (uint32_t)"assert"[j];
    if (a) return true;
    if (cj && q + 7 <= k) {
      bool x = true;
      for (uint32_t j = 0; j < 7 && x; ++j) x = B.at(i0 + q + j) == (uint32_t)"EXPECT_"[j];
      if (x) return true;
    }
  }
  return false;
}

// Token codes of the sinks: a punctuation byte is itself; the others are above 0xFF.
constexpr uint32_t T_NUM = 0x100, T_STR = 0x101, T_LIT = 0x102, T_ID = 0x103, T_KW = 0x104, T_IS = 0x105, T_IN = 0x106,
                   T_NOT = 0x107, T_ASSERT = 0x108, T_SASSERT = 0x109;

// Identifier tokens: keyword, literal name or identifier, by the keyword table of the blind lexer.
__device__ __forceinline__ uint32_t lx_ident_code(const BlindKw* kw, const uint8_t* kind, uint32_t fam, const LxName& n) {
  const uint32_t kk = blind_kw_kind(kw, kind, n.lo, n.hi, n.k);
  if (kk & (fam == 1 ? KW_PY : KW_CJ)) {
    if (lx_is(n, lx_name("assert"))) return T_ASSERT;
    if (fam == 1 && lx_is(n, lx_name("is"))) return T_IS;
    if (fam == 1 && lx_is(n, lx_name("in"))) return T_IN;
    if (fam == 1 && lx_is(n, lx_name("not"))) return T_NOT;
    if (fam == 2 && lx_is(n, lx_name("static_assert"))) return T_SASSERT;
    return T_KW;
  }
  return (kk & (fam == 1 ? KW_PY_LIT : KW_CJ_LIT)) ? T_LIT : T_ID;
}

// Operand state of Magic Number: 0 empty, 1 a sign, 2 a sign and a number or a number (magic when it ends so), 3 anything else.
__device__ __forceinline__ uint32_t lx_operand(uint32_t os, uint32_t t) {
  if (t == T_NUM) return os <= 1 ? 2u : 3u;
  if ((t == '-' || t == '+') && os == 0) return 1u;
  return 3u;
}

// Code-line facts: Mystery Guest and the local names (section 25).  WRITE: hashes the names into out.
template <bool WRITE>
struct LineSink {
  const BlindKw* kw; const uint8_t* kind; uint32_t fam;
  unsigned long long* out;
  bool guest = false, pend_call = false;
  uint32_t pst = 0, n = 0;                                 // PY: 0 start, 1 name, 2 ',', 3 '=', 4 names, 5 none
  int32_t depth = 0;                                       // CJ: the first depth-0 lone '=' (cst 0 search, 1 pending, 2 found)
  uint32_t nt = 0, cst = 0, prev = 0, ci0 = 0, ck = 0;
  bool bad = false, cand = false;
  __device__ __forceinline__ void name_hash(LineBytes& B, uint32_t i0, uint32_t k, uint32_t slot) {
    BlindHash h{0, 0, 0};
    for (uint32_t j = 0; j < k; ++j) h.byte(B.at(i0 + j));
    out[slot] = mix_hash(canon61(h.acc), h.len);
  }
  // token t; (i0, k): the identifier's bytes when t == T_ID
  __device__ __forceinline__ void tok(LineBytes* B, uint32_t t, uint32_t i0, uint32_t k) {
    if (pend_call && t == '(') guest = true;
    pend_call = false;
    if (fam == 1) {
      if (t == T_ID && (pst == 0 || pst == 2)) {
        if (WRITE) name_hash(*B, i0, k, n);
        ++n; pst = 1;
      } else if (pst == 1 && t == ',') pst = 2;
      else if (pst == 1 && t == '=') pst = 3;
      else if (pst == 3) pst = t == '=' ? 5u : 4u;
      else if (pst < 3) pst = 5;
      return;
    }
    if (cst == 1) cst = t == '=' ? 0u : 2u;
    if (cst == 0 && depth == 0 && t == '=' &&
        !(prev == '=' || prev == '!' || prev == '<' || prev == '>' || prev == '+' || prev == '-' || prev == '*' || prev == '/' ||
          prev == '%' || prev == '&' || prev == '|' || prev == '^')) {
      cst = 1;
      cand = nt >= 2 && prev == T_ID && !bad;
    }
    bad = bad || t == '(' || t == '.' || t == '[';
    if (t == '(' || t == '[' || t == '{') ++depth;
    else if (t == ')' || t == ']' || t == '}') --depth;
    ++nt;
    prev = t;
    if (t == T_ID && cst == 0) { ci0 = i0; ck = k; }
  }
  __device__ __forceinline__ void number() { tok(nullptr, T_NUM, 0, 0); }
  __device__ __forceinline__ void string() { tok(nullptr, T_STR, 0, 0); }
  __device__ __forceinline__ void punct(uint32_t c) { tok(nullptr, c, 0, 0); }
  __device__ __forceinline__ void ident(LineBytes& B, uint32_t, uint32_t i0, uint32_t k, unsigned long long lo, unsigned long long hi) {
    const LxName nm{lo, hi, k};
    const uint32_t t = lx_ident_code(kw, kind, fam, nm);
    bool call = false;
    if (t == T_ID) {
      if (fam == 1) {
        call = lx_is(nm, lx_name("open")) || lx_is(nm, lx_name("urlopen")) || lx_is(nm, lx_name("connect")) ||
               lx_is(nm, lx_name("read_csv")) || lx_is(nm, lx_name("read_excel")) || lx_is(nm, lx_name("read_json")) ||
               lx_is(nm, lx_name("read_parquet")) || lx_is(nm, lx_name("loadtxt")) || lx_is(nm, lx_name("genfromtxt")) ||
               lx_is(nm, lx_name("imread")) || lx_is(nm, lx_name("listdir"));
      } else {
        call = lx_is(nm, lx_name("fopen")) || lx_is(nm, lx_name("freopen")) || lx_is(nm, lx_name("open")) ||
               lx_is(nm, lx_name("getConnection"));
        if (lx_is(nm, lx_name("ifstream")) || lx_is(nm, lx_name("ofstream")) || lx_is(nm, lx_name("fstream")) ||
            lx_is(nm, lx_name("File")) || lx_is(nm, lx_name("FileReader")) || lx_is(nm, lx_name("FileWriter")) ||
            lx_is(nm, lx_name("FileInputStream")) || lx_is(nm, lx_name("FileOutputStream")) ||
            lx_is(nm, lx_name("RandomAccessFile")) || lx_is(nm, lx_name("Files")))
          guest = true;
      }
    }
    tok(&B, t, i0, k);
    pend_call = call;
  }
  // the count of names the line assigns, after its last token (WRITE: the C-family name is hashed here)
  __device__ __forceinline__ uint32_t names(LineBytes& B) {
    if (fam == 1) return pst == 3 || pst == 4 ? n : 0u;
    if (cst && cand) {
      if (WRITE) name_hash(B, ci0, ck, 0);
      return 1;
    }
    return 0;
  }
};

// The assertion statement of one line (section 25), token by token over the lines of its walk.
enum : uint32_t { CK_NONE, CK_UNITTEST, CK_NUMPY, CK_GTEST, CK_CASSERT, CK_STATIC, CK_JCALL, CK_PYASSERT, CK_JASSERT };
enum : uint32_t { PH_FIND, PH_PEND, PH_LIST, PH_AFTER, PH_EXPR, PH_DONE };
struct StmtSink {
  const BlindKw* kw; const uint8_t* kind; uint32_t fam, ext;
  uint32_t phase = PH_FIND, ck = CK_NONE, arity = 0, sub = 0, prev = 0;
  int32_t depth = 0;
  bool stmt = false, magic = false, subhit = false, msg = false, kwmsg = false, kwerr = false, anylit = false;
  bool first_str = false, last_str = false, lt1 = false, expl_lt = false, line_bs = false, line_tok = false;
  uint32_t nargs = 0, npos = 0, after = 0;
  // the current argument
  uint32_t ti = 0, a0 = 0, t0 = 0, kwst = 0, os = 0, os_prev = 0, ins = 0, eqs = 0;
  bool arg_magic = false, arg_sub = false;

  __device__ __forceinline__ void end_operand(uint32_t t) {
    const uint32_t o = ((t == '=' && prev == '!') || (t == T_IN && prev == T_NOT)) ? os_prev : os;
    if (o == 2) arg_magic = true;
    os = os_prev = 0;
  }
  // a token of an operand list at its level (calls: inside the argument; statements: the expression)
  __device__ __forceinline__ void operand_tok(uint32_t t) {
    const bool py = fam == 1;
    if (t == '<' || t == '>' || t == '=' || (py && (t == T_IS || t == T_IN || (t == T_NOT && prev == T_IS))))
      end_operand(t);
    else { os_prev = os; os = lx_operand(os, t); }
  }
  __device__ __forceinline__ void close_arg() {
    if (os == 2) arg_magic = true;
    if (ti) {
      const bool kwarg = fam == 1 && kwst == 2 && ti >= 2;
      if (!kwarg) {
        ++npos;
        magic = magic || arg_magic;
        anylit = anylit || (ti == 1 && t0 == T_LIT);
      } else if (a0 == 2) kwmsg = true;
      else if (a0 == 3) kwerr = true;
      if (nargs == 0) {
        first_str = ti == 1 && t0 == T_STR;
        if (sub == 1) subhit = subhit || arg_sub || ins == 3 || eqs == 4;
      }
      last_str = ti == 1 && t0 == T_STR;
      ++nargs;
    }
    ti = a0 = t0 = kwst = os = os_prev = ins = eqs = 0;
    arg_magic = arg_sub = false;
  }
  // the token t of the current argument; d = the depth before it (1: the argument's own level), ida: identifier facts
  // (1 msg, 2 err_msg, 4 isinstance, 8 equals)
  __device__ __forceinline__ void arg_tok(uint32_t t, int32_t d, uint32_t ida) {
    const bool py = fam == 1, level = d == 1, closer = t == ')' || t == ']' || t == '}';
    if (ti == 0) {
      t0 = t;
      a0 = t == T_ID ? ((ida & 1) ? 2u : (ida & 2) ? 3u : 1u) : 0u;
      kwst = t == T_ID ? 1u : 0u;
      ins = (py && t == T_ID && (ida & 4)) ? 1u : 0u;
    } else if (ti == 1) {
      kwst = kwst == 1 && t == '=' ? 2u : 0u;
      ins = ins == 1 && t == '(' ? 2u : 0u;
    } else {
      if (ti == 2 && kwst == 2 && t == '=') kwst = 0;
      if (ins == 2 && closer && d == 2) ins = 3;
      else if (ins == 3) ins = 0;
    }
    if (level) {
      operand_tok(t);
      if (t == '=' && (prev == '=' || prev == '!' || prev == '<' || prev == '>')) arg_sub = true;
      if (py && (t == '<' || t == '>' || t == T_IS || t == T_IN)) arg_sub = true;
    }
    if (ext == 4) {
      if (eqs == 3) { if (closer && d == 2) eqs = 4; }
      else if (level) eqs = t == '.' ? 1u : (eqs == 1 && t == T_ID && (ida & 8)) ? 2u : (eqs == 2 && t == '(') ? 3u : 0u;
    }
    ++ti;
  }
  __device__ __forceinline__ void classify(LineBytes& B, uint32_t i0, const LxName& n) {
    const bool py = fam == 1;
    ck = CK_NONE; arity = 0;
    if (py) {
      if (lx_pre(n, lx_name("assert_")) && n.k > 7) {
        ck = (lx_pre(n, lx_name("assert_called")) || lx_pre(n, lx_name("assert_awaited")) || lx_is(n, lx_name("assert_any_call")) ||
              lx_is(n, lx_name("assert_has_calls")) || lx_is_long(B, i0, n, "assert_not_called")) ? CK_NONE : CK_NUMPY;
      } else if (prev == '.' && lx_pre(n, lx_name("assert"))) {
        if (!(lx_pre(n, lx_name("assertRaises")) || lx_pre(n, lx_name("assertWarns")) || lx_is(n, lx_name("assertLogs")) ||
              lx_is(n, lx_name("assertNoLogs")))) {
          ck = CK_UNITTEST;
          arity = (lx_is(n, lx_name("assertTrue")) || lx_is(n, lx_name("assertFalse")) || lx_is(n, lx_name("assertIsNone")) ||
                   lx_is(n, lx_name("assertIsNotNone")) || lx_is(n, lx_name("assert_"))) ? 1u
                  : (lx_is_long(B, i0, n, "assertAlmostEqual") || lx_is_long(B, i0, n, "assertNotAlmostEqual") ||
                     lx_is_long(B, i0, n, "assertAlmostEquals") || lx_is_long(B, i0, n, "assertNotAlmostEquals")) ? 3u : 2u;
        }
      }
    } else if (lx_pre(n, lx_name("EXPECT_")) || lx_pre(n, lx_name("ASSERT_"))) {
      ck = CK_GTEST;
    } else if (ext == 4 && lx_pre(n, lx_name("assert"))) {
      ck = CK_JCALL;
      arity = (lx_is(n, lx_name("assertTrue")) || lx_is(n, lx_name("assertFalse")) || lx_is(n, lx_name("assertNull")) ||
               lx_is(n, lx_name("assertNotNull"))) ? 1u : 2u;
    }
    sub = (lx_is(n, lx_name("assertTrue")) || lx_is(n, lx_name("assertFalse")) || lx_is(n, lx_name("assert_")) ||
           lx_is(n, lx_name("EXPECT_TRUE")) || lx_is(n, lx_name("EXPECT_FALSE")) || lx_is(n, lx_name("ASSERT_TRUE")) ||
           lx_is(n, lx_name("ASSERT_FALSE"))) ? 1u
          : (lx_is(n, lx_name("assertEqual")) || lx_is(n, lx_name("assertEquals")) || lx_is(n, lx_name("assertNotEqual")) ||
             lx_is(n, lx_name("assertNotEquals")) || lx_is(n, lx_name("assertIs")) || lx_is(n, lx_name("assertIsNot")) ||
             lx_is(n, lx_name("EXPECT_EQ")) || lx_is(n, lx_name("EXPECT_NE")) || lx_is(n, lx_name("ASSERT_EQ")) ||
             lx_is(n, lx_name("ASSERT_NE"))) ? 2u : 0u;
  }
  __device__ __forceinline__ void tok(uint32_t t, uint32_t ida) {
    line_tok = true;
    line_bs = t == '\\';
    const bool py = fam == 1;
    if (phase == PH_PEND) {
      if (t == '(') { phase = PH_LIST; depth = 1; stmt = true; prev = t; return; }
      phase = PH_FIND;
    }
    if (phase == PH_FIND) {
      if (t == T_ASSERT && (py || ext == 4)) { phase = PH_EXPR; stmt = true; ck = py ? CK_PYASSERT : CK_JASSERT; }
      else if (t == T_ASSERT && !py) { phase = PH_PEND; ck = CK_CASSERT; sub = 0; }
      else if (t == T_SASSERT && !py) { phase = PH_PEND; ck = CK_STATIC; sub = 0; }
      else if (ida & 16) phase = PH_PEND;                  // (classified by ident)
    } else if (phase == PH_LIST) {
      const bool closer = t == ')' || t == ']' || t == '}';
      if (closer && depth == 1) {
        close_arg();
        depth = 0;
        phase = ck == CK_GTEST ? PH_AFTER : PH_DONE;
      } else if (t == ',' && depth == 1) {
        close_arg();
      } else {
        arg_tok(t, depth, ida);
        if (t == '(' || t == '[' || t == '{') ++depth;
        else if (closer) --depth;
      }
    } else if (phase == PH_AFTER) {
      if (after == 0) lt1 = t == '<';
      else { expl_lt = lt1 && t == '<'; phase = PH_DONE; }
      ++after;
    } else if (phase == PH_EXPR) {
      if (ck == CK_JASSERT && depth == 0 && t == ';') phase = PH_DONE;
      else if (depth == 0 && !msg && (py ? t == ',' : t == ':')) { msg = true; if (os == 2) arg_magic = true; }
      else {
        if (!msg && depth == 0) operand_tok(t);
        if (t == '(' || t == '[' || t == '{') ++depth;
        else if (t == ')' || t == ']' || t == '}') --depth;
      }
    }
    prev = t;
  }
  __device__ __forceinline__ void number() { tok(T_NUM, 0); }
  __device__ __forceinline__ void string() { tok(T_STR, 0); }
  __device__ __forceinline__ void punct(uint32_t c) { tok(c, 0); }
  __device__ __forceinline__ void ident(LineBytes& B, uint32_t, uint32_t i0, uint32_t k, unsigned long long lo, unsigned long long hi) {
    const LxName n{lo, hi, k};
    const uint32_t t = lx_ident_code(kw, kind, fam, n);
    uint32_t ida = 0;
    if (phase == PH_FIND && t == T_ID) {
      if (lx_has_assert(B, i0, k, fam == 2)) { classify(B, i0, n); ida = 16; }
    } else if (phase == PH_PEND && t == T_ID) {            // a pending name that is not called: this one may be
      if (lx_has_assert(B, i0, k, fam == 2)) { phase = PH_FIND; classify(B, i0, n); ida = 16; }
    } else if (phase == PH_LIST && t == T_ID) {
      ida = (lx_is(n, lx_name("msg")) ? 1u : 0u) | (lx_is(n, lx_name("err_msg")) ? 2u : 0u) | (lx_is(n, lx_name("isinstance")) ? 4u : 0u) |
            (lx_is(n, lx_name("equals")) ? 8u : 0u);
    }
    tok(t, ida);
  }
  __device__ __forceinline__ void begin_line() { line_tok = line_bs = false; }
  // after each line of the walk: the first line ends the search; a PY assert ends at a depth-0 line end not behind a backslash
  __device__ __forceinline__ void end_line(bool first) {
    if (first && (phase == PH_FIND || phase == PH_PEND)) phase = PH_DONE;
    if (phase == PH_EXPR && ck == CK_PYASSERT && depth == 0 && !(line_tok && line_bs)) phase = PH_DONE;
  }
  __device__ __forceinline__ bool done() const { return phase == PH_DONE; }
  // LX_* of the statement, once the walk has ended (a list cut by the body end or the line cap ends there)
  __device__ __forceinline__ uint32_t result() {
    if (!stmt) return 0;
    if (phase == PH_LIST) close_arg();
    bool expl = false, counted = true;
    if (ck == CK_PYASSERT || ck == CK_JASSERT) {
      if (!msg && os == 2) arg_magic = true;
      magic = arg_magic;
      expl = msg;
    } else if (ck == CK_UNITTEST) expl = npos > arity || kwmsg;
    else if (ck == CK_NUMPY) expl = kwmsg || kwerr;
    else if (ck == CK_GTEST) expl = expl_lt;
    else if (ck == CK_STATIC) expl = nargs >= 2;
    else if (ck == CK_JCALL) expl = nargs > arity && (first_str || last_str);
    else if (ck == CK_NONE) counted = false;
    const bool sb = (sub == 1 && subhit) || (sub == 2 && anylit);
    return LX_STMT | (counted && !expl ? LX_UNEXPL : 0) | (magic ? LX_MAGIC : 0) | (sb ? LX_SUB : 0);
  }
};

struct LexBody {
  const tsm_smell_test* tests; uint32_t n_tests; const unsigned long long* line_base; const uint8_t* ext;
  const uint8_t* kind; const SmellLine* L; uint8_t* lx_flag; uint32_t* lx_end;
};

__global__ void __launch_bounds__(256) k_lex_body(LexBody a) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  const uint32_t lt = (1u << lane) - 1u;
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < a.n_tests; t += warps) {
    const tsm_smell_test r = a.tests[t];
    const uint32_t b = (uint32_t)a.line_base[r.file] + (uint32_t)r.line, bend = b + (uint32_t)r.body_lines;
    const bool py = a.ext[r.file] == 1;
    uint32_t hend = bend;                                  // the header statement: b and the kind-2 lines after it
    for (uint32_t base = b + 1; base < bend; base += 32) {
      const uint32_t l = base + lane;
      const uint32_t m = __ballot_sync(0xffffffffu, l < bend && a.kind[l] != 2);
      if (m) { hend = base + __ffs(m) - 1; break; }
    }
    uint32_t dqc = 0, sqc = 0;
    for (uint32_t base = b; base < bend; base += 32) {
      const uint32_t l = base + lane;
      const bool valid = l < bend, inbody = valid && l >= hend;
      const uint32_t bits = valid ? a.L[l].bits : 0;
      const uint32_t dm = __ballot_sync(0xffffffffu, inbody && (bits & SL_DQ)), sm = __ballot_sync(0xffffffffu, inbody && (bits & SL_SQ));
      const bool doc = py && ((bits & SL_DOCSTART) || ((dqc + __popc(dm & lt)) & 1) || ((sqc + __popc(sm & lt)) & 1));
      dqc += __popc(dm); sqc += __popc(sm);
      const bool code = inbody && !(bits & (SL_BLANK | SL_COMMENT)) && !doc;
      if (valid) {
        a.lx_flag[l] = (uint8_t)(l < hend ? LB_COUNTED : code ? (LB_COUNTED | LB_CODE) : 0);
        a.lx_end[l] = bend;
      }
    }
  }
}

template <bool WRITE>
__global__ void __launch_bounds__(256) k_lex_lines(DiffSide d, uint32_t n, unsigned long long total, const uint8_t* state,
                                                   const uint8_t* lx_flag, const uint32_t* lx_end, uint8_t* lflag, uint32_t* ncnt,
                                                   const unsigned long long* nbase, unsigned long long* names) {
  __shared__ BlindKw kw[BLIND_KW_SLOTS];
  __shared__ uint8_t kind[BLIND_KW_SLOTS];
  for (uint32_t t = threadIdx.x; t < BLIND_KW_SLOTS; t += blockDim.x) { kw[t] = c_blind_kw[t]; kind[t] = c_blind_kind[t]; }
  __syncthreads();
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const uint32_t fl = lx_flag[i];
  if (WRITE ? ncnt[i] == 0 : fl == 0) {
    if (!WRITE) { lflag[i] = 0; ncnt[i] = 0; }
    return;
  }
  const uint32_t f = blind_file(d.line_base, n, i), ext = d.ext[f], fam = blind_family(ext);
  const uint8_t* g = d.arena + (uint32_t)d.off[f];
  const uint32_t fb = (uint32_t)d.line_base[f];
  const auto line_start = [&](uint32_t l) { return l == fb ? 0u : d.line_end[l - 1] + 1u; };
  uint32_t out = 0, cnt = 0;
  if (fl & LB_CODE) {
    LineSink<WRITE> ls{kw, kind, fam, WRITE ? names + nbase[i] : nullptr};
    LineBytes B{g, 1u, 0};
    blind_lex(B, line_start((uint32_t)i), d.line_end[i], fam, state[i], ls);
    cnt = ls.names(B);
    if (ls.guest) out |= LX_GUEST;
  }
  if (WRITE) return;
  if ((fl & LB_COUNTED) && d.line_flag[i]) {
    StmtSink s{kw, kind, fam, ext};
    const uint32_t lim = min(lx_end[i], (uint32_t)i + LEX_STMT_LINES);
    for (uint32_t l = (uint32_t)i; l < lim && !s.done(); ++l) {
      LineBytes B{g, 1u, 0};
      s.begin_line();
      blind_lex(B, line_start(l), d.line_end[l], fam, state[l], s);
      s.end_line(l == (uint32_t)i);
    }
    out |= s.result();
  }
  lflag[i] = (uint8_t)out;
  ncnt[i] = cnt;
}

struct LexTests {
  const tsm_smell_test* tests; uint32_t n_tests; const unsigned long long* line_base;
  const uint8_t* lflag; const unsigned long long* nbase; const unsigned long long* names;
  unsigned long long* gset;                                // [2 * names]: LEX_EMPTY, the sets of the tests of many names
  uint8_t* line_lsmell; tsm_lex_test* out;
};

__global__ void __launch_bounds__(256) k_lex_tests(LexTests a) {
  __shared__ unsigned long long s_set[8][LEX_SET_SLOTS];
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < a.n_tests; t += warps) {
    const tsm_smell_test r = a.tests[t];
    const uint32_t b = (uint32_t)a.line_base[r.file] + (uint32_t)r.line, bend = b + (uint32_t)r.body_lines;
    uint32_t nst = 0, nun = 0, nmg = 0;
    for (uint32_t base = b; base < bend; base += 32) {
      const uint32_t l = base + lane;
      const uint32_t x = l < bend ? a.lflag[l] : 0;
      nst += __popc(__ballot_sync(0xffffffffu, x & LX_STMT));
      nun += __popc(__ballot_sync(0xffffffffu, x & LX_UNEXPL));
      nmg += __popc(__ballot_sync(0xffffffffu, x & LX_MAGIC));
    }
    const unsigned long long n0 = a.nbase[b], nn = a.nbase[bend] - n0;
    const bool small = nn <= LEX_SET_SLOTS / 2;
    unsigned long long* set = small ? s_set[threadIdx.x >> 5] : a.gset + 2 * n0;
    const unsigned long long slots = small ? LEX_SET_SLOTS : 2 * nn;
    if (small)
      for (uint32_t k = lane; k < LEX_SET_SLOTS; k += 32) set[k] = LEX_EMPTY;
    __syncwarp();
    uint32_t nloc = 0;
    bool sentinel = false;                                 // a name whose hash is LEX_EMPTY counts once, outside the set
    for (unsigned long long t0 = 0; t0 < nn; t0 += 32) {
      const unsigned long long idx = t0 + lane;
      const unsigned long long h = idx < nn ? a.names[n0 + idx] : LEX_EMPTY;
      bool fresh = false;
      if (idx < nn && h != LEX_EMPTY) {
        unsigned long long q = __umul64hi(h, slots);       // home slot: h * slots / 2^64
        for (;;) {
          const unsigned long long prev = atomicCAS(set + q, LEX_EMPTY, h);
          if (prev == LEX_EMPTY) { fresh = true; break; }
          if (prev == h) break;
          if (++q == slots) q = 0;
        }
      }
      nloc += __popc(__ballot_sync(0xffffffffu, fresh));
      sentinel = sentinel || __any_sync(0xffffffffu, idx < nn && h == LEX_EMPTY);
    }
    nloc += sentinel ? 1u : 0u;
    __syncwarp();
    const bool roulette = nun >= 2, obscure = nloc > LEX_OBSCURE_LOCALS;
    uint32_t ninst = 0, smells = 0;
    for (uint32_t base = b; base < bend; base += 32) {
      const uint32_t l = base + lane;
      uint32_t ls = 0;
      if (l < bend) {
        const uint32_t x = a.lflag[l];
        ls = (roulette && (x & LX_UNEXPL) ? LS_ROULETTE : 0) | (x & LX_MAGIC ? LS_MAGIC : 0) | (x & LX_SUB ? LS_SUB : 0) |
             (x & LX_GUEST ? LS_GUEST : 0) | (l == b && obscure ? LS_OBSCURE : 0);
        a.line_lsmell[l] = (uint8_t)ls;
      }
      ninst += __reduce_add_sync(0xffffffffu, __popc(ls));
      smells |= __reduce_or_sync(0xffffffffu, ls);
    }
    if (lane == 0) a.out[t] = tsm_lex_test{(int32_t)nst, (int32_t)nun, (int32_t)nmg, (int32_t)nloc, smells, (int32_t)ninst};
  }
}

}  // namespace tsm
