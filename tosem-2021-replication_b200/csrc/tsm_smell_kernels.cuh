// tsm_smell_kernels.cuh - test smells (docs/SPEC.md section 18) from the line records, the section-10 line kinds and the case
// spans of tsm_case_kernels.cuh (k_case_heads, xscan, k_case_lines).  Lines are global indices (< 2^32).
//
//   k_smell_lines   one thread per line, 8 bytes per load: every per-line fact the tests need (SmellLine), the patterns of
//                   sleepy and print from one Shift-And automaton over a 256-entry shared table with a 64-bit state, and on
//                   assertion lines the stripped-line bytes_hash and the redundant form.  On a header line it also decides
//                   whether the case is a test: tflag[case] (numbered by xscan into dense test records).
//   k_smell_tests   persistent warps, one test at a time, 32 lines per round: the header statement end and the body end by
//                   ballots (PY: a kind-1, non-comment line indented at most as the header; C family and Java: a warp scan of
//                   the brace deltas), the docstring state by a parity scan of ballots, the line-level instances, then the
//                   duplicate assertions by comparing every assertion hash with every earlier one of the test through
//                   shuffles, 32 x 32 per tile pair (O(A^2 / 32) per test); lane 0 walks the '@' lines above the header.
//   k_smell_churn   persistent warps, one test of one side of revision pairs at a time, 32 body lines per round: per smell the
//                   instance lines and those the revision adds or removes (docs/SPEC.md section 19), by ballots; <true> also
//                   those of the five lexical smells (section 26) in the same walk.
#pragma once
#include "tsm_device.cuh"
#include "tsm_diff_kernels.cuh"

namespace tsm {

// SmellLine::bits
constexpr uint32_t SL_BLANK = 1u << 0, SL_COMMENT = 1u << 1, SL_DOCSTART = 1u << 2, SL_EMPTYOK = 1u << 3, SL_OPEN = 1u << 4,
                   SL_DQ = 1u << 5, SL_SQ = 1u << 6, SL_AT = 1u << 7, SL_DECO_IGN = 1u << 8, SL_HDR_IGN = 1u << 9,
                   SL_COND = 1u << 10, SL_EXC = 1u << 11, SL_SLEEP = 1u << 12, SL_PRINT = 1u << 13, SL_SKIPCALL = 1u << 14,
                   SL_ASSERT = 1u << 15, SL_REDUNDANT = 1u << 16;
// smell bits (tsm_smell_test::smells, line_smell): the order of docs/SPEC.md section 18 and TSM_SMELL_* of tosemscan.h
constexpr uint32_t SM_EMPTY = 1u << 0, SM_FREE = 1u << 1, SM_DUP = 1u << 2, SM_REDUNDANT = 1u << 3, SM_COND = 1u << 4,
                   SM_EXC = 1u << 5, SM_SLEEP = 1u << 6, SM_PRINT = 1u << 7, SM_IGNORED = 1u << 8;

struct SmellLine { uint32_t bits; int32_t brace; uint32_t indent; uint32_t pad; unsigned long long hash; };

// Shift-And patterns (62 state bits).  Some are suffixes whose prefix is checked at the match: `_for(` and
// `_until(` need `sleep` before them, `out.print` and `err.print` need `System.`.  The print family needs a byte outside
// [A-Za-z0-9_] (or the line start) before it; `print(` preceded by such a `p` is `pprint(`.
#define TSM_SMELL_PATTERNS "print(\0printf(\0puts(\0cout\0cerr\0sleep(\0_for(\0_until(\0out.print\0err.print\0"
constexpr int kSmellPats = 10;
__constant__ char kSmellPat[] = TSM_SMELL_PATTERNS;

__device__ __forceinline__ uint32_t sm_byte(const uint8_t* g, uint32_t q) { return __ldg(g + q); }

__device__ __forceinline__ bool sm_at(const uint8_t* g, uint32_t q, uint32_t hi, const char* lit) {   // lit occurs at q, inside [.., hi)
  for (uint32_t k = 0; lit[k]; ++k)
    if (q + k >= hi || sm_byte(g, q + k) != (uint8_t)lit[k]) return false;
  return true;
}
__device__ __forceinline__ bool sm_has(const uint8_t* g, uint32_t s, uint32_t e, const char* lit) {
  for (uint32_t q = s; q < e; ++q)
    if (sm_at(g, q, e, lit)) return true;
  return false;
}
__device__ __forceinline__ bool sm_is(const uint8_t* g, uint32_t s, uint32_t e, const char* lit) {     // [s, e) == lit
  uint32_t k = 0;
  for (; lit[k]; ++k)
    if (s + k >= e || sm_byte(g, s + k) != (uint8_t)lit[k]) return false;
  return s + k == e;
}
__device__ __forceinline__ void sm_trim(const uint8_t* g, uint32_t& s, uint32_t& e) {
  while (s < e && is_w(sm_byte(g, s))) ++s;
  while (e > s && is_w(sm_byte(g, e - 1))) --e;
}
__device__ __forceinline__ bool sm_constant(const uint8_t* g, uint32_t s, uint32_t e) {
  return sm_is(g, s, e, "True") || sm_is(g, s, e, "False") || sm_is(g, s, e, "true") || sm_is(g, s, e, "false") ||
         sm_is(g, s, e, "None") || sm_is(g, s, e, "nullptr") || sm_is(g, s, e, "NULL") || sm_is(g, s, e, "0") || sm_is(g, s, e, "1");
}
__device__ __forceinline__ bool sm_ident_before(const uint8_t* g, uint32_t s, uint32_t q) {   // byte q-1 exists and is [A-Za-z0-9_]
  return q > s && is_ident(sm_byte(g, q - 1));
}

// The redundant form of SPEC section 18 on the stripped assertion line [a0, a1); fp / lp = its first '(' and last ')'.
__device__ bool sm_redundant(const uint8_t* g, uint32_t a0, uint32_t a1, uint32_t fp, uint32_t lp) {
  if (a1 - a0 > 6 && sm_at(g, a0, a1, "assert") && is_w(sm_byte(g, a0 + 6))) {
    uint32_t s = a0 + 6, e = a1;
    sm_trim(g, s, e);
    if (sm_constant(g, s, e)) return true;
  }
  if (fp == 0xFFFFFFFFu || lp == 0xFFFFFFFFu || lp <= fp) return false;
  uint32_t x0 = fp + 1, x1 = lp;
  sm_trim(g, x0, x1);
  if (sm_constant(g, x0, x1)) return true;
  int depth = 0;
  uint32_t commas = 0, cpos = 0;
  for (uint32_t q = x0; q < x1; ++q) {
    const uint32_t c = sm_byte(g, q);
    if (c == '(' || c == '[' || c == '{') ++depth;
    else if (c == ')' || c == ']' || c == '}') --depth;
    else if (c == ',' && depth == 0) { if (++commas > 1) return false; cpos = q; }
  }
  if (commas != 1) return false;
  uint32_t p0 = x0, p1 = cpos, q0 = cpos + 1, q1 = x1;
  sm_trim(g, p0, p1); sm_trim(g, q0, q1);
  if (p1 == p0 || p1 - p0 != q1 - q0) return false;
  for (uint32_t k = 0; k < p1 - p0; ++k)
    if (sm_byte(g, p0 + k) != sm_byte(g, q0 + k)) return false;
  return true;
}

// The test-header forms of SPEC section 18 on the stripped header [a0, a1) of line [s, e).
__device__ bool sm_test_header(const uint8_t* g, uint32_t s, uint32_t e, uint32_t a0, uint32_t a1, uint32_t ext) {
  if (ext == 1) {
    uint32_t q = a0;
    if (sm_at(g, q, a1, "async")) {
      q += 5;
      const uint32_t q0 = q;
      while (q < a1 && is_w(sm_byte(g, q))) ++q;
      if (q == q0) return false;
    }
    if (!sm_at(g, q, a1, "def")) return false;
    q += 3;
    const uint32_t q0 = q;
    while (q < a1 && is_w(sm_byte(g, q))) ++q;
    return q > q0 && sm_at(g, q, a1, "test");
  }
  if (ext == 4) return sm_has(g, s, e, "void") && sm_has(g, s, e, "(");
  return sm_at(g, a0, a1, "TEST(") || sm_at(g, a0, a1, "TEST_F(") || sm_at(g, a0, a1, "TEST_P(") || sm_at(g, a0, a1, "TYPED_TEST(") ||
         sm_at(g, a0, a1, "TYPED_TEST_P(") || sm_at(g, a0, a1, "BOOST_AUTO_TEST_CASE(") ||
         sm_at(g, a0, a1, "BOOST_FIXTURE_TEST_CASE(") || sm_at(g, a0, a1, "BOOST_DATA_TEST_CASE(");
}

// head[l] = 1 on header lines, case_of = xscan(head): tflag[case] = 1 when the case's header opens a test.
__global__ void __launch_bounds__(256) k_smell_lines(DiffSide d, int32_t n, unsigned long long total, const uint32_t* head,
                                                     const unsigned long long* case_of, SmellLine* out, uint32_t* tflag) {
  __shared__ unsigned long long tab[256];
  __shared__ unsigned long long s_init, s_final;
  if (threadIdx.x == 0) {
    unsigned long long init = 0, fin = 0;
    uint32_t bit = 0, k = 0;
    for (int p = 0; p < kSmellPats; ++p) {
      init |= 1ull << bit;
      while (kSmellPat[k]) { ++k; ++bit; }
      fin |= 1ull << (bit - 1);
      ++k;
    }
    s_init = init; s_final = fin;
  }
  {
    unsigned long long t = 0;
    uint32_t bit = 0;
    for (uint32_t k = 0; k < sizeof(kSmellPat) - 1; ++k) {
      if (!kSmellPat[k]) continue;
      if ((uint8_t)kSmellPat[k] == threadIdx.x) t |= 1ull << bit;
      ++bit;
    }
    tab[threadIdx.x] = t;
  }
  __syncthreads();
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const unsigned long long INIT = s_init, FINAL = s_final;
  int lo = 0, hi = n;                                   // file of line i: line_base[lo] <= i < line_base[hi]
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (d.line_base[mid] <= i) lo = mid; else hi = mid; }
  const uint8_t* g = d.arena + (uint32_t)d.off[lo];
  const uint32_t ext = d.ext[lo];
  const uint32_t e = d.line_end[i];
  const uint32_t s = (i == d.line_base[lo]) ? 0u : d.line_end[i - 1] + 1u;
  uint32_t a0 = 0xFFFFFFFFu, a1 = 0, fp = 0xFFFFFFFFu, lp = 0xFFFFFFFFu, ind = 0, dqr = 0, sqr = 0, dqp = 0, sqp = 0;
  int32_t brace = 0;
  bool lead = true, open = false, other = false, sleepy = false, print = false;
  unsigned long long D = 0;
  for (uint32_t wb = s & ~7u; wb < e; wb += 8) {
    unsigned long long w = __ldg(reinterpret_cast<const unsigned long long*>(g + wb));
    const uint32_t k0 = wb < s ? s - wb : 0, k1 = min(8u, e - wb);
    w >>= 8 * k0;
    for (uint32_t k = k0; k < k1; ++k, w >>= 8) {
      const uint32_t c = (uint32_t)(w & 0xFF), q = wb + k;
      if (lead && (c == 0x20 || c == 0x09)) ++ind; else lead = false;
      if (!is_w(c)) { if (a0 == 0xFFFFFFFFu) a0 = q; a1 = q + 1; }
      if (c == '{') { ++brace; open = true; }
      else if (c == '}') --brace;
      else if (c == '(') { if (fp == 0xFFFFFFFFu) fp = q; }
      else if (c == ')') lp = q;
      if (!is_w(c) && c != '{' && c != '}' && c != '(' && c != ')' && c != ';' && c != ':') other = true;
      if (c == '"') ++dqr; else { dqp ^= (dqr / 3) & 1; dqr = 0; }
      if (c == '\'') ++sqr; else { sqp ^= (sqr / 3) & 1; sqr = 0; }
      D = ((D << 1) | INIT) & tab[c];
      if (D & FINAL) {
        const unsigned long long m = D & FINAL;
        // final bits in pattern order: print( 5, printf( 12, puts( 17, cout 21, cerr 25, sleep( 31, _for( 36, _until( 43,
        // out.print 52, err.print 61
        if (m & (1ull << 5)) {
          const uint32_t st = q - 5;
          if (!sm_ident_before(g, s, st) || (sm_byte(g, st - 1) == 'p' && !sm_ident_before(g, s, st - 1))) print = true;
        }
        if ((m & (1ull << 12)) && !sm_ident_before(g, s, q - 6)) print = true;
        if ((m & (1ull << 17)) && !sm_ident_before(g, s, q - 4)) print = true;
        if ((m & (1ull << 21)) && !sm_ident_before(g, s, q - 3)) print = true;
        if ((m & (1ull << 25)) && !sm_ident_before(g, s, q - 3)) print = true;
        if (m & (1ull << 31)) sleepy = true;
        if ((m & (1ull << 36)) && q - 4 >= s + 5 && sm_at(g, q - 9, q, "sleep")) sleepy = true;
        if ((m & (1ull << 43)) && q - 6 >= s + 5 && sm_at(g, q - 11, q, "sleep")) sleepy = true;
        if ((m & ((1ull << 52) | (1ull << 61))) && q - 8 >= s + 7 && sm_at(g, q - 15, q, "System.")) print = true;
      }
    }
  }
  dqp ^= (dqr / 3) & 1;
  sqp ^= (sqr / 3) & 1;
  SmellLine r{};
  r.brace = brace; r.indent = ind;
  uint32_t b = (open ? SL_OPEN : 0) | (dqp ? SL_DQ : 0) | (sqp ? SL_SQ : 0) | (sleepy ? SL_SLEEP : 0) | (print ? SL_PRINT : 0);
  if (a0 == 0xFFFFFFFFu) {
    b |= SL_BLANK | SL_EMPTYOK;
  } else {
    const bool py = ext == 1;
    if (py ? sm_at(g, a0, a1, "#") : (sm_at(g, a0, a1, "//") || sm_at(g, a0, a1, "/*") || sm_at(g, a0, a1, "*"))) b |= SL_COMMENT;
    if (sm_at(g, a0, a1, "\"\"\"") || sm_at(g, a0, a1, "'''")) b |= SL_DOCSTART;
    if (!other || sm_is(g, a0, a1, "pass")) b |= SL_EMPTYOK;
    uint32_t t = a0;                                    // first token: behind the leading W and '}' bytes
    while (t < a1 && (is_w(sm_byte(g, t)) || sm_byte(g, t) == '}')) ++t;
    uint32_t te = t;
    while (te < a1 && te - t < 8 && is_ident(sm_byte(g, te))) ++te;
    if (te == a1 || !is_ident(sm_byte(g, te))) {
      if (sm_is(g, t, te, "if") || sm_is(g, t, te, "elif") || sm_is(g, t, te, "for") || sm_is(g, t, te, "while") || sm_is(g, t, te, "switch"))
        b |= SL_COND;
      if (sm_is(g, t, te, "try") || sm_is(g, t, te, "except") || sm_is(g, t, te, "catch") || sm_is(g, t, te, "raise") || sm_is(g, t, te, "throw"))
        b |= SL_EXC;
    }
    if (py && (sm_at(g, a0, a1, "self.skipTest(") || sm_at(g, a0, a1, "pytest.skip("))) b |= SL_SKIPCALL;
    if (sm_byte(g, a0) == '@') {
      b |= SL_AT;
      if (py ? sm_has(g, s, e, "skip") : (ext == 4 && (sm_has(g, s, e, "@Ignore") || sm_has(g, s, e, "@Disabled")))) b |= SL_DECO_IGN;
    }
    if (head[i]) {
      if (ext == 4 ? (sm_has(g, s, e, "@Ignore") || sm_has(g, s, e, "@Disabled")) : (ext != 1 && sm_has(g, s, e, "DISABLED_"))) b |= SL_HDR_IGN;
      tflag[case_of[i]] = sm_test_header(g, s, e, a0, a1, ext) ? 1u : 0u;
    }
    if (d.line_flag[i]) {
      b |= SL_ASSERT;
      unsigned long long hacc = 0; uint32_t hr = 0;     // Mersenne-61 of the stripped line (SPEC section 3, k_classify's recurrence)
      for (uint32_t q = a0; q < a1; ++q) {
        hacc = fold61(hacc + rotl61((unsigned long long)sm_byte(g, q), hr));
        hr += 8; if (hr >= 61) hr -= 61;
      }
      r.hash = mix_hash(canon61(hacc), a1 - a0);
      if (sm_redundant(g, a0, a1, fp, lp)) b |= SL_REDUNDANT;
    }
  }
  r.bits = b;
  out[i] = r;
}

struct SmellArgs {
  const unsigned long long* line_base; uint32_t n_files; const uint8_t* ext;
  const uint8_t* kind; const uint32_t* head; const uint32_t* first; uint32_t n_cases;
  const uint32_t* tflag; const unsigned long long* tidx; const SmellLine* L;
  unsigned long long* a_hash; uint32_t* a_line;             // [lines]: a test's assertion lines, packed from its header line on
  uint16_t* line_smell; tsm_smell_test* out;
};

__global__ void __launch_bounds__(256) k_smell_tests(SmellArgs a) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  const uint32_t lt = (1u << lane) - 1u, le = lt | (1u << lane);
  for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < a.n_cases; c += warps) {
    if (!a.tflag[c]) continue;
    const uint32_t b = a.first[c];
    uint32_t lo = 0, hi = a.n_files;                       // file of line b
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (a.line_base[mid] <= b) lo = mid; else hi = mid; }
    const uint32_t fb = (uint32_t)a.line_base[lo], fe = (uint32_t)a.line_base[lo + 1];
    const uint32_t e = c + 1 < a.n_cases && a.first[c + 1] < fe ? a.first[c + 1] : fe;
    const bool py = a.ext[lo] == 1;
    uint32_t hs = e;                                       // end of the header statement: the first line after b not of kind 2
    for (uint32_t base = b + 1; base < e; base += 32) {
      const uint32_t l = base + lane;
      const uint32_t m = __ballot_sync(0xffffffffu, l < e && a.kind[l] != 2);
      if (m) { hs = base + __ffs(m) - 1; break; }
    }
    uint32_t bend = e;
    if (py) {
      const uint32_t ind = a.L[b].indent;
      for (uint32_t base = hs; base < e; base += 32) {
        const uint32_t l = base + lane;
        bool p = false;
        if (l < e) { const SmellLine& r = a.L[l]; p = a.kind[l] == 1 && !(r.bits & SL_COMMENT) && r.indent <= ind; }
        const uint32_t m = __ballot_sync(0xffffffffu, p);
        if (m) { bend = base + __ffs(m) - 1; break; }
      }
    } else {
      long long run = 0;
      bool opened = false;
      for (uint32_t base = b; base < e; base += 32) {
        const uint32_t l = base + lane;
        long long v = 0;
        bool op = false;
        if (l < e) { v = a.L[l].brace; op = (a.L[l].bits & SL_OPEN) != 0; }
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
          const long long u = __shfl_up_sync(0xffffffffu, v, k);
          if (lane >= (uint32_t)k) v += u;
        }
        const uint32_t om = __ballot_sync(0xffffffffu, op);
        const bool o = opened || (om & le);
        const uint32_t m = __ballot_sync(0xffffffffu, l < e && o && run + v <= 0);
        if (m) { bend = base + __ffs(m); break; }
        run += __shfl_sync(0xffffffffu, v, 31);
        opened = opened || om;
      }
    }
    const uint32_t hend = min(hs, bend);
    uint32_t na = 0, ninst = 0, smells = 0, dqc = 0, sqc = 0;
    bool notempty = false;
    for (uint32_t base = b; base < bend; base += 32) {
      const uint32_t l = base + lane;
      const bool valid = l < bend, inbody = valid && l >= hend;
      const uint32_t bits = valid ? a.L[l].bits : 0;
      const uint32_t dm = __ballot_sync(0xffffffffu, inbody && (bits & SL_DQ)), sm = __ballot_sync(0xffffffffu, inbody && (bits & SL_SQ));
      const bool doc = py && ((bits & SL_DOCSTART) || ((dqc + __popc(dm & lt)) & 1) || ((sqc + __popc(sm & lt)) & 1));
      dqc += __popc(dm); sqc += __popc(sm);
      const bool code = inbody && !(bits & (SL_BLANK | SL_COMMENT)) && !doc;
      const bool isa = (bits & SL_ASSERT) && (code || (valid && l < hend));
      uint32_t ls = 0;
      if (isa && (bits & SL_REDUNDANT)) ls |= SM_REDUNDANT;
      if (code) {
        if (bits & SL_COND) ls |= SM_COND;
        if (bits & SL_EXC) ls |= SM_EXC;
        if (bits & SL_SLEEP) ls |= SM_SLEEP;
        if (bits & SL_PRINT) ls |= SM_PRINT;
        if (py && (bits & SL_SKIPCALL)) ls |= SM_IGNORED;
      }
      if (__any_sync(0xffffffffu, code && !(bits & SL_EMPTYOK))) notempty = true;
      const uint32_t am = __ballot_sync(0xffffffffu, isa);
      if (isa) {
        const uint32_t slot = b + na + __popc(am & lt);
        a.a_hash[slot] = a.L[l].hash;
        a.a_line[slot] = l;
      }
      na += __popc(am);
      if (valid) a.line_smell[l] = (uint16_t)ls;
      ninst += __reduce_add_sync(0xffffffffu, __popc(ls));
      smells |= __reduce_or_sync(0xffffffffu, ls);
    }
    __syncwarp();
    uint32_t ndup = 0;
    for (uint32_t t0 = 0; t0 < na; t0 += 32) {             // tile of assertion lines t0 .. t0 + 31 against all earlier ones
      const uint32_t idx = t0 + lane;
      const bool have = idx < na;
      const unsigned long long h = have ? a.a_hash[b + idx] : 0ull;
      bool dup = false;
      for (uint32_t p0 = 0; p0 < t0; p0 += 32) {
        const unsigned long long hp = a.a_hash[b + p0 + lane];
#pragma unroll 8
        for (int k = 0; k < 32; ++k) dup |= __shfl_sync(0xffffffffu, hp, k) == h;
      }
#pragma unroll 8
      for (int k = 0; k < 32; ++k) {                        // (every lane shuffles: the shuffle is not behind the lane test)
        const unsigned long long x = __shfl_sync(0xffffffffu, h, k);
        dup |= (uint32_t)k < lane && x == h;
      }
      dup = dup && have;
      if (dup) { const uint32_t l = a.a_line[b + idx]; a.line_smell[l] = (uint16_t)(a.line_smell[l] | SM_DUP); }
      ndup += __popc(__ballot_sync(0xffffffffu, dup));
    }
    __syncwarp();
    if (lane == 0) {
      const uint32_t ext = a.ext[lo];
      bool ign = ext != 1 && (a.L[b].bits & SL_HDR_IGN);
      for (uint32_t q = b; q > fb && !a.head[q - 1] && (a.L[q - 1].bits & SL_AT); --q)
        if (a.L[q - 1].bits & SL_DECO_IGN) ign = true;
      uint32_t hb = ign ? SM_IGNORED : 0;
      if (na == 0) hb |= SM_FREE | (notempty ? 0 : SM_EMPTY);
      a.line_smell[b] = (uint16_t)(a.line_smell[b] | hb);
      smells |= hb | (ndup ? SM_DUP : 0);
      a.out[a.tidx[c]] = tsm_smell_test{(int32_t)lo, (int32_t)(b - fb), (int32_t)(bend - b), (int32_t)na, smells,
                                        (int32_t)(ninst + ndup + __popc(hb))};
    }
  }
}

// Smell churn of one side of the revision pairs (docs/SPEC.md section 19).  mark / rank: this side's edit marks and kept ranks;
// other_smell / other_by_rank: the line_smell of the other side and its kept line of every rank.
struct ChurnSide {
  const unsigned long long* line_base; const tsm_smell_test* tests; uint32_t n_tests;
  const uint16_t* line_smell; const uint8_t* mark; const unsigned long long* rank; const unsigned long long* case_of;
  const uint16_t* other_smell; const uint32_t* other_by_rank; tsm_test_churn* out;
};

// The lexical smells of one side (docs/SPEC.md section 26): its line_lsmell, the other side's, and one record per test.
struct LexChurnSide { const uint8_t* line_lsmell; const uint8_t* other_lsmell; tsm_lex_churn* out; };

// Persistent warps, one test at a time, 32 body lines per round: the instances of a line are its smell bits, its churned
// instances the bits the corresponding line of the other side lacks (all of them on a deleted or inserted line).  Lane k < 9
// counts smell k from one ballot per smell and kind.  kLex: the line's TSM_LSMELL_* bits join above the nine (bit 9 + k),
// looked up through the same kept rank, and lanes 9..13 count them into x.out (x is unused otherwise).
template <bool kLex>
__global__ void __launch_bounds__(256) k_smell_churn(ChurnSide s, LexChurnSide x) {
  constexpr uint32_t K = kLex ? TSM_N_SMELLS + TSM_N_LSMELLS : TSM_N_SMELLS;
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < s.n_tests; t += warps) {
    const tsm_smell_test r = s.tests[t];
    const uint32_t b = (uint32_t)s.line_base[r.file] + (uint32_t)r.line, e = b + (uint32_t)r.body_lines;
    uint32_t ni = 0, nc = 0;
    for (uint32_t base = b; base < e; base += 32) {
      const uint32_t l = base + lane;
      uint32_t bits = 0, churn = 0;
      if constexpr (!kLex) {
        if (l < e && (bits = s.line_smell[l]) != 0)
          churn = s.mark[l] ? bits : bits & ~(uint32_t)s.other_smell[s.other_by_rank[s.rank[l]]];
      } else if (l < e && (bits = s.line_smell[l] | (uint32_t)x.line_lsmell[l] << TSM_N_SMELLS) != 0) {
        if (s.mark[l]) {
          churn = bits;
        } else {
          const uint32_t m = s.other_by_rank[s.rank[l]];
          churn = bits & ~(s.other_smell[m] | (uint32_t)x.other_lsmell[m] << TSM_N_SMELLS);
        }
      }
#pragma unroll
      for (uint32_t k = 0; k < K; ++k) {
        const uint32_t mi = __ballot_sync(0xffffffffu, (bits >> k) & 1u), mc = __ballot_sync(0xffffffffu, (churn >> k) & 1u);
        if (lane == k) { ni += __popc(mi); nc += __popc(mc); }
      }
    }
    tsm_test_churn* o = s.out + t;
    if (lane == 0) o->case_idx = (int32_t)s.case_of[b];
    if (lane < TSM_N_SMELLS) { o->instances[lane] = (int32_t)ni; o->churned[lane] = (int32_t)nc; }
    if constexpr (kLex)
      if (lane >= TSM_N_SMELLS && lane < K) {
        x.out[t].instances[lane - TSM_N_SMELLS] = (int32_t)ni;
        x.out[t].churned[lane - TSM_N_SMELLS] = (int32_t)nc;
      }
  }
}

}  // namespace tsm
