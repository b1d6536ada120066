// tsm_link_kernels.cuh - test-to-code links (docs/SPEC.md section 27): the production functions and classes each section-18 test
// of a test file calls, resolved by name within its repository, from the tests of the smell stage (tsm_smell_kernels.cuh), the
// code lines of k_lex_body (tsm_lexsmell_kernels.cuh) and the lexer states of the blind front (tsm_blind_kernels.cuh).  Lines
// are global indices (< 2^32).
//
//   k_link_pick   one thread per test of the smell stage: 1 for a test of a test file (role != 0); an xscan numbers them and
//                 k_link_gather copies them to the dense test list that the kernels below index.
//   k_link_mark   one warp per test: ltest[l] = the test of each of its code lines (else LK_NONE).
//   k_link_lines  one thread per line, lexing with blind_lex: on a production line the definition it holds (DefSink), on a test
//                 code line the calls (CallSink).  Count-then-write: the first pass counts, two xscans place definitions and
//                 calls in line order, the second pass (WRITE) hashes the names and writes the entries.
//   k_link_defs   one thread per definition: the name key (grp, name) and the focal key (grp, stem, name) into one open-addressing
//                 table of 16-B keys (128-bit atomicCAS, at most half full): count, kind mask and first definition (atomicMin).
//   k_link_calls  one thread per call: the name key is looked up; a defined name inserts the link key (test, name) into a second
//                 table (calls by atomicAdd, first call by atomicMin of the call's index), and a link's first insertion adds one
//                 to its (test file, name) key, to the name's linking tests and to the test's links.
//   k_link_first  one thread per call: 1 for the first call of its link.  Calls are numbered in line order and tests own
//                 disjoint line ranges in test order, so the xscan of these flags lists the links in (test, first call) order
//                 without a sort.
//   k_link_emit   one thread per first call: the link record, its target (the one definition, else the first focal one) and the
//                 target's tests and calls (atomicAdd).
//   k_link_tests  persistent warps, one test at a time: the counts over its links, Eager Test and Lazy Test.
//   k_link_out    one thread per definition: its record.
#pragma once
#include "tsm_device.cuh"
#include "tsm_blind_kernels.cuh"
#include "tsm_lexsmell_kernels.cuh"

namespace tsm {

constexpr uint32_t LK_NONE = 0xFFFFFFFFu;
constexpr uint32_t LK_FUNC = 1, LK_CLASS = 2;              // definition kinds, and the bits of a name's kind mask
constexpr uint32_t LK_EAGER = 1, LK_LAZY = 2;              // TSM_LINK_EAGER / TSM_LINK_LAZY
constexpr uint32_t LKB_FUNC = 1, LKB_FOCAL = 2, LKB_LAZY = 4;   // per-link facts that k_link_tests sums

struct __align__(16) LinkKey { unsigned long long hash, tag; };   // tag 0: an empty slot

// The name key of repository g, the focal key of its stem s (s >= 0), the link key of test t, the (test file f, name) key.
__device__ __forceinline__ unsigned long long lk_name_tag(uint32_t g) { return (unsigned long long)(g + 1) << 32; }
__device__ __forceinline__ unsigned long long lk_focal_tag(uint32_t g, int32_t s) { return lk_name_tag(g) | (uint32_t)(s + 1); }
__device__ __forceinline__ unsigned long long lk_link_tag(uint32_t t) { return (unsigned long long)t + 1; }
__device__ __forceinline__ unsigned long long lk_file_tag(uint32_t f) { return (1ull << 32) | (f + 1ull); }

__device__ __forceinline__ uint32_t lk_home(const LinkKey& k, uint32_t mask) {
  unsigned long long x = k.hash ^ (k.tag * 0x9E3779B97F4A7C15ull);
  x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ull; x ^= x >> 32;
  return (uint32_t)x & mask;
}
// The slot of k, claimed when absent (fresh: by this call).  A key, once set, never changes: the CAS's answer decides.
__device__ __forceinline__ uint32_t lk_insert(LinkKey* tab, uint32_t mask, const LinkKey& k, bool& fresh) {
  const LinkKey empty{0, 0};
  for (uint32_t s = lk_home(k, mask);; s = (s + 1) & mask) {
    const LinkKey was = atomicCAS(&tab[s], empty, k);
    if (was.tag == 0) { fresh = true; return s; }
    if (was.hash == k.hash && was.tag == k.tag) { fresh = false; return s; }
  }
}
// The slot of k, or LK_NONE; only in a launch behind every insertion of k's kind.
__device__ __forceinline__ uint32_t lk_find(const LinkKey* tab, uint32_t mask, const LinkKey& k) {
  for (uint32_t s = lk_home(k, mask);; s = (s + 1) & mask) {
    const LinkKey x = tab[s];
    if (x.tag == 0) return LK_NONE;
    if (x.hash == k.hash && x.tag == k.tag) return s;
  }
}

// bytes_hash (SPEC section 3) of the k bytes at i0.
__device__ __forceinline__ unsigned long long lk_hash(LineBytes& B, uint32_t i0, uint32_t k) {
  BlindHash h{0, 0, 0};
  for (uint32_t j = 0; j < k; ++j) h.byte(B.at(i0 + j));
  return mix_hash(canon61(h.acc), h.len);
}

// Token codes of the link sinks: a punctuation byte is itself.  LT_KWX: a keyword behind which no function is defined.
constexpr uint32_t LT_ID = 0x100, LT_KW = 0x101, LT_KWX = 0x102, LT_OTHER = 0x103;
__device__ __forceinline__ uint32_t lk_ident_code(const BlindKw* kw, const uint8_t* kind, uint32_t fam, const LxName& n) {
  const uint32_t kk = blind_kw_kind(kw, kind, n.lo, n.hi, n.k);
  if (kk & (fam == 1 ? KW_PY : KW_CJ)) {
    const bool x = lx_is(n, lx_name("return")) || lx_is(n, lx_name("new")) || lx_is(n, lx_name("delete")) ||
                   lx_is(n, lx_name("throw")) || lx_is(n, lx_name("else")) || lx_is(n, lx_name("case")) ||
                   lx_is(n, lx_name("goto")) || lx_is(n, lx_name("sizeof")) || lx_is(n, lx_name("typeid")) ||
                   lx_is(n, lx_name("alignof")) || lx_is(n, lx_name("decltype")) || lx_is(n, lx_name("co_return")) ||
                   lx_is(n, lx_name("co_yield")) || lx_is(n, lx_name("co_await"));
    return x ? LT_KWX : LT_KW;
  }
  return (kk & (fam == 1 ? KW_PY_LIT : KW_CJ_LIT)) ? LT_OTHER : LT_ID;
}

// The definition of one production line (section 27): result() gives its kind (0 none, LK_FUNC, LK_CLASS) and name bytes.
struct DefSink {
  const BlindKw* kw; const uint8_t* kind; uint32_t fam;
  // PY: 0 start, 1 after `async`, 2 after `def`, 3 after `class`, 4 function found, 6 class found, 5 none
  // CJ class rule: 0 modifiers, 1 after `enum`, 2 after a class keyword, 3 name (its next token pending), 4 found, 5 none
  uint32_t cst = 0, ci0 = 0, ck = 0;
  // CJ function rule: 0 searching, 1 an identifier at depth 0 (its next token pending), 2 decided (fok)
  uint32_t fst = 0, fi0 = 0, fk = 0, prev = 0, prev2 = 0, iprev = 0, iprev2 = 0, last = 0;
  int32_t depth = 0;
  bool eq = false, ieq = false, fok = false;

  __device__ __forceinline__ void tok(uint32_t t, uint32_t i0, uint32_t k, const LxName& n) {
    const bool kwd = t == LT_KW || t == LT_KWX;
    if (fam == 1) {
      if (cst == 0 && kwd && lx_is(n, lx_name("async"))) cst = 1;
      else if (cst <= 1 && kwd && lx_is(n, lx_name("def"))) cst = 2;
      else if (cst == 0 && kwd && lx_is(n, lx_name("class"))) cst = 3;
      else if ((cst == 2 || cst == 3) && t == LT_ID) { ci0 = i0; ck = k; cst = cst == 2 ? 4u : 6u; }
      else if (cst < 4) cst = 5;
      return;
    }
    if (cst == 3) cst = t == ';' ? 5u : 4u;
    else if (cst < 3) {
      if (cst == 0 && kwd &&
          (lx_is(n, lx_name("public")) || lx_is(n, lx_name("protected")) || lx_is(n, lx_name("private")) ||
           lx_is(n, lx_name("static")) || lx_is(n, lx_name("final")) || lx_is(n, lx_name("abstract")) ||
           lx_is(n, lx_name("export")))) {
      } else if (cst == 0 && kwd && lx_is(n, lx_name("enum"))) cst = 1;
      else if (kwd && ((cst == 0 && (lx_is(n, lx_name("class")) || lx_is(n, lx_name("struct")) || lx_is(n, lx_name("interface")))) ||
                       (cst == 1 && (lx_is(n, lx_name("class")) || lx_is(n, lx_name("struct"))))))
        cst = 2;
      else if ((cst == 1 || cst == 2) && t == LT_ID) { cst = 3; ci0 = i0; ck = k; }
      else cst = 5;
    }
    if (fst == 1) {
      if (t == '(') {
        fst = 2;
        fok = !ieq && (iprev == LT_ID || iprev == LT_KW || iprev == '*' || iprev == '&' || iprev == '>' ||
                       (iprev == ':' && iprev2 == ':'));
      } else fst = 0;
    }
    if (fst == 0 && t == LT_ID && depth == 0) { fst = 1; fi0 = i0; fk = k; iprev = prev; iprev2 = prev2; ieq = eq; }
    if (t == '(' || t == '[' || t == '{') ++depth;
    else if (t == ')' || t == ']' || t == '}') --depth;
    eq = eq || t == '=';
    prev2 = prev; prev = t; last = t;
  }
  __device__ __forceinline__ void number() { tok(LT_OTHER, 0, 0, LxName{0, 0, 0}); }
  __device__ __forceinline__ void string() { tok(LT_OTHER, 0, 0, LxName{0, 0, 0}); }
  __device__ __forceinline__ void punct(uint32_t c) { tok(c, 0, 0, LxName{0, 0, 0}); }
  __device__ __forceinline__ void ident(LineBytes&, uint32_t, uint32_t i0, uint32_t k, unsigned long long lo, unsigned long long hi) {
    const LxName n{lo, hi, k};
    tok(lk_ident_code(kw, kind, fam, n), i0, k, n);
  }
  // after the line's last token
  __device__ __forceinline__ uint32_t result(uint32_t& i0, uint32_t& k) const {
    if (fam == 1) {
      if (cst != 4 && cst != 6) return 0;
      i0 = ci0; k = ck;
      return cst == 4 ? LK_FUNC : LK_CLASS;
    }
    if (cst == 3 || cst == 4) { i0 = ci0; k = ck; return LK_CLASS; }
    if (fst == 2 && fok && last != ';') { i0 = fi0; k = fk; return LK_FUNC; }
    return 0;
  }
};

struct LinkDef { unsigned long long key; uint32_t line, file, off, len, kind, pad; };   // a definition: name hash, global line
struct LinkCall { unsigned long long key; uint32_t line, pos; };                        // a call: name hash, global line, byte

// The calls of one test code line (section 27): an identifier whose next token on the line is `(`, not behind PY `def` or
// `class`.  WRITE: each call's name hash, line and byte into out[n].
template <bool WRITE>
struct CallSink {
  const BlindKw* kw; const uint8_t* kind; uint32_t fam;
  LineBytes* B; LinkCall* out; uint32_t line;
  uint32_t n = 0, pi0 = 0, pk = 0;
  bool pend = false, defkw = false;
  __device__ __forceinline__ void tok(uint32_t t) {
    if (pend && t == '(') {
      if (WRITE) out[n] = LinkCall{lk_hash(*B, pi0, pk), line, pi0};
      ++n;
    }
    pend = false;
  }
  __device__ __forceinline__ void number() { tok(LT_OTHER); defkw = false; }
  __device__ __forceinline__ void string() { tok(LT_OTHER); defkw = false; }
  __device__ __forceinline__ void punct(uint32_t c) { tok(c); defkw = false; }
  __device__ __forceinline__ void ident(LineBytes&, uint32_t, uint32_t i0, uint32_t k, unsigned long long lo, unsigned long long hi) {
    const LxName nm{lo, hi, k};
    const uint32_t t = lk_ident_code(kw, kind, fam, nm);
    tok(t);
    if (t == LT_ID && !defkw) { pend = true; pi0 = i0; pk = k; }
    defkw = fam == 1 && t == LT_KW && (lx_is(nm, lx_name("def")) || lx_is(nm, lx_name("class")));
  }
};

__global__ void __launch_bounds__(256) k_link_pick(const tsm_smell_test* tests, uint32_t nt, const uint8_t* role, uint32_t* flag) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nt) flag[t] = role[tests[t].file] != 0;
}

__global__ void __launch_bounds__(256) k_link_gather(const tsm_smell_test* tests, uint32_t nt, const uint32_t* flag,
                                                     const unsigned long long* pos, tsm_smell_test* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nt && flag[t]) out[pos[t]] = tests[t];
}

__global__ void __launch_bounds__(256) k_link_mark(const tsm_smell_test* tests, uint32_t nt, const unsigned long long* line_base,
                                                   const uint8_t* lx_flag, uint32_t* ltest) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < nt; t += warps) {
    const tsm_smell_test r = tests[t];
    const uint32_t b = (uint32_t)line_base[r.file] + (uint32_t)r.line, bend = b + (uint32_t)r.body_lines;
    for (uint32_t l = b + lane; l < bend; l += 32)
      if (lx_flag[l] & LB_CODE) ltest[l] = t;
  }
}

// Count pass (WRITE false): dcnt / ccnt of every line (a test code line holds calls only, a production line at most one
// definition).  Write pass: the entries at dbase / cbase.
template <bool WRITE>
__global__ void __launch_bounds__(256) k_link_lines(DiffSide d, uint32_t n, unsigned long long total, const uint8_t* state,
                                                    const uint8_t* role, const uint32_t* ltest, uint32_t* dcnt, uint32_t* ccnt,
                                                    const unsigned long long* dbase, const unsigned long long* cbase,
                                                    LinkDef* defs, LinkCall* calls) {
  __shared__ BlindKw kw[BLIND_KW_SLOTS];
  __shared__ uint8_t kind[BLIND_KW_SLOTS];
  for (uint32_t t = threadIdx.x; t < BLIND_KW_SLOTS; t += blockDim.x) { kw[t] = c_blind_kw[t]; kind[t] = c_blind_kind[t]; }
  __syncthreads();
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const bool test_line = ltest[i] != LK_NONE;
  if (WRITE && (test_line ? ccnt[i] : dcnt[i]) == 0) return;
  const uint32_t f = blind_file(d.line_base, n, i), fam = blind_family(d.ext[f]);
  if (!WRITE && (fam == 0 || (!test_line && role[f]))) { dcnt[i] = 0; ccnt[i] = 0; return; }
  const uint8_t* g = d.arena + (uint32_t)d.off[f];
  const uint32_t fb = (uint32_t)d.line_base[f];
  const uint32_t s = i == fb ? 0u : d.line_end[i - 1] + 1u, e = d.line_end[i];
  LineBytes B{g, 1u, 0};
  if (test_line) {
    CallSink<WRITE> cs{kw, kind, fam, &B, WRITE ? calls + cbase[i] : nullptr, (uint32_t)i};
    blind_lex(B, s, e, fam, state[i], cs);
    if (!WRITE) { ccnt[i] = cs.n; dcnt[i] = 0; }
    return;
  }
  DefSink ds{kw, kind, fam};
  blind_lex(B, s, e, fam, state[i], ds);
  uint32_t i0 = 0, k = 0;
  const uint32_t kd = ds.result(i0, k);
  if (!WRITE) { dcnt[i] = kd ? 1u : 0u; ccnt[i] = 0; return; }
  defs[dbase[i]] = LinkDef{lk_hash(B, i0, k), (uint32_t)i, f, i0, k, kd, 0};
}

struct LinkTables {
  LinkKey* name; uint32_t name_mask;                       // name and focal keys
  uint32_t* n_defs; uint32_t* kmask; uint32_t* first;      // per slot of `name`: definitions, kind mask, first definition
  uint32_t* n_tests;                                       //   tests linking the name (name keys)
  LinkKey* link; uint32_t link_mask;                       // link and (test file, name) keys
  uint32_t* calls; uint32_t* first_call;                   // per slot of `link`: calls and first call (link keys), tests
                                                           //   (in calls) of the (test file, name) keys
};

__global__ void __launch_bounds__(256) k_link_defs(const LinkDef* defs, uint32_t nd, const uint16_t* grp, const int32_t* stem,
                                                   LinkTables T, uint32_t* dslot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nd) return;
  const LinkDef df = defs[i];
  const uint32_t g = grp[df.file];
  bool fresh;
  const uint32_t s = lk_insert(T.name, T.name_mask, LinkKey{df.key, lk_name_tag(g)}, fresh);
  atomicAdd(&T.n_defs[s], 1u);
  atomicOr(&T.kmask[s], df.kind);
  atomicMin(&T.first[s], i);
  dslot[i] = s;
  const int32_t st = stem[df.file];
  if (st >= 0) atomicMin(&T.first[lk_insert(T.name, T.name_mask, LinkKey{df.key, lk_focal_tag(g, st)}, fresh)], i);
}

__global__ void __launch_bounds__(256) k_link_calls(const LinkCall* calls, uint32_t nc, const uint32_t* ltest, const tsm_smell_test* tests,
                                                    const uint16_t* grp, LinkTables T, uint32_t* cslot, uint32_t* tlinks) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  const LinkCall c = calls[i];
  const uint32_t t = ltest[c.line], f = (uint32_t)tests[t].file;
  const uint32_t ns = lk_find(T.name, T.name_mask, LinkKey{c.key, lk_name_tag(grp[f])});
  uint32_t ls = LK_NONE;
  if (ns != LK_NONE) {
    bool fresh;
    ls = lk_insert(T.link, T.link_mask, LinkKey{ns, lk_link_tag(t)}, fresh);
    atomicAdd(&T.calls[ls], 1u);
    atomicMin(&T.first_call[ls], i);
    if (fresh) {
      atomicAdd(&T.calls[lk_insert(T.link, T.link_mask, LinkKey{ns, lk_file_tag(f)}, fresh)], 1u);
      atomicAdd(&T.n_tests[ns], 1u);
      atomicAdd(&tlinks[t], 1u);
    }
  }
  cslot[i] = ls;
}

__global__ void __launch_bounds__(256) k_link_first(const uint32_t* cslot, uint32_t nc, LinkTables T, uint32_t* flag) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  const uint32_t ls = cslot[i];
  flag[i] = ls != LK_NONE && T.first_call[ls] == i;
}

struct LinkEmit {
  const LinkCall* calls; uint32_t nc; const uint32_t* cslot; const uint32_t* flag; const unsigned long long* lpos;
  const uint32_t* ltest; const tsm_smell_test* tests; const uint16_t* grp; const int32_t* stem; const unsigned long long* line_base;
  const LinkDef* defs; LinkTables T;
  tsm_link* links; uint8_t* lbits; uint32_t* dtests; uint32_t* dcalls;
};

__global__ void __launch_bounds__(256) k_link_emit(LinkEmit a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.nc || !a.flag[i]) return;
  const LinkCall c = a.calls[i];
  const uint32_t ls = a.cslot[i], ns = (uint32_t)a.T.link[ls].hash, t = a.ltest[c.line], f = (uint32_t)a.tests[t].file;
  const uint32_t nd = a.T.n_defs[ns], first = a.T.first[ns], calls = a.T.calls[ls];
  const int32_t st = a.stem[f];
  const uint32_t fs = st >= 0 ? lk_find(a.T.name, a.T.name_mask, LinkKey{a.T.name[ns].hash, lk_focal_tag(a.grp[f], st)}) : LK_NONE;
  const uint32_t target = nd == 1 ? first : fs != LK_NONE ? a.T.first[fs] : LK_NONE;
  const bool func = a.T.kmask[ns] & LK_FUNC;
  const uint32_t fc = a.T.calls[lk_find(a.T.link, a.T.link_mask, LinkKey{ns, lk_file_tag(f)})];
  const unsigned long long p = a.lpos[i];
  a.links[p] = tsm_link{(int32_t)t, (int32_t)first, (int32_t)target, (int32_t)nd, (int32_t)calls,
                        (int32_t)(c.line - (uint32_t)a.line_base[f]), (int32_t)c.pos};
  a.lbits[p] = (uint8_t)((func ? LKB_FUNC : 0) | (fs != LK_NONE ? LKB_FOCAL : 0) | (func && fc >= 2 ? LKB_LAZY : 0));
  if (target != LK_NONE) {
    atomicAdd(&a.dtests[target], 1u);
    atomicAdd(&a.dcalls[target], calls);
  }
}

struct LinkTests {
  const tsm_smell_test* tests; uint32_t nt; const unsigned long long* line_base; const unsigned long long* cbase;
  const unsigned long long* lbase;
  const tsm_link* links; const uint8_t* lbits; tsm_link_test* out;
};

__global__ void __launch_bounds__(256) k_link_tests(LinkTests a) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < a.nt; t += warps) {
    const unsigned long long b = a.lbase[t], e = a.lbase[t + 1];
    uint32_t linked = 0, nfunc = 0, nfocal = 0, lazy = 0;
    for (unsigned long long j = b + lane; j < e; j += 32) {
      const uint32_t x = a.lbits[j];
      linked += (uint32_t)a.links[j].calls;
      nfunc += (x & LKB_FUNC) != 0;
      nfocal += (x & LKB_FOCAL) != 0;
      lazy |= x & LKB_LAZY;
    }
    linked = __reduce_add_sync(0xffffffffu, linked);
    nfunc = __reduce_add_sync(0xffffffffu, nfunc);
    nfocal = __reduce_add_sync(0xffffffffu, nfocal);
    lazy = __reduce_or_sync(0xffffffffu, lazy);
    if (lane == 0) {
      const tsm_smell_test r = a.tests[t];
      const uint32_t lb = (uint32_t)a.line_base[r.file] + (uint32_t)r.line;   // (calls lie on the test's own code lines only)
      a.out[t] = tsm_link_test{r.file, r.line, (int32_t)(a.cbase[lb + (uint32_t)r.body_lines] - a.cbase[lb]), (int32_t)linked, (int32_t)(e - b), (int32_t)nfunc,
                               (int32_t)nfocal, (nfunc >= 2 ? LK_EAGER : 0u) | (lazy ? LK_LAZY : 0u)};
    }
  }
}

__global__ void __launch_bounds__(256) k_link_out(const LinkDef* defs, uint32_t nd, const uint32_t* dslot, const unsigned long long* line_base,
                                                  LinkTables T, const uint32_t* dtests, const uint32_t* dcalls, tsm_link_def* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nd) return;
  const LinkDef df = defs[i];
  out[i] = tsm_link_def{(int32_t)df.file, (int32_t)(df.line - (uint32_t)line_base[df.file]), (int32_t)df.off, (int32_t)df.len,
                        (int32_t)df.kind, (int32_t)dtests[i], (int32_t)T.n_tests[dslot[i]], (int32_t)dcalls[i]};
}

}  // namespace tsm
