// tsm_scan_walk.cuh - k_scan, THE hot kernel of the corpus scan (docs/SPEC.md sections 2-5, 7; DESIGN.md section 3): one warp
// per (file, 4 KiB chunk) work unit, the chunk staged global -> shared by one 1-D TMA bulk copy (cp.async.bulk + mbarrier),
// every source byte read from HBM exactly once.  Per chunk:
//
//   walk     every lane takes the 17 words of its own 136-byte stripe (all 32 lanes busy whatever the line lengths are):
//            multi-pattern Shift-And automaton, one LUT lookup per byte.  '\n' is one of its patterns (state bit 31), so the
//            OR of a word's eight states says for free whether the word holds a newline: there is no newline pass over every
//            byte.  The OR of the states since the last newline word stays in a REGISTER and is stored in front of every word
//            (one STS); the Mersenne-61 running hash prefix is checkpointed every 4 words;
//   mixed    a word that holds a newline AND a pattern end (a few per chunk) is re-walked byte by byte by a dense pass that
//            splits its states between the line that ends in it and the line that starts;
//   records  only the words that hold a newline (~ 1 in 5) are looked at again: a dense pass (one lane per such word, SWAR
//            for the newline bytes) turns them into one 16-bit record per LINE;
//   finish   one line per lane, no inner loops: one hash prefix per line (the one behind its newline; the one in front of
//            the line is the neighbour lane's), pattern flags from the word's stored OR, per-file counters, the candidate
//            (assertion line) list for k_classify; with TSM_SCAN_LINE_HASHES the line's record (hash, end, flag) as well.
//
// Table addresses are formed by IMAD (FMA pipe) instead of LEA (ALU pipe), and the walk is a rolled loop: the kernel is
// latency / issue bound and sensitive to its instruction-cache footprint (profiles/h100_variants.txt).  Where its cycles go:
// profiles/h100_phases.txt (the TSM_PHASE_CLOCKS build variant).
// There is no reference kernel: the reference ships data only (SURVEY.md section 0).  Rules cite docs/SPEC.md.
#pragma once
#include "tsm_scan_kernels.cuh"

namespace tsm {

#ifndef TSM_SCAN2_WARPS
#define TSM_SCAN2_WARPS 11
#endif
#ifndef TSM_SCAN2_CTAS
#define TSM_SCAN2_CTAS 2
#endif
#ifndef TSM_WALK_UNROLL
#define TSM_WALK_UNROLL 1         // H100: 1.5 % (C2) / 1.9 % (C4) less k_scan time than 2 (profiles/h100_variants.txt)
#endif
constexpr int SCAN2_WARPS = TSM_SCAN2_WARPS, SCAN2_CTAS_PER_SM = TSM_SCAN2_CTAS, WALK_UNROLL = TSM_WALK_UNROLL;

// ---- per-warp shared memory --------------------------------------------------------------------
constexpr uint32_t NWORD = BUF / 8;                      // 544 words of 8 bytes, 17 per stripe
constexpr uint32_t O2_ARUN = BUF;                        // u32[NWORD + 1]  OR of the states since the last newline word, in front of every word
constexpr uint32_t SLOT_TAIL = NWORD;                    //                 (+ one slot: the line that ends with the data)
constexpr uint32_t RW2_PER_STRIPE = 4;                   // hash-prefix checkpoint behind words 3, 7, 11 and 15 of every stripe
constexpr uint32_t O2_RW = O2_ARUN + ((NWORD + 1) * 4 + 7) / 8 * 8;   // u64[32 * RW2_PER_STRIPE]
constexpr uint32_t O2_WENT = O2_RW + 32 * RW2_PER_STRIPE * 8;         // u16[WENT_CAP]   newline words in order (bit 15: mixed)
constexpr uint32_t WENT_CAP = NWORD + 8;
constexpr uint32_t LCAP = 512;                           // line records per window
constexpr uint32_t O2_LTAB = O2_WENT + WENT_CAP * 2;     // u16[LCAP]       line records; consumed ones are reused for the candidate list
constexpr uint32_t O2_BASE = O2_LTAB + (LCAP + 8) * 2;   // u64[33]         hash prefix at every stripe start (+ total)
constexpr uint32_t Q2_CAP = 64;
constexpr uint32_t O2_Q = O2_BASE + 34 * 8;              // u16[Q2_CAP]     mixed words
constexpr uint32_t O2_CTL = O2_Q + Q2_CAP * 2;           // u32 queue length, u32 mbarrier phase, u64 mbarrier
constexpr uint32_t WARP_SMEM2 = ((O2_CTL + 16 + 127) / 128) * 128;
// Phase clocks: a build variant (-DTSM_PHASE_CLOCKS=1, read by tools/phase_clocks.py) in which lane 0 of every warp
// adds the SM-clock cycles of each phase of the chunk loop into a per-CTA table, flushed to g_scan_phase_clk at exit.
#ifndef TSM_PHASE_CLOCKS
#define TSM_PHASE_CLOCKS 0
#endif
enum ScanPhase { PH_WAIT, PH_ZERO, PH_WALK, PH_SCANS, PH_MIXED, PH_RECORDS, PH_FINISH, PH_LONG, PH_FLUSH, PH_N };
#if TSM_PHASE_CLOCKS
__device__ unsigned long long g_scan_phase_clk[PH_N];
#endif
struct PhaseClock {
#if TSM_PHASE_CLOCKS
  uint32_t* tab;                                         // per CTA, shared memory
  long long t;
  __device__ __forceinline__ void mark(int ph, int lane) {
    const long long now = clock64();
    if (lane == 0) atomicAdd(tab + ph, (uint32_t)(now - t));
    t = now;
  }
#else
  __device__ __forceinline__ void mark(int, int) {}
#endif
};

// per CTA in front of the warps: automaton table (1 KB), per-language masks + LutRef (128 B), rotations of '\n' (61 x 8 B)
// (+ the phase-clock table in that build variant)
constexpr uint32_t O2_T0A = LUT_BYTES;
constexpr uint32_t O2_PHASE = LUT_BYTES + 512;
constexpr uint32_t CTA_BYTES2 = LUT_BYTES + 512 + (TSM_PHASE_CLOCKS ? 128 : 0);
constexpr uint32_t SCAN2_SMEM = CTA_BYTES2 + SCAN2_WARPS * WARP_SMEM2;
constexpr uint32_t O2_LUTB = SCAN2_SMEM;                 // Rev-B trigger table (only the TSM_SCAN_REV_B instantiation): 256 x u32 behind the warps
constexpr uint32_t SCAN2_SMEM_B = SCAN2_SMEM + 1024;
static_assert(O2_RW % 8 == 0 && O2_WENT % 8 == 0 && O2_LTAB % 2 == 0 && O2_BASE % 8 == 0 && O2_Q % 4 == 0 && O2_CTL % 8 == 0, "alignment");
static_assert(SCAN2_CTAS_PER_SM * (SCAN2_SMEM_B + 1024) <= 233472, "shared memory per SM (228 KB, 1 KB reserved per CTA)");
// line record: bits 0..12 position of the line's end in the buffer, 13 = first newline of its word (the word's stored
// OR is the line's), 14 = the word is mixed, 15 = no newline: the unterminated last line of a file
constexpr uint32_t LR_POS = 0x1FFFu, LR_FIRST = 0x2000u, LR_MIXED = 0x4000u, LR_VIRT = 0x8000u;

// Rev-B triggers (docs/SPEC.md section 4b; second automaton word, only in the TSM_SCAN_REV_B instantiation):
//   bits 0..5 `_CHECK`   bits 6..14 `TESTEQUAL`   bits 15..18 `FAIL`
constexpr uint32_t B2_FIRST = (1u << 0) | (1u << 6) | (1u << 15), B2_FIN = (1u << 5) | (1u << 14) | (1u << 18);
constexpr uint32_t REVB_BIT = 1u;                        // in the stored ORs: bit 0 (a non-final state of `assert`) = "a Rev-B trigger ended"

// Table entry of byte `idx`.  The address is formed by an integer multiply-add whose factor (4) the compiler
// cannot see: IMAD runs on the FMA pipe, the LEA it replaces on the ALU pipe.  Both operands come from shared memory
// (LutRef, written by the kernel prologue), so the compiler keeps them in registers for the whole pass instead of
// forming the table address again for every word.
struct LutRef { uint32_t four, base; };                  // 4 (from a launch parameter) and the table's shared-window address
__device__ __forceinline__ LutRef lut_ref() { return LutRef{scan_lut()[256 + 12], scan_lut()[256 + 13]}; }
template <bool REVB>
__device__ __forceinline__ void lut_at(uint32_t idx, LutRef t, uint32_t& v, uint32_t& v2) {
  uint32_t addr;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(addr) : "r"(idx), "r"(t.four), "r"(t.base));
  asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  if (REVB) asm("ld.shared.u32 %0, [%1+%2];" : "=r"(v2) : "r"(addr), "n"(O2_LUTB));
}

struct Auto { uint32_t D, D2; };                         // automaton state (D2: the Rev-B word, unused otherwise)

// One automaton step; returns the states that count for the OR of a line (Rev-B: bit 0 = a Rev-B trigger ended).
template <bool REVB>
__device__ __forceinline__ uint32_t step1(Auto& a, uint32_t byte, LutRef t) {
  uint32_t m, m2 = 0;
  lut_at<REVB>(byte, t, m, m2);
  a.D = ((a.D + a.D) | B_FIRST) & m;
  if (!REVB) return a.D;
  a.D2 = ((a.D2 + a.D2) | B2_FIRST) & m2;
  return (a.D & ~REVB_BIT) | ((a.D2 & B2_FIN) ? REVB_BIT : 0u);
}

// Eight automaton steps over one 8-byte word; A collects every state of the word.
template <bool REVB>
__device__ __forceinline__ void step8b(unsigned long long w, Auto& a, uint32_t& A, LutRef t) {
  const uint32_t lo = (uint32_t)w, hi = (uint32_t)(w >> 32);
  uint32_t A2 = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    uint32_t m, m2 = 0;
    lut_at<REVB>(__byte_perm(k < 4 ? lo : hi, 0, 0x4440 + (k & 3)), t, m, m2);
    a.D = ((a.D + a.D) | B_FIRST) & m;
    A |= a.D;
    if (REVB) { a.D2 = ((a.D2 + a.D2) | B2_FIRST) & m2; A2 |= a.D2; }
  }
  if (REVB) A = (A & ~REVB_BIT) | ((A2 & B2_FIN) ? REVB_BIT : 0u);
}

__device__ __forceinline__ uint32_t nl8_of(unsigned long long w) {       // bit b = byte b of w is '\n'
  return nl_word((uint32_t)w) | (nl_word((uint32_t)(w >> 32)) << 4);
}
__device__ __forceinline__ unsigned long long low_mask(uint32_t b) {    // the b low bytes, b in 0..8
  return b >= 8u ? ~0ull : ((1ull << (8u * b)) - 1ull);
}
__device__ __forceinline__ unsigned long long ror3_61(unsigned long long r) { return (r >> 3) + ((r & 7ull) << 58); }

struct WalkOut { uint32_t nlw, tail; };                  // bit k: word k of the stripe holds a newline; states since the stripe's last newline word

// The walk: every lane takes the 17 words of its own 136-byte stripe (all 32 lanes busy whatever the line
// lengths are; the bytes outside the chunk's staged range are zeros).  Per word: 8 automaton steps, the
// Mersenne-61 running prefix R_k = R_{k-1} * 2^-64 + w_k, one store of the running OR.  Then one warp scan
// turns the stripe totals into the absolute hash prefix at every stripe start.
template <bool REVB>
__device__ __noinline__ WalkOut walk2(uint8_t* wb, uint32_t fin, int lane) {
  const uint32_t pos0 = (uint32_t)lane * STRIPE;
  const uint8_t* sp = wb + pos0;
  uint32_t* ar = reinterpret_cast<uint32_t*>(wb + O2_ARUN) + (uint32_t)lane * 17u;
  unsigned long long* rw = reinterpret_cast<unsigned long long*>(wb + O2_RW) + (uint32_t)lane * RW2_PER_STRIPE;
  const LutRef t = lut_ref();
  Auto au{0u, 0u};
  if (lane) {                                            // state in front of the stripe: no state looks back more than 8 bytes
    uint32_t A = 0;                                      // (the longest pattern, Rev B's TESTEQUAL, has 9)
    step8b<REVB>(*reinterpret_cast<const unsigned long long*>(sp - 8), au, A, t);
  }
  unsigned long long R = 0;
  uint32_t run = 0, nlr = 0;                             // nlr: newline-word bits, the newest word in bit 0
  auto word = [&](uint32_t k) {                          // word k of the stripe
    const unsigned long long w = *reinterpret_cast<const unsigned long long*>(sp + 8u * k);
    uint32_t A = 0;
    step8b<REVB>(w, au, A, t);
    R = ror3_61(R) + fold61(w);                          // lazily reduced: stays below 2^63
    ar[k] = run;
    nlr = __funnelshift_l(A, nlr, 1);                    // bit 31 of A: the word holds a newline
    const bool nl = (int32_t)A < 0;
    if (nl && (A & fin)) {                               // rare: a pattern ends in a newline word
      const uint32_t slot = atomicAdd(reinterpret_cast<uint32_t*>(wb + O2_CTL), 1u);
      if (slot < Q2_CAP) reinterpret_cast<uint16_t*>(wb + O2_Q)[slot] = (uint16_t)((uint32_t)lane * 17u + k);
    }
    run = nl ? 0u : (run | A);
  };
#pragma unroll 1
  for (uint32_t g = 0; g < 4; ++g) {
#pragma unroll WALK_UNROLL
    for (uint32_t k = 0; k < 4; ++k) word(4u * g + k);
    rw[g] = R;
  }
  word(16);                                              // (no checkpoint behind the 17th word)
  // stripe totals (frame of the stripe's last word) -> absolute frame -> exclusive scan
  unsigned long long incl = rotl61(canon61(R), (3u * (17u * (uint32_t)lane + 16u)) % 61u);
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl = fold61(incl + t);
  }
  unsigned long long excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = 0;
  unsigned long long* sbase = reinterpret_cast<unsigned long long*>(wb + O2_BASE);
  sbase[lane] = excl;
  if (lane == 31) sbase[32] = incl;
  return WalkOut{__brev(nlr) >> 15, run};
}

// A mixed word (newline + pattern end), byte by byte: the states in front of its first newline belong to the
// line that ends there (word entry i), the states behind its last newline to the line that ends at the next
// entry.  Lines inside the word are walked by the finish pass itself (LR_MIXED asks for it).
template <bool REVB>
__device__ __noinline__ void resolve_mixed(uint8_t* wb, uint32_t g, uint32_t i, uint32_t n_went) {
  const LutRef t = lut_ref();
  Auto au{0u, 0u};
  uint32_t A = 0;
  step8b<REVB>(*reinterpret_cast<const unsigned long long*>(wb + 8u * g - 8u), au, A, t);   // g >= 2: the first 16 bytes are zeros
  unsigned long long w = *reinterpret_cast<const unsigned long long*>(wb + 8u * g);
  uint32_t pre = 0, post = 0, seen = 0;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const uint32_t d = step1<REVB>(au, (uint32_t)w & 0xFFu, t);
    const uint32_t m = (uint32_t)((int32_t)au.D >> 31);  // all ones at a newline
    pre |= d & ~seen;
    seen |= m;
    post = (post | d) & ~m;
    w >>= 8;
  }
  uint32_t* arun = reinterpret_cast<uint32_t*>(wb + O2_ARUN);
  const uint16_t* went = reinterpret_cast<const uint16_t*>(wb + O2_WENT);
  atomicOr(arun + g, pre);
  const uint32_t tgt = i + 1u < n_went ? ((uint32_t)went[i + 1u] & 0x3FFu) : SLOT_TAIL;
  atomicOr(arun + tgt, post);
}

__device__ __forceinline__ void emit_header(const ScanParams& p, uint32_t f, uint32_t line_off, uint32_t len, uint32_t fl) {
  const uint32_t slot = atomicAdd(&p.ctrl->n_hev, 1u);
  if (slot < p.hev_cap) p.hev[slot] = tsm_header_event{f, line_off, len, (fl >> 2) & 1u};
  else p.ctrl->overflow = 1;
}

// Does the stripped line [s, e) start with the n <= 7 bytes of `pat` (little-endian in a u64)?  With need_ws the
// byte behind them must be a blank that lies inside the stripped line (SPEC section 5, `class`).
template <typename Bytes>
__device__ __noinline__ bool starts_with8(Bytes lb, uint32_t s, uint32_t e, unsigned long long pat, uint32_t n, bool need_ws) {
  uint32_t r;
  while (s + 8 <= e && (r = lb.spaces8(s)) != 0) { s += r; if (r < 8) break; }
  while (s < e && is_w(lb(s))) ++s;
  if (s + n + (need_ws ? 1u : 0u) > e) return false;
  const unsigned long long v = lb.load8(s);              // readable 8 bytes past any line (SmemByte, HbmByte)
  if ((v & low_mask(n)) != pat) return false;
  if (need_ws) {
    const uint32_t c = (uint32_t)(v >> (8u * n)) & 0xFFu;
    if (c != 0x20 && c != 0x09) return false;
    for (uint32_t q = s + n + 1; q < e; ++q)
      if (!is_w(lb(q))) return true;
    return false;
  }
  return true;
}

// Flags of a finished line (SPEC sections 4 / 5) from the OR of its automaton states; adds it to the per-file counters.
template <bool REVB, typename Bytes>
__device__ __forceinline__ uint32_t line_flags2(uint32_t s, uint32_t e, uint32_t A, uint32_t g1, uint32_t g2, int ext, Bytes lb, Accum& ac) {
  if (ext == 0) return 0;
  uint32_t fl = (A & (AF_ASSERT | AF_EXPECT | (REVB ? REVB_BIT : 0u))) ? LF_CAND : 0;
  bool hdr;
  if (ext == TSM_EXT_PY) {
    hdr = (A & g1) != 0;
    if (!hdr && (A & g2)) hdr = starts_with8(lb, s, e, 0x7373616C63ull, 5, true);           // "class" + blank
  } else {
    hdr = (A & g1) != 0 && (A & g2) != 0;
  }
  if (hdr) { fl |= LF_HDR; if ((A & B_F) && starts_with8(lb, s, e, 0x465F54534554ull, 6, false)) fl |= LF_FIX; }   // "TEST_F"
  ac.asserts += fl & LF_CAND;
  ac.hdrs += (fl >> 1) & 1u;
  ac.fixes += (fl >> 2) & 1u;
  return fl;
}

struct FinishState {                                     // carried from one window of line records to the next (by value: no local memory)
  Accum ac;                                              // the chunk's per-file counters
  uint32_t prev_last;                                    // newline in front of the next line
  unsigned long long prevP;                              // hash prefix of the bytes [0, prev_last]
  uint32_t lh_base, lh_done;                             // TSM_SCAN_LINE_HASHES: the chunk's region of the staging arrays, records written
};

// Finish pass over the n line records of the window: one lane per line, no inner loops.  The hash of a line is
// the difference of two prefixes: the one behind its own newline minus the newline byte, and the one behind the
// newline in front of it, which is the neighbour lane's.  A line belongs to the chunk its first byte lies in
// (start < lim).  The starts of the assertion lines are compacted (u16 each) over the records already consumed
// and go to the global candidate list at the end of the window.
template <bool REVB>
__device__ __noinline__ FinishState finish_lines2(const ScanParams& p, uint8_t* wb, const uint32_t* lc, uint32_t n, uint32_t lim,
                                                  bool skip_first, uint32_t f, uint32_t cb, int ext, int lane, FinishState fs) {
  uint16_t* ltab = reinterpret_cast<uint16_t*>(wb + O2_LTAB);
  const uint32_t* arun = reinterpret_cast<const uint32_t*>(wb + O2_ARUN);
  const unsigned long long* t0a = reinterpret_cast<const unsigned long long*>(scan_lut()) + O2_T0A / 8;
  const uint32_t g1 = lc[1], g2 = lc[2];
  const SmemByte lb{wb};
  const bool want_hev = (p.flags & TSM_SCAN_HEADER_EVENTS) != 0, want_lh = (p.flags & TSM_SCAN_LINE_HASHES) != 0;
  Accum a = fs.ac;
  uint32_t nc = 0, lh_done = fs.lh_done;
  uint32_t prev_last = fs.prev_last;
  unsigned long long prevP = fs.prevP;
  for (uint32_t base = 0; base < n; base += 32) {        // uniform trip count
    const uint32_t j = base + (uint32_t)lane;
    const bool valid = j < n;
    const uint32_t rec = valid ? (uint32_t)ltab[j] : 0u;
    const uint32_t e = rec & LR_POS;
    const bool isv = (rec & LR_VIRT) != 0;
    const uint32_t g = min(e >> 3, NWORD - 1u), b1 = e - 8u * g + (isv ? 0u : 1u);   // bytes of word g up to and including the newline
    // ---- Pn: hash prefix of the bytes [0, e] (SPEC section 3; lazily reduced, < 2^62 + 8)
    const uint32_t l = g / 17u, i = g - 17u * l, c0 = i >> 2, ns = i & 3u;
    unsigned long long R = 0;
    if (c0) R = *reinterpret_cast<const unsigned long long*>(wb + O2_RW + 8u * (l * RW2_PER_STRIPE + c0 - 1u));
    const unsigned long long* wp = reinterpret_cast<const unsigned long long*>(wb) + (g - ns);   // words since the checkpoint
#pragma unroll
    for (uint32_t t = 0; t < 3u; ++t)
      if (ns > t) R = ror3_61(R) + fold61(wp[t]);
    const unsigned long long w = *reinterpret_cast<const unsigned long long*>(wb + 8u * g);
    const uint32_t r3g = (3u * g) % 61u;
    const unsigned long long X = ror3_61(R) + fold61(w & low_mask(b1));
    unsigned long long Pn = *reinterpret_cast<const unsigned long long*>(wb + O2_BASE + 8u * l) + rotl61(fold61(fold61(X)), r3g);
    // ---- Pe: the same without the newline byte
    uint32_t r8e = r3g + 8u * (e & 7u);
    if (r8e >= 61u) r8e -= 61u;
    const unsigned long long Pe = isv ? Pn : Pn + M61 - t0a[r8e];
    uint32_t s = __shfl_up_sync(0xffffffffu, e, 1) + 1u;
    unsigned long long Ps = __shfl_up_sync(0xffffffffu, Pn, 1);
    if (lane == 0) { s = prev_last + 1u; Ps = prevP; }
    const int src = base + 32u <= n ? 31 : (int)(n - 1u - base);         // the round's last record
    prev_last = __shfl_sync(0xffffffffu, e, src);
    prevP = __shfl_sync(0xffffffffu, Pn, src);
    const bool owned = valid && s < lim && !(s == PRE && skip_first);
    uint32_t fl = 0;
    unsigned long long lh = 0;
    if (owned) {
      const unsigned long long hr = canon61(Pe + 4ull * M61 - Ps);       // bytes [s, e), weighted from position 0
      const uint32_t sh = (8u * s) % 61u;
      unsigned long long h = rotl61(hr, sh ? 61u - sh : 0u);
      uint32_t len = e - s;
      if (len && lb(e - 1u) == 0x0D) {                   // drop one trailing CR: subtract 0x0D * 256^(len-1)
        --len;
        const unsigned long long cr = rotl61(0x0Dull, (8u * len) % 61u);
        h = h >= cr ? h - cr : h + M61 - cr;
      }
      a.lines++;
      lh = mix_hash(h, len);
      a.digest += lh;
      uint32_t A = 0;
      if (rec & LR_FIRST) A = arun[isv ? SLOT_TAIL : g];
      else if (rec & LR_MIXED) {                         // a line inside a mixed word: its own states
        Auto au{0u, 0u};
        const LutRef t = lut_ref();
        for (uint32_t q = s; q < e; ++q) A |= step1<REVB>(au, lb(q), t);
      }
      fl = line_flags2<REVB>(s, e, A, g1, g2, ext, lb, a);
      if (want_hev && (fl & LF_HDR)) emit_header(p, f, cb + s - PRE, e - s, fl);
    }
    if (want_lh) {                                       // the line's record, in line order inside the chunk's region
      const uint32_t mo = __ballot_sync(0xffffffffu, owned);
      const uint32_t slot = fs.lh_base + lh_done + __popc(mo & ((1u << lane) - 1u));
      if (owned && slot < p.lh_cap) {
        p.lh_hash[slot] = lh;
        p.lh_end[slot] = cb + e - PRE;
        p.lh_flag[slot] = (uint8_t)(fl & LF_CAND);
      }
      lh_done += __popc(mo);
    }
    __syncwarp();                                        // every record of the round is read: the list may grow over them
    const uint32_t mc = __ballot_sync(0xffffffffu, fl & LF_CAND);
    if (fl & LF_CAND) ltab[nc + __popc(mc & ((1u << lane) - 1u))] = (uint16_t)s;
    nc += __popc(mc);
  }
  __syncwarp();
  if (nc && p.cand_cap) {                                // candidates of the window to their global list
    const uint32_t cbase = warp_reserve(&p.ctrl->n_cand, nc, lane);
    for (uint32_t i = (uint32_t)lane; i < nc; i += 32) {
      const uint32_t slot = cbase + i;
      if (slot < p.cand_cap) p.cand[slot] = ((unsigned long long)f << 32) | (cb + (uint32_t)ltab[i] - PRE);
      else p.ctrl->overflow = 1;
    }
  }
  __syncwarp();
  fs.ac = a;
  fs.prev_last = prev_last;
  fs.prevP = prevP;
  fs.lh_done = lh_done;
  return fs;
}

// Slow path: the line that starts at file byte s of this chunk but ends behind the staged bytes (rare).  Lane 0 walks
// it straight from HBM with the walk's automaton step and hash recurrence and finishes it as finish_lines2 does: its
// candidate, header event and line record are written here.  Everything goes in and out by value: no argument of
// this call lives in local memory.
template <bool REVB>
__device__ __noinline__ Accum long_line(const ScanParams& p, const uint32_t* lc, uint32_t f, uint32_t size, int ext,
                                        uint32_t s, uint32_t lh_slot, Accum ac) {
  const HbmByte lb{p.arena + (uint32_t)p.off[f]};
  uint32_t e = s;
  while (e < size && lb(e) != '\n') ++e;                 // (e > s: byte s is no newline)
  const uint32_t k0 = s >> 3, k1 = (e - 1u) >> 3;        // the words the line touches
  const LutRef t = lut_ref();
  Auto au{0u, 0u};
  uint32_t A = 0;
  unsigned long long R = 0;
#pragma unroll 1
  for (uint32_t k = k0; k <= k1; ++k) {                  // bytes outside the line become zeros, as in the staged chunk
    unsigned long long w = __ldg(reinterpret_cast<const unsigned long long*>(lb.b) + k);
    if (k == k0) w &= ~0ull << (8u * (s & 7u));
    if (k == k1) w &= low_mask(e - 8u * k);
    uint32_t Aw = 0;
    step8b<REVB>(w, au, Aw, t);
    A |= Aw;
    R = ror3_61(R) + fold61(w);
  }
  // value of the bytes [s, e): R * 2^(64 (k1 - k0)) / 2^(8 (s & 7))
  unsigned long long h = rotl61(canon61(R), (3u * (k1 - k0) + 61u * 8u - 8u * (s & 7u)) % 61u);
  uint32_t len = e - s;
  if (lb(e - 1u) == 0x0D) {                              // drop one trailing CR: subtract 0x0D * 256^(len-1)
    --len;
    const unsigned long long cr = rotl61(0x0Dull, (8u * len) % 61u);
    h = h >= cr ? h - cr : h + M61 - cr;
  }
  const unsigned long long lh = mix_hash(h, len);
  ac.lines++;
  ac.digest += lh;
  const uint32_t fl = line_flags2<REVB>(s, e, A, lc[1], lc[2], ext, lb, ac);
  if ((fl & LF_CAND) && p.cand_cap) {
    const uint32_t slot = atomicAdd(&p.ctrl->n_cand, 1u);
    if (slot < p.cand_cap) p.cand[slot] = ((unsigned long long)f << 32) | s;
    else p.ctrl->overflow = 1;
  }
  if ((fl & LF_HDR) && (p.flags & TSM_SCAN_HEADER_EVENTS)) emit_header(p, f, s, e - s, fl);
  if ((p.flags & TSM_SCAN_LINE_HASHES) && lh_slot < p.lh_cap) {   // the chunk's last line
    p.lh_hash[lh_slot] = lh;
    p.lh_end[lh_slot] = e;
    p.lh_flag[lh_slot] = (uint8_t)(fl & LF_CAND);
  }
  return ac;
}

template <bool REVB>
__device__ __forceinline__ void process_chunk2(const ScanParams& p, const uint32_t* lc, uint8_t* wb, uint32_t uslot, uint32_t f,
                                               uint32_t cb, uint32_t size, int ext, int lane, PhaseClock& pc) {
  const uint32_t ce = min(cb + CH, size);
  const uint32_t le = min(ce + EXT, size);
  const uint32_t lim = PRE + (ce - cb);                  // buffer position just past the owned bytes
  const uint32_t lim2 = PRE + (le - cb);                 // ... past the staged bytes
  const bool skip_first = (cb != 0) && (wb[PRE - 1] != '\n');   // chunk starts inside a foreign line
  __syncwarp();
  // ---- everything outside the staged range [PRE, lim2) becomes zeros: no pass has to mask its loads
  //      (a zero byte is no newline, matches no pattern and adds nothing to the hash prefix)
  if (lane < 2) reinterpret_cast<unsigned long long*>(wb)[lane] = 0ull;
  {
    const uint32_t za = (lim2 + 7u) & ~7u;
    if ((uint32_t)lane < za - lim2) wb[lim2 + lane] = 0;
    for (uint32_t q = za + 8u * (uint32_t)lane; q < BUF; q += 256u) *reinterpret_cast<unsigned long long*>(wb + q) = 0ull;
  }
  if (lane == 0) *reinterpret_cast<uint32_t*>(wb + O2_CTL) = 0u;
  __syncwarp();
  pc.mark(PH_ZERO, lane);
  const WalkOut wo = walk2<REVB>(wb, lc[0], lane);
  pc.mark(PH_WALK, lane);
  // ---- newline words behind the owned bytes: only the first one matters (it ends the last owned line)
  const uint32_t w0 = 17u * (uint32_t)lane, lim_w = (lim + 7u) >> 3;
  const uint32_t ownbits = lim_w <= w0 ? 0u : (lim_w - w0 >= 17u ? 0x1FFFFu : (1u << (lim_w - w0)) - 1u);
  const uint32_t extbits = wo.nlw & ~ownbits;
  const uint32_t gx = __reduce_min_sync(0xffffffffu, extbits ? w0 + (uint32_t)__ffs((int)extbits) - 1u : 0xFFFFu);
  uint32_t kept = wo.nlw & ownbits;
  if (gx - w0 < 17u) kept |= 1u << (gx - w0);
  // ---- states of a line that spans stripes: OR of the stripe tails back to the stripe of its first byte;
  //      and the positions of the kept newline words in the entry table (two scans, one loop)
  uint32_t tv = wo.tail, tf = wo.nlw != 0u;
  const uint32_t cnt = __popc(kept);
  uint32_t incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t uv = __shfl_up_sync(0xffffffffu, tv, d), uf = __shfl_up_sync(0xffffffffu, tf, d);
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) { if (!tf) tv |= uv; tf |= uf; incl += t; }
  }
  uint32_t carry = __shfl_up_sync(0xffffffffu, tv, 1);
  if (lane == 0) carry = 0;
  const uint32_t tail_all = __shfl_sync(0xffffffffu, tv, 31);
  const uint32_t n_went = __shfl_sync(0xffffffffu, incl, 31), ebase = incl - cnt;
  uint16_t* went = reinterpret_cast<uint16_t*>(wb + O2_WENT);
  uint32_t* arun = reinterpret_cast<uint32_t*>(wb + O2_ARUN);
  {
    uint32_t b = kept, idx = ebase;
    while (b) { went[idx++] = (uint16_t)(w0 + (uint32_t)__ffs((int)b) - 1u); b &= b - 1u; }
    if (wo.nlw) arun[w0 + (uint32_t)__ffs((int)wo.nlw) - 1u] |= carry;
    if (lane == 0) arun[SLOT_TAIL] = tail_all;
  }
  __syncwarp();
  pc.mark(PH_SCANS, lane);
  // ---- mixed words
  {
    const uint32_t nq_all = *reinterpret_cast<const uint32_t*>(wb + O2_CTL);
    const uint16_t* q = reinterpret_cast<const uint16_t*>(wb + O2_Q);
    if (nq_all <= Q2_CAP) {
      for (uint32_t base = 0; base < nq_all; base += 32) {
        const uint32_t t = base + (uint32_t)lane;
        const uint32_t g = t < nq_all ? (uint32_t)q[t] : 0u;
        const uint32_t l = g / 17u, k = g - 17u * l;
        const uint32_t m = __shfl_sync(0xffffffffu, kept, (int)l), eb = __shfl_sync(0xffffffffu, ebase, (int)l);
        const bool act = t < nq_all && ((m >> k) & 1u);
        const uint32_t i = eb + __popc(m & ((1u << k) - 1u));
        if (act) resolve_mixed<REVB>(wb, g, i, n_went);
        __syncwarp();
        if (act) went[i] |= 0x8000u;
        __syncwarp();
      }
    } else if (lc[0]) {                                  // queue overflow: take every newline word as mixed
      for (uint32_t base = 0; base < n_went; base += 32) {
        const uint32_t i = base + (uint32_t)lane;
        if (i < n_went) resolve_mixed<REVB>(wb, (uint32_t)went[i] & 0x3FFu, i, n_went);
        __syncwarp();
        if (i < n_went) went[i] |= 0x8000u;
        __syncwarp();
      }
    }
  }
  pc.mark(PH_MIXED, lane);
  // ---- newline words -> one record per line (dense: one lane per newline word, SWAR for the newline bytes),
  //      finished window by window (one window unless the chunk has more than ~LCAP lines)
  uint16_t* ltab = reinterpret_cast<uint16_t*>(wb + O2_LTAB);
  FinishState fs{{0, 0, 0, 0, 0}, PRE - 1u, 0ull, 0u, 0u};   // (the 16 bytes in front of the chunk are zeros)
  const bool want_lh = (p.flags & TSM_SCAN_LINE_HASHES) != 0;
  if (want_lh) {                                         // one region for the chunk's line records: newlines of the kept words + 1
    uint32_t tot = 0;
    for (uint32_t j = (uint32_t)lane; j < n_went; j += 32)
      tot += __popc(nl8_of(*reinterpret_cast<const unsigned long long*>(wb + 8u * ((uint32_t)went[j] & 0x3FFu))));
    tot = __reduce_add_sync(0xffffffffu, tot) + 1u;
    uint32_t base = 0;
    if (lane == 0) {
      base = atomicAdd(&p.ctrl->n_lh, tot);
      if (base + tot > p.lh_cap) p.ctrl->lh_overflow = 1;
      p.unit_out[uslot] = base;
    }
    fs.lh_base = __shfl_sync(0xffffffffu, base, 0);
  }
  uint32_t n_rec = 0, last_nl = PRE - 1u;
  for (uint32_t base = 0; base < n_went; base += 32) {
    const uint32_t j = base + (uint32_t)lane;
    const uint32_t ge = j < n_went ? (uint32_t)went[j] : 0u;
    const uint32_t g = ge & 0x3FFu;
    uint32_t m = j < n_went ? nl8_of(*reinterpret_cast<const unsigned long long*>(wb + 8u * g)) : 0u;
    const uint32_t c = __popc(m);
    uint32_t in2 = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, in2, d);
      if (lane >= d) in2 += t;
    }
    if (base + 32u >= n_went) {                          // position of the chunk's last newline
      const uint32_t lastl = n_went - 1u - base;
      last_nl = __shfl_sync(0xffffffffu, 8u * g + 31u - (uint32_t)__clz((int)(m | 1u)), (int)lastl);
    }
    uint32_t off = n_rec + in2 - c;
    uint32_t rec = 8u * g + LR_FIRST + ((ge >> 15) << 14);
    while (m) {
      ltab[off++] = (uint16_t)(rec + (uint32_t)__ffs((int)m) - 1u);
      rec &= ~LR_FIRST;
      m &= m - 1u;
    }
    n_rec += __shfl_sync(0xffffffffu, in2, 31);
    __syncwarp();
    if (n_rec + 256u > LCAP && base + 32u < n_went) {    // the next round may not fit: finish what is there
      pc.mark(PH_RECORDS, lane);
      fs = finish_lines2<REVB>(p, wb, lc, n_rec, lim, skip_first, f, cb, ext, lane, fs);
      pc.mark(PH_FINISH, lane);
      n_rec = 0;
    }
  }
  // ---- the line behind the last newline: ends with the file (virtual record), lies in the next chunk, or is long
  const uint32_t tail_start = last_nl + 1u;
  bool tail_long = false;
  if (tail_start < lim && !(skip_first && n_went == 0u)) {
    if (le == size) {                                    // unterminated last line of the file (the data ends at lim2)
      if (tail_start < lim2) { if (lane == 0) ltab[n_rec] = (uint16_t)(lim2 | LR_VIRT | LR_FIRST); ++n_rec; }
    } else tail_long = true;
  }
  __syncwarp();
  pc.mark(PH_RECORDS, lane);
  if (n_rec) fs = finish_lines2<REVB>(p, wb, lc, n_rec, lim, skip_first, f, cb, ext, lane, fs);
  pc.mark(PH_FINISH, lane);
  Accum ac = fs.ac;
  if (tail_long && lane == 0) ac = long_line<REVB>(p, lc, f, size, ext, cb + tail_start - PRE, fs.lh_base + fs.lh_done, ac);
  pc.mark(PH_LONG, lane);
  // ---- per-file counters: warp reduce (the digest as three partial sums: low halves keep their carries),
  //      then one store (single-chunk file) or one atomic per counter
  ac.lines = __reduce_add_sync(0xffffffffu, ac.lines);
  ac.asserts = __reduce_add_sync(0xffffffffu, ac.asserts);
  ac.hdrs = __reduce_add_sync(0xffffffffu, ac.hdrs);
  ac.fixes = __reduce_add_sync(0xffffffffu, ac.fixes);
  {
    const uint32_t dlo = (uint32_t)ac.digest, dhi = (uint32_t)(ac.digest >> 32);
    const unsigned long long s0 = __reduce_add_sync(0xffffffffu, dlo & 0xFFFFu);
    const unsigned long long s1 = __reduce_add_sync(0xffffffffu, dlo >> 16);
    const unsigned long long s2 = __reduce_add_sync(0xffffffffu, dhi);
    ac.digest = s0 + (s1 << 16) + (s2 << 32);
  }
  if (want_lh && lane == 0) p.unit_lines[uslot] = ac.lines;
  if (lane == 0) {
    tsm_file_stat* st = p.stats + f;
    if (size <= CH) {                                    // sole owner of the record: plain store
      *st = tsm_file_stat{ac.lines, ac.asserts, ac.hdrs, ac.fixes, ac.digest};
    } else {
      if (ac.lines) atomicAdd(&st->n_lines, ac.lines);
      if (ac.asserts) atomicAdd(&st->n_assert, ac.asserts);
      if (ac.hdrs) atomicAdd(&st->n_headers, ac.hdrs);
      if (ac.fixes) atomicAdd(&st->n_fixture, ac.fixes);
      if (ac.digest) atomicAdd(reinterpret_cast<unsigned long long*>(&st->digest), ac.digest);
    }
  }
  pc.mark(PH_FLUSH, lane);
}

template <bool REVB>
__global__ void __launch_bounds__(SCAN2_WARPS * 32, SCAN2_CTAS_PER_SM) k_scan_t(const __grid_constant__ ScanParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t* lut_all = reinterpret_cast<uint32_t*>(smem);  // [0,256) the automaton table, then 3 x 4 per-language masks, the opaque 4
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut_all[i] = c_lut[i];
  if (threadIdx.x < 12) {                                // per language (PY, C family, none): pattern ends that count, then the header groups
    const int t = threadIdx.x, lang = t >> 2, q = t & 3;
    const uint32_t g1 = lang == 0 ? PY_G1 : CJ_G1, g2 = lang == 0 ? PY_G2 : CJ_G2;
    const uint32_t v = q == 0 ? (AF_ASSERT | AF_EXPECT | g1 | g2 | B_F | (REVB ? REVB_BIT : 0u)) : (q == 1 ? g1 : (q == 2 ? g2 : 0u));
    lut_all[256 + t] = lang == 2 ? 0u : v;
  }
  if (threadIdx.x == 12) lut_all[256 + 12] = p.four;
  if (threadIdx.x == 13) lut_all[256 + 13] = smem_u32(lut_all);
  if (REVB) for (int i = threadIdx.x; i < 256; i += blockDim.x) lut_all[O2_LUTB / 4 + i] = c_lut_b[i];
  PhaseClock pc;
#if TSM_PHASE_CLOCKS
  pc.tab = reinterpret_cast<uint32_t*>(smem + O2_PHASE);
  if (threadIdx.x < PH_N) pc.tab[threadIdx.x] = 0u;
#endif
  if (threadIdx.x >= 32 && threadIdx.x < 32 + 61)        // rotations of the newline byte: 0x0A * 2^r mod 2^61-1
    reinterpret_cast<unsigned long long*>(smem + O2_T0A)[threadIdx.x - 32] = rotl61(0x0Aull, threadIdx.x - 32);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* wb = smem + CTA_BYTES2 + warp * WARP_SMEM2;
  uint64_t* bar = reinterpret_cast<uint64_t*>(wb + O2_CTL + 8);
  uint32_t* phase = reinterpret_cast<uint32_t*>(wb + O2_CTL + 4);   // (in shared memory: as a register it spilled in the Rev-B kernel)
  if (lane == 0) { mbar_init(bar, 1); fence_mbar_init(); *phase = 0u; }
  __syncwarp();
  const uint32_t n_units = p.slab->n_units;
  Unit cur = claim_unit(p, n_units, lane);
#if TSM_PHASE_CLOCKS
  pc.t = clock64();
#endif
  while (cur.u < n_units) {                              // (no CTA-wide chunk start: with the walk as one rolled loop the hot code fits the
                                                         //  instruction cache and the barrier only costs)
    fence_proxy_async();                                 // this warp's zero fill and reads of the last chunk come first
    __syncwarp();
    if (lane == 0) issue_load(p, wb, bar, cur.fo, cur.size, cur.cb);
    const Unit nxt = claim_unit(p, n_units, lane);       // metadata of the next unit arrives during this chunk
    const uint32_t ph = *phase;
    while (!mbar_try_wait(bar, ph)) {}
    __syncwarp();
    if (lane == 0) *phase = ph ^ 1u;
    pc.mark(PH_WAIT, lane);
    const uint32_t lang = cur.ext == 0 ? 2u : (cur.ext == TSM_EXT_PY ? 0u : 1u);
    process_chunk2<REVB>(p, lut_all + 256u + 4u * lang, wb, p.unit_base + cur.u, cur.f, cur.cb, cur.size, cur.ext, lane, pc);
    __syncwarp();
    cur = nxt;
  }
#if TSM_PHASE_CLOCKS
  __syncthreads();
  if (threadIdx.x < PH_N) atomicAdd(&g_scan_phase_clk[threadIdx.x], (unsigned long long)pc.tab[threadIdx.x]);
#endif
}

// The two instantiations: canonical Rev A (the hot path, what bench.py times) and Rev B (TSM_SCAN_REV_B).
template __global__ void k_scan_t<false>(const __grid_constant__ ScanParams);
template __global__ void k_scan_t<true>(const __grid_constant__ ScanParams);

}  // namespace tsm
