// tsm_scan_kernels.cuh - hand-written sm_90a kernels of the corpus scan (docs/SPEC.md, DESIGN.md), part 1:
//
//   k_plan      files -> (file, 4 KiB chunk) work units                         [tiny]
//   (k_scan     the hot kernel: tsm_scan_walk.cuh; this file holds the small helpers it uses)
//   k_classify  one thread per candidate: statement, last identifier, category (S5), events, the
//               cross-file aggregate into a shared-memory privatised [group][category] table, and
//               the totals of the per-file records.
//
// There is no reference kernel: the reference ships data only (SURVEY.md section 0).  Rules cite
// docs/SPEC.md, which cites the artefacts.
#pragma once
#include "tsm_device.cuh"

namespace tsm {

__constant__ uint32_t c_lut[256];                       // automaton table (tsm_device.cuh; built by tsm_create)
__constant__ uint32_t c_lut_b[256];                     // Rev-B trigger table (tsm_scan_walk.cuh)
__constant__ uint32_t c_elut[256];                      // bare-assert operator automaton (k_classify)
// category tables: read once per block of k_classify into shared memory (coalesced, hence plain device memory)
__device__ uint8_t c_cat_slot[TSM_CAT_SLOTS];            // perfect hash slot -> category id
__device__ uint16_t c_cat_off[TSM_CAT_NAMED + 1];
__device__ char c_cat_blob[TSM_CAT_BLOB_LEN + 1];

// ================================================================================= k_plan
// One lane per file: units = ceil(len / CH); the warp reserves a contiguous range of the unit
// table with one atomic.  Unit order is irrelevant for the results (all outputs are sums or sets).
__global__ void k_plan(ScanParams p) {
  const int f = p.f_begin + blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) p.ctrl->cls_done = p.ctrl->n_cand;   // everything found so far has been classified
  uint32_t nu = 0;
  if (f < p.f_end) {
    nu = ((uint32_t)p.len[f] + CH - 1) / CH;
    if (nu != 1) p.stats[f] = tsm_file_stat{0, 0, 0, 0, 0};   // several chunks add into it (one chunk: k_scan stores), none leave it zero
  }
  uint32_t incl = nu;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
  uint32_t base = 0;
  if (lane == 31 && total) base = atomicAdd(&p.slab->n_units, total);
  base = __shfl_sync(0xffffffffu, base, 31);
  uint32_t at = p.unit_base + base + incl - nu;
  for (uint32_t u = 0; u < nu; ++u, ++at) {
    if (at < p.unit_cap) { p.unit_file[at] = (uint32_t)f; p.unit_begin[at] = u * CH; }
    else p.ctrl->overflow = 1;
  }
}

// ================================================================================= helpers of k_scan
// SWAR: 4-bit mask of the bytes equal to '\n' in a 32-bit word.
__device__ __forceinline__ uint32_t nl_word(uint32_t w) {
  const uint32_t y = w ^ 0x0A0A0A0Au;
  const uint32_t t = (y & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
  const uint32_t z = ~(t | y | 0x7F7F7F7Fu);            // 0x80 in every byte that was '\n'
  return (z * 0x00204081u) >> 28;                        // gather the four flag bits: 7+21, 15+14, 23+7, 31+0 -> 28..31
}
// number of leading 0x20 bytes among the 8 bytes of w
__device__ __forceinline__ uint32_t spaces_of(unsigned long long w) {
  const unsigned long long x = w ^ 0x2020202020202020ull, k7 = 0x7F7F7F7F7F7F7F7Full;
  const unsigned long long nz = (((x & k7) + k7) | x) & ~k7;             // 0x80 in every byte that is not a space
  return nz ? ((uint32_t)__ffsll((long long)nz) - 1u) >> 3 : 8u;
}
// Byte sources of the line rules (line_flags2, starts_with8): a byte, the 8 bytes at any alignment, their leading spaces.
struct SmemByte {                                        // the staged chunk
  const uint8_t* b;
  __device__ __forceinline__ uint32_t operator()(uint32_t i) const { return b[i]; }
  // the 8 bytes at i, any alignment (shared memory is readable 8 bytes past any line of the buffer)
  __device__ __forceinline__ unsigned long long load8(uint32_t i) const {
    const uint32_t a = i & ~7u, sh = 8u * (i & 7u);
    const unsigned long long lo = *reinterpret_cast<const unsigned long long*>(b + a);
    const unsigned long long hi = *reinterpret_cast<const unsigned long long*>(b + a + 8);
    return sh ? (lo >> sh) | (hi << (64u - sh)) : lo;
  }
  __device__ __forceinline__ uint32_t spaces8(uint32_t i) const { return spaces_of(load8(i)); }
};
struct HbmByte {                                         // a file in HBM (long lines), b 8-byte aligned
  const uint8_t* b;
  __device__ __forceinline__ uint32_t operator()(uint32_t i) const { return __ldg(b + i); }
  // the 8 bytes at i from two aligned loads, which read up to byte i + 15, i.e. up to 15 bytes past the line end.  That
  // is readable: every device arena has 4 096 B of slack behind off[n] (tsm_create allocates max_arena + 4096,
  // side_upload ab + 4096).
  __device__ __forceinline__ unsigned long long load8(uint32_t i) const {
    const unsigned long long* w = reinterpret_cast<const unsigned long long*>(b) + (i >> 3);
    const uint32_t sh = 8u * (i & 7u);
    const unsigned long long lo = __ldg(w), hi = __ldg(w + 1);
    return sh ? (lo >> sh) | (hi << (64u - sh)) : lo;
  }
  __device__ __forceinline__ uint32_t spaces8(uint32_t i) const { return spaces_of(load8(i)); }
};
struct Accum { uint32_t lines, asserts, hdrs, fixes; unsigned long long digest; };

// Append `n` list entries with one atomic; returns the base slot (broadcast from lane 0).
__device__ __forceinline__ uint32_t warp_reserve(uint32_t* counter, uint32_t n, int lane) {
  uint32_t base = 0;
  if (lane == 0 && n) base = atomicAdd(counter, n);
  return __shfl_sync(0xffffffffu, base, 0);
}

// The automaton table of k_scan sits at the start of the dynamic shared memory: a compile-time address.
__device__ __forceinline__ const uint32_t* scan_lut() {
  extern __shared__ __align__(128) uint8_t smem[];
  return reinterpret_cast<const uint32_t*>(smem);
}

// Stage the bytes [max(cb-16,0), min(cb+CH+EXT, size)) of a file so that file byte cb sits at buf+PRE.
__device__ __forceinline__ void issue_load(const ScanParams& p, uint8_t* buf, uint64_t* bar, uint32_t fo,
                                           uint32_t size, uint32_t cb) {
  const uint32_t lb = cb ? cb - PRE : 0u;
  const uint32_t le = min(cb + CH + EXT, size);
  const uint32_t bytes = (le - lb + 15u) & ~15u;          // the pad up to the 128-B file boundary is readable
  mbar_expect_tx(bar, bytes);
  bulk_load(buf + PRE - (cb - lb), p.arena + (size_t)fo + lb, bytes, bar);
}

struct Unit { uint32_t u, f, cb, fo, size; int ext; };

// Claim the next work unit and fetch its metadata (4 dependent global loads: issued one chunk
// ahead so that their latency hides behind the current chunk).
__device__ __forceinline__ Unit claim_unit(const ScanParams& p, uint32_t n_units, int lane) {
  Unit x{0, 0, 0, 0, 0, 0};
  if (lane == 0) x.u = atomicAdd(&p.slab->work, 1u);
  x.u = __shfl_sync(0xffffffffu, x.u, 0);
  if (x.u < n_units) {
    x.f = p.unit_file[p.unit_base + x.u];
    x.cb = p.unit_begin[p.unit_base + x.u];
    x.fo = (uint32_t)p.off[x.f];
    x.size = (uint32_t)p.len[x.f];
    x.ext = p.ext[x.f];
  }
  return x;
}

// ================================================================================= k_classify
// One thread per candidate line, exactly SPEC sections 4 and 6.  The statement T ends at the first '(';
// one pass over its bytes (8-byte loads, one shared-memory class lookup per byte) finds the
// stripped start, the right-stripped end and the last identifier L; everything else (gtest stem,
// bare-assert operators, table lookup of L, statement hash) touches only the few bytes it needs.
constexpr uint32_t CC_W = 1, CC_IDENT = 2, CC_STOP = 4;  // byte classes: blank, [A-Za-z0-9_], '(' or LF
constexpr uint32_t CLS_CAT_OFF_N = (TSM_CAT_NAMED + 2) & ~1u;            // u16 entries (even count keeps the blob 4-byte aligned)
constexpr uint32_t CLS_CAT_WORDS = ((TSM_CAT_SLOTS + 2 * CLS_CAT_OFF_N + TSM_CAT_BLOB_LEN + 15) / 16) * 4;   // (keeps the queue 16-byte aligned)
constexpr uint32_t CLS_SMEM_BASE = 4 * (512 + CLS_CAT_WORDS + 4 * 1024 + 4);   // bytes in front of the histogram (tables + BQ_CAP queue)
constexpr uint32_t E_FIRST = (1u << 0) | (1u << 5) | (1u << 9) | (1u << 17) | (1u << 21) | (1u << 23) | (1u << 25) |
                             (1u << 27) | (1u << 29) | (1u << 30);

struct FileBytes {                                       // 8-byte buffered reader over one file in HBM
  const unsigned long long* base; uint32_t cur_blk; unsigned long long w;
  // the first words of the candidate line, fetched by independent loads up front: one HBM / L2 latency per
  // candidate instead of one per step of the parse
  uint32_t blk0; unsigned long long w0, w1, w2, w3;
  __device__ __forceinline__ FileBytes(const uint8_t* b, uint32_t first_byte)
      : base(reinterpret_cast<const unsigned long long*>(b)), cur_blk(0xFFFFFFFFu), w(0), blk0(first_byte >> 3) {
    w0 = __ldg(base + blk0); w1 = __ldg(base + blk0 + 1); w2 = __ldg(base + blk0 + 2); w3 = __ldg(base + blk0 + 3);
  }
  __device__ __forceinline__ unsigned long long word(uint32_t blk) const {
    const uint32_t d = blk - blk0;
    if (d < 4u) return d < 2u ? (d == 0u ? w0 : w1) : (d == 2u ? w2 : w3);
    return __ldg(base + blk);
  }
  __device__ __forceinline__ uint32_t get(uint32_t i) {
    const uint32_t blk = i >> 3;
    if (blk != cur_blk) { w = word(blk); cur_blk = blk; }
    return (uint32_t)(w >> (8u * (i & 7u))) & 0xFFu;
  }
  // the 8 bytes at file offset i (unaligned), little-endian
  __device__ __forceinline__ unsigned long long get8(uint32_t i) const {
    const uint32_t blk = i >> 3, sh = 8u * (i & 7u);
    const unsigned long long lo = word(blk);
    if (sh == 0) return lo;
    return (lo >> sh) | (word(blk + 1) << (64u - sh));
  }
};

__device__ __forceinline__ unsigned long long low_bytes(unsigned long long v, uint32_t n) {   // keep n <= 8 bytes
  return n >= 8 ? v : (v & ((1ull << (8u * n)) - 1ull));
}

// gtest stem table (SPEC section 6 rule 1): stem = bytes after "EXPECT_" / "ASSERT_", n = its length
__device__ __forceinline__ int stem_lookup(FileBytes& rd, uint32_t s, uint32_t n) {
  if (n < 2 || n > 9) return 0;
  const unsigned long long v = low_bytes(rd.get8(s), n);
  const uint32_t c9 = n == 9 ? rd.get(s + 8) : 0u;
  switch (n) {
    case 2:
      if (v == 0x5145ull) return 1;            // EQ
      if (v == 0x454Eull) return 2;            // NE
      if (v == 0x5447ull) return 5;            // GT
      if (v == 0x4547ull) return 6;            // GE
      if (v == 0x544Cull) return 7;            // LT
      if (v == 0x454Cull) return 8;            // LE
      return 0;
    case 4:
      if (v == 0x45555254ull) return 3;        // TRUE
      if (v == 0x5241454Eull) return 9;        // NEAR
      return 0;
    case 5:
      if (v == 0x45534C4146ull) return 4;      // FALSE
      if (v == 0x574F524854ull) return 12;     // THROW
      return 0;
    case 8: return v == 0x51455F54414F4C46ull ? 10 : 0;                 // FLOAT_EQ
    case 9: return (v == 0x455F454C42554F44ull && c9 == 'Q') ? 11 : 0;   // DOUBLE_EQ
    default: return 0;
  }
}

// SPEC section 6 rule 2 on e = T[7:] of a bare "assert <expr>": one Shift-And pass over e for the ten
// operator patterns (table built in tsm_api.cu), 8 bytes per step:
//  " not " 0-4 | " in " 5-8 | " is not " 9-16 | "True" 17-20 | "==" 21-22 | "!=" 23-24 | "<=" 25-26 |
//  ">=" 27-28 | "<" 29 | ">" 30   (final bits 4, 8, 16, 20, 22, 24, 26, 28, 29, 30)
__device__ __forceinline__ int bare_assert_category(FileBytes& rd, uint32_t e0, uint32_t en, const uint32_t* elut, int deflt = 3,
                                                    bool not_prefix = true) {
  if (not_prefix && en >= 4 && (uint32_t)rd.get8(e0) == 0x20746F6Eu) return 2;        // "not "
  uint32_t D = 0, A = 0;
  for (uint32_t a = 0; a < en; a += 8) {                 // bytes behind the end become zeros (match nothing)
    unsigned long long w = rd.get8(e0 + a);
    if (en - a < 8) w &= (1ull << (8u * (en - a))) - 1ull;
    const uint32_t lo = (uint32_t)w, hi = (uint32_t)(w >> 32);
#pragma unroll
    for (int k = 0; k < 4; ++k) { D = ((D + D) | E_FIRST) & elut[__byte_perm(lo, 0, 0x4440 + k)]; A |= D; }
#pragma unroll
    for (int k = 0; k < 4; ++k) { D = ((D + D) | E_FIRST) & elut[__byte_perm(hi, 0, 0x4440 + k)]; A |= D; }
  }
  if (((A & (1u << 4)) && (A & (1u << 8))) || (A & (1u << 16))) return 4;   // not ... in / is not
  if (A & (1u << 20)) return 3;                          // True
  if (A & (1u << 22)) return 1;                          // ==
  if (A & (1u << 24)) return 2;                          // !=
  if (A & (1u << 26)) return 8;                          // <=
  if (A & (1u << 28)) return 6;                          // >=
  if (A & (1u << 29)) return 7;                          // <
  if (A & (1u << 30)) return 5;                          // >
  return deflt;
}

// Is the identifier [s, s + n) of the file the name `name` (Rev-B rules, docs/SPEC.md section 4b; rare path)?
__device__ __noinline__ bool ident_eq(FileBytes& rd, uint32_t s, uint32_t n, const char* name, uint32_t len) {
  if (n != len) return false;
  for (uint32_t k = 0; k < len; ++k)
    if (rd.get(s + k) != (uint8_t)name[k]) return false;
  return true;
}

constexpr uint32_t BQ_CAP = 1024;                        // bare-assert expressions a block of k_classify defers (16 B each)

#ifndef TSM_CLS_MINB
#define TSM_CLS_MINB 1
#endif
template <bool REVB>
__global__ void __launch_bounds__(256, TSM_CLS_MINB) k_classify_t(ScanParams p) {
  extern __shared__ __align__(16) uint32_t csm[];        // byte classes, operator table, category tables, deferral queue, [n_groups][K] histogram
  uint32_t* cls = csm;
  uint32_t* elut = csm + 256;
  uint8_t* cat_slot = reinterpret_cast<uint8_t*>(csm + 512);             // copies of the constant tables: the lanes of a
  uint16_t* cat_off = reinterpret_cast<uint16_t*>(cat_slot + TSM_CAT_SLOTS);   // warp look up different names (divergent
  uint8_t* cat_blob = reinterpret_cast<uint8_t*>(cat_off + CLS_CAT_OFF_N);     // constant-memory reads would serialise)
  uint4* bq = reinterpret_cast<uint4*>(csm + 512 + CLS_CAT_WORDS);       // deferred bare asserts: file, e0, en, event slot
  uint32_t* bqn = csm + 512 + CLS_CAT_WORDS + 4 * BQ_CAP;
  uint32_t* hist = bqn + 4;
  const bool use_smem = p.n_groups <= 16;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    const uint32_t c = (uint32_t)i;
    cls[i] = (is_w(c) ? CC_W : 0u) | (is_ident(c) ? CC_IDENT : 0u) | ((c == '(' || c == '\n') ? CC_STOP : 0u);
    elut[i] = c_elut[i];
  }
  for (int i = threadIdx.x; i < TSM_CAT_SLOTS; i += blockDim.x) cat_slot[i] = c_cat_slot[i];
  for (int i = threadIdx.x; i < TSM_CAT_NAMED + 1; i += blockDim.x) cat_off[i] = c_cat_off[i];
  for (int i = threadIdx.x; i < TSM_CAT_BLOB_LEN; i += blockDim.x) cat_blob[i] = (uint8_t)c_cat_blob[i];
  if (use_smem) for (int i = threadIdx.x; i < p.n_groups * TSM_K; i += blockDim.x) hist[i] = 0;
  if (threadIdx.x == 0) *bqn = 0;
  __syncthreads();
  auto count = [&](uint32_t f, int cat) {                // cross-file aggregate: [group][category]
    const uint32_t g = p.grp ? p.grp[f] : 0u;
    if (use_smem) atomicAdd(&hist[g * TSM_K + cat], 1u);
    else {
      atomicAdd(&p.counts[(size_t)g * TSM_K + cat], 1ull);
      atomicAdd(&p.counts[(size_t)p.n_groups * TSM_K + cat], 1ull);
    }
  };
  const uint32_t n = min(p.ctrl->n_cand, p.cand_cap), n0 = min(p.ctrl->cls_done, n);   // this launch: candidates [n0, n)
  const bool want_ev = (p.flags & TSM_SCAN_ASSERT_EVENTS) != 0;
  constexpr bool revb = REVB;                            // (two instantiations: the Rev-B rules stay out of the canonical kernel)
  for (uint32_t i = n0 + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long cd = p.cand[i];
    const uint32_t f = (uint32_t)(cd >> 32), line_off = (uint32_t)cd;
    const uint32_t size = (uint32_t)p.len[f];
    FileBytes rd(p.arena + (size_t)(uint32_t)p.off[f], line_off);
    // ---- T = [t0, last): skip the indentation, find the first '(' / LF a word at a time (SWAR),
    //      strip blanks backwards; L = the identifier run that ends at `last`
    uint32_t q = line_off;
    while (q < size && (cls[rd.get(q)] & CC_W)) ++q;     // LF is not blank: stops at the line end too
    const uint32_t t0 = q;
    uint32_t stop = size;
    for (uint32_t wb = t0 & ~7u; wb < size; wb += 8) {
      unsigned long long w = rd.word(wb >> 3);
      const unsigned long long x1 = w ^ 0x2828282828282828ull, x2 = w ^ 0x0A0A0A0A0A0A0A0Aull;
      const unsigned long long k7 = 0x7F7F7F7F7F7F7F7Full;
      unsigned long long z = (~(((x1 & k7) + k7) | x1 | k7)) | (~(((x2 & k7) + k7) | x2 | k7));   // 0x80 per '(' or LF
      if (wb < t0) z &= ~0ull << (8u * (t0 - wb));
      if (z) { stop = wb + ((uint32_t)__ffsll((long long)z) - 1u) / 8u; break; }
    }
    stop = min(stop, size);
    uint32_t last = stop;
    while (last > t0 && (cls[rd.get(last - 1)] & CC_W)) --last;
    uint32_t Ls = last;
    while (Ls > t0 && (cls[rd.get(Ls - 1)] & CC_IDENT)) --Ls;
    uint32_t tlen = last - t0;                           // (Rev B may lengthen the statement of the event; the rules see Rev A's)
    const uint32_t tlen_a = tlen, Ln = last - Ls;
    // ---- category (SPEC section 6), first match wins
    int cat = 0;
    bool done = false;
    uint32_t def_e0 = 0, def_en = 0;                     // def_en != 0: category decided by the deferred operator pass
    if (revb) {                                          // ---- Rev B (SPEC section 4b): one more stem, the bare forms by their operators, full statements
      const bool macro = ident_eq(rd, Ls, Ln, "BOOST_CHECK", 11) || ident_eq(rd, Ls, Ln, "NTA_CHECK", 9);
      const bool bare6 = tlen == 6 && low_bytes(rd.get8(t0), 6) == 0x747265737361ull;
      const bool full = macro || p.ext[f] == TSM_EXT_JAVA;
      uint32_t fe = last;                                // end of the stripped line
      if (full || ((macro || bare6) && stop < size && rd.get(stop) == '(')) {
        uint32_t le = stop;
        while (le < size && rd.get(le) != '\n') ++le;
        fe = le;
        while (fe > t0 && (cls[rd.get(fe - 1)] & CC_W)) --fe;
      }
      if (ident_eq(rd, Ls, Ln, "BOOST_CHECK_EQUAL", 17)) { cat = 1; done = true; }
      else if ((macro || bare6) && stop < size && rd.get(stop) == '(') {
        uint32_t x = stop + 1;
        while (x < fe && (cls[rd.get(x)] & CC_W)) ++x;
        if (x < fe && rd.get(x) == '!' && !(x + 1 < fe && rd.get(x + 1) == '=')) cat = 4;
        else cat = bare_assert_category(rd, x, fe > x ? fe - x : 0u, elut, macro ? 0 : 3, false);
        done = true;
      }
      if (full) tlen = fe - t0;                          // the event carries the Rev-B statement (the rules above used Rev A's T)
    }
    if (Ln >= 7) {                                       // rule 1: EXPECT_x / ASSERT_x
      const unsigned long long h7 = low_bytes(rd.get8(Ls), 7);
      if (h7 == 0x5F544345505845ull || h7 == 0x5F545245535341ull) { cat = stem_lookup(rd, Ls + 7, Ln - 7); done = true; }
    }
    if (!done && tlen_a >= 6) {                          // rule 2: T == "assert" or T starts with "assert "
      const unsigned long long h = rd.get8(t0);
      const bool a6 = low_bytes(h, 6) == 0x747265737361ull;
      if (a6 && tlen_a == 6) { cat = 3; done = true; }
      else if (a6 && tlen_a >= 8 && ((h >> 48) & 0xFF) == 0x20) {
        done = true;
        def_e0 = t0 + 7; def_en = tlen_a - 7;            // e = T[7:]: the operator pass runs later, with every lane busy
      }
    }
    if (!done && Ln >= 6) {                              // rules 3-5 on L
      const unsigned long long h = rd.get8(Ls);
      if (low_bytes(h, 6) == 0x747265737361ull) {
        if (Ln == 7 && ((h >> 48) & 0xFF) == '_') cat = 3;
        else {
          cat = TSM_CAT_OTHER;
          uint32_t hh = 0x811C9DC5u;                       // FNV-1a of L, 8 bytes per load
          for (uint32_t j = 0; j < Ln; j += 8) {
            unsigned long long w = rd.get8(Ls + j);
            const uint32_t nb = min(8u, Ln - j);
#pragma unroll
            for (uint32_t k = 0; k < 8; ++k) {
              if (k < nb) hh = (hh ^ ((uint32_t)w & 0xFFu)) * 0x01000193u;
              w >>= 8;
            }
          }
          const int id = cat_slot[(hh * TSM_CAT_HASH_MULT) >> 23];
          if (id && (uint32_t)(cat_off[id + 1] - cat_off[id]) == Ln) {
            const uint8_t* name = cat_blob + cat_off[id];
            bool ok = true;
            for (uint32_t j = 0; j < Ln; j += 8) {
              unsigned long long w = rd.get8(Ls + j);
              const uint32_t nb = min(8u, Ln - j);
              for (uint32_t k = 0; k < nb; ++k) { ok &= ((uint32_t)w & 0xFFu) == (uint32_t)name[j + k]; w >>= 8; }
            }
            if (ok) cat = id;
          }
        }
      }
    }
    // ---- event, then aggregate (or defer)
    uint32_t ev_slot = 0xFFFFFFFFu;
    if (want_ev) {
      unsigned long long hacc = 0; uint32_t hr = 0;     // Mersenne-61 of T (SPEC section 3)
      for (uint32_t j = 0; j < tlen; ++j) {
        hacc = fold61(hacc + rotl61((unsigned long long)rd.get(t0 + j), hr));
        hr += 8; if (hr >= 61) hr -= 61;
      }
      const uint32_t slot = atomicAdd(&p.ctrl->n_aev, 1u);
      if (slot < p.aev_cap) {
        tsm_assert_event ev;
        ev.file = f; ev.line_off = line_off; ev.stmt_off = t0;
        ev.stmt_len = (uint16_t)min(tlen, 65535u); ev.cat = (uint16_t)cat;      // (patched by the deferred pass)
        ev.ident_off = Ls; ev.ident_len = (uint16_t)min(Ln, 65535u); ev.pad = 0;
        ev.stmt_hash = mix_hash(canon61(hacc), tlen);
        p.aev[slot] = ev;
        ev_slot = slot;
      } else p.ctrl->overflow = 1;
    }
    if (def_en) {
      const uint32_t slot = atomicAdd(bqn, 1u);
      if (slot < BQ_CAP) { bq[slot] = make_uint4(f, def_e0, def_en, ev_slot); continue; }
      cat = bare_assert_category(rd, def_e0, def_en, elut);              // queue full: decide here
      if (ev_slot != 0xFFFFFFFFu) p.aev[ev_slot].cat = (uint16_t)cat;
    }
    count(f, cat);
  }
  // ---- deferred bare asserts: the block's queue, one expression per thread (the inline version kept 3 of 32
  //      lanes busy for ~50 bytes of serial automaton each)
  __syncthreads();
  {
    const uint32_t nq = min(*bqn, BQ_CAP);
    for (uint32_t t = threadIdx.x; t < nq; t += blockDim.x) {
      const uint4 e = bq[t];
      FileBytes rd(p.arena + (size_t)(uint32_t)p.off[e.x], e.y);
      const int cat = bare_assert_category(rd, e.y, e.z, elut);
      if (e.w != 0xFFFFFFFFu) p.aev[e.w].cat = (uint16_t)cat;
      count(e.x, cat);
    }
  }
  // ---- totals of the per-file records (lines, assertion lines, headers, fixture headers) behind the table
  if (p.cls_last) {
    unsigned long long t0 = 0, t1 = 0, t2 = 0, t3 = 0;
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < p.n_files; f += gridDim.x * blockDim.x) {
      const tsm_file_stat s = p.stats[f];
      t0 += s.n_lines; t1 += s.n_assert; t2 += s.n_headers; t3 += s.n_fixture;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      t0 += __shfl_xor_sync(0xffffffffu, t0, d); t1 += __shfl_xor_sync(0xffffffffu, t1, d);
      t2 += __shfl_xor_sync(0xffffffffu, t2, d); t3 += __shfl_xor_sync(0xffffffffu, t3, d);
    }
    if ((threadIdx.x & 31) == 0) {
      unsigned long long* tot = p.counts + (size_t)(p.n_groups + 1) * TSM_K;
      if (t0) atomicAdd(&tot[0], t0);
      if (t1) atomicAdd(&tot[1], t1);
      if (t2) atomicAdd(&tot[2], t2);
      if (t3) atomicAdd(&tot[3], t3);
    }
  }
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i < p.n_groups * TSM_K; i += blockDim.x) {
      const uint32_t v = hist[i];
      if (v) {
        atomicAdd(&p.counts[i], (unsigned long long)v);
        atomicAdd(&p.counts[(size_t)p.n_groups * TSM_K + (i & (TSM_K - 1))], (unsigned long long)v);
      }
    }
  }
}

template __global__ void k_classify_t<false>(ScanParams);
template __global__ void k_classify_t<true>(ScanParams);

}  // namespace tsm
