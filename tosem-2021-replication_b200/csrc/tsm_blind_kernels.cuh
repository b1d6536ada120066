// tsm_blind_kernels.cuh - the lexer of the blind clones (docs/SPEC.md section 21): the blind form of every line, from the line
// records (tsm_lines_kernels.cuh), hashed without being materialised, and the compaction of the kept lines that the clone
// kernels (tsm_clone_kernels.cuh) then group.  Lines are global indices (< 2^32).
//
// Block comments and triple-quoted strings span lines, so the lexer state at a line's start depends on the lines above it:
//   k_blind_state    one thread per line, 8 bytes per load: the line's transfer function over its family's cross-line states
//                    (PY: code, inside """, inside '''; CJ: code, inside /* */; tag 0: none), 2 bits per state in a u8.  A line
//                    without a byte that can open or close such a state (PY: a quote; CJ: '*') is the identity, found by a
//                    SWAR test of its words before any lexing.
//   k_blind_scan     one warp per file, 32 lines per round: an exclusive scan of the transfer functions under composition from
//                    the code state at the file's first line (any file length; the carry is the state), in place.
//   k_blind_lines    one thread per line: lexes the line from its start state and feeds the blind bytes, separators included,
//                    into the Mersenne-61 recurrence of SPEC section 3 (blind_hash = bytes_hash of the blind form); kept = the
//                    form is not empty.  Keywords: an open-addressing table of BLIND_KW_SLOTS names in shared memory.
//   xscan(kept)      rank of every kept line;
//   k_blind_compact  the kept lines' blind_hash, assertion flag and original index to their rank;
//   k_blind_files    one warp per file: kept_base (the rank of the file's first line) and its kept assertion lines.
#pragma once
#include "tsm_device.cuh"
#include "tsm_diff_kernels.cuh"

namespace tsm {

constexpr uint32_t BLIND_NONE = 0xFFFFFFFFu;
constexpr uint8_t BLIND_IDENTITY = 0 | (1 << 2) | (2 << 4);   // state s -> bits [2s, 2s + 2)

// Keyword table: every name zero-padded to 16 bytes (lo = bytes 0-7, little-endian), an empty slot has lo = 0.  kind: which
// family keeps the name verbatim, or reads it as a literal (placeholder N).
constexpr uint32_t BLIND_KW_SLOTS = 512;
constexpr uint8_t KW_PY = 1, KW_CJ = 2, KW_PY_LIT = 4, KW_CJ_LIT = 8;
struct BlindKw { unsigned long long lo, hi; };
__device__ BlindKw c_blind_kw[BLIND_KW_SLOTS];
__device__ uint8_t c_blind_kind[BLIND_KW_SLOTS];

#define TSM_BLIND_PY_KEYWORDS \
  "and as assert async await break class continue def del elif else except finally for from global if import in is lambda " \
  "nonlocal not or pass raise return try while with yield"
#define TSM_BLIND_CJ_KEYWORDS \
  "_ _Alignas _Alignof _Atomic _Bool _Complex _Generic _Imaginary _Noreturn _Static_assert _Thread_local abstract alignas alignof " \
  "and and_eq asm assert auto bitand bitor bool boolean break byte case catch char char16_t char32_t char8_t class co_await " \
  "co_return co_yield compl concept const const_cast consteval constexpr constinit continue decltype default delete do double " \
  "dynamic_cast else enum explicit export extends extern final finally float for friend goto if implements import inline " \
  "instanceof int interface long mutable namespace native new noexcept not not_eq operator or or_eq package private protected " \
  "public register reinterpret_cast requires restrict return short signed sizeof static static_assert static_cast strictfp struct " \
  "super switch synchronized template this thread_local throw throws transient try typedef typeid typename union unsigned using " \
  "virtual void volatile wchar_t while xor xor_eq"
#define TSM_BLIND_PY_LITERALS "True False None"
#define TSM_BLIND_CJ_LITERALS "true false null nullptr"

__host__ __device__ __forceinline__ uint32_t blind_kw_home(unsigned long long lo, unsigned long long hi) {
  return (uint32_t)(((lo ^ (hi * 0x9E3779B97F4A7C15ull)) * 0xBF58476D1CE4E5B9ull) >> 55);   // 9 bits
}

// The table of the four lists above (host side, for tsm_create).
static inline void blind_keyword_table(BlindKw* kw, uint8_t* kind) {
  for (uint32_t i = 0; i < BLIND_KW_SLOTS; ++i) { kw[i] = BlindKw{0, 0}; kind[i] = 0; }
  const char* lists[4] = {TSM_BLIND_PY_KEYWORDS, TSM_BLIND_CJ_KEYWORDS, TSM_BLIND_PY_LITERALS, TSM_BLIND_CJ_LITERALS};
  const uint8_t bits[4] = {KW_PY, KW_CJ, KW_PY_LIT, KW_CJ_LIT};
  for (int l = 0; l < 4; ++l)
    for (const char* p = lists[l]; *p;) {
      unsigned long long lo = 0, hi = 0;
      uint32_t k = 0;
      for (; *p && *p != ' '; ++p, ++k) {
        if (k < 8) lo |= (unsigned long long)(uint8_t)*p << (8 * k);
        else hi |= (unsigned long long)(uint8_t)*p << (8 * (k - 8));
      }
      while (*p == ' ') ++p;
      uint32_t s = blind_kw_home(lo, hi);
      while (kw[s].lo && !(kw[s].lo == lo && kw[s].hi == hi)) s = (s + 1) & (BLIND_KW_SLOTS - 1);
      kw[s] = BlindKw{lo, hi};
      kind[s] |= bits[l];
    }
}

__device__ __forceinline__ uint32_t blind_family(uint32_t ext) { return ext == 1 ? 1u : (ext - 2u) < 5u ? 2u : 0u; }
__device__ __forceinline__ bool is_digit(uint32_t c) { return (c - '0') < 10u; }
__device__ __forceinline__ bool blind_ident(uint32_t c) { return is_ident(c) || c == '$' || c >= 0x80; }

// The bytes of one line, read through one cached 8-byte word (the lexer moves forward; a lookahead over a word boundary
// costs one reload).  Only positions inside the line are read.
struct LineBytes {
  const uint8_t* g; uint32_t wb; unsigned long long w;
  __device__ __forceinline__ uint32_t at(uint32_t q) {
    const uint32_t b = q & ~7u;
    if (b != wb) { wb = b; w = __ldg(reinterpret_cast<const unsigned long long*>(g + b)); }
    return (uint32_t)(w >> (8 * (q & 7))) & 0xFFu;
  }
};

// bytes_hash (SPEC section 3) of a byte string fed one byte at a time.
struct BlindHash {
  unsigned long long acc; uint32_t r, len;
  __device__ __forceinline__ void byte(uint32_t c) {
    acc = fold61(acc + rotl61((unsigned long long)c, r));
    r += 8; if (r >= 61) r -= 61;
    ++len;
  }
  __device__ __forceinline__ void token(uint32_t c) { if (len) byte(' '); byte(c); }
};

// Index behind the delimiter that closes state st of family fam, searched from i; BLIND_NONE when the line holds none.
__device__ __forceinline__ uint32_t blind_close(LineBytes& B, uint32_t i, uint32_t e, uint32_t fam, uint32_t st) {
  if (fam == 2) {
    for (; i + 1 < e; ++i)
      if (B.at(i) == '*' && B.at(i + 1) == '/') return i + 2;
    return BLIND_NONE;
  }
  const uint32_t q = st == 1 ? '"' : '\'';
  while (i < e) {
    const uint32_t c = B.at(i);
    if (c == '\\') i += 2;
    else if (c == q && i + 2 < e && B.at(i + 1) == q && B.at(i + 2) == q) return i + 3;
    else ++i;
  }
  return BLIND_NONE;
}

// The literal whose quote is at i: the index behind it; st = the state after it (a PY triple-quoted literal left open).
__device__ __forceinline__ uint32_t blind_string(LineBytes& B, uint32_t i, uint32_t e, uint32_t fam, uint32_t& st) {
  const uint32_t q = B.at(i);
  st = 0;
  if (fam == 1 && i + 2 < e && B.at(i + 1) == q && B.at(i + 2) == q) {
    const uint32_t s = q == '"' ? 1u : 2u, j = blind_close(B, i + 3, e, 1, s);
    if (j == BLIND_NONE) { st = s; return e; }
    return j;
  }
  for (uint32_t j = i + 1; j < e;) {
    const uint32_t c = B.at(j);
    if (c == '\\') j += 2;
    else if (c == q) return j + 1;
    else ++j;
  }
  return e;
}

// The keyword kind (KW_*) of an identifier of k bytes whose first 16 are (lo, hi): 0 when it is no name of the table.
__device__ __forceinline__ uint32_t blind_kw_kind(const BlindKw* kw, const uint8_t* kind, unsigned long long lo, unsigned long long hi,
                                                  uint32_t k) {
  uint32_t kk = 0;
  if (k <= 16)
    for (uint32_t sl = blind_kw_home(lo, hi); kw[sl].lo; sl = (sl + 1) & (BLIND_KW_SLOTS - 1))
      if (kw[sl].lo == lo && kw[sl].hi == hi) { kk = kind[sl]; break; }
  return kk;
}

// Token sinks of blind_lex, one call per token: number(), string(), ident(B, fam, i0, k, lo, hi) for the identifier of k bytes
// at i0 whose first 16 bytes are (lo, hi), punct(c) for any other byte.  NoSink only follows the state; BlindSink feeds the
// blind form into h, looking keywords up in (kw, kind).
struct NoSink {
  __device__ __forceinline__ void number() {}
  __device__ __forceinline__ void string() {}
  __device__ __forceinline__ void ident(LineBytes&, uint32_t, uint32_t, uint32_t, unsigned long long, unsigned long long) {}
  __device__ __forceinline__ void punct(uint32_t) {}
};
struct BlindSink {
  BlindHash h; const BlindKw* kw; const uint8_t* kind;
  __device__ __forceinline__ void number() { h.token('N'); }
  __device__ __forceinline__ void string() { h.token('S'); }
  __device__ __forceinline__ void ident(LineBytes&, uint32_t fam, uint32_t, uint32_t k, unsigned long long lo, unsigned long long hi) {
    const uint32_t kk = blind_kw_kind(kw, kind, lo, hi, k);
    if (kk & (fam == 1 ? KW_PY : KW_CJ)) {
      if (h.len) h.byte(' ');
      for (uint32_t j = 0; j < k; ++j) h.byte((uint32_t)((j < 8 ? lo >> (8 * j) : hi >> (8 * (j - 8))) & 0xFFu));
    } else {
      h.token((kk & (fam == 1 ? KW_PY_LIT : KW_CJ_LIT)) ? 'N' : 'I');
    }
  }
  __device__ __forceinline__ void punct(uint32_t c) { h.token(c); }
};

// Lexes line [s, e) of family fam (1 PY, 2 CJ) from state st, hands every token that begins on it to sink, and returns the
// state at its end.  The one copy of the lexing rules of docs/SPEC.md section 21.
template <typename Sink>
__device__ uint32_t blind_lex(LineBytes& B, uint32_t s, uint32_t e, uint32_t fam, uint32_t st, Sink& sink) {
  uint32_t i = s;
  if (st) {
    i = blind_close(B, s, e, fam, st);
    if (i == BLIND_NONE) return st;
  }
  while (i < e) {
    const uint32_t c = B.at(i), nx = i + 1 < e ? B.at(i + 1) : 0x100u;
    if (is_w(c)) { ++i; continue; }
    if (fam == 1 ? c == '#' : (c == '/' && nx == '/')) break;
    if (fam == 2 && c == '/' && nx == '*') {
      i = blind_close(B, i + 2, e, 2, 1);
      if (i == BLIND_NONE) return 1;
      continue;
    }
    if (is_digit(c) || (c == '.' && is_digit(nx))) {            // pp-number
      uint32_t prev = c;
      for (++i; i < e; ++i) {
        const uint32_t d = B.at(i);
        const bool exp = (prev | 0x20u) == 'e' || (prev | 0x20u) == 'p';
        if (!(is_ident(d) || d == '.' || ((d == '+' || d == '-') && exp) || (fam == 2 && d == '\'' && i + 1 < e && is_ident(B.at(i + 1)))))
          break;
        prev = d;
      }
      sink.number();
      continue;
    }
    if (blind_ident(c)) {
      unsigned long long lo = 0, hi = 0;
      const uint32_t i0 = i;
      bool pyp = true;                                          // every byte one of rRbBuUfF
      for (uint32_t d = c; i < e && blind_ident(d = B.at(i)); ++i) {
        const uint32_t k = i - i0;
        if (k < 8) lo |= (unsigned long long)d << (8 * k);
        else if (k < 16) hi |= (unsigned long long)d << (8 * (k - 8));
        const uint32_t l = d | 0x20u;
        pyp = pyp && (l == 'r' || l == 'b' || l == 'u' || l == 'f');
      }
      const uint32_t k = i - i0;
      if (i < e && (B.at(i) == '"' || B.at(i) == '\'')) {
        const bool prefix = fam == 1 ? pyp && k <= 2
                                     : k <= 3 && (lo == 'L' || lo == 'u' || lo == 'U' || lo == 0x3875u || lo == 'R' || lo == 0x524Cu ||
                                                  lo == 0x5275u || lo == 0x5255u || lo == 0x523875u);
        if (prefix) {
          uint32_t st2;
          i = blind_string(B, i, e, fam, st2);
          sink.string();
          if (st2) return st2;
          continue;
        }
      }
      sink.ident(B, fam, i0, k, lo, hi);
      continue;
    }
    if (c == '"' || c == '\'') {
      uint32_t st2;
      i = blind_string(B, i, e, fam, st2);
      sink.string();
      if (st2) return st2;
      continue;
    }
    sink.punct(c);
    ++i;
  }
  return 0;
}

// High bit of every byte of w that equals c (exact for the lowest such byte; a byte above one may be flagged too: the test
// below is only a filter).
__device__ __forceinline__ unsigned long long bytes_eq(unsigned long long w, uint32_t c) {
  const unsigned long long x = w ^ (0x0101010101010101ull * c);
  return (x - 0x0101010101010101ull) & ~x & 0x8080808080808080ull;
}

// File of line i: line_base[lo] <= i < line_base[lo + 1].
__device__ __forceinline__ uint32_t blind_file(const unsigned long long* line_base, uint32_t n, unsigned long long i) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (line_base[mid] <= i) lo = mid; else hi = mid; }
  return lo;
}

__global__ void __launch_bounds__(256) k_blind_state(DiffSide d, uint32_t n, unsigned long long total, uint8_t* fn) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const uint32_t f = blind_file(d.line_base, n, i), fam = blind_family(d.ext[f]);
  uint8_t out = BLIND_IDENTITY;
  if (fam) {
    const uint8_t* g = d.arena + (uint32_t)d.off[f];
    const uint32_t e = d.line_end[i], s = i == d.line_base[f] ? 0u : d.line_end[i - 1] + 1u;
    bool any = false;
    for (uint32_t wb = s & ~7u; wb < e && !any; wb += 8) {
      const unsigned long long w = __ldg(reinterpret_cast<const unsigned long long*>(g + wb));
      unsigned long long m = fam == 1 ? bytes_eq(w, '"') | bytes_eq(w, '\'') : bytes_eq(w, '*');
      if (wb < s) m &= ~0ull << (8 * (s - wb));
      if (e - wb < 8) m &= (1ull << (8 * (e - wb))) - 1;
      any = m != 0;
    }
    if (any) {
      LineBytes B{g, 1u, 0};
      NoSink ns;
      out = (uint8_t)(blind_lex(B, s, e, fam, 0, ns) | (blind_lex(B, s, e, fam, 1, ns) << 2) | ((fam == 1 ? blind_lex(B, s, e, fam, 2, ns) : 2u) << 4));
    }
  }
  fn[i] = out;
}

__device__ __forceinline__ uint32_t blind_apply(uint32_t f, uint32_t s) { return (f >> (2 * s)) & 3u; }
__device__ __forceinline__ uint32_t blind_then(uint32_t a, uint32_t b) {   // b after a
  return blind_apply(b, a & 3u) | (blind_apply(b, (a >> 2) & 3u) << 2) | (blind_apply(b, (a >> 4) & 3u) << 4);
}

// One warp per file: fn[l] (transfer function of line l) becomes the state at the start of line l.
__global__ void __launch_bounds__(256) k_blind_scan(const unsigned long long* line_base, uint32_t n, uint8_t* fn) {
  const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (f >= n) return;
  const unsigned long long b = line_base[f], e = line_base[f + 1];
  uint32_t carry = 0;
  for (unsigned long long l0 = b; l0 < e; l0 += 32) {
    const unsigned long long l = l0 + lane;
    uint32_t incl = l < e ? fn[l] : BLIND_IDENTITY;
#pragma unroll
    for (uint32_t k = 1; k < 32; k <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, incl, k);
      if (lane >= k) incl = blind_then(o, incl);
    }
    const uint32_t excl = __shfl_up_sync(0xffffffffu, incl, 1), all = __shfl_sync(0xffffffffu, incl, 31);
    if (l < e) fn[l] = (uint8_t)(lane ? blind_apply(excl, carry) : carry);
    carry = blind_apply(all, carry);
  }
}

__global__ void __launch_bounds__(256) k_blind_lines(DiffSide d, uint32_t n, unsigned long long total, const uint8_t* state,
                                                     unsigned long long* bhash, uint32_t* kept) {
  __shared__ BlindKw kw[BLIND_KW_SLOTS];
  __shared__ uint8_t kind[BLIND_KW_SLOTS];
  for (uint32_t t = threadIdx.x; t < BLIND_KW_SLOTS; t += blockDim.x) { kw[t] = c_blind_kw[t]; kind[t] = c_blind_kind[t]; }
  __syncthreads();
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const uint32_t f = blind_file(d.line_base, n, i), fam = blind_family(d.ext[f]);
  const uint8_t* g = d.arena + (uint32_t)d.off[f];
  const uint32_t e = d.line_end[i], s = i == d.line_base[f] ? 0u : d.line_end[i - 1] + 1u;
  BlindSink sk{BlindHash{0, 0, 0}, kw, kind};
  BlindHash& h = sk.h;
  if (fam) {
    LineBytes B{g, 1u, 0};
    blind_lex(B, s, e, fam, state[i], sk);
  } else {                                                      // tag 0: the content without its W bytes
    for (uint32_t wb = s & ~7u; wb < e; wb += 8) {
      unsigned long long w = __ldg(reinterpret_cast<const unsigned long long*>(g + wb));
      const uint32_t k0 = wb < s ? s - wb : 0, k1 = min(8u, e - wb);
      w >>= 8 * k0;
      for (uint32_t k = k0; k < k1; ++k, w >>= 8)
        if (!is_w((uint32_t)(w & 0xFF))) h.byte((uint32_t)(w & 0xFF));
    }
  }
  bhash[i] = mix_hash(canon61(h.acc), h.len);
  kept[i] = h.len != 0;
}

__global__ void __launch_bounds__(256) k_blind_compact(const uint32_t* kept, const unsigned long long* rank, const unsigned long long* bhash,
                                                       const uint8_t* line_flag, unsigned long long total, unsigned long long* kline,
                                                       unsigned long long* khash, uint8_t* kflag) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= total || !kept[i]) return;
  const unsigned long long r = rank[i];
  kline[r] = i; khash[r] = bhash[i]; kflag[r] = line_flag[i];
}

// One warp per file f <= n: kept_base[f] = the kept lines before the file, kassert[f] = its kept assertion lines (f < n).
__global__ void __launch_bounds__(256) k_blind_files(const unsigned long long* line_base, uint32_t n, const unsigned long long* rank,
                                                     const uint8_t* kflag, unsigned long long* kept_base, uint32_t* kassert) {
  const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (f > n) return;
  const unsigned long long b = rank[line_base[f]];
  if (lane == 0) kept_base[f] = b;
  if (f == n) return;
  const unsigned long long e = rank[line_base[f + 1]];
  uint32_t a = 0;
  for (unsigned long long l = b + lane; l < e; l += 32) a += kflag[l] != 0;
#pragma unroll
  for (int k = 16; k; k >>= 1) a += __shfl_xor_sync(0xffffffffu, a, k);
  if (lane == 0) kassert[f] = a;
}

}  // namespace tsm
