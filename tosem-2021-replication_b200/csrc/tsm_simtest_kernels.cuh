// Similar tests (docs/SPEC.md section 23): the pairs of section-18 tests whose sequences of kept blind lines (section 21) have
// a Dice-over-LCS score of at least P %.  An exact prefix filter over tokens (h, j) - the j-th occurrence of blind hash h in a
// test - in a global rare-first order gives the candidates; a virtual candidate space over the posting lists of the prefix
// tokens is walked in chunks, and each candidate that passes the size filter and whose list is the first token both prefixes
// share is verified by a bit-parallel LCS, one warp per candidate.
#pragma once
#include "tsm_device.cuh"

namespace tsm {

constexpr unsigned long long ST_EMPTY = ~0ull;            // empty slot of the token tables
constexpr uint32_t ST_CHUNK = 1u << 22;                   // virtual candidates per enumeration launch = survivor buffer entries
constexpr uint32_t ST_NONE = 0xFFFFFFFFu;

struct StToken { uint32_t cnt, hslot, j, pslot; };        // a prefix token: order key (cnt, hslot, j), its posting list

// Slot of key h in an open-addressing table of mask + 1 slots (keys ST_EMPTY when free); h == ST_EMPTY has slot mask + 1.
__device__ __forceinline__ uint32_t st_insert(unsigned long long* key, uint32_t mask, unsigned long long h) {
  if (h == ST_EMPTY) return mask + 1;
  uint32_t s = (uint32_t)((h * 0x9E3779B97F4A7C15ull) >> 32) & mask;
  for (;;) {
    const unsigned long long old = atomicCAS(&key[s], ST_EMPTY, h);
    if (old == ST_EMPTY || old == h) return s;
    s = (s + 1) & mask;
  }
}

// One thread per test: its first kept line kbeg, kept lines kk, prefix length q (0 unless compared) and, on the kept lines of a
// compared test, ktest = the test.  kmax: the largest kk of a compared test.
__global__ void __launch_bounds__(256) k_st_tests(const tsm_smell_test* tests, uint32_t nt, const unsigned long long* line_base,
                                                  const unsigned long long* rank, uint32_t min_lines, uint32_t P, uint32_t* kbeg,
                                                  uint32_t* kk, uint32_t* q, uint32_t* ktest, uint32_t* kmax) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const tsm_smell_test x = tests[t];
  const unsigned long long l0 = line_base[x.file] + (uint32_t)x.line;
  const uint32_t b = (uint32_t)rank[l0], e = (uint32_t)rank[l0 + (uint32_t)x.body_lines], k = e - b;
  kbeg[t] = b;
  kk[t] = k;
  const bool cmp = k >= min_lines;
  const uint32_t alpha = (uint32_t)(((unsigned long long)P * k + (199u - P)) / (200u - P));   // ceil(P k / (200 - P)) <= k
  q[t] = cmp ? k - alpha + 1u : 0u;
  if (!cmp) return;
  atomicMax(kmax, k);
  for (uint32_t i = b; i < e; ++i) ktest[i] = t;
}

// One thread per kept line of a compared test: its hash's slot in the count table, and the count of that hash.
__global__ void __launch_bounds__(256) k_st_count(const unsigned long long* khash, const uint32_t* ktest, uint32_t nk,
                                                  unsigned long long* key, uint32_t mask, uint32_t* cnt, uint2* eord) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nk || ktest[i] == ST_NONE) return;
  const uint32_t s = st_insert(key, mask, khash[i]);
  eord[i].y = s;
  atomicAdd(&cnt[s], 1u);
}
__global__ void __launch_bounds__(256) k_st_order(const uint32_t* ktest, uint32_t nk, const uint32_t* cnt, uint2* eord) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nk || ktest[i] == ST_NONE) return;
  eord[i].x = cnt[eord[i].y];
}

// One thread per kept line i of a compared test t: its token (h, j) and its rank among t's tokens in the order (cnt, hslot, j).
// A token of rank < q[t] is in the prefix: written at pbase[t] + rank and counted in its posting list (pkey on hslot << 32 | j).
__global__ void __launch_bounds__(256) k_st_prefix(const uint32_t* ktest, uint32_t nk, const uint2* eord, const uint32_t* kbeg,
                                                   const uint32_t* kk, const uint32_t* q, const unsigned long long* pbase,
                                                   unsigned long long* pkey, uint32_t pmask, uint32_t* pcnt, StToken* tok,
                                                   uint32_t* ptest) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nk) return;
  const uint32_t t = ktest[i];
  if (t == ST_NONE) return;
  const uint2 me = eord[i];
  const uint32_t b = kbeg[t], e = b + kk[t];
  uint32_t r = 0, j = 0;
  for (uint32_t x = b; x < e; ++x) {
    const uint2 o = eord[x];
    if (o.y == me.y) j += x < i;
    else r += o.x < me.x || (o.x == me.x && o.y < me.y);
  }
  r += j;
  if (r >= q[t]) return;
  const unsigned long long idx = pbase[t] + r;
  const uint32_t ps = st_insert(pkey, pmask, (unsigned long long)me.y << 32 | j);
  tok[idx] = StToken{me.x, me.y, j, ps};
  ptest[idx] = t;
  atomicAdd(&pcnt[ps], 1u);
}

// One thread per prefix token (np = pbase[nt] of them): its test into its posting list, mem[mbase[list] ...].
__global__ void __launch_bounds__(256) k_st_lists(const StToken* tok, const uint32_t* ptest, const unsigned long long* np,
                                                  const unsigned long long* mbase, uint32_t* cursor, uint32_t* mem) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= *np) return;
  const uint32_t ps = tok[i].pslot;
  mem[mbase[ps] + atomicAdd(&cursor[ps], 1u)] = ptest[i];
}

// The candidates of a list of m tests, m (m - 1) / 2, scanned exclusively into cbase[n + 1] (tile sums, k_xscan_top, apply).
__device__ __forceinline__ unsigned long long st_pairs_of(uint32_t m) { return (unsigned long long)m * (m ? m - 1u : 0u) / 2u; }
// Tile sums and apply of an exclusive scan of per-list u64 counts cnt(i), as the xscan of tsm_lines_kernels.cuh.
template <typename Cnt> __device__ __forceinline__ void st_csums(Cnt cnt, uint32_t n, unsigned long long* bsum) {
  __shared__ unsigned long long sh[8];
  const uint32_t i0 = blockIdx.x * XS_TILE + threadIdx.x * 4u;
  unsigned long long s = 0;
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) if (i0 + k < n) s += cnt(i0 + k);
  s = block_sum(s, sh);
  if (threadIdx.x == 0) bsum[blockIdx.x] = s;
}
template <typename Cnt> __device__ __forceinline__ void st_capply(Cnt cnt, uint32_t n, const unsigned long long* bsum, unsigned long long* out) {
  __shared__ unsigned long long wsum[8];
  const uint32_t i0 = blockIdx.x * XS_TILE + threadIdx.x * 4u;
  unsigned long long v[4], s = 0;
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) { v[k] = i0 + k < n ? cnt(i0 + k) : 0ull; s += v[k]; }
  unsigned long long incl = s;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
  if (lane == 31) wsum[w] = incl;
  __syncthreads();
  unsigned long long off = bsum[blockIdx.x] + incl - s;
  for (int k = 0; k < w; ++k) off += wsum[k];
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) { if (i0 + k < n) out[i0 + k] = off; off += v[k]; }
  if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = bsum[gridDim.x];
}
__global__ void __launch_bounds__(256) k_st_csums(const uint32_t* pcnt, uint32_t n, unsigned long long* bsum) {
  st_csums([=](uint32_t i) { return st_pairs_of(pcnt[i]); }, n, bsum);
}
__global__ void __launch_bounds__(256) k_st_capply(const uint32_t* pcnt, uint32_t n, const unsigned long long* bsum, unsigned long long* out) {
  st_capply([=](uint32_t i) { return st_pairs_of(pcnt[i]); }, n, bsum, out);
}

struct StEnum {
  const unsigned long long* cbase; uint32_t n_lists;      // candidates before each list [n_lists + 1]
  const unsigned long long* mbase; const uint32_t* mem;   // the tests of each list
  const uint32_t* kk; const uint32_t* q; const unsigned long long* pbase; const StToken* tok;
  uint32_t P;
  uint2* surv; uint32_t* n_surv;
};

__device__ __forceinline__ bool st_less(const StToken& a, const StToken& b) {
  return a.cnt != b.cnt ? a.cnt < b.cnt : a.hslot != b.hslot ? a.hslot < b.hslot : a.j < b.j;
}

// The candidate pair of tests x and y of list s: kept (appended to the survivors) when it passes the size filter and the
// list's token is the first token the two prefixes share.
__device__ __forceinline__ void st_keep(const StEnum& a, uint32_t s, uint32_t x, uint32_t y) {
  const uint32_t ta = min(x, y), tb = max(x, y);
  const uint32_t ka = a.kk[ta], kb = a.kk[tb];
  if (200ull * min(ka, kb) < (unsigned long long)a.P * (ka + kb)) return;
  const StToken* pa = a.tok + a.pbase[ta];
  const StToken* pb = a.tok + a.pbase[tb];
  const uint32_t qa = a.q[ta], qb = a.q[tb];
  uint32_t ia = 0, ib = 0, first = ST_NONE;
  while (ia < qa && ib < qb) {
    const StToken u = pa[ia], w = pb[ib];
    if (st_less(u, w)) ++ia;
    else if (st_less(w, u)) ++ib;
    else { first = u.pslot; break; }
  }
  if (first != s) return;
  a.surv[atomicAdd(a.n_surv, 1u)] = make_uint2(ta, tb);
}

// Grid-stride over the virtual candidates [c0, c0 + n): candidate v is the pair (i, j), i < j, of the list whose range of
// cbase holds v.  Kept when it passes the size filter and the list's token is the first token the two prefixes share.
__global__ void __launch_bounds__(256) k_st_enum(StEnum a, unsigned long long c0, unsigned long long n) {
  for (unsigned long long v = c0 + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; v < c0 + n;
       v += (unsigned long long)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = a.n_lists - 1;                  // the last list s with cbase[s] <= v (it holds v)
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo + 1) / 2;
      if (a.cbase[mid] <= v) lo = mid; else hi = mid - 1;
    }
    const uint32_t s = lo;
    const unsigned long long r = v - a.cbase[s];
    unsigned long long j = (unsigned long long)((1.0 + sqrt(1.0 + 8.0 * (double)r)) * 0.5);
    while (j * (j - 1) / 2 > r) --j;
    while ((j + 1) * j / 2 <= r) ++j;
    const unsigned long long i = r - j * (j - 1) / 2;
    st_keep(a, s, a.mem[a.mbase[s] + i], a.mem[a.mbase[s] + j]);
  }
}

// LCS of the pattern pat[m] and the text txt[n] (Allison-Dix / Hyyro over 64-bit words), computed by one warp.  The match mask
// of a text element is built by ballots, 32 pattern elements each.  m <= 64: V in a register of every lane.  Otherwise lane w of
// a block of 32 words holds word w - in a register when m <= 2048, else in the warp's scratch vs - and the carries between the
// words of a block come from one 32-bit addition of the lanes' generate and propagate ballots.
__device__ __forceinline__ uint32_t st_lcs(const unsigned long long* pat, uint32_t m, const unsigned long long* txt, uint32_t n, unsigned long long* vs,
                           uint32_t lane) {
  const uint32_t FULL = 0xffffffffu;
  const uint32_t W = (m + 63) >> 6;
  if (W == 1) {
    const bool v0 = lane < m, v1 = lane + 32 < m;
    const unsigned long long p0 = v0 ? pat[lane] : 0ull, p1 = v1 ? pat[lane + 32] : 0ull;
    unsigned long long V = ~0ull;
    for (uint32_t r = 0; r < n; r += 32) {
      const unsigned long long t = r + lane < n ? txt[r + lane] : 0ull;
      const uint32_t ne = min(32u, n - r);
      for (uint32_t e = 0; e < ne; ++e) {
        const unsigned long long y = __shfl_sync(FULL, t, (int)e);
        const unsigned long long pm = (unsigned long long)__ballot_sync(FULL, v0 && p0 == y) |
                                      (unsigned long long)__ballot_sync(FULL, v1 && p1 == y) << 32;
        V = (V + (V & pm)) | (V & ~pm);
      }
    }
    return m - (uint32_t)__popcll(V & (m == 64 ? ~0ull : (1ull << m) - 1ull));
  }
  const uint32_t nbk = (W + 31) >> 5;
  unsigned long long Vr = ~0ull;
  if (nbk > 1) {
    for (uint32_t w = lane; w < nbk * 32; w += 32) vs[w] = ~0ull;
    __syncwarp();
  }
  for (uint32_t r = 0; r < n; r += 32) {
    const unsigned long long t = r + lane < n ? txt[r + lane] : 0ull;
    const uint32_t ne = min(32u, n - r);
    for (uint32_t e = 0; e < ne; ++e) {
      const unsigned long long y = __shfl_sync(FULL, t, (int)e);
      uint32_t cin = 0;
      for (uint32_t bk = 0; bk < nbk; ++bk) {
        const uint32_t w0 = bk * 32, nw = min(32u, W - w0);
        unsigned long long pm = 0;
#pragma unroll 8
        for (uint32_t wi = 0; wi < nw; ++wi) {
          const uint32_t q0 = (w0 + wi) * 64 + lane, q1 = q0 + 32;
          const uint32_t lo = __ballot_sync(FULL, q0 < m && pat[q0] == y), hi = __ballot_sync(FULL, q1 < m && pat[q1] == y);
          if (lane == wi) pm = lo | (unsigned long long)hi << 32;
        }
        const bool act = lane < nw;
        const unsigned long long v = nbk == 1 ? Vr : (act ? vs[w0 + lane] : ~0ull);
        const unsigned long long s1 = v + (v & pm);
        const uint32_t G = __ballot_sync(FULL, act && s1 < v), Pp = __ballot_sync(FULL, act && s1 == ~0ull);
        const unsigned long long x = (unsigned long long)(G | Pp), S = x + G + cin;
        const uint32_t carry = (((uint32_t)S ^ (uint32_t)x ^ G) >> lane) & 1u;   // the carry into this lane's word
        const unsigned long long nv = (s1 + carry) | (v & ~pm);
        if (nbk == 1) Vr = nv;
        else if (act) vs[w0 + lane] = nv;
        cin = (uint32_t)(S >> 32);
      }
    }
  }
  uint32_t ones = 0;
  for (uint32_t bk = 0; bk < nbk; ++bk) {
    const uint32_t w = bk * 32 + lane;
    if (w >= W) continue;
    const unsigned long long v = nbk == 1 ? Vr : vs[w];
    const uint32_t lo = w * 64u;
    ones += (uint32_t)__popcll(v & (m >= lo + 64 ? ~0ull : (1ull << (m - lo)) - 1ull));
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) ones += __shfl_xor_sync(FULL, ones, d);
  __syncwarp();
  return m - ones;
}

// Persistent warps over the survivors: the shorter sequence (a on a tie) is the pattern.  A passing pair is appended to pairs.
__global__ void __launch_bounds__(256) k_st_verify(const uint2* surv, const uint32_t* n_surv, const uint32_t* kbeg, const uint32_t* kk,
                                                   const unsigned long long* khash, uint32_t P, unsigned long long* scratch,
                                                   uint32_t slot_words, tsm_similar_pair* pairs, uint32_t* n_pairs) {
  const uint32_t lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t ns = *n_surv;
  unsigned long long* vs = scratch ? scratch + (size_t)warp * slot_words : nullptr;
  for (uint32_t c = warp; c < ns; c += warps) {
    const uint2 ab = surv[c];
    const uint32_t ka = kk[ab.x], kb = kk[ab.y];
    const bool a_pat = ka <= kb;
    const uint32_t p = a_pat ? ab.x : ab.y, o = a_pat ? ab.y : ab.x;
    const uint32_t lcs = st_lcs(khash + kbeg[p], kk[p], khash + kbeg[o], kk[o], vs, lane);
    if (lane == 0 && 200ull * lcs >= (unsigned long long)P * (ka + kb))
      pairs[atomicAdd(n_pairs, 1u)] = tsm_similar_pair{(int32_t)ab.x, (int32_t)ab.y, lcs,
                                                       (uint32_t)(120000ull * lcs / ((unsigned long long)ka + kb))};
  }
}

// ------------------------------------------------------------------------------------- SPEC section 24 similar-test churn
// One warp per matched test (old test o, new test n): same[k] = 1 when neither body holds a marked line (deleted in the old
// body, inserted in the new), the bodies have equal body_lines and the two sequences of kept blind hashes are equal.  A
// test's kept lines are [rank[l0], rank[l0 + body_lines]) of its side's blind front, l0 its header line.
struct ScChangeSide {
  const tsm_smell_test* tests; const unsigned long long* line_base; const uint8_t* mark; const unsigned long long* rank;
  const unsigned long long* khash;
};
__global__ void __launch_bounds__(256) k_sc_change(ScChangeSide o, ScChangeSide w, const uint2* match, uint32_t n, uint8_t* same) {
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += warps) {
    const uint2 m = match[k];
    const tsm_smell_test to = o.tests[m.x], tn = w.tests[m.y];
    const unsigned long long lo = o.line_base[to.file] + (uint32_t)to.line, ln = w.line_base[tn.file] + (uint32_t)tn.line;
    const unsigned long long bo = o.rank[lo], bn = w.rank[ln];
    const uint32_t ko = (uint32_t)(o.rank[lo + (uint32_t)to.body_lines] - bo), kn = (uint32_t)(w.rank[ln + (uint32_t)tn.body_lines] - bn);
    bool eq = to.body_lines == tn.body_lines && ko == kn;
    const uint32_t nb = (uint32_t)to.body_lines;
    for (uint32_t i0 = 0; eq && i0 < nb; i0 += 32) {     // (eq and the bounds are the same in every lane)
      const uint32_t i = i0 + lane;
      eq = !__any_sync(FULL, i < nb && (o.mark[lo + i] | w.mark[ln + i]));
    }
    const unsigned long long* ho = o.khash + bo;
    const unsigned long long* hn = w.khash + bn;
    for (uint32_t i0 = 0; eq && i0 < ko; i0 += 32) {
      const uint32_t i = i0 + lane;
      eq = __all_sync(FULL, i >= ko || ho[i] == hn[i]);
    }
    if (lane == 0) same[k] = eq;
  }
}

// One thread per prefix token: the dirty tests of each posting list, dcnt[list].
__global__ void __launch_bounds__(256) k_sc_dirty(const StToken* tok, const uint32_t* ptest, const unsigned long long* np,
                                                  const uint8_t* dirty, uint32_t* dcnt) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= *np || !dirty[ptest[i]]) return;
  atomicAdd(&dcnt[tok[i].pslot], 1u);
}

// k_st_lists with the dirty tests of every list first: a dirty test takes the next of the list's first dcnt slots, a clean
// one the next slot behind them.
__global__ void __launch_bounds__(256) k_sc_lists(const StToken* tok, const uint32_t* ptest, const unsigned long long* np,
                                                  const unsigned long long* mbase, const uint8_t* dirty, const uint32_t* dcnt,
                                                  uint32_t* dcur, uint32_t* ccur, uint32_t* mem) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= *np) return;
  const uint32_t ps = tok[i].pslot, t = ptest[i];
  mem[mbase[ps] + (dirty[t] ? atomicAdd(&dcur[ps], 1u) : dcnt[ps] + atomicAdd(&ccur[ps], 1u))] = t;
}

// The restricted candidates of a list of m tests whose first d are dirty: the pairs (i, j), i < d, i < j < m, row i
// (m - 1 - i of them) starting at sc_row(m, i) = i m - i (i + 1) / 2; d m - d (d + 1) / 2 in all (m (m - 1) / 2 when d = m).
__device__ __forceinline__ unsigned long long sc_row(uint32_t m, unsigned long long i) { return i * m - i * (i + 1) / 2; }
__global__ void __launch_bounds__(256) k_sc_csums(const uint32_t* pcnt, const uint32_t* dcnt, uint32_t n, unsigned long long* bsum) {
  st_csums([=](uint32_t i) { return sc_row(pcnt[i], dcnt[i]); }, n, bsum);
}
__global__ void __launch_bounds__(256) k_sc_capply(const uint32_t* pcnt, const uint32_t* dcnt, uint32_t n, const unsigned long long* bsum,
                                                   unsigned long long* out) {
  st_capply([=](uint32_t i) { return sc_row(pcnt[i], dcnt[i]); }, n, bsum, out);
}

// k_st_enum over the restricted space: candidate v is the pair (i, j) of the list whose range of cbase holds v, i found from
// the row offsets (the root of i^2 - (2m - 1) i + 2r = 0, then corrected), with the same filters; so every pair of tests of
// which at least one is dirty is kept once, and no pair of two clean tests is looked at.
__global__ void __launch_bounds__(256) k_sc_enum(StEnum a, const uint32_t* pcnt, const uint32_t* dcnt, unsigned long long c0,
                                                 unsigned long long n) {
  for (unsigned long long v = c0 + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; v < c0 + n;
       v += (unsigned long long)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = a.n_lists - 1;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo + 1) / 2;
      if (a.cbase[mid] <= v) lo = mid; else hi = mid - 1;
    }
    const uint32_t s = lo, m = pcnt[s], d = dcnt[s];
    const unsigned long long r = v - a.cbase[s];
    const double b = 2.0 * m - 1.0, disc = b * b - 8.0 * (double)r;
    unsigned long long i = (unsigned long long)fmax(0.0, (b - sqrt(fmax(disc, 0.0))) * 0.5);
    if (i >= d) i = d - 1;
    while (i > 0 && sc_row(m, i) > r) --i;
    while (i + 1 < d && sc_row(m, i + 1) <= r) ++i;
    const unsigned long long j = i + 1 + (r - sc_row(m, i));
    st_keep(a, s, a.mem[a.mbase[s] + i], a.mem[a.mbase[s] + j]);
  }
}

}  // namespace tsm
