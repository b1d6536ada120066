// tsm_edit_kernels.cuh - assertion edits of revision pairs (docs/SPEC.md section 17): which deleted assertion line became which
// inserted one, from the line records of both sides, the edit marks of the DIFF_MARKS diff and the kept ranks of k_case_kept +
// xscan.  Lines are global indices of one side (< 2^32).  An entry is a changed assertion line of a traced pair; its key
// (pair << 32 | kept rank) names its hunk over the whole batch (the k-th kept line of new corresponds to the k-th of old).
//
//   k_edit_flag     one thread per line: flag[l] = 1 for a deleted (old side) / inserted (new side) assertion line of a traced pair.
//   xscan(flag)     the entry index of every flagged line: entries are in global line order.
//   k_edit_compact  one thread per line: entry = (key, stripped bytes) and the k_classify candidate (pair << 32 | line start).
//   k_edit_ranges   one thread per old entry: the new entries with its key (binary search; both lists are sorted by key).
//   k_edit_score    one warp per old entry of at most EDIT_SHORT_WORDS * 64 stripped bytes (the pattern): its match masks
//                   Peq[c] in shared memory, then one lane per candidate runs the bit-parallel LCS (Allison-Dix / Hyyro) over
//                   the inserted line with V in registers.  Candidates with score >= 30000 are appended to `kept`.
//   k_edit_score_long  the same for longer patterns, one warp per pattern, with Peq and each lane's V in a global slot of
//                   (256 + 32) * W words (W = ceil(len / 64)); the add carries from word to word.
#pragma once
#include "tsm_device.cuh"

namespace tsm {

constexpr uint32_t EDIT_SHORT_WORDS = 4;                  // patterns of up to 256 bytes take the register path
constexpr uint32_t EDIT_SCORE_MIN = 30000;                // 50 % on git's 60000 scale
constexpr uint32_t EDIT_WARPS = 4;                        // warps per block of k_edit_score (8 KiB of Peq each)

struct EditLine { unsigned long long key; uint32_t beg, len; };   // key; stripped line at arena[beg, beg + len)
struct EditCand { uint32_t old_e, new_e, score, pad; };           // a kept candidate: old and new entry, score

struct EditSide {                                         // one side's line records and marks
  const uint8_t* arena; const int32_t* off; const unsigned long long* line_base; uint32_t n_files;
  const uint32_t* line_end; const uint8_t* flag; const uint8_t* mark; const uint8_t* traced;
};

__device__ __forceinline__ uint32_t edit_file_of(const EditSide& s, uint32_t l) {   // line_base[f] <= l < line_base[f + 1]
  uint32_t lo = 0, hi = s.n_files;
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s.line_base[mid] <= l) lo = mid; else hi = mid; }
  return lo;
}

__global__ void __launch_bounds__(256) k_edit_flag(EditSide s, uint32_t total, uint32_t* flag) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= total) return;
  flag[l] = s.mark[l] && s.flag[l] && s.traced[edit_file_of(s, l)];
}

__global__ void __launch_bounds__(256) k_edit_compact(EditSide s, uint32_t total, const uint32_t* flag, const unsigned long long* pos,
                                                      const unsigned long long* rank, EditLine* out, unsigned long long* cand) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= total || !flag[l]) return;
  const uint32_t f = edit_file_of(s, l);
  const uint32_t start = l == s.line_base[f] ? 0u : s.line_end[l - 1] + 1u;
  const uint8_t* a = s.arena + (uint32_t)s.off[f];
  uint32_t b = start, e = s.line_end[l];
  while (b < e && is_w(a[b])) ++b;
  while (e > b && is_w(a[e - 1])) --e;
  const unsigned long long k = pos[l];
  out[k] = EditLine{((unsigned long long)f << 32) | rank[l], (uint32_t)s.off[f] + b, e - b};
  cand[k] = ((unsigned long long)f << 32) | start;
}

__global__ void __launch_bounds__(256) k_edit_ranges(const EditLine* olds, uint32_t n_old, const EditLine* news, uint32_t n_new,
                                                     uint2* range) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_old) return;
  const unsigned long long key = olds[i].key;
  uint32_t lo = 0, hi = n_new;                             // first new entry with key >= key
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (news[mid].key < key) lo = mid + 1; else hi = mid; }
  uint32_t e = lo, top = n_new;                            // first new entry with key > key
  while (e < top) { const uint32_t mid = (e + top) >> 1; if (news[mid].key <= key) e = mid + 1; else top = mid; }
  range[i] = make_uint2(lo, e);
}

__device__ __forceinline__ void edit_keep(uint32_t i, uint32_t j, uint32_t lcs, uint32_t la, uint32_t lb, EditCand* kept,
                                          uint32_t cap, uint32_t* n_kept) {
  const uint32_t score = la + lb ? (uint32_t)(120000ull * lcs / (la + lb)) : 0u;   // (an assertion line is never empty)
  if (score < EDIT_SCORE_MIN) return;
  const uint32_t slot = atomicAdd(n_kept, 1u);
  if (slot < cap) kept[slot] = EditCand{i, j, score, 0};
}

// The bytes arena[beg, beg + len) one at a time, read 8 at a time (the arena has 4 KiB of padding behind the last file).
template <typename F>
__device__ __forceinline__ void edit_bytes(const uint8_t* arena, uint32_t beg, uint32_t len, F&& fn) {
  const uint32_t end = beg + len;
  for (uint32_t q = beg & ~7u; q < end; q += 8) {
    unsigned long long w = __ldg(reinterpret_cast<const unsigned long long*>(arena + q));
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) {
      if (q + k >= beg && q + k < end) fn((uint32_t)(w & 0xFFu));
      w >>= 8;
    }
  }
}

// lcs of the pattern (match masks peq[c * W + w], m bytes) and the text arena[beg, beg + len): V in registers.
template <int W>
__device__ __forceinline__ uint32_t edit_lcs_regs(const unsigned long long* peq, uint32_t m, const uint8_t* arena, uint32_t beg, uint32_t len) {
  unsigned long long V[W];
#pragma unroll
  for (int w = 0; w < W; ++w) V[w] = ~0ull;
  edit_bytes(arena, beg, len, [&](uint32_t c) {
    const unsigned long long* p = peq + c * W;
    unsigned long long carry = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const unsigned long long v = V[w], pm = p[w], u = v & pm;
      const unsigned long long s1 = v + u, s2 = s1 + carry;
      carry = (s1 < v) | (s2 < s1);
      V[w] = s2 | (v & ~pm);
    }
  });
  uint32_t ones = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    const uint32_t lo = (uint32_t)w * 64u;
    const unsigned long long mask = m >= lo + 64 ? ~0ull : (m > lo ? (1ull << (m - lo)) - 1ull : 0ull);
    ones += (uint32_t)__popcll(V[w] & mask);
  }
  return m - ones;
}

template <int W>
__device__ __forceinline__ void edit_warp(unsigned long long* peq, uint32_t i, const EditLine& a, const uint2 r, const EditLine* news,
                                          const uint8_t* arena_old, const uint8_t* arena_new, EditCand* kept, uint32_t cap,
                                          uint32_t* n_kept, uint32_t lane) {
  for (uint32_t x = lane; x < 256u * W; x += 32) peq[x] = 0;
  __syncwarp();
  for (uint32_t q = lane; q < a.len; q += 32) atomicOr(&peq[(uint32_t)arena_old[a.beg + q] * W + (q >> 6)], 1ull << (q & 63));
  __syncwarp();
  for (uint32_t j = r.x + lane; j < r.y; j += 32) {
    const EditLine b = news[j];
    edit_keep(i, j, edit_lcs_regs<W>(peq, a.len, arena_new, b.beg, b.len), a.len, b.len, kept, cap, n_kept);
  }
  __syncwarp();                                            // every lane is done with peq before the next pattern clears it
}

// ids: the old entries of at most EDIT_SHORT_WORDS words with candidates; persistent warps, one pattern at a time.
__global__ void __launch_bounds__(EDIT_WARPS * 32) k_edit_score(const uint32_t* ids, uint32_t n_ids, const EditLine* olds, const EditLine* news,
                                                                const uint2* range, const uint8_t* arena_old, const uint8_t* arena_new,
                                                                EditCand* kept, uint32_t cap, uint32_t* n_kept) {
  __shared__ unsigned long long s_peq[EDIT_WARPS][256 * EDIT_SHORT_WORDS];
  const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warps = gridDim.x * EDIT_WARPS;
  unsigned long long* peq = s_peq[wib];
  for (uint32_t t = blockIdx.x * EDIT_WARPS + wib; t < n_ids; t += warps) {
    const uint32_t i = ids[t];
    const EditLine a = olds[i];
    const uint2 r = range[i];
    if (a.len <= 64) edit_warp<1>(peq, i, a, r, news, arena_old, arena_new, kept, cap, n_kept, lane);
    else if (a.len <= 128) edit_warp<2>(peq, i, a, r, news, arena_old, arena_new, kept, cap, n_kept, lane);
    else edit_warp<4>(peq, i, a, r, news, arena_old, arena_new, kept, cap, n_kept, lane);
  }
}

// ids[t] (t < n_ids): old entries longer than the register path; slot_base[t]: the word offset of its slot in `scratch`
// ((256 + 32) * W words: Peq, then V of each lane word-major), which the host zeroed.
__global__ void __launch_bounds__(128) k_edit_score_long(const uint32_t* ids, const unsigned long long* slot_base, uint32_t n_ids,
                                                         const EditLine* olds, const EditLine* news, const uint2* range,
                                                         const uint8_t* arena_old, const uint8_t* arena_new, unsigned long long* scratch, EditCand* kept,
                                                         uint32_t cap, uint32_t* n_kept) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= n_ids) return;
  const uint32_t i = ids[t];
  const EditLine a = olds[i];
  const uint2 r = range[i];
  const uint32_t W = (a.len + 63) >> 6;
  unsigned long long* peq = scratch + slot_base[t];
  unsigned long long* V = peq + 256ull * W;
  for (uint32_t q = lane; q < a.len; q += 32) atomicOr(&peq[(size_t)arena_old[a.beg + q] * W + (q >> 6)], 1ull << (q & 63));
  __syncwarp();
  __threadfence_block();
  for (uint32_t j0 = r.x; j0 < r.y; j0 += 32) {            // the whole warp per round (lanes without a candidate idle)
    const uint32_t j = j0 + lane;
    if (j >= r.y) break;
    const EditLine b = news[j];
    for (uint32_t w = 0; w < W; ++w) V[(size_t)w * 32 + lane] = ~0ull;
    edit_bytes(arena_new, b.beg, b.len, [&](uint32_t c) {
      const unsigned long long* p = peq + (size_t)c * W;
      unsigned long long carry = 0;
      for (uint32_t w = 0; w < W; ++w) {
        const unsigned long long v = V[(size_t)w * 32 + lane], pm = p[w], u = v & pm;
        const unsigned long long s1 = v + u, s2 = s1 + carry;
        carry = (s1 < v) | (s2 < s1);
        V[(size_t)w * 32 + lane] = s2 | (v & ~pm);
      }
    });
    uint32_t ones = 0;
    for (uint32_t w = 0; w < W; ++w) {
      const uint32_t lo = w * 64u;
      const unsigned long long mask = a.len >= lo + 64 ? ~0ull : (1ull << (a.len - lo)) - 1ull;
      ones += (uint32_t)__popcll(V[(size_t)w * 32 + lane] & mask);
    }
    edit_keep(i, j, a.len - ones, a.len, b.len, kept, cap, n_kept);
  }
}

}  // namespace tsm
