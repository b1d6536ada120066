// tsm_clone_kernels.cuh - duplicated test code (docs/SPEC.md section 15): the maximal classes of repeated windows of n
// lines, from the line records (tsm_lines_kernels.cuh) and the n-gram keys of k_ngrams.  Positions are global line
// indices (< 2^32: the scan's staging arrays hold at most 0xFFFFFFF0 lines).
//
// Grouping without a global sort:
//   k_clone_insert   one thread per line: is a window of n lines starting there (inside its file, not all empty)?  Its
//                    key goes into an open-addressing table (slot = key & mask, linear probing; key 0 marks an empty slot,
//                    so a window whose key is 0 takes the side slot mask + 1): count (atomicAdd) and first position
//                    (atomicMax of ~p) in one 16-byte slot.  slot_of[p] = its slot.
//   k_clone_preds    per duplicated window: pred_lo / pred_hi of its slot = min / max of the slot of p - 1 (NONE when p - 1
//                    is no window of the same file).  Slot ids depend on insertion order but are only compared for equality.
//   k_clone_heads    per duplicated window: its group extends one to the left (pred_lo == pred_hi != NONE with the same
//                    count) -> ext[p]; else p is the head of a class when it is the group's first position -> head[p].
//   xscan(head)      class numbers in representative order; xscan(dup) the prefix counts of the coverage.
//   k_clone_classes  per head: rep / size of its class, slot -> class, classes of more than 32 fragments listed.
//   xscan(size)      class_base.
//   k_clone_length   persistent warps, one class at a time: 32 ext flags per ballot from the representative on.
// Members and coverage:
//   k_clone_scatter  every window of a head slot to its class segment (per-class cursor); the segments are then sorted:
//   k_clone_sort_warp   up to 32 fragments in registers (one warp per class),
//   k_clone_sort_cta    more, one CTA per class: up to SIM_SMEM_LINES in shared memory, larger ones in tiles through
//                       global memory (bitonic_merge_tiles, as k_sim_sort does for large files).
//   k_clone_cover    one warp per file: line l is duplicated iff C[l+1] - C[max(b, l-n+1)] > 0.
#pragma once
#include "tsm_device.cuh"
#include "tsm_similar_kernels.cuh"

namespace tsm {

constexpr uint32_t CLONE_NONE = 0xFFFFFFFFu;
constexpr uint32_t CLONE_WARP_MAX = 32;                   // classes of up to this many fragments are sorted by one warp
constexpr uint8_t CW_FILE_HEAD = 1;                        // wflag: the line is the first line of its file

struct CloneSlot { unsigned long long key; uint32_t count, nfirst; };   // nfirst = ~(first position)
static_assert(sizeof(CloneSlot) == 16, "one sector-aligned 16-byte slot per probe");

// Content of line i (SPEC section 3: the line minus one trailing CR) is empty.
__device__ __forceinline__ bool line_empty(const uint8_t* file, const uint32_t* line_end, unsigned long long first, unsigned long long i) {
  const uint32_t end = line_end[i], start = i == first ? 0u : line_end[i - 1] + 1u;
  return end == start || (end == start + 1 && file[start] == 0x0D);
}

// SKIP_EMPTY: a window of n empty lines is no window (read from arena, off and line_end).  The blind clones
// (tsm_blind_kernels.cuh) group compacted kept lines, none of them empty, and pass no bytes.
template <bool SKIP_EMPTY>
__global__ void __launch_bounds__(256) k_clone_insert(const unsigned long long* key, const unsigned long long* line_base, uint32_t n_files,
                                                      const uint32_t* line_end, const uint8_t* arena, const int32_t* off, uint32_t total,
                                                      uint32_t n, CloneSlot* table, uint32_t mask, uint32_t* slot_of, uint8_t* wflag) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  uint32_t lo = 0, hi = n_files;                           // file of line p: line_base[lo] <= p < line_base[hi]
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (line_base[mid] <= p) lo = mid; else hi = mid; }
  const unsigned long long b = line_base[lo], e = line_base[lo + 1];
  uint32_t s = CLONE_NONE;
  if ((unsigned long long)p + n <= e) {
    bool empty = SKIP_EMPTY;
    if (SKIP_EMPTY) {
      const uint8_t* file = arena + off[lo];
      for (uint32_t k = 0; k < n && empty; ++k) empty = line_empty(file, line_end, b, (unsigned long long)p + k);
    }
    if (!empty) {
      const unsigned long long k = key[p];
      if (k == 0) s = mask + 1;
      else
        for (s = (uint32_t)k & mask;; s = (s + 1) & mask) {   // a stale 0 only costs a CAS: a key, once set, never changes
          const unsigned long long have = table[s].key;
          if (have == k) break;
          if (have == 0) {
            const unsigned long long was = atomicCAS(&table[s].key, 0ull, k);
            if (was == 0 || was == k) break;
          }
        }
      atomicAdd(&table[s].count, 1u);
      atomicMax(&table[s].nfirst, ~p);
    }
  }
  slot_of[p] = s;
  wflag[p] = p == b ? CW_FILE_HEAD : 0;
}

__global__ void __launch_bounds__(256) k_clone_preds(const CloneSlot* table, const uint32_t* slot_of, const uint8_t* wflag, uint32_t total,
                                                     uint32_t* pred_lo, uint32_t* pred_hi) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const uint32_t s = slot_of[p];
  if (s == CLONE_NONE || table[s].count < 2) return;
  const uint32_t v = (wflag[p] & CW_FILE_HEAD) ? CLONE_NONE : slot_of[p - 1];
  atomicMin(&pred_lo[s], v);
  atomicMax(&pred_hi[s], v);
}

__global__ void __launch_bounds__(256) k_clone_heads(const CloneSlot* table, const uint32_t* slot_of, const uint32_t* pred_lo,
                                                     const uint32_t* pred_hi, uint32_t total, uint32_t* dup, uint32_t* head, uint8_t* ext) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const uint32_t s = slot_of[p];
  uint32_t d = 0, h = 0;
  bool x = false;
  if (s != CLONE_NONE) {
    const uint32_t cnt = table[s].count;
    if (cnt >= 2) {
      const uint32_t lo = pred_lo[s];
      d = 1;
      x = lo == pred_hi[s] && lo != CLONE_NONE && table[lo].count == cnt;
      h = !x && ~table[s].nfirst == p;
    }
  }
  dup[p] = d; head[p] = h; ext[p] = x;
}

__global__ void __launch_bounds__(256) k_clone_classes(const uint32_t* head, const unsigned long long* cls_idx, const uint32_t* slot_of,
                                                       const CloneSlot* table, uint32_t total, uint32_t* rep, uint32_t* size,
                                                       uint32_t* slot_class, uint32_t* big, uint32_t* n_big) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total || !head[p]) return;
  const uint32_t c = (uint32_t)cls_idx[p], s = slot_of[p], cnt = table[s].count;
  rep[c] = p; size[c] = cnt; slot_class[s] = c;
  if (cnt > CLONE_WARP_MAX) big[atomicAdd(n_big, 1u)] = c;
}

// Persistent warps over the *n_classes classes: L = n + r, r = the run of ext flags behind the representative.
__global__ void __launch_bounds__(256) k_clone_length(const uint32_t* rep, const uint8_t* ext, uint32_t total, uint32_t n,
                                                      const unsigned long long* n_classes, uint32_t* class_len) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  const uint32_t nc = (uint32_t)*n_classes;
  for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < nc; c += warps) {
    const unsigned long long p1 = (unsigned long long)rep[c] + 1;
    uint32_t r = 0;
    for (;;) {
      const unsigned long long q = p1 + r + lane;
      const uint32_t stop = __ballot_sync(0xffffffffu, q >= total || !ext[q]);
      if (stop) { r += __ffs(stop) - 1; break; }
      r += 32;
    }
    if (lane == 0) class_len[c] = n + r;
  }
}

__global__ void __launch_bounds__(256) k_clone_scatter(const uint32_t* slot_of, const uint32_t* slot_class, const unsigned long long* class_base,
                                                       uint32_t total, uint32_t* cursor, unsigned long long* member) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const uint32_t s = slot_of[p];
  if (s == CLONE_NONE) return;
  const uint32_t c = slot_class[s];
  if (c == CLONE_NONE) return;
  member[class_base[c] + atomicAdd(&cursor[c], 1u)] = p;
}

// One warp per class of up to 32 fragments: a bitonic sort across the lanes.
__global__ void __launch_bounds__(256) k_clone_sort_warp(const unsigned long long* class_base, uint32_t n_classes, unsigned long long* member) {
  const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (c >= n_classes) return;
  const unsigned long long b = class_base[c];
  const uint32_t m = (uint32_t)(class_base[c + 1] - b);
  if (m > CLONE_WARP_MAX) return;
  unsigned long long v = lane < m ? member[b + lane] : ~0ull;
#pragma unroll
  for (uint32_t k = 2; k <= 32; k <<= 1)
#pragma unroll
    for (uint32_t j = k >> 1; j; j >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, v, j);
      v = (((lane & j) == 0) == ((lane & k) == 0)) ? min(v, o) : max(v, o);
    }
  if (lane < m) member[b + lane] = v;
}

// CTAs over the listed classes of more than 32 fragments (dynamic shared memory SIM_SORT_SMEM); wk_w: the sort's companion
// array (bitonic_pass moves a u32 with every key; its values are not used).
__global__ void __launch_bounds__(SIM_SORT_THREADS) k_clone_sort_cta(const unsigned long long* class_base, const uint32_t* big, const uint32_t* n_big,
                                                                     unsigned long long* member, uint32_t* wk_w) {
  extern __shared__ __align__(16) uint8_t clone_smem[];
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(clone_smem);
  uint32_t* sw = reinterpret_cast<uint32_t*>(clone_smem + SIM_SMEM_LINES * sizeof(unsigned long long));
  const uint32_t nb = *n_big;
  for (uint32_t i = blockIdx.x; i < nb; i += gridDim.x) {
    const uint32_t c = big[i];
    const unsigned long long b = class_base[c];
    const uint32_t m = (uint32_t)(class_base[c + 1] - b);
    unsigned long long* gk = member + b;
    uint32_t* gw = wk_w + b;
    if (m <= SIM_SMEM_LINES) {
      const uint32_t n2 = pow2_at_least(m);
      for (uint32_t t = threadIdx.x; t < m; t += blockDim.x) sk[t] = gk[t];
      __syncthreads();
      for (uint32_t k = 2; k <= n2; k <<= 1)
        for (uint32_t j = k >> 1; j; j >>= 1) bitonic_pass(sk, sw, m, n2, k, j);
      for (uint32_t t = threadIdx.x; t < m; t += blockDim.x) gk[t] = sk[t];
      __syncthreads();
      continue;
    }
    for (uint32_t t0 = 0; t0 < m; t0 += SIM_SMEM_LINES) {   // tiles in shared memory, then the passes that span tiles
      const uint32_t mt = min(SIM_SMEM_LINES, m - t0);
      for (uint32_t t = threadIdx.x; t < mt; t += blockDim.x) sk[t] = gk[t0 + t];
      __syncthreads();
      for (uint32_t k = 2; k <= SIM_SMEM_LINES; k <<= 1)
        for (uint32_t j = k >> 1; j; j >>= 1) bitonic_pass(sk, sw, mt, SIM_SMEM_LINES, k, j);
      for (uint32_t t = threadIdx.x; t < mt; t += blockDim.x) gk[t0 + t] = sk[t];
      __syncthreads();
    }
    bitonic_merge_tiles(gk, gw, m, pow2_at_least(m), sk, sw);
  }
}

// One warp per file: its duplicated lines and duplicated assertion lines.
__global__ void __launch_bounds__(256) k_clone_cover(const unsigned long long* line_base, uint32_t n_files, const unsigned long long* cover,
                                                     const uint8_t* line_flag, uint32_t n, uint32_t* file_dup, uint32_t* file_dup_assert) {
  const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (f >= n_files) return;
  const unsigned long long b = line_base[f], e = line_base[f + 1];
  uint32_t d = 0, a = 0;
  for (unsigned long long l = b + lane; l < e; l += 32) {
    const unsigned long long lo = l + 1 >= b + n ? l + 1 - n : b;
    if (cover[l + 1] > cover[lo]) { ++d; a += line_flag[l] != 0; }
  }
#pragma unroll
  for (int k = 16; k; k >>= 1) { d += __shfl_xor_sync(0xffffffffu, d, k); a += __shfl_xor_sync(0xffffffffu, a, k); }
  if (lane == 0) { file_dup[f] = d; file_dup_assert[f] = a; }
}

}  // namespace tsm
