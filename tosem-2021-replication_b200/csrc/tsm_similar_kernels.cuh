// tsm_similar_kernels.cuh - rename similarity (docs/SPEC.md section 13): per file the multiset of its lines as a sorted list
// of distinct (line hash, total weight), and `common` of candidate (old file, new file) pairs over those lists.
//
// Input: the line records of both sides (tsm_lines_kernels.cuh, one k_scan pass per side).  Per side:
//   k_sim_sort      one CTA per file: the weight of every line (its bytes, +1 for the LF, -1 for the CR of a CRLF), a
//                   bitonic sort of (hash, weight) by hash and the merge of equal hashes.  Files of up to SIM_SMEM_LINES
//                   lines sort in shared memory; larger ones sort 4 096-line tiles in shared memory and run the passes
//                   whose distance spans tiles in global memory.  Each file's distinct list lands at its line_base
//                   (weights as running sums), its length in cnt.
//   xscan(cnt)      offsets of the dense CSR.
//   k_sim_compact   one warp per file: the list to its CSR place, running sums back to weights.
// Then k_similarity: persistent warps draw candidates from an atomic counter; the lanes take the entries of the shorter
// list, binary-search the longer one and sum min(w, w') into an int64 `common`.
#pragma once
#include "tsm_device.cuh"

namespace tsm {

constexpr uint32_t SIM_SMEM_LINES = 4096;                 // lines a CTA sorts in shared memory (a tile of the large-file sort)
constexpr uint32_t SIM_SORT_THREADS = 256;
constexpr uint32_t SIM_SORT_SMEM = SIM_SMEM_LINES * (sizeof(unsigned long long) + sizeof(uint32_t)) + 64;
constexpr uint32_t SIM_GRAB = 8;                           // candidates a warp takes per atomic

// Weight of line i of file f (docs/SPEC.md section 13): git's diffcore-delta counts every byte and skips the CR of a CRLF.
__device__ __forceinline__ uint32_t line_weight(const uint8_t* file, uint32_t flen, const uint32_t* line_end, unsigned long long first,
                                                unsigned long long i) {
  const uint32_t end = line_end[i], start = i == first ? 0u : line_end[i - 1] + 1u;
  uint32_t w = end - start;
  if (end < flen) w += (end > start && file[end - 1] == 0x0D) ? 0u : 1u;
  return w;
}

// One pass (stage k, distance j) of an ascending bitonic sort of key/w[0, m) padded with +inf to n2 (a power of two).
// The first pass of a stage compares mirrored positions (i with i ^ (k - 1)), so every exchange puts the smaller key
// first and a padding entry never moves: pairs that reach past m are skipped instead of stored.
__device__ __forceinline__ void bitonic_pass(unsigned long long* key, uint32_t* w, uint32_t m, uint32_t n2, uint32_t k, uint32_t j) {
  for (uint32_t t = threadIdx.x; t < n2 / 2; t += blockDim.x) {
    const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
    const uint32_t p = j == k / 2 ? (i ^ (k - 1)) : (i | j);
    if (p >= m) continue;
    const unsigned long long a = key[i], b = key[p];
    if (a > b) {
      key[i] = b; key[p] = a;
      const uint32_t x = w[i]; w[i] = w[p]; w[p] = x;
    }
  }
  __syncthreads();
}

__device__ __forceinline__ uint32_t pow2_at_least(uint32_t n) { return n <= 1 ? 1u : 1u << (32 - __clz(n - 1)); }

// The rest of an ascending bitonic sort of gk/gw[0, n) in global memory (n > SIM_SMEM_LINES, n2 = pow2_at_least(n)) whose
// tiles of SIM_SMEM_LINES are already sorted: the passes of distance >= a tile over global memory, the passes inside a tile
// in shared memory (sk / sw: one tile).  Called by the whole CTA.
__device__ __forceinline__ void bitonic_merge_tiles(unsigned long long* gk, uint32_t* gw, uint32_t n, uint32_t n2,
                                                    unsigned long long* sk, uint32_t* sw) {
  for (uint32_t k = 2 * SIM_SMEM_LINES; k <= n2; k <<= 1) {
    for (uint32_t j = k >> 1; j >= SIM_SMEM_LINES; j >>= 1) bitonic_pass(gk, gw, n, n2, k, j);
    for (uint32_t t0 = 0; t0 < n; t0 += SIM_SMEM_LINES) {   // the passes inside a tile (j < tile, never the mirror pass)
      const uint32_t m = min(SIM_SMEM_LINES, n - t0);
      for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) { sk[i] = gk[t0 + i]; sw[i] = gw[t0 + i]; }
      __syncthreads();
      for (uint32_t j = SIM_SMEM_LINES >> 1; j; j >>= 1) bitonic_pass(sk, sw, m, SIM_SMEM_LINES, k, j);
      for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) { gk[t0 + i] = sk[i]; gw[t0 + i] = sw[i]; }
      __syncthreads();
    }
  }
}

// Inclusive block scan of two u32 per thread (256 threads); tot = the block's totals.
__device__ __forceinline__ uint2 block_scan2(uint2 v, uint2* sh, uint2& tot) {
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t x = __shfl_up_sync(0xffffffffu, v.x, d), y = __shfl_up_sync(0xffffffffu, v.y, d);
    if (lane >= d) { v.x += x; v.y += y; }
  }
  if (lane == 31) sh[wi] = v;
  __syncthreads();
  uint2 off = make_uint2(0, 0);
  tot = make_uint2(0, 0);
  for (int k = 0; k < (int)(SIM_SORT_THREADS / 32); ++k) {
    if (k < wi) { off.x += sh[k].x; off.y += sh[k].y; }
    tot.x += sh[k].x; tot.y += sh[k].y;
  }
  __syncthreads();
  return make_uint2(v.x + off.x, v.y + off.y);
}

// key/w[0, n) sorted: run r of equal keys -> out_key[r], out_cum[r] = the weight of runs 0..r; returns the run count.
__device__ uint32_t merge_runs(const unsigned long long* key, const uint32_t* w, uint32_t n, unsigned long long* out_key,
                               uint32_t* out_cum, uint2* sh) {
  uint32_t runs = 0, cum = 0;
  for (uint32_t b = 0; b < n; b += SIM_SORT_THREADS) {
    const uint32_t i = b + threadIdx.x;
    const bool in = i < n;
    const unsigned long long k = in ? key[i] : 0ull;
    const bool head = in && (i == 0 || key[i - 1] != k), tail = in && (i + 1 == n || key[i + 1] != k);
    uint2 tot;
    const uint2 incl = block_scan2(make_uint2(head ? 1u : 0u, in ? w[i] : 0u), sh, tot);
    const uint32_t r = runs + incl.x - 1;
    if (head) out_key[r] = k;
    if (tail) out_cum[r] = cum + incl.y;
    runs += tot.x; cum += tot.y;
  }
  return runs;
}

// One CTA per file; dynamic shared memory SIM_SORT_SMEM.  wk_key / wk_w: global work space of the large-file sort (the
// file's lines at its line_base); out_key / out_cum: the distinct list at line_base; cnt[f]: its length.
__global__ void __launch_bounds__(SIM_SORT_THREADS) k_sim_sort(const uint8_t* arena, const int32_t* off, const int32_t* len,
                                                              const unsigned long long* line_base, const unsigned long long* line_hash,
                                                              const uint32_t* line_end, unsigned long long* wk_key, uint32_t* wk_w,
                                                              unsigned long long* out_key, uint32_t* out_cum, uint32_t* cnt) {
  extern __shared__ __align__(16) uint8_t sim_smem[];
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(sim_smem);
  uint32_t* sw = reinterpret_cast<uint32_t*>(sim_smem + SIM_SMEM_LINES * sizeof(unsigned long long));
  uint2* sh = reinterpret_cast<uint2*>(sim_smem + SIM_SMEM_LINES * (sizeof(unsigned long long) + sizeof(uint32_t)));
  const uint32_t f = blockIdx.x;
  const unsigned long long b0 = line_base[f];
  const uint32_t n = (uint32_t)(line_base[f + 1] - b0);
  const uint8_t* file = arena + off[f];
  const uint32_t flen = (uint32_t)len[f];
  if (n <= SIM_SMEM_LINES) {                                // shared-memory path
    const uint32_t n2 = pow2_at_least(n);
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      sk[i] = line_hash[b0 + i];
      sw[i] = line_weight(file, flen, line_end, b0, b0 + i);
    }
    __syncthreads();
    for (uint32_t k = 2; k <= n2; k <<= 1)
      for (uint32_t j = k >> 1; j; j >>= 1) bitonic_pass(sk, sw, n, n2, k, j);
    const uint32_t runs = merge_runs(sk, sw, n, out_key + b0, out_cum + b0, sh);
    if (threadIdx.x == 0) cnt[f] = runs;
    return;
  }
  // global path: tiles of SIM_SMEM_LINES sorted in shared memory, the passes of distance >= a tile over global memory
  unsigned long long* gk = wk_key + b0;
  uint32_t* gw = wk_w + b0;
  const uint32_t n2 = pow2_at_least(n);
  for (uint32_t t0 = 0; t0 < n; t0 += SIM_SMEM_LINES) {
    const uint32_t m = min(SIM_SMEM_LINES, n - t0);
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
      sk[i] = line_hash[b0 + t0 + i];
      sw[i] = line_weight(file, flen, line_end, b0, b0 + t0 + i);
    }
    __syncthreads();
    for (uint32_t k = 2; k <= SIM_SMEM_LINES; k <<= 1)
      for (uint32_t j = k >> 1; j; j >>= 1) bitonic_pass(sk, sw, m, SIM_SMEM_LINES, k, j);
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) { gk[t0 + i] = sk[i]; gw[t0 + i] = sw[i]; }
    __syncthreads();
  }
  bitonic_merge_tiles(gk, gw, n, n2, sk, sw);
  const uint32_t runs = merge_runs(gk, gw, n, out_key + b0, out_cum + b0, sh);
  if (threadIdx.x == 0) cnt[f] = runs;
}

// One warp per file: the distinct list from line_base[f] to its CSR place dbase[f], running sums back to weights.
__global__ void k_sim_compact(const unsigned long long* line_base, const uint32_t* cnt, const unsigned long long* dbase, uint32_t n_files,
                              const unsigned long long* s_key, const uint32_t* s_cum, unsigned long long* d_key, uint32_t* d_w) {
  const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (f >= n_files) return;
  const unsigned long long src = line_base[f], dst = dbase[f];
  const uint32_t n = cnt[f];
  for (uint32_t r = lane; r < n; r += 32) {
    d_key[dst + r] = s_key[src + r];
    d_w[dst + r] = s_cum[src + r] - (r ? s_cum[src + r - 1] : 0u);
  }
}

// common[c] = sum over the hashes h shared by old file cand_old[c] and new file cand_new[c] of min(W_old(h), W_new(h)).
// Persistent warps take SIM_GRAB candidates per atomic on *next (zeroed by the caller).
__global__ void __launch_bounds__(256) k_similarity(const unsigned long long* key_a, const uint32_t* w_a, const unsigned long long* base_a,
                                                    const unsigned long long* key_b, const uint32_t* w_b, const unsigned long long* base_b,
                                                    const int32_t* cand_old, const int32_t* cand_new, unsigned long long n_cand,
                                                    unsigned long long* next, long long* common) {
  const uint32_t lane = threadIdx.x & 31;
  for (;;) {
    unsigned long long c0 = 0;
    if (lane == 0) c0 = atomicAdd(next, (unsigned long long)SIM_GRAB);
    c0 = __shfl_sync(0xffffffffu, c0, 0);
    if (c0 >= n_cand) return;
    const unsigned long long c1 = min(c0 + SIM_GRAB, n_cand);
    for (unsigned long long c = c0; c < c1; ++c) {
      const int32_t i = cand_old[c], j = cand_new[c];
      const unsigned long long* ks = key_a + base_a[i];
      const uint32_t* ws = w_a + base_a[i];
      uint32_t ns = (uint32_t)(base_a[i + 1] - base_a[i]);
      const unsigned long long* kl = key_b + base_b[j];
      const uint32_t* wl = w_b + base_b[j];
      uint32_t nl = (uint32_t)(base_b[j + 1] - base_b[j]);
      if (ns > nl) {
        const unsigned long long* tk = ks; ks = kl; kl = tk;
        const uint32_t* tw = ws; ws = wl; wl = tw;
        const uint32_t tn = ns; ns = nl; nl = tn;
      }
      long long acc = 0;
      for (uint32_t s = lane; s < ns; s += 32) {
        const unsigned long long h = ks[s];
        uint32_t lo = 0, hi = nl;                            // first entry >= h
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (kl[mid] < h) lo = mid + 1; else hi = mid; }
        if (lo < nl && kl[lo] == h) acc += (long long)min(ws[s], wl[lo]);
      }
#pragma unroll
      for (int d = 16; d; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
      if (lane == 0) common[c] = acc;
    }
  }
}

}  // namespace tsm
