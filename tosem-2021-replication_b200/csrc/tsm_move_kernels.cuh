// tsm_move_kernels.cuh - moved code of revision pairs (docs/SPEC.md section 20, git's `--color-moved=blocks`), from the line
// records of both sides and the edit marks of the DIFF_MARKS diff.  Lines are global indices of one side (< 2^32: the scan's
// staging arrays hold at most 0xFFFFFFF0 lines).  A run is a maximal sequence of changed lines of one file on one side.
//
//   k_move_lines    one thread per line, 8 bytes per load: the changed flag, whether the line starts or ends its run, and on a
//                   changed line its alphanumeric bytes.  xscan of the counts gives alnum(x .. y) in O(1); xscan of the
//                   changed flags numbers the entries, xscan of the run starts numbers the runs.
//   k_move_compact  one thread per line: the changed lines in line order (the entries) and the first / end line of every run.
//   k_move_insert   one thread per entry: the entry's (step, hash) into one open-addressing table shared by both sides
//                   (linear probing, 16-byte keys claimed by one 128-bit CAS; step + 1 in the key, so 0 marks an empty slot),
//                   counting the old and the new entries of every slot.  xscan of each side's counts gives its segments.
//   k_move_scatter  one thread per entry: each slot's entries of one side into its segment (order inside a segment is free).
//   k_move_reach    persistent warps, one deleted entry d at a time, lanes over the inserted entries e of its slot.  (d, e) is
//                   skipped when (d-1, e-1) continues its diagonal; else the diagonal's length D is walked (by the lane up to
//                   32 lines, then by the whole warp, 32 lines a round) and every (d+i, e+i), i < D, gets
//                   atomicMax((D-i) << 32 | ~partner) on both sides: the longest reach, ties to the smallest partner.
//                   The work is the number of matching (deleted, inserted) pairs of a step: quadratic in a line that repeats
//                   on both sides (blank lines, `}`), as git's own candidate lists are.
//   k_move_starts   one thread per entry: does a block start there if the walk reaches it (L(x) > 0 and alnum(x .. x+L(x)-1)
//                   >= 20)?  Pass 0 flags those lines, xscan numbers them, pass 1 lists them in line order.  A line that starts no
//                   block moves the walk on by one line, so from x the walk goes straight to the first listed line at or after x.
//   k_move_runs     one thread per run, in run order: the greedy walk of section 20 step 5, one step per block (from x to the
//                   first listed line y >= x of the run, then to y + L(y)).  Pass 0 counts the run's blocks, xscan places them,
//                   pass 1 writes them, so the blocks come out in line order.
//   k_move_mark     one thread per entry: its block (binary search of the block starts), bit 1 of its mark, and the block's
//                   assertion lines, added once per warp and block.
#pragma once
#include "tsm_device.cuh"
#include "tsm_diff_kernels.cuh"

namespace tsm {

constexpr uint8_t MV_CHANGED = 1, MV_HEAD = 2, MV_LAST = 4;   // k_move_lines flags
constexpr uint32_t MV_LANE_WALK = 32;                        // diagonal lines a lane walks alone before the warp takes over
constexpr uint32_t MV_MIN_ALNUM = 20;                        // git's COLOR_MOVED_MIN_ALNUM_COUNT

struct __align__(16) MoveKey { unsigned long long hash, step; };   // step = grp + 1; {0, 0} is an empty slot

__device__ __forceinline__ bool mv_alnum(uint32_t c) { return (c - '0' < 10u) || ((c | 0x20u) - 'a' < 26u); }

__device__ __forceinline__ uint32_t mv_file(const unsigned long long* line_base, int32_t n, unsigned long long l) {
  int lo = 0, hi = n;                                        // line_base[lo] <= l < line_base[hi]
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (line_base[mid] <= l) lo = mid; else hi = mid; }
  return (uint32_t)lo;
}

__global__ void __launch_bounds__(256) k_move_lines(DiffSide d, int32_t n, uint32_t total, const uint8_t* mark, uint8_t* flag,
                                                    uint32_t* alnum, uint32_t* changed, uint32_t* head) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= total) return;
  const bool c = mark[l] != 0;
  uint8_t f = 0;
  uint32_t a = 0;
  if (c) {
    const uint32_t lo = mv_file(d.line_base, n, l);
    const unsigned long long fb = d.line_base[lo], fe = d.line_base[lo + 1];
    f = MV_CHANGED;
    if (l == fb || !mark[l - 1]) f |= MV_HEAD;
    if (l + 1 == fe || !mark[l + 1]) f |= MV_LAST;
    const uint8_t* g = d.arena + (uint32_t)d.off[lo];
    const uint32_t e = d.line_end[l], s = l == fb ? 0u : d.line_end[l - 1] + 1u;
    for (uint32_t wb = s & ~7u; wb < e; wb += 8) {
      unsigned long long w = __ldg(reinterpret_cast<const unsigned long long*>(g + wb));
      const uint32_t k0 = wb < s ? s - wb : 0, k1 = min(8u, e - wb);
      w >>= 8 * k0;
      for (uint32_t k = k0; k < k1; ++k, w >>= 8) a += mv_alnum((uint32_t)(w & 0xFF));
    }
  }
  flag[l] = f; alnum[l] = a; changed[l] = c; head[l] = (f & MV_HEAD) != 0;
}

__global__ void __launch_bounds__(256) k_move_compact(const uint8_t* flag, uint32_t total, const unsigned long long* eidx,
                                                      const unsigned long long* ridx, uint32_t* ent, uint32_t* run_first, uint32_t* run_end) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= total) return;
  const uint8_t f = flag[l];
  if (!(f & MV_CHANGED)) return;
  ent[eidx[l]] = l;
  const uint32_t r = (uint32_t)ridx[l + 1] - 1;              // (the run of a changed line: the run starts up to and including it)
  if (f & MV_HEAD) run_first[r] = l;
  if (f & MV_LAST) run_end[r] = l + 1;
}

__device__ __forceinline__ uint32_t mv_slot(unsigned long long h, unsigned long long step, uint32_t mask) {
  const unsigned long long x = h ^ (step * 0x9E3779B97F4A7C15ull);
  return (uint32_t)(x ^ (x >> 32)) & mask;
}

__global__ void __launch_bounds__(256) k_move_insert(const uint32_t* ent, uint32_t ne, const unsigned long long* hash,
                                                     const unsigned long long* line_base, int32_t n, const uint16_t* grp, MoveKey* table,
                                                     uint32_t mask, uint32_t* cnt, uint32_t* slot_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ne) return;
  const uint32_t l = ent[i];
  const MoveKey k{hash[l], (unsigned long long)grp[mv_file(line_base, n, l)] + 1};
  const MoveKey empty{0, 0};
  uint32_t s = mv_slot(k.hash, k.step, mask);
  for (;; s = (s + 1) & mask) {                              // a key, once set, never changes: the CAS's answer decides
    const MoveKey was = atomicCAS(&table[s], empty, k);
    if (was.step == 0 || (was.hash == k.hash && was.step == k.step)) break;
  }
  atomicAdd(&cnt[s], 1u);
  slot_of[i] = s;
}

__global__ void __launch_bounds__(256) k_move_scatter(const uint32_t* ent, const uint32_t* slot_of, uint32_t ne, const unsigned long long* base,
                                                      uint32_t* cursor, uint32_t* seg, uint32_t* seg_slot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ne) return;
  const uint32_t s = slot_of[i];
  const unsigned long long p = base[s] + atomicAdd(&cursor[s], 1u);
  seg[p] = ent[i];
  if (seg_slot) seg_slot[p] = s;
}

struct MoveSide {                                            // one side's line hashes, run structure and reach
  const unsigned long long* hash; const uint8_t* flag; const unsigned long long* ridx; const uint32_t* run_end;
  unsigned long long* best;                                  // (L << 32 | ~partner), 0 = no match
};
__device__ __forceinline__ uint32_t mv_run_end(const MoveSide& s, uint32_t x) { return s.run_end[(uint32_t)s.ridx[x + 1] - 1]; }

__device__ __forceinline__ void mv_put(const MoveSide& o, const MoveSide& nw, uint32_t d, uint32_t e, uint32_t k, uint32_t D) {
  const unsigned long long len = (unsigned long long)(D - k) << 32;
  atomicMax(&o.best[d + k], len | (uint32_t)~(e + k));
  atomicMax(&nw.best[e + k], len | (uint32_t)~(d + k));
}

__global__ void __launch_bounds__(256) k_move_reach(MoveSide o, MoveSide nw, const uint32_t* seg_old, const uint32_t* seg_old_slot,
                                                    uint32_t n_old, const uint32_t* seg_new, const unsigned long long* new_base) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_old; i += warps) {
    const uint32_t d = seg_old[i], s = seg_old_slot[i];
    const unsigned long long b = new_base[s], be = new_base[s + 1];
    if (b == be) continue;
    const uint32_t dend = mv_run_end(o, d);
    const bool dhead = (o.flag[d] & MV_HEAD) != 0;
    const unsigned long long hprev = dhead ? 0ull : o.hash[d - 1];
    for (unsigned long long j0 = b; j0 < be; j0 += 32) {
      const unsigned long long j = j0 + lane;
      uint32_t e = 0, eend = 0, D = 0;
      bool start = false;
      if (j < be) {
        e = seg_new[j];
        start = dhead || (nw.flag[e] & MV_HEAD) || nw.hash[e - 1] != hprev;
        if (start) {
          eend = mv_run_end(nw, e);
          D = 1;
          while (D < MV_LANE_WALK && d + D < dend && e + D < eend && o.hash[d + D] == nw.hash[e + D]) ++D;
          if (D < MV_LANE_WALK)
            for (uint32_t k = 0; k < D; ++k) mv_put(o, nw, d, e, k, D);
        }
      }
      for (uint32_t m = __ballot_sync(0xffffffffu, start && D == MV_LANE_WALK); m; m &= m - 1) {   // long diagonals: the whole warp
        const int ld = __ffs(m) - 1;
        const uint32_t ee = __shfl_sync(0xffffffffu, e, ld), ee_end = __shfl_sync(0xffffffffu, eend, ld);
        uint32_t L = MV_LANE_WALK;
        for (;;) {
          const uint32_t q = L + lane;
          const bool stop = d + q >= dend || ee + q >= ee_end || o.hash[d + q] != nw.hash[ee + q];
          const uint32_t bs = __ballot_sync(0xffffffffu, stop);
          if (bs) { L += __ffs(bs) - 1; break; }
          L += 32;
        }
        for (uint32_t k = lane; k < L; k += 32) mv_put(o, nw, d, ee, k, L);
      }
    }
  }
}

// PASS 0: start[i] = 1 when entry i (line ent[i]) would start a block.  PASS 1: starts[sidx[i]] = ent[i] for those entries.
template <int PASS>
__global__ void __launch_bounds__(256) k_move_starts(const uint32_t* ent, uint32_t ne, const unsigned long long* best,
                                                     const unsigned long long* apre, uint32_t* start, const unsigned long long* sidx,
                                                     uint32_t* starts) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ne) return;
  if (PASS) {
    if (start[i]) starts[sidx[i]] = ent[i];
    return;
  }
  const uint32_t x = ent[i], L = (uint32_t)(best[x] >> 32);
  start[i] = L && apre[x + L] - apre[x] >= MV_MIN_ALNUM;
}

// One run per thread: from x (the run's first line) to y, the first listed start at or after x (its entry number eidx[x] counts
// the entries before x, sidx[eidx[x]] the starts among them); y inside the run -> block [y, y+L(y)) with partner(y), x = y + L(y);
// else the run is done.  PASS 0 counts the blocks into cnt[r]; PASS 1 writes them from base[r] on.
template <int PASS>
__global__ void __launch_bounds__(256) k_move_runs(const uint32_t* run_first, const uint32_t* run_end, uint32_t n_runs,
                                                   const unsigned long long* best, const unsigned long long* eidx,
                                                   const unsigned long long* sidx, uint32_t ne, const uint32_t* starts, uint32_t* cnt,
                                                   const unsigned long long* base, tsm_move_block* out) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_runs) return;
  const uint32_t end = run_end[r];
  const unsigned long long n_starts = sidx[ne];
  unsigned long long at = PASS ? base[r] : 0;
  uint32_t nb = 0;
  for (uint32_t x = run_first[r]; x < end;) {
    const unsigned long long k = sidx[eidx[x]];
    if (k >= n_starts) break;
    const uint32_t y = starts[k];
    if (y >= end) break;
    const unsigned long long v = best[y];
    const uint32_t L = (uint32_t)(v >> 32);
    if (PASS) out[at++] = tsm_move_block{(int64_t)y, (int64_t)(uint32_t)~(uint32_t)v, (int32_t)L, 0};
    ++nb;
    x = y + L;
  }
  if (!PASS) cnt[r] = nb;
}

// One thread per entry: the block that holds line x is the last one starting at or before it, if it reaches x.
__global__ void __launch_bounds__(256) k_move_mark(const uint32_t* ent, uint32_t ne, tsm_move_block* blocks, uint32_t nb,
                                                   const uint8_t* line_flag, uint8_t* mark) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t b = 0xFFFFFFFFu;
  bool a = false;
  if (i < ne && nb) {
    const uint32_t x = ent[i];
    uint32_t lo = 0, hi = nb;                                 // first block starting after x
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint32_t)blocks[mid].line <= x) lo = mid + 1; else hi = mid; }
    if (lo && x < (uint32_t)blocks[lo - 1].line + (uint32_t)blocks[lo - 1].n_lines) {
      b = lo - 1;
      mark[x] |= 2;
      a = line_flag[x] != 0;
    }
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, b);   // lanes of the same block add their count once
  const uint32_t n = __popc(__ballot_sync(0xffffffffu, a) & peers);
  if (b != 0xFFFFFFFFu && n && (threadIdx.x & 31) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&blocks[b].n_assert, (int32_t)n);
}

}  // namespace tsm
