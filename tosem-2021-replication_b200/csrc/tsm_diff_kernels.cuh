// tsm_diff_kernels.cuh - S8 revision-pair churn (docs/SPEC.md section 8): per (old, new) pair the number of
// added / removed lines = |new| - LCS, |old| - LCS over the SPEC section 3 line-hash sequences, and the canonical
// edit script's hunks.  Pins: Important-files/ML-Testing-v1.xlsx!projects:R1 (`cloc = added + removed`); no revision
// history ships, so parity is against the oracle's O(n*m) DP and its serial Myers script.  The line records (hash,
// flag per line, in file order) come from k_scan (tsm_scan_walk.cuh, tsm_lines_kernels.cuh).
//
//   k_diff_small    warp per pair, the common case in ONE kernel: common prefix / suffix trim by ballots, the middle
//                   hash sequences staged in shared memory, the greedy furthest-reaching D-path search with the
//                   diagonals of one D across the lanes and V in REGISTERS (neighbour diagonals by shuffle), the rows
//                   of V kept in shared memory, the canonical backtrack by lane 0.  Four sizes (DS_SIZES: staged lines,
//                   largest distance, pairs per SM), each fed by the list the size before it leaves; a pair none of
//                   them holds (middle above 4 096 lines, distance above 127) is left to the two kernels below
//   k_myers         warp per pair: the same search with V in global scratch (any size)
//   k_myers_trace   the same with one row of V kept per D in global memory, then the backtrack
//
// k_diff_small and k_myers_trace have two more variants (DiffMode): DIFF_EMIT also lists the changed assertion lines
// (SPEC section 8) for k_classify, DIFF_MARKS marks every deleted and inserted line (SPEC section 14) for k_blame.  The
// variant with neither is the same code as before they existed.
#pragma once
#include "tsm_scan_kernels.cuh"

namespace tsm {

struct DiffSide {                   // one corpus (old or new) on the device
  const uint8_t* arena; const int32_t* off; const int32_t* len;
  uint32_t* n_lines;                // [n]
  const unsigned long long* line_base;   // [n+1] exclusive prefix of n_lines
  uint32_t* line_end;               // [total lines] file-relative end of each line (position of its LF or EOF)
  unsigned long long* line_hash;    // [total lines]
  const uint8_t* ext;               // [n] S1 tags (NULL = all 0), only read when line_flag != NULL
  uint8_t* line_flag;               // [total lines] 1 = assertion line (SPEC section 4); NULL = not wanted
};

// Where the DIFF_EMIT variants put the changed assertion lines: side 0 = deleted lines of `old`, side 1 = inserted lines of `new`,
// each as (pair << 32 | file-relative line start), the candidate format of k_classify.  n[s] is the n_cand of the Ctrl that
// k_classify reads for side s; it counts every line, also those past cap[s], so that the host sees an overflow.
// The DIFF_MARKS variants use mark[] only: mark[0][g] = 1 for every deleted line g of `old`, mark[1][g] = 1 for every
// inserted line g of `new` (global line indices, zeroed by the host).
struct AssertSink {
  unsigned long long* list[2];
  uint32_t* n[2];
  uint32_t cap[2];
  const uint32_t* line_end[2];      // DiffSide::line_end of each side
  uint8_t* mark[2];
};

enum DiffMode { DIFF_PLAIN = 0, DIFF_EMIT = 1, DIFF_MARKS = 2 };

// Candidate of line g (global line index) of pair pr, whose file starts at line `first` of its side.
__device__ __forceinline__ unsigned long long sink_key(const AssertSink& s, int side, int pr, unsigned long long first,
                                                       unsigned long long g) {
  return ((unsigned long long)(uint32_t)pr << 32) | (g == first ? 0u : s.line_end[side][g - 1] + 1u);
}
__device__ __forceinline__ void sink_put(const AssertSink& s, int side, unsigned long long key) {   // one lane
  const uint32_t slot = atomicAdd(s.n[side], 1u);
  if (slot < s.cap[side]) s.list[side][slot] = key;
}
// Every flagged line of the run [g0, g0 + cnt) (flags q[0 .. cnt)): the whole warp, one atomic per 32 lines.
__device__ __forceinline__ void sink_run(const AssertSink& s, int side, int pr, unsigned long long first, unsigned long long g0,
                                         const uint8_t* q, int cnt, int lane) {
  for (int i0 = 0; i0 < cnt; i0 += 32) {
    const int i = i0 + lane;
    const bool f = i < cnt && q[i] != 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, f);
    if (!bal) continue;
    const uint32_t base = warp_reserve(s.n[side], (uint32_t)__popc(bal), lane);
    const uint32_t slot = base + (uint32_t)__popc(bal & ((1u << lane) - 1u));
    if (f && slot < s.cap[side]) s.list[side][slot] = sink_key(s, side, pr, first, g0 + (unsigned long long)i);
  }
}

// Mark the run [0, cnt) of p: the whole warp.
__device__ __forceinline__ void mark_run(uint8_t* p, int cnt, int lane) {
  for (int i = lane; i < cnt; i += 32) p[i] = 1;
}

// Follow a diagonal while the lines are equal.  Four positions are compared per round trip to HBM / L2 (the loads
// of one round do not depend on each other); the clamped indices keep speculative reads inside the sequences.
__device__ __forceinline__ void snake_gmem(const unsigned long long* a, const unsigned long long* b, int n, int m, int& x, int& y) {
  while (x < n && y < m) {
    const int r = min(n - x, m - y);
    const unsigned long long a0 = a[x], b0 = b[y];
    const unsigned long long a1 = a[x + min(1, r - 1)], b1 = b[y + min(1, r - 1)];
    const unsigned long long a2 = a[x + min(2, r - 1)], b2 = b[y + min(2, r - 1)];
    const unsigned long long a3 = a[x + min(3, r - 1)], b3 = b[y + min(3, r - 1)];
    int t = 0;
    if (a0 == b0) { t = 1; if (r > 1 && a1 == b1) { t = 2; if (r > 2 && a2 == b2) { t = 3; if (r > 3 && a3 == b3) t = 4; } } }
    x += t; y += t;
    if (t < 4) break;
  }
}

__host__ __device__ constexpr uint32_t ds_rows(int dcap) { return (uint32_t)((dcap + 1) * (dcap + 2) / 2); }
__host__ __device__ constexpr uint32_t ds_warp_bytes(int hcap, int dcap) { return (uint32_t)hcap * 8u + ds_rows(dcap) * 4u + (uint32_t)hcap; }

// Four sizes of the same kernel, k_diff_small<hcap, dcap, warps, MODE>, launched in this order: lines of both middles
// staged per warp, largest distance, warps per block, and the blocks per SM that the launch asks for.  The rows of V
// ((dcap+1)(dcap+2)/2 ints) and the staged middle (9 B per line) fix the shared memory per pair, hence the pairs in
// flight per SM: most pairs are small, the few large ones decide the tail.
struct DiffSmallSize {
  int hcap, dcap, warps, per_sm;
  constexpr uint32_t smem() const { return (uint32_t)warps * ds_warp_bytes(hcap, dcap); }   // dynamic shared memory per block
};
constexpr DiffSmallSize DS_SIZES[] = {
    {512, 31, 8, 4},      //  6.6 KB per pair: 32 pairs per SM
    {1024, 63, 2, 6},     // 17.3 KB per pair: 12 pairs per SM
    {4096, 63, 1, 5},     // 44.3 KB per pair:  5 pairs per SM
    {4096, 127, 1, 3},    // 68.3 KB per pair:  3 pairs per SM (a handful of far-apart pairs)
};
constexpr int DS_N = (int)(sizeof(DS_SIZES) / sizeof(DS_SIZES[0]));
constexpr bool ds_sizes_fit() {   // per_sm blocks of each size in the 228 KB of an SM, 1 KB reserved per block
  for (const DiffSmallSize& s : DS_SIZES)
    if (s.per_sm * (s.smem() + 1024) > 233472) return false;
  return true;
}
static_assert(ds_sizes_fit(), "pairs per SM");

// One pair start to finish; false = left to the next size (middle longer than HCAP lines or distance above DCAP).
//   * V of row d lives in REGISTERS: entry j (diagonal k = -d + 2 j) in lane j % 32, register j / 32.  Row d + 1 needs
//     entries j - 1 and j of row d: the lane's own register and the neighbour lane's (lane 0: lane 31 of the register
//     below) - two shuffles, no memory;
//   * a snake (run of equal lines along a diagonal) is followed four steps by its own lane; what is still running then
//     is finished by the whole warp, 32 lines per step: a long unchanged stretch costs a few ballots, not hundreds of
//     dependent loads;
//   * the assertion-line flags of the middle are staged next to the hashes: the backtrack reads shared memory only.
template <int HCAP, int DCAP, int MODE>
__device__ __forceinline__ bool diff_one(uint8_t* mine, int pr, int lane,
    const unsigned long long* ha, const unsigned long long* la, const uint8_t* fa,
    const unsigned long long* hb, const unsigned long long* lb, const uint8_t* fb,
    long long* added, long long* removed, tsm_diff_detail* detail, const AssertSink& sink) {
  constexpr int NQ = (DCAP + 32) / 32;                    // row entries per lane
  unsigned long long* sa = reinterpret_cast<unsigned long long*>(mine);
  int32_t* rows = reinterpret_cast<int32_t*>(mine + HCAP * 8);
  uint8_t* sfa = mine + HCAP * 8 + ds_rows(DCAP) * 4;
  const unsigned long long* a = ha + la[pr];
  const unsigned long long* b = hb + lb[pr];
  const uint8_t* qa = fa ? fa + la[pr] : nullptr;
  const uint8_t* qb = fb ? fb + lb[pr] : nullptr;
  int n = (int)(la[pr + 1] - la[pr]), m = (int)(lb[pr + 1] - lb[pr]);
  const int n0 = n, m0 = m;
  int pre = 0;
  while (true) {
    const int i = pre + lane;
    const uint32_t mk = __ballot_sync(0xffffffffu, !(i < n && i < m && a[i] == b[i]));
    if (mk) { pre += __ffs(mk) - 1; break; }
    pre += 32;
  }
  a += pre; b += pre; n -= pre; m -= pre;
  if (detail) { qa += pre; qb += pre; }
  int suf = 0;
  while (true) {
    const int i = suf + lane;
    const uint32_t mk = __ballot_sync(0xffffffffu, !(i < n && i < m && a[n - 1 - i] == b[m - 1 - i]));
    if (mk) { suf += __ffs(mk) - 1; break; }
    suf += 32;
  }
  n -= suf; m -= suf;
  long long h_add = 0, h_del = 0, h_mod = 0, a_as = 0, r_as = 0;
  int D = 0;
  if (n == 0 || m == 0) {                                 // one pure hunk (or none)
    D = n + m;
    if (detail) {
      int ca = 0, cb = 0;
      for (int i = lane; i < n; i += 32) ca += qa[i] != 0;
      for (int i = lane; i < m; i += 32) cb += qb[i] != 0;
#pragma unroll
      for (int k = 16; k; k >>= 1) { ca += __shfl_xor_sync(0xffffffffu, ca, k); cb += __shfl_xor_sync(0xffffffffu, cb, k); }
      if (n) { h_del = 1; r_as = ca; }
      if (m) { h_add = 1; a_as = cb; }
      if constexpr (MODE == DIFF_EMIT) {
        sink_run(sink, 0, pr, la[pr], la[pr] + pre, qa, n, lane);
        sink_run(sink, 1, pr, lb[pr], lb[pr] + pre, qb, m, lane);
      }
    }
  } else {
    if (n + m > HCAP) return false;
    unsigned long long* sb = sa + n;
    uint8_t* sfb = sfa + n;
    __syncwarp();                                         // (the previous pair's backtrack is done with the buffers)
#pragma unroll 8                                          // (independent loads: eight in flight per lane)
    for (int i = lane; i < n; i += 32) sa[i] = a[i];
#pragma unroll 8
    for (int i = lane; i < m; i += 32) sb[i] = b[i];
    if (detail) {
#pragma unroll 8
      for (int i = lane; i < n; i += 32) sfa[i] = qa[i];
#pragma unroll 8
      for (int i = lane; i < m; i += 32) sfb[i] = qb[i];
    }
    __syncwarp();
    bool found = false;
    int xv[NQ];                                           // row d - 1, entries lane + 32 q
#pragma unroll
    for (int q = 0; q < NQ; ++q) xv[q] = 0;
    for (int d = 0; d <= DCAP && d <= n + m; ++d) {
      bool hit = false;
#pragma unroll
      for (int q = NQ - 1; q >= 0; --q) {                 // downwards: entry (lane 0, q) reads row d - 1 of register q - 1
        if (32 * q > d) continue;                         // (warp-uniform)
        const int j = lane + 32 * q, k = -d + 2 * j;
        const int up = __shfl_up_sync(0xffffffffu, xv[q], 1);
        const int wrap = __shfl_sync(0xffffffffu, q ? xv[q ? q - 1 : 0] : 0, 31);
        const int xm = lane ? up : wrap;                  // V[k - 1]
        const bool act = j <= d;
        int x = 0, y = 0;
        bool run = false;                                 // the snake is still going
        if (act) {
          if (d) {
            const bool down = (k == -d) || (k != d && xm < xv[q]);
            x = down ? xv[q] : xm + 1;
          }
          y = x - k;
          int t = 0;
          while (t < 4 && x < n && y < m && sa[x] == sb[y]) { ++x; ++y; ++t; }
          run = t == 4;
        }
        uint32_t going = __ballot_sync(0xffffffffu, run);
        while (going) {                                   // finish the long snakes with the whole warp, one diagonal at a time
          const int src = __ffs(going) - 1;
          int bx = __shfl_sync(0xffffffffu, x, src), by = __shfl_sync(0xffffffffu, y, src);
          while (true) {
            const int ix = bx + lane, iy = by + lane;
            const uint32_t ne = __ballot_sync(0xffffffffu, !(ix < n && iy < m && sa[ix] == sb[iy]));
            const int adv = ne ? __ffs(ne) - 1 : 32;
            bx += adv; by += adv;
            if (ne) break;
          }
          if (lane == src) { x = bx; y = by; }
          going &= going - 1;
        }
        if (act) {
          xv[q] = x;
          if (detail) rows[d * (d + 1) / 2 + j] = x;
          hit |= x >= n && y >= m;
        }
      }
      if (__any_sync(0xffffffffu, hit)) { D = d; found = true; break; }
    }
    if (!found) return false;
    __syncwarp();
    if (detail && lane == 0) {                            // canonical backtrack: edits from the last to the first
      int x = n, y = m;
      bool in_hunk = false, has_add = false, has_del = false;
      for (int d = D; d >= 1; --d) {
        const int k = x - y;
        const int32_t* P = rows + (d - 1) * d / 2;
        const bool down = (k == -d) || (k != d && P[(k - 1 + d - 1) / 2] < P[(k + 1 + d - 1) / 2]);
        const int pk = down ? k + 1 : k - 1;
        const int px = P[(pk + d - 1) / 2], py = px - pk;
        const int midx = down ? px : px + 1;
        if (in_hunk && x - midx > 0) {
          if (has_add && has_del) ++h_mod; else if (has_add) ++h_add; else ++h_del;
          has_add = has_del = false;
        }
        in_hunk = true;
        if (down) { has_add = true; a_as += sfb[py] != 0; }
        else { has_del = true; r_as += sfa[px] != 0; }
        if constexpr (MODE == DIFF_EMIT) {
          if (down && sfb[py]) sink_put(sink, 1, sink_key(sink, 1, pr, lb[pr], lb[pr] + pre + py));
          if (!down && sfa[px]) sink_put(sink, 0, sink_key(sink, 0, pr, la[pr], la[pr] + pre + px));
        }
        if constexpr (MODE == DIFF_MARKS) {                // bit 1 of the staged flag, written out by the warp below
          if (down) sfb[py] |= 2;
          else sfa[px] |= 2;
        }
        x = px; y = py;
      }
      if (in_hunk) { if (has_add && has_del) ++h_mod; else if (has_add) ++h_add; else ++h_del; }
    }
    if constexpr (MODE == DIFF_MARKS) {
      __syncwarp();
      uint8_t* ma = sink.mark[0] + la[pr] + pre;
      uint8_t* mb = sink.mark[1] + lb[pr] + pre;
#pragma unroll 1
      for (int i = lane; i < n; i += 32) if (sfa[i] & 2) ma[i] = 1;
#pragma unroll 1
      for (int i = lane; i < m; i += 32) if (sfb[i] & 2) mb[i] = 1;
    }
  }
  if constexpr (MODE == DIFF_MARKS)
    if (n == 0 || m == 0) {
      mark_run(sink.mark[0] + la[pr] + pre, n, lane);
      mark_run(sink.mark[1] + lb[pr] + pre, m, lane);
    }
  if (lane == 0) {
    const long long lcs = ((long long)(n + m) - D) / 2 + pre + suf;
    removed[pr] = n0 - lcs;
    added[pr] = m0 - lcs;
    if (detail) detail[pr] = tsm_diff_detail{h_add, h_del, h_mod, a_as, r_as};
  }
  return true;
}

// Persistent warps, pairs handed out by an atomic counter (their cost varies by two orders of magnitude).  The pairs
// are todo_in[0 .. *n_in) when todo_in is given, else 0 .. n_all; what this size cannot finish goes to todo_out.
template <int HCAP, int DCAP, int WARPS, int MODE>
__global__ void __launch_bounds__(WARPS * 32) k_diff_small(
    const unsigned long long* ha, const unsigned long long* la, const uint8_t* fa,
    const unsigned long long* hb, const unsigned long long* lb, const uint8_t* fb,
    const int32_t* todo_in, const uint32_t* n_in, int32_t n_all, uint32_t* work,
    long long* added, long long* removed, tsm_diff_detail* detail, int32_t* todo_out, uint32_t* n_out, AssertSink sink) {
  extern __shared__ __align__(16) uint8_t ds_smem[];
  const int lane = threadIdx.x & 31;
  uint8_t* mine = ds_smem + (threadIdx.x >> 5) * ds_warp_bytes(HCAP, DCAP);
  const uint32_t limit = n_in ? *n_in : (uint32_t)n_all;
  while (true) {
    uint32_t slot = 0;
    if (lane == 0) slot = atomicAdd(work, 1u);
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (slot >= limit) return;
    const int pr = todo_in ? todo_in[slot] : (int)slot;
    if (!diff_one<HCAP, DCAP, MODE>(mine, pr, lane, ha, la, fa, hb, lb, fb, added, removed, detail, sink) && lane == 0)
      todo_out[atomicAdd(n_out, 1u)] = pr;
  }
}

// Edit distance D (insertions + deletions) of hash sequences a[0..n) and b[0..m); one warp per pair.
// V (furthest x per diagonal) lives in global scratch of 2*(n+m)+3 ints per pair.
__global__ void k_myers(const unsigned long long* ha, const unsigned long long* la, const unsigned long long* hb,
                        const unsigned long long* lb, int32_t n_pairs, int32_t* vbuf, const unsigned long long* vbase,
                        long long* added, long long* removed, const int32_t* todo) {
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (slot >= n_pairs) return;
  const int pr = todo ? todo[slot] : slot;                // `todo`: the pairs k_diff_small left over (vbase is indexed by slot)
  const unsigned long long* a = ha + la[pr];
  const unsigned long long* b = hb + lb[pr];
  int n = (int)(la[pr + 1] - la[pr]), m = (int)(lb[pr + 1] - lb[pr]);
  const int n0 = n, m0 = m;
  // common prefix
  int pre = 0;
  while (true) {
    const int i = pre + lane;
    const bool ne = !(i < n && i < m && a[i] == b[i]);
    const uint32_t mk = __ballot_sync(0xffffffffu, ne);
    if (mk) { pre += __ffs(mk) - 1; break; }
    pre += 32;
  }
  a += pre; b += pre; n -= pre; m -= pre;
  int suf = 0;
  while (true) {
    const int i = suf + lane;
    const bool ne = !(i < n && i < m && a[n - 1 - i] == b[m - 1 - i]);
    const uint32_t mk = __ballot_sync(0xffffffffu, ne);
    if (mk) { suf += __ffs(mk) - 1; break; }
    suf += 32;
  }
  n -= suf; m -= suf;
  int D = 0;
  if (n == 0 || m == 0) D = n + m;
  else {
    int32_t* V = vbuf + vbase[slot] + (n + m + 1);        // V[k], k in [-(n+m)-1, n+m+1]
    if (lane == 0) V[1] = 0;
    __syncwarp();
    bool done = false;
    for (D = 0; D <= n + m && !done; ++D) {
      bool hit = false;
      for (int k = -D + 2 * lane; k <= D; k += 64) {
        int x;
        if (k == -D || (k != D && V[k - 1] < V[k + 1])) x = V[k + 1]; else x = V[k - 1] + 1;
        int y = x - k;
        snake_gmem(a, b, n, m, x, y);
        V[k] = x;
        if (x >= n && y >= m) hit = true;
      }
      __syncwarp();
      done = __any_sync(0xffffffffu, hit);
    }
    --D;                                                  // the loop increments once more after the hit
  }
  if (lane == 0) {
    const long long lcs = ((long long)(n + m) - D) / 2 + pre + suf;
    removed[pr] = n0 - lcs;
    added[pr] = m0 - lcs;
  }
}

// Hunks and their classification (docs/SPEC.md section 8): the same search with one row of V kept per D
// (row d holds the diagonals -d, -d+2, ..., d), then the canonical backtrack by lane 0.
// trace_base[pr] = first int of pair pr's rows, sized (D+1)(D+2)/2 from the distances of k_myers.
// The DIFF_MARKS variant marks the whole middle (between the common prefix and suffix) of a pair it does not trace.
template <int MODE>
__global__ void k_myers_trace(const unsigned long long* ha, const unsigned long long* la, const uint8_t* fa,
                              const unsigned long long* hb, const unsigned long long* lb, const uint8_t* fb,
                              int32_t pair0, int32_t n_pairs, int32_t* trace, const unsigned long long* trace_base,
                              const long long* added, const long long* removed, long long max_d, tsm_diff_detail* detail,
                              const int32_t* todo, AssertSink sink) {
  const int slot = pair0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (slot >= pair0 + n_pairs) return;
  const int pr = todo ? todo[slot] : slot;                // trace_base is indexed by slot
  if constexpr (MODE != DIFF_MARKS)
    if (added[pr] + removed[pr] > max_d) return;           // too far apart to keep the rows of V: the host reports one hunk
  const unsigned long long* a = ha + la[pr];
  const unsigned long long* b = hb + lb[pr];
  const uint8_t* qa = fa + la[pr];
  const uint8_t* qb = fb + lb[pr];
  int n = (int)(la[pr + 1] - la[pr]), m = (int)(lb[pr + 1] - lb[pr]);
  int pre = 0;
  while (true) {
    const int i = pre + lane;
    const uint32_t mk = __ballot_sync(0xffffffffu, !(i < n && i < m && a[i] == b[i]));
    if (mk) { pre += __ffs(mk) - 1; break; }
    pre += 32;
  }
  a += pre; b += pre; qa += pre; qb += pre; n -= pre; m -= pre;
  int suf = 0;
  while (true) {
    const int i = suf + lane;
    const uint32_t mk = __ballot_sync(0xffffffffu, !(i < n && i < m && a[n - 1 - i] == b[m - 1 - i]));
    if (mk) { suf += __ffs(mk) - 1; break; }
    suf += 32;
  }
  n -= suf; m -= suf;
  if constexpr (MODE == DIFF_MARKS)
    if (added[pr] + removed[pr] > max_d) {
      mark_run(sink.mark[0] + la[pr] + pre, n, lane);
      mark_run(sink.mark[1] + lb[pr] + pre, m, lane);
      return;
    }
  long long h_add = 0, h_del = 0, h_mod = 0, a_as = 0, r_as = 0;
  if (n == 0 || m == 0) {                                 // one pure hunk (or none)
    int ca = 0, cb = 0;
    for (int i = lane; i < n; i += 32) ca += qa[i] != 0;
    for (int i = lane; i < m; i += 32) cb += qb[i] != 0;
#pragma unroll
    for (int k = 16; k; k >>= 1) { ca += __shfl_xor_sync(0xffffffffu, ca, k); cb += __shfl_xor_sync(0xffffffffu, cb, k); }
    if (n) { h_del = 1; r_as = ca; }
    if (m) { h_add = 1; a_as = cb; }
    if constexpr (MODE == DIFF_EMIT) {
      sink_run(sink, 0, pr, la[pr], la[pr] + pre, qa, n, lane);
      sink_run(sink, 1, pr, lb[pr], lb[pr] + pre, qb, m, lane);
    }
    if constexpr (MODE == DIFF_MARKS) {
      mark_run(sink.mark[0] + la[pr] + pre, n, lane);
      mark_run(sink.mark[1] + lb[pr] + pre, m, lane);
    }
  } else {
    int32_t* R = trace + trace_base[slot];
    int D = 0;
    bool done = false;
    for (int d = 0; !done; ++d) {
      int32_t* row = R + (size_t)d * (d + 1) / 2;
      const int32_t* P = R + (size_t)(d - 1) * d / 2;     // previous row, entry (kk + d - 1) / 2
      bool hit = false;
      for (int k = -d + 2 * lane; k <= d; k += 64) {
        int x;
        if (d == 0) x = 0;
        else {
          const bool down = (k == -d) || (k != d && P[(k - 1 + d - 1) / 2] < P[(k + 1 + d - 1) / 2]);
          x = down ? P[(k + 1 + d - 1) / 2] : P[(k - 1 + d - 1) / 2] + 1;
        }
        int y = x - k;
        snake_gmem(a, b, n, m, x, y);
        row[(k + d) / 2] = x;
        if (x >= n && y >= m) hit = true;
      }
      __syncwarp();
      done = __any_sync(0xffffffffu, hit);
      D = d;
    }
    if (lane == 0) {                                      // canonical backtrack: edits from the last to the first
      int x = n, y = m;
      bool in_hunk = false, has_add = false, has_del = false;
      for (int d = D; d >= 1; --d) {
        const int k = x - y;
        const int32_t* P = R + (size_t)(d - 1) * d / 2;
        const bool down = (k == -d) || (k != d && P[(k - 1 + d - 1) / 2] < P[(k + 1 + d - 1) / 2]);
        const int pk = down ? k + 1 : k - 1;
        const int px = P[(pk + d - 1) / 2], py = px - pk;
        const int midx = down ? px : px + 1;
        if (in_hunk && x - midx > 0) {
          if (has_add && has_del) ++h_mod; else if (has_add) ++h_add; else ++h_del;
          has_add = has_del = false;
        }
        in_hunk = true;
        if (down) { has_add = true; a_as += qb[py] != 0; }
        else { has_del = true; r_as += qa[px] != 0; }
        if constexpr (MODE == DIFF_EMIT) {
          if (down && qb[py]) sink_put(sink, 1, sink_key(sink, 1, pr, lb[pr], lb[pr] + pre + py));
          if (!down && qa[px]) sink_put(sink, 0, sink_key(sink, 0, pr, la[pr], la[pr] + pre + px));
        }
        if constexpr (MODE == DIFF_MARKS) {
          if (down) sink.mark[1][lb[pr] + pre + py] = 1;
          else sink.mark[0][la[pr] + pre + px] = 1;
        }
        x = px; y = py;
      }
      if (in_hunk) { if (has_add && has_del) ++h_mod; else if (has_add) ++h_add; else ++h_del; }
    }
  }
  if (lane == 0) detail[pr] = tsm_diff_detail{h_add, h_del, h_mod, a_as, r_as};
}

}  // namespace tsm
