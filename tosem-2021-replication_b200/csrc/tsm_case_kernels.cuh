// tsm_case_kernels.cuh - test-case churn of revision pairs (docs/SPEC.md section 16), from the line records of both sides,
// the header events k_scan writes beside them and the edit marks of the DIFF_MARKS diff.  Lines are global indices of one
// side (< 2^32: the scan's staging arrays hold at most 0xFFFFFFF0 lines).
//
//   k_case_heads   one thread per header event: the event's line (binary search of line_end inside its file) -> head[l] = 1.
//   k_case_kept    one thread per line: kept[l] = 1 when the script neither deletes nor inserts line l.
//   xscan(head)    the case of every header line, cases numbered in line order; xscan(kept) the kept rank of every line.  Per
//                  pair both sides keep equally many lines, so the ranks of the two sides line up over the whole batch.
//   k_case_lines   one thread per line: first[case] = its header line; on the old side old_by_rank[rank] = the kept line.
//   k_case_reduce  persistent warps, one case at a time, 32 lines per round: lines, assertion lines, changed lines and changed
//                  assertion lines; on the new side the step-1 match through old_by_rank.
#pragma once
#include "tsm_device.cuh"

namespace tsm {

__global__ void __launch_bounds__(256) k_case_heads(const tsm_header_event* ev, uint32_t n_ev, const unsigned long long* line_base,
                                                    const uint32_t* line_end, uint32_t* head) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_ev) return;
  const tsm_header_event e = ev[i];
  unsigned long long lo = line_base[e.file], hi = line_base[e.file + 1];   // the file's first line that ends at or after line_off
  while (lo < hi) {
    const unsigned long long mid = (lo + hi) >> 1;
    if (line_end[mid] < e.line_off) lo = mid + 1; else hi = mid;
  }
  head[lo] = 1;
}

__global__ void __launch_bounds__(256) k_case_kept(const uint8_t* mark, uint32_t total, uint32_t* kept) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < total) kept[l] = mark[l] == 0;
}

__global__ void __launch_bounds__(256) k_case_lines(const uint32_t* head, const uint32_t* kept, const unsigned long long* case_of,
                                                    const unsigned long long* rank, uint32_t total, uint32_t* first, uint32_t* old_by_rank) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= total) return;
  if (head[l]) first[case_of[l]] = l;
  if (old_by_rank && kept[l]) old_by_rank[rank[l]] = l;
}

struct CaseSide {                                          // one side's line records, marks and cases
  const unsigned long long* line_base; uint32_t n_files;
  const uint8_t* flag; const uint8_t* mark;
  const uint32_t* first; uint32_t n_cases;
};

// Old side: old_by_rank == nullptr, match = -1.  New side: a case whose header line is kept matches the old case that starts
// at the corresponding old line (old_head / old_case_of of the old side), if one does.
__global__ void __launch_bounds__(256) k_case_reduce(CaseSide s, const unsigned long long* rank, const uint32_t* old_by_rank,
                                                     const uint32_t* old_head, const unsigned long long* old_case_of, tsm_case* out) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < s.n_cases; c += warps) {
    const uint32_t b = s.first[c];
    uint32_t lo = 0, hi = s.n_files;                       // file of line b: line_base[lo] <= b < line_base[lo + 1]
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s.line_base[mid] <= b) lo = mid; else hi = mid; }
    const unsigned long long fe = s.line_base[lo + 1];
    const unsigned long long e = c + 1 < s.n_cases && s.first[c + 1] < fe ? s.first[c + 1] : fe;
    uint32_t na = 0, nc = 0, nca = 0;
    for (unsigned long long q = b + lane; q < e; q += 32) {
      const bool a = s.flag[q] != 0, m = s.mark[q] != 0;
      na += a; nc += m; nca += a && m;
    }
#pragma unroll
    for (int k = 16; k; k >>= 1) {
      na += __shfl_xor_sync(0xffffffffu, na, k);
      nc += __shfl_xor_sync(0xffffffffu, nc, k);
      nca += __shfl_xor_sync(0xffffffffu, nca, k);
    }
    if (lane == 0) {
      int32_t match = -1;
      if (old_by_rank && !s.mark[b]) {
        const uint32_t ol = old_by_rank[rank[b]];
        if (old_head[ol]) match = (int32_t)old_case_of[ol];
      }
      out[c] = tsm_case{(int32_t)lo, (int32_t)(b - s.line_base[lo]), (int32_t)(e - b), (int32_t)na, (int32_t)nc, (int32_t)nca, match};
    }
  }
}

}  // namespace tsm
