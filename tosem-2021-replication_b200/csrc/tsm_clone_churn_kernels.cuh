// tsm_clone_churn_kernels.cuh - clone churn along a revision history (docs/SPEC.md section 22): which fragments of the
// clone classes of each revision (section 15, or section 21 over kept lines) a step's edit marks (section 14) touch.
//
// The pairs of a step are diffed as views of the two revisions already on the device:
//   k_churn_gather   one thread per view line: the line hash and assertion flag of its revision line (file pair_file[k],
//                    line j), so that the diff of tsm_diff_pairs_marks runs over the pairs without a second upload or scan.
//   k_churn_marks    one thread per view line: its mark onto the revision line, in a zeroed byte per revision line.
// Then per revision, over the units the classes are numbered in (lines, or kept lines under --blind):
//   k_churn_units    one thread per unit: marked, and marked assertion line (u32 each, for xscan); with kept_line the unit's
//                    revision line is kept_line[u].
//   xscan            P and PA, the prefix sums of both.
//   k_churn_frags    one thread per fragment: changed = P[m + L] - P[m] (and the same over PA), then its state.
//   k_churn_classes  persistent warps, one class at a time, 32 fragments per round: three ballots and popcounts give the kept,
//                    edited and whole counts, then the side's status rule.
#pragma once
#include "tsm_device.cuh"

namespace tsm {

// Fragment states and class statuses (tosemscan.h TSM_FRAG_* / TSM_CLONE_*).
constexpr uint8_t FRAG_KEPT = 0, FRAG_EDITED = 1, FRAG_WHOLE = 2;
constexpr uint8_t CLS_UNTOUCHED = 0, CLS_CHANGED = 1, CLS_REMOVED = 2, CLS_DIVERGED = 3, CLS_DROPPED = 4, CLS_CREATED = 5,
                  CLS_COPIED = 6, CLS_JOINED = 7;

// The pair of view line v: view_base[k] <= v < view_base[k + 1] (view_base ascending, n_pairs + 1 entries).
__device__ __forceinline__ uint32_t churn_pair_of(const unsigned long long* view_base, uint32_t n_pairs, unsigned long long v) {
  uint32_t lo = 0, hi = n_pairs;
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (view_base[mid] <= v) lo = mid; else hi = mid; }
  return lo;
}

// View line v -> its revision line: pair k's file f = pair_file[k] (>= 0 whenever the pair has lines on this side).
__device__ __forceinline__ unsigned long long churn_rev_line(const unsigned long long* view_base, uint32_t n_pairs, const int32_t* pair_file,
                                                             const unsigned long long* rev_base, unsigned long long v) {
  const uint32_t k = churn_pair_of(view_base, n_pairs, v);
  return rev_base[pair_file[k]] + (v - view_base[k]);
}

__global__ void __launch_bounds__(256) k_churn_gather(const unsigned long long* view_base, uint32_t n_pairs, const int32_t* pair_file,
                                                      const unsigned long long* rev_base, const unsigned long long* rev_hash,
                                                      const uint8_t* rev_flag, unsigned long long total, unsigned long long* hash,
                                                      uint8_t* flag) {
  const unsigned long long v = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= total) return;
  const unsigned long long g = churn_rev_line(view_base, n_pairs, pair_file, rev_base, v);
  hash[v] = rev_hash[g];
  flag[v] = rev_flag[g];
}

__global__ void __launch_bounds__(256) k_churn_marks(const unsigned long long* view_base, uint32_t n_pairs, const int32_t* pair_file,
                                                     const unsigned long long* rev_base, const uint8_t* view_mark, unsigned long long total,
                                                     uint8_t* rev_mark) {
  const unsigned long long v = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= total || !view_mark[v]) return;
  rev_mark[churn_rev_line(view_base, n_pairs, pair_file, rev_base, v)] = 1;
}

// unit_line: NULL = unit u is revision line u; unit_flag: the assertion flag of every unit.
__global__ void __launch_bounds__(256) k_churn_units(const uint8_t* rev_mark, const unsigned long long* unit_line, const uint8_t* unit_flag,
                                                     uint32_t n_units, uint32_t* marked, uint32_t* marked_assert) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_units) return;
  const uint32_t m = rev_mark[unit_line ? unit_line[u] : u];
  marked[u] = m;
  marked_assert[u] = m & (unit_flag[u] ? 1u : 0u);
}

__global__ void __launch_bounds__(256) k_churn_frags(const unsigned long long* class_base, const uint32_t* class_len, uint32_t n_classes,
                                                     const unsigned long long* member, unsigned long long n_members,
                                                     const unsigned long long* P, const unsigned long long* PA, uint32_t* changed,
                                                     uint32_t* changed_assert, uint8_t* state) {
  const unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_members) return;
  uint32_t lo = 0, hi = n_classes;                         // class of fragment j: class_base[lo] <= j < class_base[lo + 1]
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (class_base[mid] <= j) lo = mid; else hi = mid; }
  const uint32_t L = class_len[lo];
  const unsigned long long m = member[j];
  const uint32_t ch = (uint32_t)(P[m + L] - P[m]);
  changed[j] = ch;
  changed_assert[j] = (uint32_t)(PA[m + L] - PA[m]);
  state[j] = ch == 0 ? FRAG_KEPT : ch == L ? FRAG_WHOLE : FRAG_EDITED;
}

// counts[3 * c + {0, 1, 2}] = kept, edited, whole fragments of class c; status[c] by the rule of the side (new_side: created,
// copied, joined, changed; else removed, diverged, dropped, changed), untouched when every fragment is kept.
__global__ void __launch_bounds__(256) k_churn_classes(const unsigned long long* class_base, uint32_t n_classes, const uint8_t* state,
                                                       bool new_side, uint32_t* counts, uint8_t* status) {
  const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n_classes; c += warps) {
    const unsigned long long b = class_base[c], e = class_base[c + 1];
    uint32_t kept = 0, edited = 0, whole = 0;
    for (unsigned long long j = b; j < e; j += 32) {
      const bool in = j + lane < e;
      const uint8_t s = in ? state[j + lane] : 0xFF;
      kept += __popc(__ballot_sync(0xffffffffu, s == FRAG_KEPT));
      edited += __popc(__ballot_sync(0xffffffffu, s == FRAG_EDITED));
      whole += __popc(__ballot_sync(0xffffffffu, s == FRAG_WHOLE));
    }
    if (lane == 0) {
      const uint32_t total = kept + edited + whole;
      uint8_t st = CLS_CHANGED;
      if (kept == total) st = CLS_UNTOUCHED;
      else if (new_side) st = whole == total ? CLS_CREATED : kept && whole ? CLS_COPIED : kept ? CLS_JOINED : CLS_CHANGED;
      else st = whole == total ? CLS_REMOVED : kept && edited ? CLS_DIVERGED : kept ? CLS_DROPPED : CLS_CHANGED;
      counts[3 * (size_t)c] = kept; counts[3 * (size_t)c + 1] = edited; counts[3 * (size_t)c + 2] = whole;
      status[c] = st;
    }
  }
}

}  // namespace tsm
