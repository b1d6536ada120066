// tsm_blame_kernels.cuh - line provenance along a revision history (docs/SPEC.md section 14).  The pairs of one batch form
// chains: pair i's old side is the new side of pair prev[i] (earlier in the batch), or, for a chain head, a file whose origins
// the host uploads.  Per pair, the k-th line of `new` that the canonical script does not insert inherits the origin of the
// k-th line of `old` that it does not delete; an inserted line j gets (label[i], j + 1).  The marks come from the DIFF_MARKS
// variants of k_diff_small / k_myers_trace (tsm_diff_kernels.cuh).
//
//   k_blame   persistent warps, one chain at a time (the host orders them longest first), its pairs in order.  Per pair two
//             passes over 32-line tiles: the origins of the kept old lines are packed by ballot and popcount into `keep`
//             (the pair's own region, indexed like its old lines), then each kept new line takes keep[rank].
#pragma once
#include "tsm_diff_kernels.cuh"

namespace tsm {

__global__ void __launch_bounds__(256) k_blame(
    const unsigned long long* la, const unsigned long long* lb, const uint8_t* del, const uint8_t* ins,
    const int32_t* prev, const int32_t* label, const tsm_origin* head, const long long* in_base,
    const int32_t* chain_pairs, const int32_t* chain_start, int32_t n_chains, uint32_t* work,
    tsm_origin* keep, tsm_origin* out) {
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  while (true) {
    uint32_t ch = 0;
    if (lane == 0) ch = atomicAdd(work, 1u);
    ch = __shfl_sync(0xffffffffu, ch, 0);
    if (ch >= (uint32_t)n_chains) return;
    for (int s = chain_start[ch]; s < chain_start[ch + 1]; ++s) {
      const int pr = chain_pairs[s];
      const unsigned long long a0 = la[pr], b0 = lb[pr];
      const int n = (int)(la[pr + 1] - a0), m = (int)(lb[pr + 1] - b0);
      const tsm_origin* src = prev[pr] >= 0 ? out + lb[prev[pr]] : head + in_base[pr];
      tsm_origin* kp = keep + a0;
      int k = 0;
      for (int t0 = 0; t0 < n; t0 += 32) {
        const int t = t0 + lane;
        const bool live = t < n && !del[a0 + t];
        const uint32_t bal = __ballot_sync(0xffffffffu, live);
        if (live) kp[k + __popc(bal & lt)] = src[t];
        k += __popc(bal);
      }
      __syncwarp();                                       // (keep and the previous pair's origins are written by other lanes)
      k = 0;
      const int32_t lab = label[pr];
      for (int j0 = 0; j0 < m; j0 += 32) {
        const int j = j0 + lane;
        const bool in = j < m;
        const bool live = in && !ins[b0 + j];
        const uint32_t bal = __ballot_sync(0xffffffffu, live);
        if (live) out[b0 + j] = kp[k + __popc(bal & lt)];
        else if (in) out[b0 + j] = tsm_origin{lab, j + 1};
        k += __popc(bal);
      }
      __syncwarp();
    }
  }
}

}  // namespace tsm
