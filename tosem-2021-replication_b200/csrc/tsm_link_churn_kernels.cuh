// tsm_link_churn_kernels.cuh - test-to-code link churn (docs/SPEC.md section 28): the links a step adds, removes, retargets and
// redefines, and the Eager / Lazy flags it introduces and removes, from the resident link stages of both revisions
// (tsm_link_kernels.cuh) and the edit marks of the changed pairs.  Lines are global indices of one revision (< 2^32).
//
//   k_lc_change   one warp per matched test of a changed pair: '=' when both bodies are equally long and no line of either is
//                 marked.
//   k_lc_calls    one thread per call of one revision, linked or not: the key (identity, name hash) into one open-addressing
//                 table of 16-B keys (lk_insert); the slot counts the calls of each side.  The identity is the new test for a
//                 new or matched test, else n_new + the old test.
//   k_lc_links    one thread per link of one revision: its index into its key's slot (behind every insertion).
//   k_lc_by_rank  one thread per new line: by_rank[kept rank] = the kept line.
//   k_lc_defmap   one thread per old definition: the new global line that corresponds to its line (the same line of an
//                 unchanged file, the kept-rank counterpart in a pair), or LK_NONE.
//   k_lc_events   persistent warps, one output test at a time (the 'D' tests in old order, then the new tests): COUNT gives the
//                 rows of each test; an xscan places them; the write pass emits them in row order (flag rows, removed links in
//                 old first-call order, the other link events in new first-call order), 32 links per round by ballot.
#pragma once
#include "tsm_link_kernels.cuh"

namespace tsm {

struct LcSlot { uint32_t calls[2], link[2]; };            // per key: the calls and the link (LK_NONE: none) of each side

__global__ void __launch_bounds__(256) k_lc_change(const tsm_smell_test* to, const tsm_smell_test* tn, const unsigned long long* obase,
                                                   const unsigned long long* nbase, const uint8_t* omark, const uint8_t* nmark,
                                                   const uint2* match, uint32_t n, uint8_t* same) {
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += warps) {
    const uint2 m = match[k];
    const tsm_smell_test a = to[m.x], b = tn[m.y];
    const unsigned long long lo = obase[a.file] + (uint32_t)a.line, ln = nbase[b.file] + (uint32_t)b.line;
    const uint32_t nb = (uint32_t)a.body_lines;
    bool eq = a.body_lines == b.body_lines;
    for (uint32_t i0 = 0; eq && i0 < nb; i0 += 32) {       // (eq and the bounds are the same in every lane)
      const uint32_t i = i0 + lane;
      eq = !__any_sync(FULL, i < nb && (omark[lo + i] | nmark[ln + i]));
    }
    if (lane == 0) same[k] = eq;
  }
}

__device__ __forceinline__ uint32_t lc_identity(uint32_t side, uint32_t t, const int32_t* omatch, uint32_t n_new) {
  return side ? t : omatch[t] >= 0 ? (uint32_t)omatch[t] : n_new + t;
}

__global__ void __launch_bounds__(256) k_lc_calls(const LinkCall* calls, uint32_t nc, const uint32_t* ltest, uint32_t side,
                                                  const int32_t* omatch, uint32_t n_new, LinkKey* tab, uint32_t mask, LcSlot* slot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  const LinkCall c = calls[i];
  bool fresh;
  const uint32_t s = lk_insert(tab, mask, LinkKey{c.key, lc_identity(side, ltest[c.line], omatch, n_new) + 1ull}, fresh);
  atomicAdd(&slot[s].calls[side], 1u);
}

__global__ void __launch_bounds__(256) k_lc_links(const tsm_link* links, uint32_t nk, const LinkDef* defs, uint32_t side,
                                                  const int32_t* omatch, uint32_t n_new, const LinkKey* tab, uint32_t mask, LcSlot* slot) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nk) return;
  const tsm_link l = links[p];
  const uint32_t s = lk_find(tab, mask, LinkKey{defs[l.name_def].key, lc_identity(side, (uint32_t)l.test, omatch, n_new) + 1ull});
  slot[s].link[side] = p;                                  // (a link's name has a call of its test: the key is present)
}

__global__ void __launch_bounds__(256) k_lc_by_rank(const uint32_t* kept, const unsigned long long* rank, uint32_t total, uint32_t* by_rank) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < total && kept[l]) by_rank[rank[l]] = l;
}

// cfile[f]: the new file of old file f (its unpaired counterpart or its pair), or -1.
__global__ void __launch_bounds__(256) k_lc_defmap(const LinkDef* defs, uint32_t nd, const int32_t* cfile, const unsigned long long* obase,
                                                   const unsigned long long* nbase, const uint8_t* omark, const unsigned long long* orank,
                                                   const unsigned long long* nrank, const uint32_t* by_rank, uint32_t* dline) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nd) return;
  const LinkDef d = defs[i];
  const int32_t fn = cfile[d.file];
  uint32_t out = LK_NONE;
  if (fn >= 0 && !omark[d.line]) out = by_rank[nrank[nbase[fn]] + (orank[d.line] - orank[obase[d.file]])];
  dline[i] = out;
}

struct LcRev {                                             // one revision's link state (links, defs and name table may be empty)
  const tsm_link* links; const unsigned long long* lbase; const tsm_link_test* tests; const LinkDef* defs;
  const LinkKey* name; uint32_t name_mask; const uint32_t* n_defs;
};

struct LcEvents {
  LcRev o, n;
  const uint2* otest; uint32_t n_out, n_new;               // per output test (old test, new test), LK_NONE where absent
  const int32_t* omatch; const LinkKey* tab; uint32_t mask; const LcSlot* slot;
  const int32_t* cfile; const uint32_t* dline;
  uint32_t* cnt; const unsigned long long* pos; tsm_link_event* out;
};

__device__ __forceinline__ int32_t lc_defs(const LcRev& r, unsigned long long key) {   // the name's definitions in r
  if (!r.name) return 0;
  const uint32_t s = lk_find(r.name, r.name_mask, LinkKey{key, lk_name_tag(0)});
  return s == LK_NONE ? 0 : (int32_t)r.n_defs[s];
}

// The event of the link pair (jo, jn) of one key (LK_NONE where a side has no link), or -1 for none.
__device__ __forceinline__ int32_t lc_kind(const LcEvents& a, uint32_t jo, uint32_t jn) {
  if (jo == LK_NONE) return TSM_LINKEV_ADDED;
  if (jn == LK_NONE) return TSM_LINKEV_REMOVED;
  const int32_t to = a.o.links[jo].target, tn = a.n.links[jn].target;
  if (to < 0 && tn < 0) return -1;
  if (to < 0 || tn < 0) return TSM_LINKEV_RETARGETED;
  const LinkDef dn = a.n.defs[tn];
  if (a.cfile[a.o.defs[to].file] != (int32_t)dn.file) return TSM_LINKEV_RETARGETED;
  return a.dline[to] == dn.line ? -1 : TSM_LINKEV_REDEFINED;
}

template <bool WRITE>
__global__ void __launch_bounds__(256) k_lc_events(LcEvents a) {
  const uint32_t FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t o = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; o < a.n_out; o += warps) {
    const uint2 t = a.otest[o];
    const uint32_t id = t.y != LK_NONE ? t.y : a.n_new + t.x;
    const uint32_t fo = t.x != LK_NONE ? a.o.tests[t.x].flags : 0u, fn = t.y != LK_NONE ? a.n.tests[t.y].flags : 0u;
    uint32_t flag_ev[2], nf = 0;
    if ((fn & ~fo) & LK_EAGER) flag_ev[nf++] = TSM_LINKEV_EAGER_INTRODUCED;
    if ((fo & ~fn) & LK_EAGER) flag_ev[nf++] = TSM_LINKEV_EAGER_REMOVED;
    if ((fn & ~fo) & LK_LAZY) flag_ev[nf++] = TSM_LINKEV_LAZY_INTRODUCED;
    if ((fo & ~fn) & LK_LAZY) flag_ev[nf++] = TSM_LINKEV_LAZY_REMOVED;
    const int32_t ot = t.x != LK_NONE ? (int32_t)t.x : -1, nt = t.y != LK_NONE ? (int32_t)t.y : -1;
    unsigned long long p = WRITE ? a.pos[o] : 0;
    if (WRITE && lane < nf)
      a.out[p + lane] = tsm_link_event{(int32_t)flag_ev[lane], -1, ot, nt, -1, -1, -1, -1, -1, -1};
    uint32_t n = nf;
    for (int side = 0; side < 2; ++side) {                 // the removed links of the old test, then the new test's events
      const LcRev& r = side ? a.n : a.o;
      const uint32_t tt = side ? t.y : t.x;
      if (tt == LK_NONE) continue;
      const unsigned long long b = r.lbase[tt], e = r.lbase[tt + 1];
      for (unsigned long long j0 = b; j0 < e; j0 += 32) {
        const unsigned long long j = j0 + lane;
        int32_t ev = -1;
        uint32_t s = 0;
        unsigned long long key = 0;
        if (j < e) {
          key = r.defs[r.links[j].name_def].key;
          s = lk_find(a.tab, a.mask, LinkKey{key, id + 1ull});
          const LcSlot x = a.slot[s];
          ev = side ? lc_kind(a, x.link[0], (uint32_t)j) : (x.link[1] == LK_NONE ? (int32_t)TSM_LINKEV_REMOVED : -1);
        }
        const uint32_t hit = __ballot_sync(FULL, ev >= 0);
        if (WRITE && ev >= 0) {
          const LcSlot x = a.slot[s];
          const bool removed = ev == TSM_LINKEV_REMOVED, added = ev == TSM_LINKEV_ADDED;
          const uint32_t gone = removed ? 1 : 0;           // the side without the link
          const int32_t cause = !(removed || added) ? -1
                                : (removed ? t.y : t.x) == LK_NONE ? TSM_LINKCAUSE_TEST
                                : x.calls[gone] == 0 ? TSM_LINKCAUSE_CALL : TSM_LINKCAUSE_DEFINITION;
          const uint32_t jo = side ? x.link[0] : (uint32_t)j, jn = side ? (uint32_t)j : LK_NONE;
          const int32_t od = jo != LK_NONE ? a.o.links[jo].n_defs : lc_defs(a.o, key);
          const int32_t nd = jn != LK_NONE ? a.n.links[jn].n_defs : lc_defs(a.n, key);
          a.out[p + n + __popc(hit & ((1u << lane) - 1))] =
              tsm_link_event{ev, cause, ot, nt, jo != LK_NONE ? (int32_t)jo : -1, jn != LK_NONE ? (int32_t)jn : -1,
                             ot >= 0 ? (int32_t)x.calls[0] : -1, nt >= 0 ? (int32_t)x.calls[1] : -1, od, nd};
        }
        n += __popc(hit);
      }
    }
    if (!WRITE && lane == 0) a.cnt[o] = n;
  }
}

}  // namespace tsm
