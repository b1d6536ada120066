// tsm_api.cu - the extern "C" boundary of libtosemscan.so (include/tosemscan.h): context, device
// memory, H2D/D2H staging and kernel launches.  No torch types, no CPU fallback.
#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <string>
#include <unordered_map>
#include <new>
#include <utility>
#include <vector>

#include "tsm_device.cuh"

#include "tsm_scan_kernels.cuh"
#include "tsm_scan_walk.cuh"
#include "tsm_reduce_kernels.cuh"
#include "tsm_diff_kernels.cuh"
#include "tsm_blame_kernels.cuh"
#include "tsm_stmt_kernels.cuh"
#include "tsm_lines_kernels.cuh"
#include "tsm_similar_kernels.cuh"
#include "tsm_clone_kernels.cuh"
#include "tsm_blind_kernels.cuh"
#include "tsm_case_kernels.cuh"
#include "tsm_edit_kernels.cuh"
#include "tsm_smell_kernels.cuh"
#include "tsm_lexsmell_kernels.cuh"
#include "tsm_link_kernels.cuh"
#include "tsm_link_churn_kernels.cuh"
#include "tsm_move_kernels.cuh"
#include "tsm_clone_churn_kernels.cuh"
#include "../host/tsm_names.hpp"
#include "tsm_simtest_kernels.cuh"

using namespace tsm;

static const char* const kNames[TSM_K] = TSM_CAT_NAMES_INIT;

// Scratch memory of the diff / statements calls: grow-only, kept by the ctx between calls (a cudaMalloc +
// cudaFree pair per buffer and call costs more than the kernels of a C5-sized batch).
struct ScratchPool {
  struct Slot { void* p; size_t cap; bool used; };
  std::vector<Slot> slots;
  void* take(size_t bytes) {
    int best = -1;
    for (int i = 0; i < (int)slots.size(); ++i)
      if (!slots[(size_t)i].used && slots[(size_t)i].cap >= bytes && (best < 0 || slots[(size_t)i].cap < slots[(size_t)best].cap)) best = i;
    if (best < 0) {
      for (size_t i = 0; i < slots.size(); ++i)           // replace a free slot that is too small rather than pile up
        if (!slots[i].used) { cudaFree(slots[i].p); slots.erase(slots.begin() + (long)i); break; }
      void* q = nullptr;
      const size_t cap = bytes + bytes / 8 + 256;
      if (cudaMalloc(&q, cap) != cudaSuccess) return nullptr;
      slots.push_back(Slot{q, cap, true});
      return q;
    }
    slots[(size_t)best].used = true;
    return slots[(size_t)best].p;
  }
  void give(void* p) { for (Slot& s : slots) if (s.p == p) s.used = false; }
  void clear() { for (Slot& s : slots) cudaFree(s.p); slots.clear(); }
};
static thread_local ScratchPool* t_pool = nullptr;        // pool of the ctx whose call runs on this thread
struct PoolScope {                                        // (restores the pool it replaced: scopes nest)
  ScratchPool* prev;
  explicit PoolScope(ScratchPool* p) : prev(t_pool) { t_pool = p; }
  ~PoolScope() { t_pool = prev; }
};

struct DevBuf {                                           // device scratch from the ctx's pool, returned on scope exit
  void* p = nullptr;
  ~DevBuf() { reset(); }
  void reset() { if (p && t_pool) t_pool->give(p); p = nullptr; }
  bool alloc(size_t bytes) { reset(); p = t_pool ? t_pool->take(bytes ? bytes : 16) : nullptr; return p != nullptr; }
  template <typename T> T* as() const { return static_cast<T*>(p); }
};

struct SyncGuard {                                        // error paths: wait for the work queued on st before the DevBufs of the
  cudaStream_t st;                                        // call hand their slots back to the pool (see CallScope)
  explicit SyncGuard(cudaStream_t s) : st(s) {}
  ~SyncGuard() { cudaStreamSynchronize(st); }
};

// The timed calls: tsm_ctx::last_ms[MS_*] holds the phases of the last call of each, which its tsm_*_last_ms returns.
enum Timed {
  MS_DIFF,    // k_scan over both sides, k_diff_small, k_myers + k_myers_trace of the last pair call (whose k_scan time is
              // its own row's for tsm_similarity and tsm_diff_pairs_assert_edits)
  MS_SIM,     // k_scan over both sides, sort / merge, k_similarity of the last tsm_similarity
  MS_CLONE,   // k_scan, grouping + classes, members + coverage of the last tsm_clones
  MS_BLIND,   // k_scan, lexing + compaction, grouping + classes, members + coverage of the last tsm_clones_blind
  MS_SMELL,   // k_scan, kinds + case spans, k_smell_lines, k_smell_tests of the last tsm_smells
  MS_CHURN,   // k_scan, smell stages, the diff, case records + k_smell_churn of the last tsm_diff_pairs_smells
  MS_EDIT,    // k_scan, the diff, compact to pairing (host clock) of the last tsm_diff_pairs_assert_edits
  MS_MOVE,    // k_scan, the diff, line flags to k_move_reach, k_move_starts to k_move_mark of the last tsm_diff_pairs_moves
  MS_BLAME,   // k_blame of the last tsm_blame_pairs
  MS_CCHURN,  // k_scan of both revisions, classes of both, the marks diff, the churn kernels of the last tsm_clone_churn
  MS_SIMTEST, // k_scan, case spans + smell stage + lexer, tokens + lists + enumeration, verification of the last tsm_similar_tests
  MS_SCHURN,  // k_scan of both revisions, fronts + marks + k_sc_change, tokens + lists + enumeration, verification of the last
              // tsm_similar_churn
  MS_LEXSMELL,// k_scan, front (case spans + smell stage), lexer states + k_lex_body + k_lex_lines, k_lex_tests of the last
              // tsm_smells_lexical
  MS_LEXCHURN,// k_scan, smell and lexical stages, the diff, case records + k_smell_churn<true> of the last
              // tsm_diff_pairs_smells_lexical
  MS_LINKS,   // k_scan, front (smell stage, lexer states, test code lines), k_link_lines, the join to the records of the last
              // tsm_test_links
  MS_LCHURN,  // k_scan of both revisions, both link fronts + marks + k_lc_change, both link joins, the churn join and emit of
              // the last tsm_link_churn
  N_TIMED
};

// tsm_ctx::h_rb: the counts a call reads back between its kernels, at fixed offsets in 256 B of pinned memory.
struct alignas(32) SideCtrl { Ctrl v; };
struct Readback {
  SideCtrl ctrl[2];                        // the Ctrl of each side's scan (line records)
  unsigned long long total[2];             // the line total of each side
  uint32_t n_todo;                         // the pairs k_diff_small leaves to k_myers
  alignas(64) unsigned long long u64[4];   // the counts of the call's own stages (clones, smells, smell churn, moves)
};
static_assert(offsetof(Readback, ctrl[1]) == 32 && offsetof(Readback, total) == 64 && offsetof(Readback, n_todo) == 80 &&
              offsetof(Readback, u64) == 128 && sizeof(Readback) <= 256, "Readback: the 256 B block");

struct tsm_ctx {
  int device = 0;
  ScratchPool pool;
  int cls_per_sm = 0; size_t cls_smem = (size_t)-1;      // resident k_classify blocks per SM at cls_smem bytes of histogram
  int sms = 0;
  int64_t max_arena = 0;
  int32_t max_files = 0, max_groups = 0;
  int64_t max_events = 0;
  // device buffers
  uint8_t* d_arena = nullptr;
  int32_t* d_off = nullptr;
  int32_t* d_len = nullptr;
  uint8_t* d_ext = nullptr;
  uint16_t* d_grp = nullptr;
  uint32_t* d_unit_file = nullptr;
  uint32_t* d_unit_begin = nullptr;
  uint32_t unit_cap = 0;
  uint8_t* d_zero = nullptr;                // one allocation, zeroed by one memset per scan: ctrl | slab | counts
  Ctrl* d_ctrl = nullptr;
  SlabCtl* d_slab = nullptr;                // [kMaxSlabs]
  cudaStream_t copy_stream = nullptr;       // H2D of arena slabs, overlapped with the scan of earlier slabs
  cudaEvent_t slab_ev[64] = {};
  cudaEvent_t ready_ev = nullptr;
  cudaEvent_t order_ev = nullptr;           // recorded behind the device work of every call (CallScope)
  static constexpr int kEvSlots = 8;
  cudaEvent_t diff_ev[kEvSlots] = {};      // around the kernels of the pair and line-record calls: slots EV_*
  Readback* h_rb = nullptr;                // 256 B pinned: what those calls read back between their kernels
  float last_ms[N_TIMED][4] = {};          // phases of the last call of each timed kind (MS_*)
  struct HostSidePair* res_pair = nullptr; // sides kept in HBM by tsm_diff_upload
  static constexpr int kMaxSlabs = 64;
  tsm_file_stat* d_stats = nullptr;
  unsigned long long* d_cand = nullptr;
  tsm_header_event* d_hev = nullptr;
  tsm_assert_event* d_aev = nullptr;
  unsigned long long* d_counts = nullptr;   // [(max_groups + 1) * K + 4]
  Ctrl* h_ctrl = nullptr;                   // pinned
  // resident corpus
  bool resident = false, scanned = false;
  int32_t n_files = 0, n_groups = 1;
  int64_t arena_bytes = 0;
  uint32_t last_flags = 0;
  int launches = 0;
  // CUDA events around the 4 scan kernels: a ring of sets so that back-to-back scans can be timed
  // per kernel without a host sync inside the timed region.
  static constexpr int kRing = 32;
  cudaEvent_t ev[kRing][5] = {};
  bool ev_used[kRing] = {};
  int ev_next = 0, ev_last = -1;
  double ms_sum[4] = {0, 0, 0, 0};
  long long ms_n = 0;
};

// Slots of tsm_ctx::diff_ev, by call and phase.  Each phase reads its slots behind a synchronisation of its own, and a later
// phase records a slot again only after that: the rows below a call's line-record row reuse slots that have been read.
//
//   phase                                  0       1       2       3       4       5       6       7       read
//   line records of side 0 / 1 (k_scan)    SCAN[0] SCAN[0]                                 SCAN[1] SCAN[1] sides_records
//   diff_core                                              SMALL   SMALL   LEFT    LEFT                    diff_core, per launch
//   tsm_similarity                                         LISTS   PAIRS   END                             at the end
//   tsm_clones                                             GROUP   MEMBERS END                             at the members / end
//   tsm_clones_blind                                       GROUP   MEMBERS END     LEX     LEX_END         at the kept count /
//                                                                                                         the members / end
//   tsm_smells (smell_stage: LINES - END)                  KINDS   LINES   TESTS   END                     at the end
//   tsm_diff_pairs_smells: smell stages    CHURN_SMELLS            LINES*  TESTS*  END*                    before the diff
//     (_lexical) lexical stages, then                                                      CHURN_LEX       at the end
//     case records + churn, behind diff    CHURN_CASES                                                     at the end
//   tsm_diff_pairs_moves, behind the diff  MOVE_FLAGS      MOVE_JOIN       MOVE_RUNS       MOVE_MARK       at the end
//   tsm_blame_pairs, behind the diff       BLAME                                                           at the end
//   tsm_clone_churn: gather, behind scans  CCHURN                                                          behind the diff
//     marks, then per side behind classes  CCHURN                                                          at each end
//   tsm_similar_tests                                      FRONT   ENUM*   VERIFY* END*    LEXED   LISTS   at the counts /
//                                                                                                         each chunk
//   tsm_smells_lexical                                     FRONT                   END     LINES   TESTS   at the test count /
//                                                                                                         the end
//   (* recorded by smell_stage, and not read in this call)
struct EvSpan { int from, to; };
constexpr EvSpan EV_SCAN[2] = {{0, 1}, {6, 7}}, EV_SMALL = {2, 3}, EV_LEFT = {4, 5};
constexpr int EV_SIM_LISTS = 2, EV_SIM_PAIRS = 3, EV_SIM_END = 4;
constexpr int EV_CLONE_GROUP = 2, EV_CLONE_MEMBERS = 3, EV_CLONE_END = 4;
constexpr int EV_BLIND_LEX = 5, EV_BLIND_LEX_END = 6;
constexpr int EV_SMELL_KINDS = 2, EV_SMELL_LINES = 3, EV_SMELL_TESTS = 4, EV_SMELL_END = 5;
constexpr EvSpan EV_CHURN_SMELLS = {0, 1}, EV_CHURN_CASES = {0, 1};   // the old side's scan slots, then the same again
constexpr EvSpan EV_CHURN_LEX = {6, 7};                                 // the new side's scan slots (diff_core leaves them)
constexpr EvSpan EV_MOVE_FLAGS = {0, 1}, EV_MOVE_JOIN = {2, 3}, EV_MOVE_RUNS = {4, 5}, EV_MOVE_MARK = {6, 7};
constexpr EvSpan EV_BLAME = {0, 1};
constexpr EvSpan EV_CCHURN = {0, 1};
constexpr int EV_LK_FRONT = 2, EV_LK_LINES = 6, EV_LK_JOIN = 7, EV_LK_END = 5;
constexpr int EV_LX_FRONT = 2, EV_LX_LINES = 6, EV_LX_TESTS = 7, EV_LX_END = 5;
constexpr int EV_LC_FROM = 2, EV_LC_TO = 5;
constexpr int EV_ST_FRONT = 2, EV_ST_ENUM = 3, EV_ST_VERIFY = 4, EV_ST_END = 5, EV_ST_LEXED = 6, EV_ST_LISTS = 7;

// The start of every call that queues device work on st: the ctx's device, the ctx's pool for the call's DevBufs, and the
// order of the ctx's calls.  A ctx orders its own work, whatever stream each call is given: the call's stream first waits
// for the ctx's order event (a wait on an event that was never recorded is a no-op), and the event is recorded on it
// behind everything the call queued, on every return path once the device is set.  status = the first failure.
// Order of a call's objects: this scope, then the DevBufs (and the HostSides that hold them), then a SyncGuard.
// Destruction runs backwards: the SyncGuard waits for st before any buffer goes back to the pool (the next call may
// reuse or free it), and the order event is recorded behind all of it.  A helper that takes DevBufs of its own
// (diff_core, diff_asserts, the tails of line_records and pair_call) synchronises st before it returns them on success;
// on an error it returns them at once, but the call then unwinds without allocating again and its SyncGuard waits for
// st before the call returns.
struct CallScope {
  tsm_ctx* c; cudaStream_t st;
  PoolScope pool;
  bool on_device;
  cudaError_t status;
  CallScope(tsm_ctx* ctx, cudaStream_t s) : c(ctx), st(s), pool(&ctx->pool) {
    status = cudaSetDevice(c->device);
    on_device = status == cudaSuccess;
    if (on_device) status = cudaStreamWaitEvent(st, c->order_ev, 0);
  }
  ~CallScope() { if (on_device) cudaEventRecord(c->order_ev, st); }
};

// Fold the elapsed times of event set `i` into the running sums (waits for it if still in flight).
static void fold_events(tsm_ctx* c, int i) {
  if (!c->ev_used[i]) return;
  if (cudaEventSynchronize(c->ev[i][4]) == cudaSuccess) {
    float ms;
    bool ok = true;
    float t[4];
    for (int k = 0; k < 4; ++k) { ok &= cudaEventElapsedTime(&ms, c->ev[i][k], c->ev[i][k + 1]) == cudaSuccess; t[k] = ms; }
    if (ok) { for (int k = 0; k < 4; ++k) c->ms_sum[k] += t[k]; c->ms_n++; }
  }
  c->ev_used[i] = false;
}

#define CU(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
  fprintf(stderr, "tosemscan: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return TSM_E_CUDA; } } while (0)

extern "C" int tsm_abi_version(void) { return TSM_ABI_VERSION; }

extern "C" const char* tsm_strerror(int s) {
  switch (s) {
    case TSM_OK: return "ok";
    case TSM_E_ARG: return "bad argument";
    case TSM_E_LAYOUT: return "corpus violates the arena layout (docs/SPEC.md section 1)";
    case TSM_E_CAPACITY: return "corpus or event list exceeds the context capacity";
    case TSM_E_CUDA: return "CUDA error (no device, allocation or launch failure)";
    case TSM_E_NOMEM: return "out of host memory";
    case TSM_E_STATE: return "call out of order";
    default: return "unknown status";
  }
}

extern "C" const char* tsm_category_name(int id) {
  if (id == TSM_CAT_OTHER) return "<other>";
  if (id < 0 || id >= TSM_CAT_NAMED) return "";
  return kNames[id];
}

static void build_lut(uint32_t* lut) {                   // the automaton table of tsm_device.cuh (bit 30 = 'F', bit 31 = newline)
  struct Pat { const char* s; int first; bool ci; };
  static const Pat pats[] = {{"assert", 0, true}, {"EXPECT_", 6, false}, {"class", 13, false}, {"def", 18, false},
                             {"test", 21, true}, {"void", 25, false}, {"{", 29, false}, {"F", 30, false}, {"\n", 31, false}};
  memset(lut, 0, 256 * sizeof(uint32_t));
  for (const Pat& p : pats)
    for (int k = 0; p.s[k]; ++k) {
      const unsigned char c = (unsigned char)p.s[k];
      lut[c] |= 1u << (p.first + k);
      if (p.ci && c >= 'a' && c <= 'z') lut[c - 32] |= 1u << (p.first + k);
    }
}

static void build_lut_b(uint32_t* lut) {                 // Rev-B triggers (tsm_scan_walk.cuh, docs/SPEC.md section 4b)
  struct Pat { const char* s; int first; };
  static const Pat pats[] = {{"_CHECK", 0}, {"TESTEQUAL", 6}, {"FAIL", 15}};
  memset(lut, 0, 256 * sizeof(uint32_t));
  for (const Pat& p : pats)
    for (int k = 0; p.s[k]; ++k) lut[(unsigned char)p.s[k]] |= 1u << (p.first + k);
}

static void build_elut(uint32_t* lut) {                  // operator patterns of SPEC section 6 rule 2
  struct Pat { const char* s; int first; };
  static const Pat pats[] = {{" not ", 0}, {" in ", 5}, {" is not ", 9}, {"True", 17}, {"==", 21}, {"!=", 23},
                             {"<=", 25}, {">=", 27}, {"<", 29}, {">", 30}};
  memset(lut, 0, 256 * sizeof(uint32_t));
  for (const Pat& p : pats)
    for (int k = 0; p.s[k]; ++k) lut[(unsigned char)p.s[k]] |= 1u << (p.first + k);
}

static void free_res_pair(tsm_ctx* c);

// f(std::integral_constant<int, I>{}) for every size I of k_diff_small (DS_SIZES), in order.
template <typename F, int... I> static void for_ds_sizes(F&& f, std::integer_sequence<int, I...>) { (f(std::integral_constant<int, I>{}), ...); }
template <typename F> static void for_ds_sizes(F&& f) { for_ds_sizes(f, std::make_integer_sequence<int, DS_N>()); }

template <int MODE> static bool diff_small_smem() {      // the dynamic shared memory limit of every k_diff_small size
  bool ok = true;
  for_ds_sizes([&](auto i) {
    constexpr DiffSmallSize s = DS_SIZES[decltype(i)::value];
    ok = ok && cudaFuncSetAttribute(k_diff_small<s.hcap, s.dcap, s.warps, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)s.smem()) == cudaSuccess;
  });
  return ok;
}

extern "C" void tsm_destroy(tsm_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaFree(c->d_arena); cudaFree(c->d_off); cudaFree(c->d_len); cudaFree(c->d_ext); cudaFree(c->d_grp);
  cudaFree(c->d_unit_file); cudaFree(c->d_unit_begin); cudaFree(c->d_zero); cudaFree(c->d_stats);
  c->pool.clear();
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  for (cudaEvent_t e : c->slab_ev) if (e) cudaEventDestroy(e);
  if (c->ready_ev) cudaEventDestroy(c->ready_ev);
  if (c->order_ev) cudaEventDestroy(c->order_ev);
  for (cudaEvent_t e : c->diff_ev) if (e) cudaEventDestroy(e);
  free_res_pair(c);
  cudaFree(c->d_cand); cudaFree(c->d_hev); cudaFree(c->d_aev);
  if (c->h_ctrl) cudaFreeHost(c->h_ctrl);
  if (c->h_rb) cudaFreeHost(c->h_rb);
  for (auto& set : c->ev) for (cudaEvent_t e : set) if (e) cudaEventDestroy(e);
  delete c;
}

extern "C" int tsm_create(tsm_ctx** out, int device, int64_t max_arena_bytes, int32_t max_files,
                          int32_t max_groups, int64_t max_events) {
  if (!out || max_arena_bytes <= 0 || max_arena_bytes >= (1ll << 31) || max_files <= 0 || max_groups <= 0)
    return TSM_E_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
    fprintf(stderr, "tosemscan: no usable CUDA device %d (there is no CPU fallback)\n", device);
    return TSM_E_CUDA;
  }
  CU(cudaSetDevice(device));
  tsm_ctx* c = new (std::nothrow) tsm_ctx;
  if (!c) return TSM_E_NOMEM;
  c->device = device;
  {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) { tsm_destroy(c); return TSM_E_CUDA; }
    c->sms = sms;
  }
  c->max_arena = (max_arena_bytes + 127) / 128 * 128;
  c->max_files = max_files;
  c->max_groups = max_groups;
  c->max_events = max_events > 0 ? max_events : c->max_arena / 32 + max_files;
  if (c->max_events > 0xFFFFFFF0ll) c->max_events = 0xFFFFFFF0ll;
  c->unit_cap = (uint32_t)(c->max_arena / CH + max_files);
  int rc = TSM_OK;
  auto A = [&](void** p, size_t bytes) { if (rc == TSM_OK && cudaMalloc(p, bytes ? bytes : 16) != cudaSuccess) rc = TSM_E_CUDA; };
  A((void**)&c->d_arena, (size_t)c->max_arena + 4096);   // slack: bulk copies round sizes up to 16 B
  A((void**)&c->d_off, sizeof(int32_t) * ((size_t)max_files + 1));
  A((void**)&c->d_len, sizeof(int32_t) * (size_t)max_files);
  A((void**)&c->d_ext, (size_t)max_files);
  A((void**)&c->d_grp, sizeof(uint16_t) * (size_t)max_files);
  A((void**)&c->d_unit_file, sizeof(uint32_t) * (size_t)c->unit_cap);
  A((void**)&c->d_unit_begin, sizeof(uint32_t) * (size_t)c->unit_cap);
  {
    const size_t slab_off = 256, counts_off = slab_off + (sizeof(SlabCtl) * tsm_ctx::kMaxSlabs + 255) / 256 * 256;
    A((void**)&c->d_zero, counts_off + sizeof(unsigned long long) * ((size_t)(max_groups + 1) * TSM_K + 4));
    c->d_ctrl = reinterpret_cast<Ctrl*>(c->d_zero);
    c->d_slab = reinterpret_cast<SlabCtl*>(c->d_zero + slab_off);
    c->d_counts = reinterpret_cast<unsigned long long*>(c->d_zero + counts_off);
  }
  if (rc == TSM_OK && cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess) rc = TSM_E_CUDA;
  for (cudaEvent_t& e : c->slab_ev) if (rc == TSM_OK && cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) rc = TSM_E_CUDA;
  if (rc == TSM_OK && cudaEventCreateWithFlags(&c->ready_ev, cudaEventDisableTiming) != cudaSuccess) rc = TSM_E_CUDA;
  if (rc == TSM_OK && cudaEventCreateWithFlags(&c->order_ev, cudaEventDisableTiming) != cudaSuccess) rc = TSM_E_CUDA;
  for (cudaEvent_t& e : c->diff_ev) if (rc == TSM_OK && cudaEventCreate(&e) != cudaSuccess) rc = TSM_E_CUDA;
  A((void**)&c->d_stats, sizeof(tsm_file_stat) * (size_t)max_files);
  A((void**)&c->d_cand, sizeof(unsigned long long) * (size_t)c->max_events);
  if (rc == TSM_OK && cudaHostAlloc((void**)&c->h_ctrl, sizeof(Ctrl) + 64, cudaHostAllocDefault) != cudaSuccess) rc = TSM_E_CUDA;
  if (rc == TSM_OK && cudaHostAlloc((void**)&c->h_rb, 256, cudaHostAllocDefault) != cudaSuccess) rc = TSM_E_CUDA;
  for (auto& set : c->ev) for (cudaEvent_t& e : set) if (rc == TSM_OK && cudaEventCreate(&e) != cudaSuccess) rc = TSM_E_CUDA;
  if (rc == TSM_OK) {
    uint32_t lut[256];
    build_lut(lut);
    static const uint8_t slot[TSM_CAT_SLOTS] = TSM_CAT_SLOT_INIT;
    static const uint16_t offs[TSM_CAT_NAMED + 1] = TSM_CAT_OFF_INIT;
    static const char blob[] = TSM_CAT_BLOB_INIT;
    uint32_t elut[256], lutb[256];
    build_elut(elut);
    build_lut_b(lutb);
    BlindKw bkw[BLIND_KW_SLOTS];
    uint8_t bkind[BLIND_KW_SLOTS];
    blind_keyword_table(bkw, bkind);
    if (cudaMemcpyToSymbol(c_lut, lut, sizeof lut) != cudaSuccess ||
        cudaMemcpyToSymbol(c_elut, elut, sizeof elut) != cudaSuccess ||
        cudaMemcpyToSymbol(c_cat_slot, slot, sizeof slot) != cudaSuccess ||
        cudaMemcpyToSymbol(c_cat_off, offs, sizeof offs) != cudaSuccess ||
        cudaMemcpyToSymbol(c_cat_blob, blob, TSM_CAT_BLOB_LEN + 1) != cudaSuccess ||
        cudaMemset(c->d_arena, 0, (size_t)c->max_arena + 4096) != cudaSuccess ||
        cudaMemcpyToSymbol(c_lut_b, lutb, sizeof lutb) != cudaSuccess ||
        cudaMemcpyToSymbol(c_blind_kw, bkw, sizeof bkw) != cudaSuccess ||
        cudaMemcpyToSymbol(c_blind_kind, bkind, sizeof bkind) != cudaSuccess ||
        cudaFuncSetAttribute(k_scan_t<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SCAN2_SMEM) != cudaSuccess ||
        cudaFuncSetAttribute(k_scan_t<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SCAN2_SMEM_B) != cudaSuccess ||
        !diff_small_smem<DIFF_PLAIN>() || !diff_small_smem<DIFF_EMIT>() || !diff_small_smem<DIFF_MARKS>() ||
        cudaFuncSetAttribute(k_sim_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIM_SORT_SMEM) != cudaSuccess ||
        cudaFuncSetAttribute(k_clone_sort_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SIM_SORT_SMEM) != cudaSuccess)
      rc = TSM_E_CUDA;
  }
  // The arena memset runs on the legacy stream and the last constant-table copy may still be in flight: a first call on
  // a non-blocking stream would not be ordered behind either.
  if (rc == TSM_OK && cudaDeviceSynchronize() != cudaSuccess) rc = TSM_E_CUDA;
  if (rc != TSM_OK) {
    fprintf(stderr, "tosemscan: tsm_create failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    tsm_destroy(c);
    return rc;
  }
  *out = c;
  return TSM_OK;
}

// Layout rules of docs/SPEC.md section 1.  check_corpus_head: the O(1) part, for the scan's corpus.  check_files: the
// per-file part over files [f0, f1) - aligned starts, every file inside [off[i], off[i+1]) (so the offsets ascend and no
// file runs into the next), and the range inside the arena (off[f1] <= off[n_files]: tsm_scan copies a slab's bytes
// [off[f0], off[f1]) before it has checked the files behind the slab) - plus, as the caller asks, every ext <= TSM_EXT_H
// (if ext is given) and check_groups.  tsm_scan checks a slab's files while the slab in front of it is on the wire.
static int check_corpus_head(const tsm_ctx* c, const tsm_corpus* k) {
  if (!k || k->n_files < 0 || k->n_groups < 1 || (k->n_files > 0 && (!k->arena || !k->off || !k->len || !k->ext)))
    return TSM_E_ARG;
  if (k->n_files > c->max_files || k->n_groups > c->max_groups) return TSM_E_CAPACITY;
  if (k->n_files == 0) return TSM_OK;
  const int64_t total = k->off[k->n_files];
  if (total < 0 || (total & (TSM_ALIGN - 1))) return TSM_E_LAYOUT;
  if (total > c->max_arena) return TSM_E_CAPACITY;
  return TSM_OK;
}
static int check_groups(const tsm_corpus* k, int32_t f0, int32_t f1) {   // every grp of files [f0, f1) below n_groups
  if (k->n_groups < 1) return TSM_E_ARG;
  if (k->grp)
    for (int32_t i = f0; i < f1; ++i)
      if (k->grp[i] >= k->n_groups) return TSM_E_LAYOUT;
  return TSM_OK;
}
static int check_files(const tsm_corpus* k, int32_t f0, int32_t f1, bool ext_rule, bool grp_rule) {
  for (int32_t i = f0; i < f1; ++i) {
    const int64_t o = k->off[i], l = k->len[i];
    if (o < 0 || (o & (TSM_ALIGN - 1)) || l < 0 || o + l > (int64_t)k->off[i + 1] || (ext_rule && k->ext && k->ext[i] > TSM_EXT_H))
      return TSM_E_LAYOUT;
  }
  if (f0 < f1 && k->off[f1] > k->off[k->n_files]) return TSM_E_LAYOUT;
  return grp_rule ? check_groups(k, f0, f1) : TSM_OK;
}

// The file index (off, len, ext, grp; NULL grp = all 0) to the ctx, which takes the corpus' sizes.
static int upload_index(tsm_ctx* c, const tsm_corpus* k, cudaStream_t st) {
  const int32_t n = k->n_files;
  c->n_files = n;
  c->n_groups = k->n_groups;
  c->arena_bytes = n ? k->off[n] : 0;
  if (n) {
    CU(cudaMemcpyAsync(c->d_off, k->off, sizeof(int32_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(c->d_len, k->len, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(c->d_ext, k->ext, (size_t)n, cudaMemcpyHostToDevice, st));
    if (k->grp) CU(cudaMemcpyAsync(c->d_grp, k->grp, sizeof(uint16_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    else CU(cudaMemsetAsync(c->d_grp, 0, sizeof(uint16_t) * (size_t)n, st));
  }
  return TSM_OK;
}

extern "C" int tsm_upload(tsm_ctx* c, const tsm_corpus* k, void* stream) {
  if (!c) return TSM_E_ARG;
  int rc = check_corpus_head(c, k);
  if (rc == TSM_OK) rc = check_files(k, 0, k->n_files, true, true);
  if (rc != TSM_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  rc = upload_index(c, k, st);
  if (rc != TSM_OK) return rc;
  if (c->n_files) CU(cudaMemcpyAsync(c->d_arena, k->arena, (size_t)c->arena_bytes, cudaMemcpyHostToDevice, st));
  c->resident = true;
  c->scanned = false;
  return TSM_OK;
}

static int ensure_event_buffers(tsm_ctx* c, uint32_t flags) {
  if ((flags & TSM_SCAN_ASSERT_EVENTS) && !c->d_aev)
    CU(cudaMalloc((void**)&c->d_aev, sizeof(tsm_assert_event) * (size_t)c->max_events));
  if ((flags & TSM_SCAN_HEADER_EVENTS) && !c->d_hev)
    CU(cudaMalloc((void**)&c->d_hev, sizeof(tsm_header_event) * (size_t)c->max_events));
  return TSM_OK;
}

static ScanParams make_params(const tsm_ctx* c, uint32_t flags) {   // the ScanParams of a scan of the ctx's corpus
  ScanParams p{};
  p.arena = c->d_arena; p.off = c->d_off; p.len = c->d_len; p.ext = c->d_ext; p.grp = c->d_grp;
  p.n_files = c->n_files; p.n_groups = c->n_groups;
  p.unit_file = c->d_unit_file; p.unit_begin = c->d_unit_begin; p.unit_cap = c->unit_cap;
  p.ctrl = c->d_ctrl; p.stats = c->d_stats;
  p.cand = c->d_cand; p.cand_cap = (uint32_t)c->max_events;
  p.hev = c->d_hev; p.hev_cap = (uint32_t)c->max_events;
  p.aev = c->d_aev; p.aev_cap = (uint32_t)c->max_events;
  p.counts = c->d_counts; p.flags = flags; p.four = 4; p.cls_last = 1;
  return p;
}

// k_scan over the slab of p, with the Rev-B triggers or without.
static void launch_k_scan(const tsm_ctx* c, const ScanParams& p, bool rev_b, cudaStream_t st) {
  if (rev_b) k_scan_t<true><<<c->sms * SCAN2_CTAS_PER_SM, SCAN2_WARPS * 32, SCAN2_SMEM_B, st>>>(p);
  else k_scan_t<false><<<c->sms * SCAN2_CTAS_PER_SM, SCAN2_WARPS * 32, SCAN2_SMEM, st>>>(p);
}

// The dynamic shared memory of k_classify over n_groups groups (their histogram is kept per block up to 16 groups) and
// one resident wave of its blocks, which loop over the candidates (the occupancy query is cached for the last size).
struct ClassifyShape { size_t smem; uint32_t wave; };
static ClassifyShape classify_shape(tsm_ctx* c, int32_t n_groups) {
  const size_t smem = CLS_SMEM_BASE + sizeof(uint32_t) * (n_groups <= 16 ? (size_t)n_groups * TSM_K : 0);
  if (c->cls_smem != smem) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_classify_t<false>, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 4;
    c->cls_per_sm = per_sm;
    c->cls_smem = smem;
  }
  return {smem, (uint32_t)(c->sms * c->cls_per_sm)};
}

static void launch_k_classify(const ScanParams& p, bool rev_b, uint32_t grid, size_t smem, cudaStream_t st) {
  if (rev_b) k_classify_t<true><<<grid, 256, smem, st>>>(p);
  else k_classify_t<false><<<grid, 256, smem, st>>>(p);
}

// One scan = [memsets] + per slab (k_plan, k_scan) + k_classify on `st`.  With host != NULL
// the arena slabs are copied on the ctx's copy stream and each slab's kernels wait for its copy only,
// so the H2D of slab s+1 overlaps the scan of slab s (the e2e path); with host == NULL the arena is
// already resident and there is a single slab.
static int launch_scan(tsm_ctx* c, uint32_t flags, cudaStream_t st, const tsm_corpus* host, bool check_files_here = false) {
  int rc = ensure_event_buffers(c, flags);
  if (rc != TSM_OK) return rc;
  ScanParams p = make_params(c, flags);
  const int n = c->n_files;
  c->launches = 0;
  CU(cudaMemsetAsync(c->d_zero, 0, (size_t)(reinterpret_cast<uint8_t*>(c->d_counts) - c->d_zero) +
                     sizeof(unsigned long long) * ((size_t)(c->n_groups + 1) * TSM_K + 4), st));   // ctrl | slab | counts
  if (n) {                                               // (k_plan zeroes the per-file records that k_scan adds into)
    // slab boundaries (file indices): one slab when resident, ~32 MiB of arena each when streaming
    std::vector<int32_t> cut{0};
    if (host) {
      int64_t slab_bytes = 32ll << 20;
      while (c->arena_bytes / slab_bytes + 1 > tsm_ctx::kMaxSlabs) slab_bytes *= 2;
      int64_t next = slab_bytes;
      for (int32_t i = 1; i < n; ++i)
        if ((int64_t)host->off[i] >= next) { cut.push_back(i); next = (int64_t)host->off[i] + slab_bytes; }
      CU(cudaEventRecord(c->ready_ev, st));               // the arena may still be read by earlier work on st
      CU(cudaStreamWaitEvent(c->copy_stream, c->ready_ev, 0));
    }
    cut.push_back(n);
    if ((int)cut.size() - 1 > tsm_ctx::kMaxSlabs) return TSM_E_LAYOUT;   // (only offsets that break the layout rules can cut this often)
    const int es = c->ev_next;
    c->ev_next = (es + 1) % tsm_ctx::kRing;
    fold_events(c, es);                                  // only blocks when 32 scans are in flight
    cudaEvent_t* ev = c->ev[es];
    CU(cudaEventRecord(ev[0], st));
    const int n_slabs = (int)cut.size() - 1;
    const bool rev_b = flags & TSM_SCAN_REV_B;
    const ClassifyShape cls = classify_shape(c, c->n_groups);
    for (int s = 0; s < n_slabs; ++s) {
      const int32_t f0 = cut[(size_t)s], f1 = cut[(size_t)s + 1];
      if (host) {
        if (check_files_here && s == 0) {                  // the first slab's files before anything of them is used ...
          const int rc0 = check_files(host, f0, f1, true, true);
          if (rc0 != TSM_OK) return rc0;
        }
        const size_t b0 = (size_t)host->off[f0], b1 = (size_t)host->off[f1];
        CU(cudaMemcpyAsync(c->d_arena + b0, host->arena + b0, b1 - b0, cudaMemcpyHostToDevice, c->copy_stream));
        CU(cudaEventRecord(c->slab_ev[s], c->copy_stream));
        CU(cudaStreamWaitEvent(st, c->slab_ev[s], 0));
        if (check_files_here && s + 1 < n_slabs) {         // ... the next slab's while this one is on the wire
          const int rc1 = check_files(host, f1, cut[(size_t)s + 2], true, true);
          if (rc1 != TSM_OK) { cudaStreamSynchronize(c->copy_stream); cudaStreamSynchronize(st); return rc1; }
        }
      }
      p.slab = c->d_slab + s; p.f_begin = f0; p.f_end = f1;
      // units of earlier slabs are bounded by (arena bytes before f0) / CH + f0
      p.unit_base = (uint32_t)((host ? (int64_t)host->off[f0] : 0) / CH + f0);
      k_plan<<<(f1 - f0 + 255) / 256, 256, 0, st>>>(p);
      CU(cudaGetLastError());
      if (s == 0 && n_slabs == 1) CU(cudaEventRecord(ev[1], st));
      launch_k_scan(c, p, rev_b, st);
      CU(cudaGetLastError());
      if (s + 1 < n_slabs) {                               // streamed scan: this slab's candidates are classified under the next
        p.cls_last = 0;                                    // slab's copy, so that only the last slab's are left behind the last copy
        launch_k_classify(p, rev_b, cls.wave, cls.smem, st);
        CU(cudaGetLastError());
        p.cls_last = 1;
      }
    }
    if (n_slabs > 1) CU(cudaEventRecord(ev[1], st));      // per-kernel split is only meaningful for one slab
    CU(cudaEventRecord(ev[2], st));
    launch_k_classify(p, rev_b, cls.wave, cls.smem, st);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ev[3], st));
    CU(cudaEventRecord(ev[4], st));                           // (slot of the former k_totals, now fused into k_classify)
    c->ev_used[es] = (n_slabs == 1);
    c->ev_last = es;
    c->launches = 3 * n_slabs;                             // k_plan + k_scan + k_classify per slab
    CU(cudaGetLastError());
  }
  c->last_flags = flags;
  c->scanned = true;
  return TSM_OK;
}

extern "C" int tsm_scan_resident(tsm_ctx* c, uint32_t flags, void* stream) {
  if (!c) return TSM_E_ARG;
  flags &= TSM_SCAN_ASSERT_EVENTS | TSM_SCAN_HEADER_EVENTS | TSM_SCAN_REV_B;
  if (!c->resident) return TSM_E_STATE;
  CallScope call(c, (cudaStream_t)stream);
  CU(call.status);
  return launch_scan(c, flags, (cudaStream_t)stream, nullptr);
}

extern "C" int tsm_device_counts(tsm_ctx* c, void** dptr, int64_t* n_int64) {
  if (!c || !dptr || !n_int64) return TSM_E_ARG;
  if (!c->scanned) return TSM_E_STATE;
  *dptr = c->d_counts;
  *n_int64 = (int64_t)(c->n_groups + 1) * TSM_K + 4;
  return TSM_OK;
}

extern "C" int tsm_last_launch_count(tsm_ctx* c) { return c ? c->launches : 0; }

#if TSM_PHASE_CLOCKS
// Build variant only (tools/phase_clocks.py): SM cycles per k_scan phase (ScanPhase order) summed over every warp and
// launch since the last reset.
extern "C" int tsm_phase_clocks(unsigned long long* out, int n, int reset) {
  if (!out || n < (int)PH_N) return TSM_E_ARG;
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpyFromSymbol(out, g_scan_phase_clk, sizeof(unsigned long long) * PH_N));
  if (reset) {
    const unsigned long long zero[PH_N] = {};
    CU(cudaMemcpyToSymbol(g_scan_phase_clk, zero, sizeof(zero)));
  }
  return TSM_OK;
}
#endif

extern "C" int tsm_last_kernel_ms(tsm_ctx* c, float* ms4) {
  if (!c || !ms4) return TSM_E_ARG;
  if (!c->scanned || c->n_files == 0 || c->ev_last < 0) return TSM_E_STATE;
  CU(cudaSetDevice(c->device));
  cudaEvent_t* ev = c->ev[c->ev_last];
  CU(cudaEventSynchronize(ev[4]));
  for (int i = 0; i < 4; ++i) CU(cudaEventElapsedTime(&ms4[i], ev[i], ev[i + 1]));
  return TSM_OK;
}

extern "C" int tsm_kernel_ms_stats(tsm_ctx* c, double* sum_ms4, int64_t* n_scans, int reset) {
  if (!c) return TSM_E_ARG;
  CU(cudaSetDevice(c->device));
  for (int i = 0; i < tsm_ctx::kRing; ++i) fold_events(c, i);
  if (sum_ms4) for (int k = 0; k < 4; ++k) sum_ms4[k] = c->ms_sum[k];
  if (n_scans) *n_scans = c->ms_n;
  if (reset) { for (double& v : c->ms_sum) v = 0; c->ms_n = 0; }
  return TSM_OK;
}

// Candidate and event lists of the size the counters of an overflowed scan reached (k_scan and k_classify count every
// entry, also those past the end of a list).  The new buffers are allocated before the old ones are freed, so that a
// failed allocation leaves the ctx as it was.
static int grow_event_buffers(tsm_ctx* c, int64_t need) {
  if (need <= c->max_events) return TSM_OK;
  if (need > 0xFFFFFFF0ll) return TSM_E_CAPACITY;
  unsigned long long* cand = nullptr;
  tsm_assert_event* aev = nullptr;
  tsm_header_event* hev = nullptr;
  const bool ok = cudaMalloc((void**)&cand, sizeof(unsigned long long) * (size_t)need) == cudaSuccess &&
                  (!c->d_aev || cudaMalloc((void**)&aev, sizeof(tsm_assert_event) * (size_t)need) == cudaSuccess) &&
                  (!c->d_hev || cudaMalloc((void**)&hev, sizeof(tsm_header_event) * (size_t)need) == cudaSuccess);
  if (!ok) {
    cudaGetLastError();                                  // (not sticky: later launches must not report it)
    cudaFree(cand); cudaFree(aev); cudaFree(hev);
    return TSM_E_CUDA;
  }
  cudaFree(c->d_cand); cudaFree(c->d_aev); cudaFree(c->d_hev);
  c->d_cand = cand; c->d_aev = aev; c->d_hev = hev;
  c->max_events = need;
  return TSM_OK;
}

// The per-file records, the count tables and the control block of the last scan to the host (synchronises).
static int download_tables(tsm_ctx* c, tsm_result* r, cudaStream_t st) {
  const int n = c->n_files, G = c->n_groups;
  unsigned long long* h_tot = reinterpret_cast<unsigned long long*>(c->h_ctrl + 1);   // pinned tail
  CU(cudaMemcpyAsync(c->h_ctrl, c->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(h_tot, c->d_counts + (size_t)(G + 1) * TSM_K, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  if (r->stats && n) CU(cudaMemcpyAsync(r->stats, c->d_stats, sizeof(tsm_file_stat) * (size_t)n, cudaMemcpyDeviceToHost, st));
  if (r->group_counts) CU(cudaMemcpyAsync(r->group_counts, c->d_counts, sizeof(int64_t) * (size_t)G * TSM_K, cudaMemcpyDeviceToHost, st));
  if (r->global_counts) CU(cudaMemcpyAsync(r->global_counts, c->d_counts + (size_t)G * TSM_K, sizeof(int64_t) * TSM_K, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int i = 0; i < 4; ++i) r->totals[i] = (int64_t)h_tot[i];
  return TSM_OK;
}

// Events (any order, file < n_files) into the canonical (file, line_off) order: a counting sort by file, then the few events
// of each file by line_off.  A comparison sort of the whole array costs milliseconds for a C5 batch; this is linear.
template <typename Event> static void sort_events_by_file(Event* ev, uint32_t m, int32_t n_files) {
  if (m < 2) return;
  std::vector<uint32_t> pos((size_t)n_files + 1, 0);
  for (uint32_t i = 0; i < m; ++i) pos[(size_t)ev[i].file + 1]++;
  for (int32_t f = 0; f < n_files; ++f) pos[(size_t)f + 1] += pos[(size_t)f];
  std::vector<Event> tmp(m);
  std::vector<uint32_t> at(pos.begin(), pos.end() - 1);
  for (uint32_t i = 0; i < m; ++i) tmp[at[ev[i].file]++] = ev[i];
  for (int32_t f = 0; f < n_files; ++f)
    if (pos[(size_t)f + 1] - pos[(size_t)f] > 1)
      std::sort(tmp.begin() + pos[(size_t)f], tmp.begin() + pos[(size_t)f + 1],
                [](const Event& a, const Event& b) { return a.line_off < b.line_off; });
  std::copy(tmp.begin(), tmp.end(), ev);
}

// tsm_download inside a call that has set the device and ordered st.
static int download(tsm_ctx* c, tsm_result* r, cudaStream_t st) {
  r->n_aev = 0; r->n_hev = 0;
  int rc = download_tables(c, r, st);
  if (rc != TSM_OK) return rc;
  if (c->h_ctrl->overflow) {                             // more candidates or events than the lists hold: grow them to the
    const Ctrl& k = *c->h_ctrl;                          // counts and scan the resident arena once more
    rc = grow_event_buffers(c, std::max<int64_t>(k.n_cand, std::max(k.n_hev, k.n_aev)));
    if (rc == TSM_OK) rc = launch_scan(c, c->last_flags, st, nullptr);
    if (rc == TSM_OK) rc = download_tables(c, r, st);
    if (rc != TSM_OK) return rc;
    if (c->h_ctrl->overflow) return TSM_E_CAPACITY;
  }
  const bool want_aev = (c->last_flags & TSM_SCAN_ASSERT_EVENTS) && r->aev, want_hev = (c->last_flags & TSM_SCAN_HEADER_EVENTS) && r->hev;
  if ((want_aev && (int64_t)c->h_ctrl->n_aev > r->aev_cap) || (want_hev && (int64_t)c->h_ctrl->n_hev > r->hev_cap)) {
    r->n_aev = c->h_ctrl->n_aev; r->n_hev = c->h_ctrl->n_hev;   // the caller's arrays are too small: both sizes, to call again
    return TSM_E_CAPACITY;
  }
  if (want_aev) {
    const uint32_t m = c->h_ctrl->n_aev;
    CU(cudaMemcpyAsync(r->aev, c->d_aev, sizeof(tsm_assert_event) * (size_t)m, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    sort_events_by_file(r->aev, m, c->n_files);
    r->n_aev = m;
  } else if (c->last_flags & TSM_SCAN_ASSERT_EVENTS) r->n_aev = c->h_ctrl->n_aev;
  if (want_hev) {
    const uint32_t m = c->h_ctrl->n_hev;
    CU(cudaMemcpyAsync(r->hev, c->d_hev, sizeof(tsm_header_event) * (size_t)m, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    sort_events_by_file(r->hev, m, c->n_files);
    r->n_hev = m;
  } else if (c->last_flags & TSM_SCAN_HEADER_EVENTS) r->n_hev = c->h_ctrl->n_hev;
  return TSM_OK;
}

extern "C" int tsm_download(tsm_ctx* c, tsm_result* r, void* stream) {
  if (!c || !r) return TSM_E_ARG;
  if (!c->scanned) return TSM_E_STATE;
  CallScope call(c, (cudaStream_t)stream);
  CU(call.status);
  return download(c, r, (cudaStream_t)stream);
}

extern "C" int tsm_scan(tsm_ctx* c, const tsm_corpus* k, tsm_result* r, uint32_t flags, void* stream) {
  if (!c || !r) return TSM_E_ARG;
  int rc = check_corpus_head(c, k);                       // (the per-file rules are checked slab by slab, under the copies)
  if (rc != TSM_OK) return rc;
  flags &= TSM_SCAN_ASSERT_EVENTS | TSM_SCAN_HEADER_EVENTS | TSM_SCAN_REV_B;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  rc = upload_index(c, k, st);                            // the index first (small), the arena slab by slab
  if (rc != TSM_OK) return rc;
  c->resident = true;
  rc = launch_scan(c, flags, st, k, true);
  if (rc != TSM_OK) { c->resident = false; c->scanned = false; return rc; }
  return download(c, r, st);
}

// ------------------------------------------------------------------------------------- S10 reduce
extern "C" int tsm_reduce(tsm_ctx* c, const uint8_t* flags, const int32_t* repo, const int32_t* case_id,
                          int32_t n_rows, int32_t n_flags, int32_t n_repos, int32_t n_cases,
                          int64_t* out, int64_t* cases_per_repo, void* stream) {
  if (!c || n_rows < 0 || n_flags < 0 || n_repos <= 0 || n_cases <= 0 || !out || (n_rows && (!flags || !repo || !case_id)))
    return TSM_E_ARG;
  for (int32_t i = 0; i < n_rows; ++i)
    if (repo[i] < 0 || repo[i] >= n_repos || case_id[i] < 0 || case_id[i] >= n_cases) return TSM_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  const size_t words = ((size_t)n_cases + 31) / 32;
  const size_t nbits = (size_t)(n_flags + 1) * n_repos * words;
  DevBuf b_flags, b_repo, b_case, b_bits, b_out;          // scratch from the ctx's pool (kept between calls)
  SyncGuard guard(st);
  if (!b_flags.alloc((size_t)n_rows * n_flags) || !b_repo.alloc(sizeof(int32_t) * (size_t)n_rows) ||
      !b_case.alloc(sizeof(int32_t) * (size_t)n_rows) || !b_bits.alloc(sizeof(uint32_t) * nbits) ||
      !b_out.alloc(sizeof(unsigned long long) * (size_t)(n_flags + 1) * n_repos))
    return TSM_E_CUDA;
  uint8_t* d_flags = b_flags.as<uint8_t>(); int32_t *d_repo = b_repo.as<int32_t>(), *d_case = b_case.as<int32_t>();
  uint32_t* d_bits = b_bits.as<uint32_t>();
  unsigned long long* d_out = b_out.as<unsigned long long>();
  int rc = TSM_OK;
  std::vector<unsigned long long> h((size_t)(n_flags + 1) * n_repos);
  {
    bool ok = true;
    if (n_rows) {
      ok &= cudaMemcpyAsync(d_flags, flags, (size_t)n_rows * n_flags, cudaMemcpyHostToDevice, st) == cudaSuccess;
      ok &= cudaMemcpyAsync(d_repo, repo, sizeof(int32_t) * (size_t)n_rows, cudaMemcpyHostToDevice, st) == cudaSuccess;
      ok &= cudaMemcpyAsync(d_case, case_id, sizeof(int32_t) * (size_t)n_rows, cudaMemcpyHostToDevice, st) == cudaSuccess;
    }
    ok &= cudaMemsetAsync(d_bits, 0, sizeof(uint32_t) * nbits, st) == cudaSuccess;
    ok &= cudaMemsetAsync(d_out, 0, sizeof(unsigned long long) * h.size(), st) == cudaSuccess;
    if (ok) ok &= launch_reduce(d_flags, d_repo, d_case, n_rows, n_flags, n_repos, n_cases, d_bits, d_out, st) == 0;
    ok &= cudaMemcpyAsync(h.data(), d_out, sizeof(unsigned long long) * h.size(), cudaMemcpyDeviceToHost, st) == cudaSuccess;
    ok &= cudaStreamSynchronize(st) == cudaSuccess;
    if (!ok) rc = TSM_E_CUDA;
  }
  if (rc != TSM_OK) return rc;
  // row 0 of the device table = "any row" (cases per repo), rows 1.. = the flags
  for (int32_t r = 0; r < n_repos; ++r) if (cases_per_repo) cases_per_repo[r] = (int64_t)h[r];
  for (int32_t f = 0; f < n_flags; ++f)
    for (int32_t r = 0; r < n_repos; ++r) out[(size_t)f * n_repos + r] = (int64_t)h[(size_t)(f + 1) * n_repos + r];
  c->launches = 2;
  return TSM_OK;
}

// ------------------------------------------------------------------------------------- host helpers
extern "C" void* tsm_host_alloc(int64_t bytes) {
  void* p = nullptr;
  if (bytes <= 0) return nullptr;
  if (cudaHostAlloc(&p, (size_t)bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return p;
}
extern "C" void tsm_host_free(void* p) { if (p) cudaFreeHost(p); }

// ------------------------------------------------------------------------------------- S8 diff
static float elapsed_ms(cudaEvent_t from, cudaEvent_t to) {   // 0 if the pair cannot be timed
  float ms = 0;
  return cudaEventElapsedTime(&ms, from, to) == cudaSuccess ? ms : 0.f;
}
static float span_ms(const tsm_ctx* c, EvSpan s) { return elapsed_ms(c->diff_ev[s.from], c->diff_ev[s.to]); }

// The phase times of the timed call t: cleared at the start of the call, copied out by its tsm_*_last_ms (n of them).
static float* clear_ms(tsm_ctx* c, Timed t) { std::fill_n(c->last_ms[t], 4, 0.f); return c->last_ms[t]; }
static int copy_ms(const tsm_ctx* c, Timed t, float* out, int n) {
  if (!c || !out) return TSM_E_ARG;
  std::copy_n(c->last_ms[t], n, out);
  return TSM_OK;
}

namespace {
struct HostSide {                                         // device image of one side of the pairs + its line records
  int32_t n = 0; size_t ab = 0; uint32_t unit_cap = 0;
  DevBuf arena, off, len, ext, grp, line_base, line_end, line_hash, line_flag;   // (grp: only for the changed assertion lines)
  DevBuf line_mark;                                       // 1 = line deleted (old side) / inserted (new side): DIFF_MARKS only
  DevBuf hev;                                             // header events of the scan, when asked for (test-case churn only)
  DevBuf unit_file, unit_begin, cnt, unit_first, bsum, zero, stats, unit_lines, unit_out, unit_line_base, s_hash, s_end, s_flag;
  std::vector<unsigned long long> base;                   // host copy of line_base (only when asked for)
  uint32_t n_units = 0;                                   // (file, chunk) work units: sum of ceil(len / 4 KiB)
  Ctrl hc{};                                              // read back behind the scan: capacity flags, lines written
  unsigned long long total = 0;                           // lines of the side
  DiffSide d{};
  int launches = 0;
  void drop_staging() { s_hash.reset(); s_end.reset(); s_flag.reset(); }
};

static ScanParams side_params(const HostSide& h) {        // the ScanParams over an uploaded side: the caller adds the rest
  ScanParams p{};
  p.arena = h.arena.as<uint8_t>(); p.off = h.off.as<int32_t>(); p.len = h.len.as<int32_t>(); p.ext = h.ext.as<uint8_t>();
  p.n_files = h.n; p.four = 4;
  return p;
}

// Exclusive scan of n u32 counts into n + 1 u64 (tsm_lines_kernels.cuh); bsum holds n / 1024 + 2 u64.
static void xscan(const uint32_t* in, uint32_t n, unsigned long long* bsum, unsigned long long* out, cudaStream_t st) {
  const uint32_t nb = (n + XS_TILE - 1) / XS_TILE;
  if (nb == 0) { cudaMemsetAsync(out, 0, sizeof(unsigned long long), st); return; }
  k_xscan_sums<<<nb, 256, 0, st>>>(in, n, bsum);
  k_xscan_top<<<1, 256, 0, st>>>(bsum, nb);
  k_xscan_apply<<<nb, 256, 0, st>>>(in, n, bsum, out);
}

int side_upload(const tsm_corpus* k, HostSide& h, cudaStream_t st) {
  const int32_t n = k->n_files;
  const size_t ab = (size_t)k->off[n];
  h.n = n; h.ab = ab;
  h.unit_cap = (uint32_t)(ab / CH + (size_t)n + 1);
  const uint32_t unit_cap = h.unit_cap;
  unsigned long long nu = 0;
  for (int32_t i = 0; i < n; ++i) nu += ((unsigned long long)(uint32_t)k->len[i] + CH - 1) / CH;
  if (nu > unit_cap) return TSM_E_LAYOUT;
  h.n_units = (uint32_t)nu;
  if (!h.arena.alloc(ab + 4096) || !h.off.alloc(sizeof(int32_t) * ((size_t)n + 1)) || !h.len.alloc(sizeof(int32_t) * (size_t)n) ||
      !h.ext.alloc((size_t)n) || !h.unit_file.alloc(sizeof(uint32_t) * unit_cap) || !h.unit_begin.alloc(sizeof(uint32_t) * unit_cap) ||
      !h.cnt.alloc(sizeof(uint32_t) * (size_t)n) || !h.unit_first.alloc(sizeof(unsigned long long) * ((size_t)n + 1)) ||
      !h.bsum.alloc(sizeof(unsigned long long) * (unit_cap / XS_TILE + 4)) || !h.zero.alloc(256 + sizeof(SlabCtl)) ||
      !h.stats.alloc(sizeof(tsm_file_stat) * (size_t)n) || !h.unit_lines.alloc(sizeof(uint32_t) * unit_cap) ||
      !h.unit_out.alloc(sizeof(uint32_t) * unit_cap) || !h.unit_line_base.alloc(sizeof(unsigned long long) * ((size_t)unit_cap + 1)) ||
      !h.line_base.alloc(sizeof(unsigned long long) * ((size_t)n + 1)))
    return TSM_E_CUDA;
  CU(cudaMemsetAsync(h.arena.as<uint8_t>() + ab, 0, 4096, st));
  CU(cudaMemcpyAsync(h.arena.p, k->arena, ab, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(h.off.p, k->off, sizeof(int32_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(h.len.p, k->len, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
  if (k->ext) CU(cudaMemcpyAsync(h.ext.p, k->ext, (size_t)n, cudaMemcpyHostToDevice, st));
  else CU(cudaMemsetAsync(h.ext.p, 0, (size_t)n, st));
  return TSM_OK;
}

// The group tags of an uploaded side (NULL = all 0), which the [group][category] tables of the changed assertion lines use.
int side_upload_grp(const tsm_corpus* k, HostSide& h, cudaStream_t st) {
  if (!h.grp.alloc(sizeof(uint16_t) * (size_t)h.n)) return TSM_E_CUDA;
  if (k->grp) CU(cudaMemcpyAsync(h.grp.p, k->grp, sizeof(uint16_t) * (size_t)h.n, cudaMemcpyHostToDevice, st));
  else CU(cudaMemsetAsync(h.grp.p, 0, sizeof(uint16_t) * (size_t)h.n, st));
  return TSM_OK;
}

// Line records in file order (docs/SPEC.md sections 2-4) of `ns` uploaded sides (the two sides of the revision pairs, or one
// corpus): per side line_base[n+1], and per line its hash, its end and whether it is an assertion line.  One pass of
// k_scan over the source (TSM_SCAN_LINE_HASHES: every chunk writes the records of its own lines into a region of the
// staging arrays), one exclusive scan of the lines per unit, one gather.  The kernels of all sides are queued before the
// host looks at anything: ONE synchronisation (capacity flags + line totals) per call instead of four per side.  The
// staging arrays are sized for 8-byte lines; a side with more lines than that is scanned a second time with the exact
// size (the first pass counted them).  scan_ms adds the device time of the k_scan launches (CUDA events on st).
// host_base: also copy line_base to the host (HostSide::base).  flags: TSM_SCAN_HEADER_EVENTS also lists the header events
// into HostSide::hev (hc.n_hev of them), sized like the staging arrays: a side has no more headers than lines.
static int side_scan_pass(tsm_ctx* c, HostSide& h, ScanParams& p, size_t cap, int side, cudaStream_t st) {
  const int32_t n = h.n;
  if (cap > 0xFFFFFFF0ull) return TSM_E_CAPACITY;
  if (!h.s_hash.alloc(sizeof(unsigned long long) * cap) || !h.s_end.alloc(sizeof(uint32_t) * cap) || !h.s_flag.alloc(cap)) return TSM_E_CUDA;
  p.lh_hash = h.s_hash.as<unsigned long long>(); p.lh_end = h.s_end.as<uint32_t>(); p.lh_flag = h.s_flag.as<uint8_t>();
  p.lh_cap = (uint32_t)cap;
  if (p.flags & TSM_SCAN_HEADER_EVENTS) {
    if (!h.hev.alloc(sizeof(tsm_header_event) * cap)) return TSM_E_CUDA;
    p.hev = h.hev.as<tsm_header_event>(); p.hev_cap = (uint32_t)cap;
  }
  CU(cudaMemsetAsync(h.zero.p, 0, 256 + sizeof(SlabCtl), st));
  k_plan_det<<<(n + 1 + 255) / 256, 256, 0, st>>>(p, h.unit_first.as<unsigned long long>());
  CU(cudaEventRecord(c->diff_ev[EV_SCAN[side].from], st));
  launch_k_scan(c, p, false, st);
  CU(cudaEventRecord(c->diff_ev[EV_SCAN[side].to], st));
  CU(cudaGetLastError());
  // lines per unit -> first line of every unit (the unit count is known on the host: units are (file, chunk) in order)
  xscan(p.unit_lines, h.n_units, h.bsum.as<unsigned long long>(), h.unit_line_base.as<unsigned long long>(), st);
  CU(cudaMemcpyAsync(&c->h_rb->ctrl[side].v, p.ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, st));   // pinned: no host stall
  CU(cudaMemcpyAsync(&c->h_rb->total[side], h.unit_line_base.as<unsigned long long>() + h.n_units, sizeof(unsigned long long),
                     cudaMemcpyDeviceToHost, st));
  h.launches += 6;
  return TSM_OK;
}

int sides_records(tsm_ctx* c, HostSide* const* sides, int ns, cudaStream_t st, float* scan_ms, bool host_base, uint32_t flags = 0) {
  if (ns < 1 || ns > 2) return TSM_E_ARG;
  ScanParams ps[2];
  size_t caps[2];
  for (int i = 0; i < ns; ++i) {
    HostSide& h = *sides[i];
    const int32_t n = h.n;
    ScanParams& p = ps[i];
    p = side_params(h);
    p.n_groups = 1;
    p.unit_file = h.unit_file.as<uint32_t>(); p.unit_begin = h.unit_begin.as<uint32_t>(); p.unit_cap = h.unit_cap;
    p.ctrl = reinterpret_cast<Ctrl*>(h.zero.as<uint8_t>()); p.slab = reinterpret_cast<SlabCtl*>(h.zero.as<uint8_t>() + 256);
    p.f_end = n;
    p.stats = h.stats.as<tsm_file_stat>();
    p.flags = TSM_SCAN_LINE_HASHES | flags;
    p.unit_lines = h.unit_lines.as<uint32_t>(); p.unit_out = h.unit_out.as<uint32_t>();
    // units in (file, chunk) order
    k_file_units<<<(n + 255) / 256, 256, 0, st>>>(p.len, (uint32_t)n, h.cnt.as<uint32_t>());
    xscan(h.cnt.as<uint32_t>(), (uint32_t)n, h.bsum.as<unsigned long long>(), h.unit_first.as<unsigned long long>(), st);
    caps[i] = h.ab / 8 + 2 * (size_t)h.unit_cap + 64;
    const int rc = side_scan_pass(c, h, p, caps[i], i, st);
    if (rc != TSM_OK) return rc;
  }
  CU(cudaStreamSynchronize(st));
  for (int i = 0; i < ns; ++i) {
    HostSide& h = *sides[i];
    h.hc = c->h_rb->ctrl[i].v; h.total = c->h_rb->total[i];
    if (scan_ms) *scan_ms += span_ms(c, EV_SCAN[i]);
    if (h.hc.overflow && !h.hc.lh_overflow) return TSM_E_CAPACITY;   // (header events overflow only with the lines that bound them)
    if (h.hc.lh_overflow) {                                // more lines than the staging arrays hold: once more, exact size
      const int rc = side_scan_pass(c, h, ps[i], (size_t)h.hc.n_lh + 64, i, st);
      if (rc != TSM_OK) return rc;
      CU(cudaStreamSynchronize(st));
      h.hc = c->h_rb->ctrl[i].v; h.total = c->h_rb->total[i];
      if (scan_ms) *scan_ms += span_ms(c, EV_SCAN[i]);
      if (h.hc.overflow || h.hc.lh_overflow) return TSM_E_CAPACITY;
    }
  }
  for (int i = 0; i < ns; ++i) {
    HostSide& h = *sides[i];
    const int32_t n = h.n;
    const ScanParams& p = ps[i];
    const unsigned long long total = h.total;
    if (!h.line_end.alloc(sizeof(uint32_t) * (size_t)total) || !h.line_hash.alloc(sizeof(unsigned long long) * (size_t)total) ||
        !h.line_flag.alloc((size_t)total))
      return TSM_E_CUDA;
    if (h.n_units)
      k_gather_lines<<<(h.n_units * 32 + 255) / 256, 256, 0, st>>>(p.unit_lines, p.unit_out, h.unit_line_base.as<unsigned long long>(), h.n_units,
                                                                     p.lh_hash, p.lh_end, p.lh_flag, h.line_hash.as<unsigned long long>(),
                                                                     h.line_end.as<uint32_t>(), h.line_flag.as<uint8_t>());
    k_line_base<<<(n + 1 + 255) / 256, 256, 0, st>>>(h.unit_first.as<unsigned long long>(), h.unit_line_base.as<unsigned long long>(),
                                                       (uint32_t)n, h.line_base.as<unsigned long long>());
    CU(cudaGetLastError());
    h.launches += 5;
    h.base.clear();
    if (host_base) {
      h.base.assign((size_t)n + 1, 0);
      CU(cudaMemcpyAsync(h.base.data(), h.line_base.p, sizeof(unsigned long long) * ((size_t)n + 1), cudaMemcpyDeviceToHost, st));
    }
    h.d.arena = h.arena.as<uint8_t>(); h.d.off = h.off.as<int32_t>(); h.d.len = h.len.as<int32_t>();
    h.d.n_lines = nullptr;
    h.d.line_base = h.line_base.as<unsigned long long>();
    h.d.line_end = h.line_end.as<uint32_t>();
    h.d.line_hash = h.line_hash.as<unsigned long long>();
    h.d.ext = h.ext.as<uint8_t>();
    h.d.line_flag = h.line_flag.as<uint8_t>();
  }
  if (host_base) {
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < ns; ++i) sides[i]->drop_staging();
  }                                                        // (else the caller drops them behind its next synchronisation:
  return TSM_OK;                                           //  the gather queued above still reads them)
}

int side_records(tsm_ctx* c, HostSide& h, cudaStream_t st, float* scan_ms, uint32_t flags = 0) {
  HostSide* one[1] = {&h};
  return sides_records(c, one, 1, st, scan_ms, true, flags);
}
}  // namespace

struct HostSidePair {
  HostSide A, B; int32_t n = 0;
  int32_t groups_a = 1, groups_b = 1; bool grp_ok = true;  // n_groups of both sides, every grp < n_groups (for the assertion tables)
};

static void free_res_pair(tsm_ctx* c) {
  if (!c->res_pair) return;
  PoolScope pool_scope(&c->pool);                          // the buffers go back to the ctx's pool
  delete c->res_pair;
  c->res_pair = nullptr;
}

// The corpora of the diff and line-record calls (n_files > 0 each): arena, off and len given, and the per-file layout rules
// of the scan.  Their grp is not part of it: only the assertion tables use it.
static int check_sides(std::initializer_list<const tsm_corpus*> sides, bool ext_rule) {
  for (const tsm_corpus* k : sides) {
    if (!k->arena || !k->off || !k->len) return TSM_E_ARG;
    const int rc = check_files(k, 0, k->n_files, ext_rule, false);
    if (rc != TSM_OK) return rc;
  }
  return TSM_OK;
}

// Both sides of the revision pairs to the device (with_grp: their group tags too, for the assertion tables).  Each side
// is sized from its own corpus: the sides of tsm_similarity may differ in files (P.n is the count of `olds`).
static int pair_upload(const tsm_corpus* olds, const tsm_corpus* news, bool with_grp, HostSidePair& P, cudaStream_t st) {
  P.n = olds->n_files;
  P.groups_a = olds->n_groups; P.groups_b = news->n_groups;
  if (with_grp) P.grp_ok = check_groups(olds, 0, P.n) == TSM_OK && check_groups(news, 0, P.n) == TSM_OK;
  int rc = side_upload(olds, P.A, st);
  if (rc == TSM_OK) rc = side_upload(news, P.B, st);
  if (rc == TSM_OK && with_grp) rc = side_upload_grp(olds, P.A, st);
  if (rc == TSM_OK && with_grp) rc = side_upload_grp(news, P.B, st);
  return rc;
}

// The line records of both uploaded sides of P (*scan_ms = k_scan over both; host_base: line_base of each side on the host too;
// flags: TSM_SCAN_HEADER_EVENTS for their header events too).
static int pair_records(tsm_ctx* c, HostSidePair& P, float* scan_ms, bool host_base, cudaStream_t st, uint32_t flags = 0) {
  *scan_ms = 0;
  P.A.launches = P.B.launches = 0;
  HostSide* both[2] = {&P.A, &P.B};
  return sides_records(c, both, 2, st, scan_ms, host_base, flags);
}

// What a revision-pair call asks of pair_call, beside the TSM_SCAN_* flags of the line records (TSM_SCAN_HEADER_EVENTS).
enum : uint32_t {
  PAIR_ANY_EXT = 1u << 16,                                 // no ext <= TSM_EXT_H rule in check_sides
  PAIR_GRP = 1u << 17,                                     // the group tags of both sides too (pair_upload's with_grp)
  PAIR_HOST_BASE = 1u << 18,                               // line_base of each side on the host too (HostSide::base)
};
static_assert((TSM_SCAN_ASSERT_EVENTS | TSM_SCAN_HEADER_EVENTS | TSM_SCAN_LINE_HASHES | TSM_SCAN_REV_B) < PAIR_ANY_EXT, "PAIR_*");

// The front of every call over uploaded revision pairs (n_files > 0 on both sides; the caller checks its own arguments and
// returns early for none): check_sides, the CallScope, both sides to the device, their line records (*scan_ms = k_scan over
// both), then tail(P, st), the call's own use of them, inside the call's SyncGuard.  The tail keeps the rule of CallScope:
// it synchronises st before it returns on success, and on an error it returns without allocating again.
template <typename Tail>
static int pair_call(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, uint32_t opts, float* scan_ms, void* stream,
                     Tail tail) {
  int rc = check_sides({olds, news}, !(opts & PAIR_ANY_EXT));
  if (rc != TSM_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  HostSidePair P;
  SyncGuard guard(st);
  rc = pair_upload(olds, news, opts & PAIR_GRP, P, st);
  if (rc == TSM_OK) rc = pair_records(c, P, scan_ms, opts & PAIR_HOST_BASE, st, opts & TSM_SCAN_HEADER_EVENTS);
  return rc != TSM_OK ? rc : tail(P, st);
}

// The diff proper over two sides whose line records exist.  k_diff_small finishes the common pairs (distance at most
// 127 lines, middle of at most 4 096 lines) start to finish - search in registers, rows of V and backtrack in shared
// memory - in the sizes of DS_SIZES, each fed on the device by the list the size before it leaves.  What all of them
// leave over (the `todo` list, normally empty) goes through k_myers (edit distance, V in global scratch) and, for `detail`,
// k_myers_trace (rows of V in global memory sized from those distances, then the canonical script: hunks, changed
// assertion lines).  A pair whose distance D needs more than TSM_DIFF_TRACE_MAX_INTS trace entries ((D+1)(D+2)/2) is
// not traced: it is reported as ONE hunk (add / del / mod by its counts) with added_assert = removed_assert = -1
// (tosemscan.h).  last_ms[MS_DIFF][1] = k_diff_small, [2] = the two kernels of the left-over pairs.
// MODE (DiffMode) picks the variant of k_diff_small and k_myers_trace: DIFF_EMIT also lists the changed assertion lines
// into the caller's sink, DIFF_MARKS marks the deleted and inserted lines into A.line_mark / B.line_mark (one zeroed byte
// per line of each side).  Both find those lines on the paths that compute the detail (the assertion flags come with it),
// so they compute it also when the caller passes none.
template <int MODE>
static int diff_core(tsm_ctx* c, HostSide& A, HostSide& B, int32_t n, int64_t* added, int64_t* removed,
                     tsm_diff_detail* detail, cudaStream_t st, AssertSink sink = {}) {
  static_assert(sizeof(long long) == sizeof(int64_t), "int64");
  static_assert(2 * DS_N * sizeof(uint32_t) <= 64, "d_ntodo: two counters per size");
  std::vector<tsm_diff_detail> own;
  if (MODE != DIFF_PLAIN && !detail) { own.resize((size_t)n); detail = own.data(); }
  if constexpr (MODE == DIFF_MARKS) {
    if (!A.line_mark.alloc((size_t)A.total) || !B.line_mark.alloc((size_t)B.total)) return TSM_E_CUDA;
    CU(cudaMemsetAsync(A.line_mark.p, 0, (size_t)A.total, st));
    CU(cudaMemsetAsync(B.line_mark.p, 0, (size_t)B.total, st));
    sink.mark[0] = A.line_mark.as<uint8_t>(); sink.mark[1] = B.line_mark.as<uint8_t>();
  }
  DevBuf d_add, d_rem, d_detail, d_todo[DS_N], d_ntodo;
  bool ok = d_add.alloc(sizeof(long long) * (size_t)n) && d_rem.alloc(sizeof(long long) * (size_t)n);
  for (DevBuf& t : d_todo) ok = ok && t.alloc(sizeof(int32_t) * (size_t)n);
  if (!ok || !d_ntodo.alloc(64) || (detail && !d_detail.alloc(sizeof(tsm_diff_detail) * (size_t)n))) return TSM_E_CUDA;
  CU(cudaMemsetAsync(d_ntodo.p, 0, 64, st));
  CU(cudaMemsetAsync(d_add.p, 0, sizeof(long long) * (size_t)n, st));     // (the first copy back covers every pair, also the ones
  CU(cudaMemsetAsync(d_rem.p, 0, sizeof(long long) * (size_t)n, st));     //  the sizes leave to k_myers / k_myers_trace)
  if (detail) CU(cudaMemsetAsync(d_detail.p, 0, sizeof(tsm_diff_detail) * (size_t)n, st));
  uint32_t* cnt = d_ntodo.as<uint32_t>();                  // [I] pairs size I left over, [DS_N + I] size I's work counter
  const uint8_t* fa = detail ? A.d.line_flag : nullptr;
  const uint8_t* fb = detail ? B.d.line_flag : nullptr;
  tsm_diff_detail* d_det = detail ? d_detail.as<tsm_diff_detail>() : nullptr;
  int32_t* const d_left = d_todo[DS_N - 1].as<int32_t>();  // what the last size leaves over
  CU(cudaEventRecord(c->diff_ev[EV_SMALL.from], st));
  for_ds_sizes([&](auto i) {                               // size I: the pairs size I - 1 left over (size 0: all n)
    constexpr int I = decltype(i)::value;
    constexpr DiffSmallSize s = DS_SIZES[I];
    k_diff_small<s.hcap, s.dcap, s.warps, MODE><<<std::min((n + s.warps - 1) / s.warps, c->sms * s.per_sm), s.warps * 32, s.smem(), st>>>(
        A.d.line_hash, A.d.line_base, fa, B.d.line_hash, B.d.line_base, fb, I ? d_todo[I - 1].as<int32_t>() : nullptr,
        I ? cnt + I - 1 : nullptr, n, cnt + DS_N + I, d_add.as<long long>(), d_rem.as<long long>(), d_det, d_todo[I].as<int32_t>(),
        cnt + I, sink);
  });
  CU(cudaEventRecord(c->diff_ev[EV_SMALL.to], st));
  CU(cudaGetLastError());
  uint32_t* pin_nt = &c->h_rb->n_todo;
  CU(cudaMemcpyAsync(pin_nt, cnt + DS_N - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(added, d_add.p, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(removed, d_rem.p, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
  if (detail) CU(cudaMemcpyAsync(detail, d_detail.p, sizeof(tsm_diff_detail) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  A.drop_staging(); B.drop_staging();
  const uint32_t nt = *pin_nt;
  float* const ms = c->last_ms[MS_DIFF];
  ms[1] = span_ms(c, EV_SMALL);
  c->launches = A.launches + B.launches + DS_N;
  ms[2] = 0;
  if (nt == 0) return TSM_OK;
  // ---- the left-over pairs: long middles, far-apart revisions
  std::vector<int32_t> todo(nt);
  CU(cudaMemcpyAsync(todo.data(), d_left, sizeof(int32_t) * (size_t)nt, cudaMemcpyDeviceToHost, st));
  for (HostSide* h : {&A, &B})
    if (h->base.empty()) {
      h->base.assign((size_t)n + 1, 0);
      CU(cudaMemcpyAsync(h->base.data(), h->line_base.p, sizeof(unsigned long long) * ((size_t)n + 1), cudaMemcpyDeviceToHost, st));
    }
  CU(cudaStreamSynchronize(st));
  std::vector<unsigned long long> vbase((size_t)nt + 1, 0);
  for (uint32_t s = 0; s < nt; ++s) {
    const size_t i = (size_t)todo[s];
    vbase[(size_t)s + 1] = vbase[s] + 2 * ((A.base[i + 1] - A.base[i]) + (B.base[i + 1] - B.base[i])) + 3;
  }
  DevBuf d_vbase, d_v;
  if (!d_vbase.alloc(sizeof(unsigned long long) * ((size_t)nt + 1)) || !d_v.alloc(sizeof(int32_t) * (size_t)vbase[nt])) return TSM_E_CUDA;
  CU(cudaMemcpyAsync(d_vbase.p, vbase.data(), sizeof(unsigned long long) * ((size_t)nt + 1), cudaMemcpyHostToDevice, st));
  CU(cudaEventRecord(c->diff_ev[EV_LEFT.from], st));
  k_myers<<<(nt * 32 + 127) / 128, 128, 0, st>>>(A.d.line_hash, A.d.line_base, B.d.line_hash, B.d.line_base, (int32_t)nt,
                                                d_v.as<int32_t>(), d_vbase.as<unsigned long long>(),
                                                d_add.as<long long>(), d_rem.as<long long>(), d_left);
  CU(cudaEventRecord(c->diff_ev[EV_LEFT.to], st));
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(added, d_add.p, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(removed, d_rem.p, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  ms[2] += span_ms(c, EV_LEFT);
  c->launches++;
  if (!detail) return TSM_OK;
  // ---- their hunks: second search with the rows of V kept; rows sized from the distances just computed,
  //      pairs processed in batches of at most 2^28 trace ints (1 GiB)
  d_v.reset();                                             // the first search's scratch is no longer needed
  DevBuf d_tbase;
  if (!d_tbase.alloc(sizeof(unsigned long long) * ((size_t)nt + 1))) return TSM_E_CUDA;
  std::vector<unsigned long long> tbase((size_t)nt + 1, 0);
  std::vector<int32_t> untraced;
  const unsigned long long kBatch = TSM_DIFF_TRACE_MAX_INTS;
  uint32_t p0 = 0;
  while (p0 < nt) {
    uint32_t p1 = p0;
    unsigned long long tot = 0;
    while (p1 < nt) {
      const int32_t i = todo[p1];
      const unsigned long long D = (unsigned long long)(added[i] + removed[i]);
      unsigned long long need = (D + 1) * (D + 2) / 2;
      if (need > kBatch) { untraced.push_back(i); need = 1; }       // k_myers_trace skips it (row table of one int)
      if (p1 > p0 && tot + need > kBatch) break;
      tbase[p1] = tot;
      tot += need;
      ++p1;
    }
    DevBuf d_trace;
    if (!d_trace.alloc(sizeof(int32_t) * (size_t)tot)) return TSM_E_CUDA;
    CU(cudaMemcpyAsync(d_tbase.as<unsigned long long>() + p0, tbase.data() + p0, sizeof(unsigned long long) * (size_t)(p1 - p0),
                       cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(c->diff_ev[EV_LEFT.from], st));
    const unsigned grid = ((p1 - p0) * 32 + 127) / 128;
    k_myers_trace<MODE><<<grid, 128, 0, st>>>(
        A.d.line_hash, A.d.line_base, A.d.line_flag, B.d.line_hash, B.d.line_base, B.d.line_flag, (int32_t)p0, (int32_t)(p1 - p0),
        d_trace.as<int32_t>(), d_tbase.as<unsigned long long>(), d_add.as<long long>(), d_rem.as<long long>(),
        (long long)TSM_DIFF_TRACE_MAX_D, d_detail.as<tsm_diff_detail>(), d_left, sink);
    CU(cudaEventRecord(c->diff_ev[EV_LEFT.to], st));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    ms[2] += span_ms(c, EV_LEFT);
    c->launches++;
    p0 = p1;
  }
  CU(cudaMemcpyAsync(detail, d_detail.p, sizeof(tsm_diff_detail) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int32_t i : untraced) {                              // too far apart to trace: one hunk, assertion counts unknown
    tsm_diff_detail d{0, 0, 0, -1, -1};
    if (added[i] && removed[i]) d.hunks_mod = 1; else if (added[i]) d.hunks_add = 1; else d.hunks_del = 1;
    detail[i] = d;
  }
  return TSM_OK;
}

// Changed assertion lines (docs/SPEC.md section 8): diff_core with the EMIT kernels, then per side ONE k_classify launch
// over the list they filled, with a ScanParams over that side's arena, tags and groups and a Ctrl of its own whose n_cand
// is the list's counter - a changed line is classified by the code, and so with the result, of a scan.  Each list holds
// one entry per line of its side, a bound known before the launch that no side can exceed.
static int classify_changed(tsm_ctx* c, HostSide* const side[2], unsigned long long* const list[2], Ctrl* const ctrl[2],
                            const uint32_t nc[2], int32_t n, int32_t n_groups, tsm_diff_asserts* out, cudaStream_t st);
static int diff_asserts(tsm_ctx* c, HostSide& A, HostSide& B, int32_t n, int32_t n_groups, int64_t* added, int64_t* removed,
                        tsm_diff_detail* detail, tsm_diff_asserts* out, cudaStream_t st) {
  HostSide* side[2] = {&A, &B};                            // side 0: deleted lines of `old`, side 1: inserted lines of `new`
  DevBuf d_list[2], d_ctrl;
  AssertSink sink{};
  if (!d_ctrl.alloc(2 * 64)) return TSM_E_CUDA;
  Ctrl* ctrl[2] = {d_ctrl.as<Ctrl>(), reinterpret_cast<Ctrl*>(d_ctrl.as<uint8_t>() + 64)};
  for (int s = 0; s < 2; ++s) {
    const unsigned long long lines = side[s]->total;
    if (lines > 0xFFFFFFF0ull) return TSM_E_CAPACITY;
    if (!d_list[s].alloc(sizeof(unsigned long long) * (size_t)(lines ? lines : 1))) return TSM_E_CUDA;
    sink.list[s] = d_list[s].as<unsigned long long>(); sink.n[s] = &ctrl[s]->n_cand; sink.cap[s] = (uint32_t)lines;
    sink.line_end[s] = side[s]->d.line_end;
  }
  CU(cudaMemsetAsync(d_ctrl.p, 0, 2 * 64, st));            // n_cand = cls_done = 0
  int rc = diff_core<DIFF_EMIT>(c, A, B, n, added, removed, detail, st, sink);
  if (rc != TSM_OK) return rc;
  Ctrl hc[2];
  for (int s = 0; s < 2; ++s) CU(cudaMemcpyAsync(&hc[s], ctrl[s], sizeof(Ctrl), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const uint32_t nc[2] = {hc[0].n_cand, hc[1].n_cand};
  if (nc[0] > sink.cap[0] || nc[1] > sink.cap[1]) return TSM_E_CAPACITY;   // (more changed lines than lines: never)
  return classify_changed(c, side, sink.list, ctrl, nc, n, n_groups, out, st);
}

// The second half of diff_asserts: per side ONE k_classify launch over the nc[s] candidates list[s] (whose Ctrl ctrl[s] has
// n_cand = nc[s], cls_done = 0), then the tables and the events (sorted into canonical order) to `out`.
static int classify_changed(tsm_ctx* c, HostSide* const side[2], unsigned long long* const list[2], Ctrl* const ctrl[2],
                            const uint32_t nc[2], int32_t n, int32_t n_groups, tsm_diff_asserts* out, cudaStream_t st) {
  DevBuf d_counts[2], d_aev[2];
  tsm_assert_event* const h_ev[2] = {out->rev, out->aev};
  const int64_t h_cap[2] = {out->rev_cap, out->aev_cap};
  int64_t* const h_counts[2] = {out->removed_counts, out->added_counts};
  const size_t table = (size_t)(n_groups + 1) * TSM_K;     // [n_groups + 1][K]: k_classify also fills the global row
  const ClassifyShape cls = classify_shape(c, n_groups);
  for (int s = 0; s < 2; ++s) {
    if (!d_counts[s].alloc(sizeof(unsigned long long) * table) ||
        (h_ev[s] && !d_aev[s].alloc(sizeof(tsm_assert_event) * (size_t)std::max(nc[s], 1u))))
      return TSM_E_CUDA;
    CU(cudaMemsetAsync(d_counts[s].p, 0, sizeof(unsigned long long) * table, st));
    if (nc[s] == 0) continue;
    const HostSide& h = *side[s];
    ScanParams p = side_params(h);
    p.grp = h.grp.as<uint16_t>(); p.n_groups = n_groups;
    p.ctrl = ctrl[s];
    p.cand = list[s]; p.cand_cap = nc[s];
    p.aev = d_aev[s].as<tsm_assert_event>(); p.aev_cap = h_ev[s] ? nc[s] : 0;
    p.counts = d_counts[s].as<unsigned long long>();
    p.flags = h_ev[s] ? TSM_SCAN_ASSERT_EVENTS : 0u;
    launch_k_classify(p, false, std::min<uint32_t>(cls.wave, (nc[s] + 255) / 256), cls.smem, st);
    CU(cudaGetLastError());
    c->launches++;
  }
  for (int s = 0; s < 2; ++s)
    if (h_counts[s]) CU(cudaMemcpyAsync(h_counts[s], d_counts[s].p, sizeof(int64_t) * (size_t)n_groups * TSM_K, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  out->n_rev = nc[0]; out->n_aev = nc[1];
  if ((h_ev[0] && nc[0] > h_cap[0]) || (h_ev[1] && nc[1] > h_cap[1])) return TSM_E_CAPACITY;   // both counts set: size and call again
  for (int s = 0; s < 2; ++s)
    if (h_ev[s] && nc[s]) CU(cudaMemcpyAsync(h_ev[s], d_aev[s].p, sizeof(tsm_assert_event) * nc[s], cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int s = 0; s < 2; ++s)
    if (h_ev[s]) sort_events_by_file(h_ev[s], nc[s], n);
  return TSM_OK;
}

// The plain and the assertion diff behind the line records of P: diff_core, or diff_asserts when `out` is given.
static int pair_run(tsm_ctx* c, HostSidePair& P, int64_t* added, int64_t* removed, tsm_diff_detail* detail,
                    tsm_diff_asserts* out, cudaStream_t st) {
  if (out) return diff_asserts(c, P.A, P.B, P.n, P.groups_a, added, removed, detail, out, st);
  return diff_core<DIFF_PLAIN>(c, P.A, P.B, P.n, added, removed, detail, st);
}

extern "C" int tsm_diff_pairs_detail(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news,
                                     int64_t* added, int64_t* removed, tsm_diff_detail* detail, void* stream) {
  if (!c || !olds || !news || !added || !removed || olds->n_files != news->n_files) return TSM_E_ARG;
  if (olds->n_files == 0) return TSM_OK;
  return pair_call(c, olds, news, detail ? 0u : PAIR_ANY_EXT, &c->last_ms[MS_DIFF][0], stream, [&](HostSidePair& P, cudaStream_t st) {
    return pair_run(c, P, added, removed, detail, nullptr, st);
  });
}

extern "C" int tsm_diff_pairs(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news,
                              int64_t* added, int64_t* removed, void* stream) {
  return tsm_diff_pairs_detail(c, olds, news, added, removed, nullptr, stream);
}

extern "C" int tsm_diff_pairs_asserts(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                      tsm_diff_detail* detail, tsm_diff_asserts* out, void* stream) {
  if (!c || !olds || !news || !added || !removed || !out || olds->n_files != news->n_files || olds->n_groups != news->n_groups)
    return TSM_E_ARG;
  const int32_t n = olds->n_files;
  int rc = check_groups(olds, 0, n);
  if (rc == TSM_OK) rc = check_groups(news, 0, n);
  if (rc != TSM_OK) return rc;
  out->n_aev = out->n_rev = 0;
  if (n == 0) {
    for (int64_t* t : {out->added_counts, out->removed_counts})
      if (t) memset(t, 0, sizeof(int64_t) * (size_t)olds->n_groups * TSM_K);
    return TSM_OK;
  }
  return pair_call(c, olds, news, PAIR_GRP, &c->last_ms[MS_DIFF][0], stream, [&](HostSidePair& P, cudaStream_t st) {
    return pair_run(c, P, added, removed, detail, out, st);
  });
}

// Resident variant (what bench.py's `value` times for config C5): the two sides go to HBM once ...
extern "C" int tsm_diff_upload(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, void* stream) {
  if (!c || !olds || !news || olds->n_files != news->n_files || olds->n_files <= 0) return TSM_E_ARG;
  int rc = check_sides({olds, news}, true);
  if (rc != TSM_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  free_res_pair(c);
  SyncGuard guard(st);
  c->res_pair = new (std::nothrow) HostSidePair;
  if (!c->res_pair) return TSM_E_NOMEM;
  rc = pair_upload(olds, news, true, *c->res_pair, st);    // (a bad grp fails tsm_diff_resident_asserts, not the upload)
  if (rc == TSM_OK) rc = cudaStreamSynchronize(st) == cudaSuccess ? TSM_OK : TSM_E_CUDA;
  if (rc != TSM_OK) { delete c->res_pair; c->res_pair = nullptr; }
  return rc;
}

// ... and every call runs the kernels over them: k_scan over both sides (line records), k_myers, k_myers_trace.
static int resident_run(tsm_ctx* c, int64_t* added, int64_t* removed, tsm_diff_detail* detail, tsm_diff_asserts* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  SyncGuard guard(st);
  const int rc = pair_records(c, *c->res_pair, &c->last_ms[MS_DIFF][0], false, st);
  return rc != TSM_OK ? rc : pair_run(c, *c->res_pair, added, removed, detail, out, st);
}

extern "C" int tsm_diff_resident(tsm_ctx* c, int64_t* added, int64_t* removed, tsm_diff_detail* detail, void* stream) {
  if (!c || !added || !removed) return TSM_E_ARG;
  if (!c->res_pair) return TSM_E_STATE;
  return resident_run(c, added, removed, detail, nullptr, stream);
}

extern "C" int tsm_diff_resident_asserts(tsm_ctx* c, int64_t* added, int64_t* removed, tsm_diff_detail* detail,
                                         tsm_diff_asserts* out, void* stream) {
  if (!c || !added || !removed || !out) return TSM_E_ARG;
  if (!c->res_pair) return TSM_E_STATE;
  if (c->res_pair->groups_a != c->res_pair->groups_b) return TSM_E_ARG;
  if (!c->res_pair->grp_ok) return TSM_E_LAYOUT;
  out->n_aev = out->n_rev = 0;
  return resident_run(c, added, removed, detail, out, stream);
}

extern "C" int tsm_diff_last_ms(tsm_ctx* c, float* ms3) { return copy_ms(c, MS_DIFF, ms3, 3); }

// ------------------------------------------------------------------------------------- SPEC section 14 line provenance
extern "C" int tsm_diff_pairs_marks(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                    tsm_diff_detail* detail, tsm_line_marks* mk, void* stream) {
  if (!c || !olds || !news || !added || !removed || !mk || !mk->line_base_old || !mk->line_base_new || olds->n_files != news->n_files)
    return TSM_E_ARG;
  const int32_t n = olds->n_files;
  mk->n_old = mk->n_new = 0;
  if (n == 0) { mk->line_base_old[0] = mk->line_base_new[0] = 0; return TSM_OK; }
  return pair_call(c, olds, news, PAIR_HOST_BASE, &c->last_ms[MS_DIFF][0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    memcpy(mk->line_base_old, P.A.base.data(), sizeof(int64_t) * ((size_t)n + 1));
    memcpy(mk->line_base_new, P.B.base.data(), sizeof(int64_t) * ((size_t)n + 1));
    mk->n_old = (int64_t)P.A.total; mk->n_new = (int64_t)P.B.total;
    if (mk->del_cap < mk->n_old || mk->ins_cap < mk->n_new) return TSM_E_CAPACITY;
    if ((mk->n_old && !mk->del) || (mk->n_new && !mk->ins)) return TSM_E_ARG;
    const int rc = diff_core<DIFF_MARKS>(c, P.A, P.B, n, added, removed, detail, st);
    if (rc != TSM_OK) return rc;
    if (mk->n_old) CU(cudaMemcpyAsync(mk->del, P.A.line_mark.p, (size_t)mk->n_old, cudaMemcpyDeviceToHost, st));
    if (mk->n_new) CU(cudaMemcpyAsync(mk->ins, P.B.line_mark.p, (size_t)mk->n_new, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return TSM_OK;
  });
}

// ------------------------------------------------------------------------------------- SPEC section 16 test-case churn
// The case spans of one side whose line records and header events exist: k_case_heads (head[l] = 1 on header lines), xscan
// of the heads (case_of: the case of every header line, cases numbered in line order) and k_case_lines (first[case] = its
// header line).  bsum holds total / XS_TILE + 4 u64.
struct CaseSpans { DevBuf head, case_of, first; uint32_t n_cases = 0; };

static int case_spans(const HostSide& h, CaseSpans& sp, DevBuf& bsum, int& launches, cudaStream_t st) {
  const uint32_t T = (uint32_t)h.total, ne = h.hc.n_hev;
  const size_t L = (size_t)h.total;
  sp.n_cases = ne;
  if (!sp.head.alloc(4 * L) || !sp.case_of.alloc(8 * (L + 1)) || !sp.first.alloc(4 * ((size_t)ne + 1))) return TSM_E_CUDA;
  CU(cudaMemsetAsync(sp.head.p, 0, 4 * L, st));
  if (ne)
    k_case_heads<<<(ne + 255) / 256, 256, 0, st>>>(h.hev.as<tsm_header_event>(), ne, h.d.line_base, h.d.line_end, sp.head.as<uint32_t>());
  xscan(sp.head.as<uint32_t>(), T, bsum.as<unsigned long long>(), sp.case_of.as<unsigned long long>(), st);
  if (T)
    k_case_lines<<<(T + 255) / 256, 256, 0, st>>>(sp.head.as<uint32_t>(), nullptr, sp.case_of.as<unsigned long long>(), nullptr, T,
                                                  sp.first.as<uint32_t>(), nullptr);
  CU(cudaGetLastError());
  launches += (ne ? 1 : 0) + (T ? 4 : 0);
  return TSM_OK;
}

// The kept rank of every line of a side behind the marks diff: k_case_kept (kept[l] = 1 on the lines the diff keeps) and its
// xscan (rank[l] = the kept lines before l; rank[total] = all of them).  kept holds total u32, rank total + 1 u64.
static void kept_ranks(const HostSide& h, DevBuf& kept, DevBuf& rank, DevBuf& bsum, cudaStream_t st) {
  const uint32_t total = (uint32_t)h.total;
  if (total) k_case_kept<<<(total + 255) / 256, 256, 0, st>>>(h.line_mark.as<uint8_t>(), total, kept.as<uint32_t>());
  xscan(kept.as<uint32_t>(), total, bsum.as<unsigned long long>(), rank.as<unsigned long long>(), st);
}

// The cases of both sides of the revision pairs: their spans before the marks diff (pair_case_spans), their records behind it
// (case_records): per side kept_ranks, k_case_lines for by_rank (the kept line of every rank: the old side's always, the new
// side's when asked for) and k_case_reduce (the new side's step-1 match reads the old side's by_rank, head and case_of).
struct PairCases { CaseSpans sp[2]; DevBuf kept[2], rank[2], by_rank[2], cases[2], bsum; };

static int pair_case_spans(const HostSidePair& P, PairCases& pc, int& launches, cudaStream_t st) {
  if (!pc.bsum.alloc(sizeof(unsigned long long) * ((size_t)std::max(P.A.total, P.B.total) / XS_TILE + 4))) return TSM_E_CUDA;
  const int rc = case_spans(P.A, pc.sp[0], pc.bsum, launches, st);
  return rc == TSM_OK ? case_spans(P.B, pc.sp[1], pc.bsum, launches, st) : rc;
}

static int case_records(tsm_ctx* c, const HostSidePair& P, PairCases& pc, bool new_by_rank, int& launches, cudaStream_t st) {
  const HostSide* side[2] = {&P.A, &P.B};
  for (int s = 0; s < 2; ++s) {
    const HostSide& h = *side[s];
    const uint32_t total = (uint32_t)h.total;
    const bool by_rank = s == 0 || new_by_rank;
    if (!pc.kept[s].alloc(sizeof(uint32_t) * (size_t)total) || !pc.rank[s].alloc(sizeof(unsigned long long) * ((size_t)total + 1)) ||
        !pc.cases[s].alloc(sizeof(tsm_case) * (size_t)pc.sp[s].n_cases) || (by_rank && !pc.by_rank[s].alloc(sizeof(uint32_t) * (size_t)total)))
      return TSM_E_CUDA;
    kept_ranks(h, pc.kept[s], pc.rank[s], pc.bsum, st);
    if (total && by_rank)
      k_case_lines<<<(total + 255) / 256, 256, 0, st>>>(pc.sp[s].head.as<uint32_t>(), pc.kept[s].as<uint32_t>(),
                                                        pc.sp[s].case_of.as<unsigned long long>(), pc.rank[s].as<unsigned long long>(),
                                                        total, pc.sp[s].first.as<uint32_t>(), pc.by_rank[s].as<uint32_t>());
    launches += total ? 4 + (by_rank ? 1 : 0) : 0;
  }
  for (int s = 0; s < 2; ++s) {
    const HostSide& h = *side[s];
    const uint32_t ne = pc.sp[s].n_cases;
    if (!ne) continue;
    const CaseSide cs{h.d.line_base, (uint32_t)P.n, h.d.line_flag, h.line_mark.as<uint8_t>(), pc.sp[s].first.as<uint32_t>(), ne};
    const bool nw = s == 1;
    k_case_reduce<<<std::min((ne + 7) / 8, (uint32_t)c->sms * 8), 256, 0, st>>>(
        cs, pc.rank[s].as<unsigned long long>(), nw ? pc.by_rank[0].as<uint32_t>() : nullptr, nw ? pc.sp[0].head.as<uint32_t>() : nullptr,
        nw ? pc.sp[0].case_of.as<unsigned long long>() : nullptr, pc.cases[s].as<tsm_case>());
    ++launches;
  }
  CU(cudaGetLastError());
  return TSM_OK;
}

// The line records of both sides with their header events (the case counts, so the capacity check comes before the diff),
// the case spans, the marks diff and the case records (csrc/tsm_case_kernels.cuh).
extern "C" int tsm_diff_pairs_cases(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                    tsm_diff_detail* detail, tsm_diff_cases* out, void* stream) {
  if (!c || !olds || !news || !added || !removed || !out || olds->n_files != news->n_files) return TSM_E_ARG;
  const int32_t n = olds->n_files;
  out->n_old = out->n_new = 0;
  if (n == 0) return TSM_OK;
  return pair_call(c, olds, news, TSM_SCAN_HEADER_EVENTS, &c->last_ms[MS_DIFF][0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    out->n_old = P.A.hc.n_hev; out->n_new = P.B.hc.n_hev;
    if (out->old_cap < out->n_old || out->new_cap < out->n_new) return TSM_E_CAPACITY;
    if ((out->n_old && !out->old_cases) || (out->n_new && !out->new_cases)) return TSM_E_ARG;
    PairCases pc;
    int launches = 0;
    int rc = pair_case_spans(P, pc, launches, st);
    if (rc == TSM_OK) rc = diff_core<DIFF_MARKS>(c, P.A, P.B, n, added, removed, detail, st);
    if (rc == TSM_OK) rc = case_records(c, P, pc, false, launches, st);
    if (rc != TSM_OK) return rc;
    tsm_case* const h_out[2] = {out->old_cases, out->new_cases};
    for (int s = 0; s < 2; ++s)
      if (pc.sp[s].n_cases) CU(cudaMemcpyAsync(h_out[s], pc.cases[s].p, sizeof(tsm_case) * pc.sp[s].n_cases, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += launches;
    return TSM_OK;
  });
}

// ------------------------------------------------------------------------------------- SPEC section 17 assertion edits
// The marks diff, then per side k_case_kept + xscan (kept ranks), k_edit_flag + xscan (entry index) and k_edit_compact: the
// changed assertion lines of the traced pairs in line order, with their hunk keys and k_classify candidates.  Those lists are
// the ones tsm_diff_pairs_asserts classifies (diff_asserts gets them from the EMIT diff), so classify_changed gives the same
// tables and events, event k of a side being its entry k.  Then k_edit_ranges, the score kernels (patterns of up to 256
// bytes in one launch, longer ones in launches whose global slots stay under kEditScratch words) and the greedy pairing on
// the host, hunk by hunk (the old entries of a hunk are one run of equal keys): its candidates sorted by score, old entry, new
// entry, then taken greedily.
static constexpr unsigned long long kEditScratch = 1ull << 25;   // 256 MiB of Peq and V slots per launch of the long path

// kept: the candidates that pass; pat: the old entries (their keys name the hunks).
static int edit_scores(tsm_ctx* c, const DevBuf* lines, const uint32_t ne[2], const uint8_t* arena_old, const uint8_t* arena_new,
                       std::vector<EditCand>& kept, std::vector<EditLine>& pat, cudaStream_t st) {
  const uint32_t no = ne[0], nn = ne[1];
  DevBuf d_range, d_ids, d_slot, d_kept, d_nk, d_scratch;
  if (!d_range.alloc(sizeof(uint2) * no)) return TSM_E_CUDA;
  k_edit_ranges<<<(no + 255) / 256, 256, 0, st>>>(lines[0].as<EditLine>(), no, lines[1].as<EditLine>(), nn, d_range.as<uint2>());
  CU(cudaGetLastError());
  std::vector<uint2> range(no);
  pat.resize(no);
  CU(cudaMemcpyAsync(range.data(), d_range.p, sizeof(uint2) * no, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(pat.data(), lines[0].p, sizeof(EditLine) * no, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  std::vector<uint32_t> ids;                               // short patterns, then long ones
  std::vector<unsigned long long> slot;                    // per long pattern: its slot in the scratch of its launch
  std::vector<std::pair<uint32_t, uint32_t>> launches;     // long launches: [first, end) of the long ids
  for (uint32_t i = 0; i < no; ++i)
    if (range[i].y > range[i].x && pat[i].len <= 64 * EDIT_SHORT_WORDS) ids.push_back(i);
  const uint32_t n_short = (uint32_t)ids.size();
  unsigned long long top = 0, need = 0;
  for (uint32_t i = 0; i < no; ++i) {
    if (range[i].y == range[i].x || pat[i].len <= 64 * EDIT_SHORT_WORDS) continue;
    const unsigned long long words = 288ull * ((pat[i].len + 63) / 64);
    if (launches.empty() || (top + words > kEditScratch && top)) { launches.push_back({(uint32_t)ids.size() - n_short, 0}); top = 0; }
    ids.push_back(i); slot.push_back(top);
    top += words;
    need = std::max(need, top);
    launches.back().second = (uint32_t)ids.size() - n_short;
  }
  if (ids.empty()) return TSM_OK;
  if (!d_ids.alloc(sizeof(uint32_t) * ids.size()) || !d_nk.alloc(sizeof(uint32_t)) ||
      (!slot.empty() && (!d_slot.alloc(sizeof(unsigned long long) * slot.size()) || !d_scratch.alloc(sizeof(unsigned long long) * need))))
    return TSM_E_CUDA;
  CU(cudaMemcpyAsync(d_ids.p, ids.data(), sizeof(uint32_t) * ids.size(), cudaMemcpyHostToDevice, st));
  if (!slot.empty()) CU(cudaMemcpyAsync(d_slot.p, slot.data(), sizeof(unsigned long long) * slot.size(), cudaMemcpyHostToDevice, st));
  uint32_t cap = std::max<uint32_t>(4096, no + nn), nk = 0;
  for (int attempt = 0; attempt < 2; ++attempt) {          // a second run when more candidates pass than the first list holds
    if (!d_kept.alloc(sizeof(EditCand) * cap)) return TSM_E_CUDA;
    CU(cudaMemsetAsync(d_nk.p, 0, sizeof(uint32_t), st));
    if (n_short)
      k_edit_score<<<std::min<uint32_t>((n_short + EDIT_WARPS - 1) / EDIT_WARPS, (uint32_t)c->sms * 16), EDIT_WARPS * 32, 0, st>>>(
          d_ids.as<uint32_t>(), n_short, lines[0].as<EditLine>(), lines[1].as<EditLine>(), d_range.as<uint2>(), arena_old, arena_new,
          d_kept.as<EditCand>(), cap, d_nk.as<uint32_t>());
    for (const auto& L : launches) {
      const uint32_t cnt = L.second - L.first;
      const unsigned long long words = slot[L.second - 1] + 288ull * ((pat[ids[n_short + L.second - 1]].len + 63) / 64);
      CU(cudaMemsetAsync(d_scratch.p, 0, sizeof(unsigned long long) * words, st));
      k_edit_score_long<<<(cnt * 32 + 127) / 128, 128, 0, st>>>(
          d_ids.as<uint32_t>() + n_short + L.first, d_slot.as<unsigned long long>() + L.first, cnt, lines[0].as<EditLine>(),
          lines[1].as<EditLine>(), d_range.as<uint2>(), arena_old, arena_new, d_scratch.as<unsigned long long>(), d_kept.as<EditCand>(), cap,
          d_nk.as<uint32_t>());
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&nk, d_nk.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += (n_short ? 1 : 0) + (int)launches.size();
    if (nk <= cap) break;
    cap = nk;
  }
  if (nk > cap) return TSM_E_CAPACITY;                     // (the second run holds every candidate of the first)
  kept.resize(nk);
  if (nk) CU(cudaMemcpyAsync(kept.data(), d_kept.p, sizeof(EditCand) * nk, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TSM_OK;
}

extern "C" int tsm_diff_pairs_assert_edits(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                           tsm_diff_detail* detail, tsm_diff_asserts* chg, tsm_assert_edit* edits, int64_t edit_cap,
                                           int64_t* n_edits, void* stream) {
  if (!c || !olds || !news || !added || !removed || !chg || !chg->aev || !chg->rev || !n_edits || edit_cap < 0 ||
      olds->n_files != news->n_files || olds->n_groups != news->n_groups)
    return TSM_E_ARG;
  const int32_t n = olds->n_files;
  int rc = check_groups(olds, 0, n);
  if (rc == TSM_OK) rc = check_groups(news, 0, n);
  if (rc != TSM_OK) return rc;
  chg->n_aev = chg->n_rev = 0;
  *n_edits = 0;
  float* const ms = clear_ms(c, MS_EDIT);
  if (n == 0) {
    for (int64_t* t : {chg->added_counts, chg->removed_counts})
      if (t) memset(t, 0, sizeof(int64_t) * (size_t)olds->n_groups * TSM_K);
    return TSM_OK;
  }
  return pair_call(c, olds, news, PAIR_GRP, &ms[0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    std::vector<tsm_diff_detail> own;
    if (!detail) { own.resize((size_t)n); detail = own.data(); }
    int rc = diff_core<DIFF_MARKS>(c, P.A, P.B, n, added, removed, detail, st);
    if (rc != TSM_OK) return rc;
    ms[1] = c->last_ms[MS_DIFF][1] + c->last_ms[MS_DIFF][2];
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<uint8_t> traced((size_t)n);
    for (int32_t i = 0; i < n; ++i) traced[(size_t)i] = detail[i].added_assert >= 0;
    HostSide* side[2] = {&P.A, &P.B};
    DevBuf d_traced, d_flag[2], d_pos[2], d_kept[2], d_rank[2], d_lines[2], d_cand[2], d_bsum, d_ctrl;
    if (!d_traced.alloc((size_t)n) || !d_ctrl.alloc(2 * 64) ||
        !d_bsum.alloc(sizeof(unsigned long long) * ((size_t)std::max(P.A.total, P.B.total) / XS_TILE + 4)))
      return TSM_E_CUDA;
    CU(cudaMemcpyAsync(d_traced.p, traced.data(), (size_t)n, cudaMemcpyHostToDevice, st));
    unsigned long long cnt[2] = {0, 0};
    EditSide es[2];
    for (int s = 0; s < 2; ++s) {
      const HostSide& h = *side[s];
      const uint32_t total = (uint32_t)h.total;
      if (!d_flag[s].alloc(sizeof(uint32_t) * total) || !d_kept[s].alloc(sizeof(uint32_t) * total) ||
          !d_pos[s].alloc(sizeof(unsigned long long) * ((size_t)total + 1)) || !d_rank[s].alloc(sizeof(unsigned long long) * ((size_t)total + 1)))
        return TSM_E_CUDA;
      es[s] = EditSide{h.d.arena, h.d.off, h.d.line_base, (uint32_t)n, h.d.line_end, h.d.line_flag, h.line_mark.as<uint8_t>(), d_traced.as<uint8_t>()};
      kept_ranks(h, d_kept[s], d_rank[s], d_bsum, st);
      if (total) k_edit_flag<<<(total + 255) / 256, 256, 0, st>>>(es[s], total, d_flag[s].as<uint32_t>());
      xscan(d_flag[s].as<uint32_t>(), total, d_bsum.as<unsigned long long>(), d_pos[s].as<unsigned long long>(), st);
      CU(cudaMemcpyAsync(&cnt[s], d_pos[s].as<unsigned long long>() + total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      c->launches += total ? 8 : 0;
    }
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    const uint32_t ne[2] = {(uint32_t)cnt[0], (uint32_t)cnt[1]};
    Ctrl hc[2] = {};
    unsigned long long* list[2];
    for (int s = 0; s < 2; ++s) {
      const uint32_t total = (uint32_t)side[s]->total;
      if (!d_lines[s].alloc(sizeof(EditLine) * std::max(ne[s], 1u)) || !d_cand[s].alloc(sizeof(unsigned long long) * std::max(ne[s], 1u)))
        return TSM_E_CUDA;
      list[s] = d_cand[s].as<unsigned long long>();
      hc[s].n_cand = ne[s];
      if (total)
        k_edit_compact<<<(total + 255) / 256, 256, 0, st>>>(es[s], total, d_flag[s].as<uint32_t>(), d_pos[s].as<unsigned long long>(),
                                                            d_rank[s].as<unsigned long long>(), d_lines[s].as<EditLine>(), list[s]);
      c->launches += total ? 1 : 0;
    }
    CU(cudaGetLastError());
    Ctrl* ctrl[2] = {d_ctrl.as<Ctrl>(), reinterpret_cast<Ctrl*>(d_ctrl.as<uint8_t>() + 64)};
    for (int s = 0; s < 2; ++s) CU(cudaMemcpyAsync(ctrl[s], &hc[s], sizeof(Ctrl), cudaMemcpyHostToDevice, st));
    const int cls_rc = classify_changed(c, side, list, ctrl, ne, n, P.groups_a, chg, st);
    if (cls_rc != TSM_OK && cls_rc != TSM_E_CAPACITY) return cls_rc;
    std::vector<EditCand> kept;
    std::vector<EditLine> pat;
    if (ne[0] && ne[1]) {
      rc = edit_scores(c, d_lines, ne, P.A.d.arena, P.B.d.arena, kept, pat, st);
      if (rc != TSM_OK) return rc;
    }
    // greedy pairing per hunk: candidates bucketed by old entry (counting sort), then each hunk's run sorted by score
    // (descending), old entry, new entry and taken in that order; each entry in at most one edit
    std::vector<uint32_t> at((size_t)ne[0] + 1, 0);
    for (const EditCand& k : kept) ++at[(size_t)k.old_e + 1];
    for (uint32_t i = 0; i < ne[0]; ++i) at[(size_t)i + 1] += at[i];
    std::vector<EditCand> by_old(kept.size());
    {
      std::vector<uint32_t> put(at.begin(), at.end() - 1);
      for (const EditCand& k : kept) by_old[put[k.old_e]++] = k;
    }
    std::vector<char> used_old(ne[0], 0), used_new(ne[1], 0);
    std::vector<tsm_assert_edit> got;
    for (uint32_t h0 = 0, h1 = 0; h0 < (uint32_t)pat.size(); h0 = h1) {
      for (h1 = h0 + 1; h1 < (uint32_t)pat.size() && pat[h1].key == pat[h0].key; ++h1) {}
      const auto b = by_old.begin() + at[h0], e = by_old.begin() + at[h1];
      std::sort(b, e, [](const EditCand& x, const EditCand& y) {
        return x.score != y.score ? x.score > y.score : (x.old_e != y.old_e ? x.old_e < y.old_e : x.new_e < y.new_e);
      });
      for (auto k = b; k != e; ++k)
        if (!used_old[k->old_e] && !used_new[k->new_e]) {
          used_old[k->old_e] = used_new[k->new_e] = 1;
          got.push_back(tsm_assert_edit{(int64_t)k->old_e, (int64_t)k->new_e, (int32_t)k->score, 0});
        }
    }
    std::sort(got.begin(), got.end(), [](const tsm_assert_edit& x, const tsm_assert_edit& y) { return x.aev < y.aev; });
    ms[2] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *n_edits = (int64_t)got.size();
    if (cls_rc == TSM_E_CAPACITY || *n_edits > edit_cap) return TSM_E_CAPACITY;   // all three counts set: size and call again
    if (*n_edits && !edits) return TSM_E_ARG;
    if (*n_edits) memcpy(edits, got.data(), sizeof(tsm_assert_edit) * got.size());
    return TSM_OK;
  });
}

extern "C" int tsm_assert_edits_last_ms(tsm_ctx* c, float* ms3) { return copy_ms(c, MS_EDIT, ms3, 3); }

// Provenance: the checks of prev and the line counts on the host, the marks diff, then ONE k_blame launch over the chains
// (pair lists in chain order, longest chain first: the long chains are the tail of the launch).
extern "C" int tsm_blame_pairs(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                               tsm_diff_detail* detail, const int32_t* prev, const int32_t* label, const tsm_origin* origin_in,
                               const int64_t* in_base, int64_t* line_base_old, int64_t* line_base_new, tsm_origin* origin_out,
                               int64_t cap, int64_t* n_lines, void* stream) {
  if (!c || !olds || !news || !added || !removed || !prev || !label || !in_base || !n_lines || olds->n_files != news->n_files)
    return TSM_E_ARG;
  const int32_t n = olds->n_files;
  *n_lines = 0;
  float* const ms = clear_ms(c, MS_BLAME);
  if (n == 0) {
    if (line_base_old) line_base_old[0] = 0;
    if (line_base_new) line_base_new[0] = 0;
    return TSM_OK;
  }
  std::vector<int32_t> next((size_t)n, -1);
  if (in_base[0] < 0) return TSM_E_ARG;
  for (int32_t i = 0; i < n; ++i) {
    const int32_t p = prev[i];
    if (p < -1 || p >= i || in_base[i + 1] < in_base[i]) return TSM_E_ARG;
    if (p >= 0) {
      if (next[(size_t)p] != -1) return TSM_E_ARG;         // a new side continues one chain only
      next[(size_t)p] = i;
    } else if (in_base[i + 1] > in_base[i] && !origin_in) {
      return TSM_E_ARG;
    }
  }
  return pair_call(c, olds, news, PAIR_HOST_BASE, &c->last_ms[MS_DIFF][0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    if (line_base_old) memcpy(line_base_old, P.A.base.data(), sizeof(int64_t) * ((size_t)n + 1));
    if (line_base_new) memcpy(line_base_new, P.B.base.data(), sizeof(int64_t) * ((size_t)n + 1));
    *n_lines = (int64_t)P.B.total;
    const std::vector<unsigned long long>& la = P.A.base;
    const std::vector<unsigned long long>& lb = P.B.base;
    for (int32_t i = 0; i < n; ++i) {                        // old side i = new side prev[i], or the head's range of origin_in
      const unsigned long long want = prev[i] >= 0 ? lb[(size_t)prev[i] + 1] - lb[(size_t)prev[i]] : (unsigned long long)(in_base[i + 1] - in_base[i]);
      if (la[(size_t)i + 1] - la[(size_t)i] != want) return TSM_E_ARG;
    }
    if (cap < *n_lines) return TSM_E_CAPACITY;
    if (*n_lines && !origin_out) return TSM_E_ARG;
    const int rc = diff_core<DIFF_MARKS>(c, P.A, P.B, n, added, removed, detail, st);
    if (rc != TSM_OK) return rc;
    // chains: heads in pair order, then stably by length, longest first
    std::vector<int32_t> heads, len;
    for (int32_t i = 0; i < n; ++i)
      if (prev[i] < 0) {
        int32_t k = 0;
        for (int32_t j = i; j >= 0; j = next[(size_t)j]) ++k;
        heads.push_back(i); len.push_back(k);
      }
    std::vector<int32_t> order_h(heads.size());
    for (size_t h = 0; h < heads.size(); ++h) order_h[h] = (int32_t)h;
    std::stable_sort(order_h.begin(), order_h.end(), [&](int32_t x, int32_t y) { return len[(size_t)x] > len[(size_t)y]; });
    const int32_t n_chains = (int32_t)heads.size();
    std::vector<int32_t> chain_pairs, chain_start;
    chain_pairs.reserve((size_t)n); chain_start.reserve((size_t)n_chains + 1);
    for (int32_t h : order_h) {
      chain_start.push_back((int32_t)chain_pairs.size());
      for (int32_t j = heads[(size_t)h]; j >= 0; j = next[(size_t)j]) chain_pairs.push_back(j);
    }
    chain_start.push_back((int32_t)chain_pairs.size());
    const size_t n_in = (size_t)in_base[n];
    DevBuf d_prev, d_label, d_head, d_in_base, d_pairs, d_start, d_work, d_keep, d_out;
    if (!d_prev.alloc(sizeof(int32_t) * (size_t)n) || !d_label.alloc(sizeof(int32_t) * (size_t)n) ||
        !d_head.alloc(sizeof(tsm_origin) * n_in) || !d_in_base.alloc(sizeof(int64_t) * ((size_t)n + 1)) ||
        !d_pairs.alloc(sizeof(int32_t) * (size_t)n) || !d_start.alloc(sizeof(int32_t) * ((size_t)n_chains + 1)) || !d_work.alloc(16) ||
        !d_keep.alloc(sizeof(tsm_origin) * (size_t)P.A.total) || !d_out.alloc(sizeof(tsm_origin) * (size_t)P.B.total))
      return TSM_E_CUDA;
    CU(cudaMemcpyAsync(d_prev.p, prev, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_label.p, label, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    if (n_in) CU(cudaMemcpyAsync(d_head.p, origin_in, sizeof(tsm_origin) * n_in, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_in_base.p, in_base, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_pairs.p, chain_pairs.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_start.p, chain_start.data(), sizeof(int32_t) * ((size_t)n_chains + 1), cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(d_work.p, 0, 16, st));
    CU(cudaEventRecord(c->diff_ev[EV_BLAME.from], st));
    k_blame<<<std::min((n_chains + 7) / 8, c->sms * 8), 256, 0, st>>>(
        P.A.d.line_base, P.B.d.line_base, P.A.line_mark.as<uint8_t>(), P.B.line_mark.as<uint8_t>(), d_prev.as<int32_t>(), d_label.as<int32_t>(),
        d_head.as<tsm_origin>(), d_in_base.as<long long>(), d_pairs.as<int32_t>(), d_start.as<int32_t>(), n_chains, d_work.as<uint32_t>(),
        d_keep.as<tsm_origin>(), d_out.as<tsm_origin>());
    CU(cudaEventRecord(c->diff_ev[EV_BLAME.to], st));
    CU(cudaGetLastError());
    c->launches++;
    if (*n_lines) CU(cudaMemcpyAsync(origin_out, d_out.p, sizeof(tsm_origin) * (size_t)*n_lines, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    ms[0] = span_ms(c, EV_BLAME);
    return TSM_OK;
  });
}

extern "C" int tsm_blame_last_ms(tsm_ctx* c, float* ms) { return copy_ms(c, MS_BLAME, ms, 1); }

// ------------------------------------------------------------------------------------- SPEC section 13 rename similarity
// Per side with line records: k_sim_sort (distinct (hash, weight) of every file at its line_base), xscan of the list
// lengths, k_sim_compact (dense CSR).  last_ms[MS_SIM][1] covers both sides.
namespace {
struct SimLists { DevBuf wk_key, wk_w, s_key, s_cum, cnt, bsum, base, key, w; };

int sim_lists(const HostSide& h, SimLists& L, cudaStream_t st) {
  const int32_t n = h.n;
  const size_t lines = (size_t)h.total;
  if (!L.wk_key.alloc(sizeof(unsigned long long) * lines) || !L.wk_w.alloc(sizeof(uint32_t) * lines) ||
      !L.s_key.alloc(sizeof(unsigned long long) * lines) || !L.s_cum.alloc(sizeof(uint32_t) * lines) ||
      !L.cnt.alloc(sizeof(uint32_t) * (size_t)n) || !L.bsum.alloc(sizeof(unsigned long long) * ((size_t)n / XS_TILE + 4)) ||
      !L.base.alloc(sizeof(unsigned long long) * ((size_t)n + 1)) || !L.key.alloc(sizeof(unsigned long long) * lines) ||
      !L.w.alloc(sizeof(uint32_t) * lines))
    return TSM_E_CUDA;
  k_sim_sort<<<n, SIM_SORT_THREADS, SIM_SORT_SMEM, st>>>(h.d.arena, h.d.off, h.d.len, h.d.line_base, h.d.line_hash, h.d.line_end,
                                                        L.wk_key.as<unsigned long long>(), L.wk_w.as<uint32_t>(),
                                                        L.s_key.as<unsigned long long>(), L.s_cum.as<uint32_t>(), L.cnt.as<uint32_t>());
  xscan(L.cnt.as<uint32_t>(), (uint32_t)n, L.bsum.as<unsigned long long>(), L.base.as<unsigned long long>(), st);
  k_sim_compact<<<(unsigned)(((size_t)n * 32 + 255) / 256), 256, 0, st>>>(h.d.line_base, L.cnt.as<uint32_t>(), L.base.as<unsigned long long>(),
                                                                          (uint32_t)n, L.s_key.as<unsigned long long>(), L.s_cum.as<uint32_t>(),
                                                                          L.key.as<unsigned long long>(), L.w.as<uint32_t>());
  CU(cudaGetLastError());
  return TSM_OK;
}
}  // namespace

extern "C" int tsm_similarity(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, const int32_t* cand_old,
                              const int32_t* cand_new, int64_t n_cand, int64_t* common, void* stream) {
  if (!c || !olds || !news || n_cand < 0 || (n_cand && (!cand_old || !cand_new || !common))) return TSM_E_ARG;
  if (olds->n_files < 0 || news->n_files < 0) return TSM_E_ARG;
  float* const ms = clear_ms(c, MS_SIM);
  if (n_cand == 0) return TSM_OK;
  CU(cudaSetDevice(c->device));
  {                                                        // the candidates, their indices and results: 16 B each on the device
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if ((uint64_t)n_cand > free_b / 16) return TSM_E_NOMEM;
  }
  for (int64_t i = 0; i < n_cand; ++i)
    if (cand_old[i] < 0 || cand_old[i] >= olds->n_files || cand_new[i] < 0 || cand_new[i] >= news->n_files) return TSM_E_ARG;
  return pair_call(c, olds, news, PAIR_ANY_EXT, &ms[0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    const size_t nc = (size_t)n_cand;
    SimLists LA, LB;
    DevBuf d_cand;
    if (!d_cand.alloc(16 * nc + 64)) { cudaGetLastError(); return TSM_E_NOMEM; }
    long long* d_common = d_cand.as<long long>();
    int32_t* d_old = reinterpret_cast<int32_t*>(d_common + nc);
    int32_t* d_new = d_old + nc;
    unsigned long long* d_next = reinterpret_cast<unsigned long long*>(d_new + nc);   // at 16 * nc bytes: 8-byte aligned
    CU(cudaMemcpyAsync(d_old, cand_old, sizeof(int32_t) * nc, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_new, cand_new, sizeof(int32_t) * nc, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(d_next, 0, sizeof(unsigned long long), st));
    CU(cudaEventRecord(c->diff_ev[EV_SIM_LISTS], st));
    int rc = sim_lists(P.A, LA, st);
    if (rc == TSM_OK) rc = sim_lists(P.B, LB, st);
    if (rc != TSM_OK) return rc;
    CU(cudaEventRecord(c->diff_ev[EV_SIM_PAIRS], st));
    const unsigned grid = (unsigned)std::min<size_t>((size_t)c->sms * 8, (nc + 8 * SIM_GRAB - 1) / (8 * SIM_GRAB));
    k_similarity<<<grid, 256, 0, st>>>(LA.key.as<unsigned long long>(), LA.w.as<uint32_t>(), LA.base.as<unsigned long long>(),
                                       LB.key.as<unsigned long long>(), LB.w.as<uint32_t>(), LB.base.as<unsigned long long>(),
                                       d_old, d_new, (unsigned long long)nc, d_next, d_common);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_SIM_END], st));
    CU(cudaMemcpyAsync(common, d_common, sizeof(int64_t) * nc, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    P.A.drop_staging(); P.B.drop_staging();
    ms[1] = elapsed_ms(c->diff_ev[EV_SIM_LISTS], c->diff_ev[EV_SIM_PAIRS]);
    ms[2] = elapsed_ms(c->diff_ev[EV_SIM_PAIRS], c->diff_ev[EV_SIM_END]);
    c->launches = P.A.launches + P.B.launches + 2 * 5 + 1;   // per side k_sim_sort, xscan (3), k_sim_compact; k_similarity
    return TSM_OK;
  });
}

extern "C" int tsm_similarity_last_ms(tsm_ctx* c, float* ms3) { return copy_ms(c, MS_SIM, ms3, 3); }

// ------------------------------------------------------------------------------------- S9 line / n-gram hashes
// The front of tsm_line_hashes and tsm_statements: the corpus' line records from one pass of the scan, and line_base[n+1]
// and *n_lines on the host - also when cap is short of the lines, which returns TSM_E_CAPACITY so that the caller can
// allocate and call again.  Then tail(S, lines, st), the call's own use of the records, inside the call's SyncGuard.
// scan_ms: the device time of the k_scan launches; flags: TSM_SCAN_HEADER_EVENTS also lists the header events (S.hev).
template <typename Tail>
static int line_records(tsm_ctx* c, const tsm_corpus* k, bool ext_rule, int64_t* line_base, int64_t cap, int64_t* n_lines,
                        void* stream, Tail tail, float* scan_ms = nullptr, uint32_t flags = 0) {
  const int32_t n = k->n_files;
  *n_lines = 0;
  line_base[0] = 0;
  if (n == 0) return TSM_OK;
  int rc = check_sides({k}, ext_rule);
  if (rc != TSM_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  HostSide S;
  SyncGuard guard(st);
  rc = side_upload(k, S, st);
  if (rc == TSM_OK) rc = side_records(c, S, st, scan_ms, flags);
  if (rc != TSM_OK) return rc;
  const unsigned long long total = S.base[(size_t)n];
  for (int32_t i = 0; i <= n; ++i) line_base[i] = (int64_t)S.base[(size_t)i];
  *n_lines = (int64_t)total;
  c->launches = S.launches;
  if ((unsigned long long)cap < total) return TSM_E_CAPACITY;
  if (total == 0) return TSM_OK;
  return tail(S, total, st);
}

extern "C" int tsm_line_hashes(tsm_ctx* c, const tsm_corpus* k, int64_t* line_base, uint64_t* line_hash, uint32_t* line_end,
                               uint8_t* line_flag, int64_t cap, int64_t* n_lines, int32_t ngram_n, uint64_t* ngram_hash,
                               void* stream) {
  if (!c || !k || !line_base || !n_lines || cap < 0 || k->n_files < 0 || ngram_n < 0 || (ngram_hash && ngram_n < 1)) return TSM_E_ARG;
  return line_records(c, k, true, line_base, cap, n_lines, stream, [&](const HostSide& S, unsigned long long total, cudaStream_t st) -> int {
    if (line_hash) CU(cudaMemcpyAsync(line_hash, S.d.line_hash, sizeof(uint64_t) * (size_t)total, cudaMemcpyDeviceToHost, st));
    if (line_end) CU(cudaMemcpyAsync(line_end, S.d.line_end, sizeof(uint32_t) * (size_t)total, cudaMemcpyDeviceToHost, st));
    if (line_flag) CU(cudaMemcpyAsync(line_flag, S.d.line_flag, (size_t)total, cudaMemcpyDeviceToHost, st));
    if (ngram_hash) {
      DevBuf d_ng;
      if (!d_ng.alloc(sizeof(unsigned long long) * (size_t)total)) { cudaStreamSynchronize(st); return TSM_E_CUDA; }
      k_ngrams<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(S.d.line_hash, S.d.line_base, (uint32_t)S.n, total, (uint32_t)ngram_n,
                                                                 d_ng.as<unsigned long long>());
      CU(cudaGetLastError());
      CU(cudaMemcpyAsync(ngram_hash, d_ng.p, sizeof(uint64_t) * (size_t)total, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      c->launches++;
    }
    CU(cudaStreamSynchronize(st));
    return TSM_OK;
  });
}

// ------------------------------------------------------------------------------------- SPEC section 10 statements
extern "C" int tsm_statements(tsm_ctx* c, const tsm_corpus* k, int64_t* line_base, uint32_t* line_end,
                              uint8_t* line_kind, int64_t cap, int64_t* n_lines, void* stream) {
  if (!c || !k || !line_base || !n_lines || cap < 0 || k->n_files < 0) return TSM_E_ARG;
  return line_records(c, k, false, line_base, cap, n_lines, stream, [&](const HostSide& S, unsigned long long total, cudaStream_t st) -> int {
    if (!line_end || !line_kind) return TSM_E_ARG;
    DevBuf d_delta, d_kind;
    if (!d_delta.alloc(sizeof(int32_t) * (size_t)total) || !d_kind.alloc((size_t)total)) return TSM_E_CUDA;
    k_line_parens<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(S.d, S.n, total, d_delta.as<int32_t>(), d_kind.as<uint8_t>());
    k_stmt_kinds<<<(S.n * 32 + 127) / 128, 128, 0, st>>>(S.d, S.n, d_delta.as<int32_t>(), d_kind.as<uint8_t>());
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(line_end, S.d.line_end, sizeof(uint32_t) * (size_t)total, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(line_kind, d_kind.p, (size_t)total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += 2;
    return TSM_OK;
  });
}

// ------------------------------------------------------------------------------------- SPEC section 15 clones
// Section 15 over T lines (T > 0) of nfu files: their hashes, per-file bases line_base[nfu + 1] and assertion flags on the
// device; with SKIP_EMPTY the window test reads the lines' bytes (arena, off, line_end).  The kernels of tsm_clone_kernels.cuh,
// with one synchronisation between the grouping and the members that reads the class and fragment counts: a short cap returns
// there, else the fragments are scattered, sorted and copied back with the coverage.  ms[0] / ms[1]: grouping + classes, members
// + coverage.  Then then(dev, st), the caller's use of the classes on the device (CloneDev), before their buffers go back to the
// pool; it is not called when there is no class.  class_out / member_out: the caller has outputs of its own sized by class_cap /
// member_cap, which the capacity rule then counts as given.
struct CloneDev {
  const unsigned long long* class_base; const uint32_t* class_len; const unsigned long long* member;   // [nc + 1], [nc], [nm]
  uint32_t nc; unsigned long long nm;
  uint32_t n_units;                                        // the lines (or kept lines) the classes are numbered in
  const unsigned long long* unit_line;                     // the line of every unit (blind: kept_line), NULL = unit u is line u
  const uint8_t* unit_flag;                                // the assertion flag of every unit
};
struct NoThen { int operator()(const CloneDev&, cudaStream_t) const { return TSM_OK; } };
template <bool SKIP_EMPTY, typename Then = NoThen>
static int clone_classes(tsm_ctx* c, const unsigned long long* hash, const unsigned long long* line_base, uint32_t nfu, uint32_t T,
                         const uint8_t* line_flag, const uint32_t* line_end, const uint8_t* arena, const int32_t* off, uint32_t n,
                         tsm_clone_result* out, float* ms, cudaStream_t st, Then then = {}, bool class_out = false,
                         bool member_out = false) {
  size_t slots = 1;                                      // a power of two, at least 2 x the windows (<= lines)
  while (slots < 2 * (size_t)T) slots <<= 1;
  const uint32_t mask = (uint32_t)(slots - 1);
  const size_t table_bytes = (slots + 1) * (sizeof(CloneSlot) + 3 * sizeof(uint32_t));
  {
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if (table_bytes > free_b) return TSM_E_NOMEM;
  }
  const size_t L = (size_t)T, nb = L / XS_TILE + 4;
  DevBuf d_key, d_slot, d_wflag, d_table, d_plo, d_phi, d_scls, d_dup, d_head, d_ext, d_cidx, d_cover, d_rep, d_size, d_cbase,
      d_big, d_nbig, d_bsum, d_len, d_cursor, d_member, d_wk, d_fdup;
  if (!d_key.alloc(8 * L) || !d_slot.alloc(4 * L) || !d_wflag.alloc(L) || !d_table.alloc(sizeof(CloneSlot) * (slots + 1)) ||
      !d_plo.alloc(4 * (slots + 1)) || !d_phi.alloc(4 * (slots + 1)) || !d_scls.alloc(4 * (slots + 1)) || !d_dup.alloc(4 * L) ||
      !d_head.alloc(4 * L) || !d_ext.alloc(L) || !d_cidx.alloc(8 * (L + 1)) || !d_cover.alloc(8 * (L + 1)) || !d_rep.alloc(4 * L) ||
      !d_size.alloc(4 * L) || !d_cbase.alloc(8 * (L + 1)) || !d_big.alloc(4 * L) || !d_nbig.alloc(4) || !d_bsum.alloc(8 * nb) ||
      !d_len.alloc(4 * L) || !d_fdup.alloc(8 * (size_t)nfu)) {
    cudaGetLastError();
    return TSM_E_NOMEM;
  }
  CloneSlot* table = d_table.as<CloneSlot>();
  uint32_t* slot_of = d_slot.as<uint32_t>();
  const unsigned grid = (unsigned)((L + 255) / 256);
  CU(cudaEventRecord(c->diff_ev[EV_CLONE_GROUP], st));
  CU(cudaMemsetAsync(d_table.p, 0, sizeof(CloneSlot) * (slots + 1), st));
  CU(cudaMemsetAsync(d_plo.p, 0xFF, 4 * (slots + 1), st));
  CU(cudaMemsetAsync(d_phi.p, 0, 4 * (slots + 1), st));
  CU(cudaMemsetAsync(d_scls.p, 0xFF, 4 * (slots + 1), st));
  CU(cudaMemsetAsync(d_size.p, 0, 4 * L, st));
  CU(cudaMemsetAsync(d_nbig.p, 0, 4, st));
  k_ngrams<<<grid, 256, 0, st>>>(hash, line_base, nfu, T, n, d_key.as<unsigned long long>());
  k_clone_insert<SKIP_EMPTY><<<grid, 256, 0, st>>>(d_key.as<unsigned long long>(), line_base, nfu, line_end, arena, off, T, n, table,
                                       mask, slot_of, d_wflag.as<uint8_t>());
  k_clone_preds<<<grid, 256, 0, st>>>(table, slot_of, d_wflag.as<uint8_t>(), T, d_plo.as<uint32_t>(), d_phi.as<uint32_t>());
  k_clone_heads<<<grid, 256, 0, st>>>(table, slot_of, d_plo.as<uint32_t>(), d_phi.as<uint32_t>(), T, d_dup.as<uint32_t>(),
                                      d_head.as<uint32_t>(), d_ext.as<uint8_t>());
  xscan(d_head.as<uint32_t>(), T, d_bsum.as<unsigned long long>(), d_cidx.as<unsigned long long>(), st);
  xscan(d_dup.as<uint32_t>(), T, d_bsum.as<unsigned long long>(), d_cover.as<unsigned long long>(), st);
  k_clone_classes<<<grid, 256, 0, st>>>(d_head.as<uint32_t>(), d_cidx.as<unsigned long long>(), slot_of, table, T, d_rep.as<uint32_t>(),
                                        d_size.as<uint32_t>(), d_scls.as<uint32_t>(), d_big.as<uint32_t>(), d_nbig.as<uint32_t>());
  xscan(d_size.as<uint32_t>(), T, d_bsum.as<unsigned long long>(), d_cbase.as<unsigned long long>(), st);
  k_clone_length<<<(unsigned)c->sms * 8, 256, 0, st>>>(d_rep.as<uint32_t>(), d_ext.as<uint8_t>(), T, n, d_cidx.as<unsigned long long>() + L,
                                                       d_len.as<uint32_t>());
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->diff_ev[EV_CLONE_MEMBERS], st));
  unsigned long long* pin = c->h_rb->u64;                 // classes, fragments, large classes
  CU(cudaMemcpyAsync(pin, d_cidx.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(pin + 1, d_cbase.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(pin + 2, d_nbig.p, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  c->launches += 15;                                     // k_ngrams, insert, preds, heads, 3 x xscan (3 each), classes, length
  const uint32_t nc = (uint32_t)pin[0], nbig = (uint32_t)(pin[2] & 0xFFFFFFFFu);
  const unsigned long long nm = pin[1];
  out->n_classes = (int64_t)nc;
  out->n_members = (int64_t)nm;
  ms[0] = elapsed_ms(c->diff_ev[EV_CLONE_GROUP], c->diff_ev[EV_CLONE_MEMBERS]);
  if ((out->class_cap < (int64_t)nc && (class_out || out->class_base || out->class_len)) || (out->member_cap < (int64_t)nm && (member_out || out->member)))
    return TSM_E_CAPACITY;
  if (nc) {
    if (!d_cursor.alloc(4 * (size_t)nc) || !d_member.alloc(8 * nm) || !d_wk.alloc(4 * nm)) { cudaGetLastError(); return TSM_E_NOMEM; }
    unsigned long long* member = d_member.as<unsigned long long>();
    CU(cudaMemsetAsync(d_cursor.p, 0, 4 * (size_t)nc, st));
    k_clone_scatter<<<grid, 256, 0, st>>>(slot_of, d_scls.as<uint32_t>(), d_cbase.as<unsigned long long>(), T, d_cursor.as<uint32_t>(), member);
    k_clone_sort_warp<<<(unsigned)(((size_t)nc * 32 + 255) / 256), 256, 0, st>>>(d_cbase.as<unsigned long long>(), nc, member);
    c->launches += 2;
    if (nbig) {
      k_clone_sort_cta<<<std::min<unsigned>(nbig, (unsigned)c->sms * 2), SIM_SORT_THREADS, SIM_SORT_SMEM, st>>>(
          d_cbase.as<unsigned long long>(), d_big.as<uint32_t>(), d_nbig.as<uint32_t>(), member, d_wk.as<uint32_t>());
      c->launches += 1;
    }
    uint32_t* fdup = d_fdup.as<uint32_t>();
    k_clone_cover<<<(unsigned)(((size_t)nfu * 32 + 255) / 256), 256, 0, st>>>(line_base, nfu, d_cover.as<unsigned long long>(),
                                                                            line_flag, n, fdup, fdup + nfu);
    c->launches += 1;
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_CLONE_END], st));
    if (out->file_dup) CU(cudaMemcpyAsync(out->file_dup, fdup, 4 * (size_t)nfu, cudaMemcpyDeviceToHost, st));
    if (out->file_dup_assert) CU(cudaMemcpyAsync(out->file_dup_assert, fdup + nfu, 4 * (size_t)nfu, cudaMemcpyDeviceToHost, st));
    if (out->class_base) CU(cudaMemcpyAsync(out->class_base, d_cbase.p, 8 * ((size_t)nc + 1), cudaMemcpyDeviceToHost, st));
    if (out->class_len) CU(cudaMemcpyAsync(out->class_len, d_len.p, 4 * (size_t)nc, cudaMemcpyDeviceToHost, st));
    if (out->member) CU(cudaMemcpyAsync(out->member, member, 8 * nm, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    ms[1] = elapsed_ms(c->diff_ev[EV_CLONE_MEMBERS], c->diff_ev[EV_CLONE_END]);
    return then(CloneDev{d_cbase.as<unsigned long long>(), d_len.as<uint32_t>(), member, nc, nm, T, nullptr, line_flag}, st);
  }
  return TSM_OK;
}

// The line records of the corpus (line_records), then clone_classes over them.
extern "C" int tsm_clones(tsm_ctx* c, const tsm_corpus* k, int32_t min_lines, tsm_clone_result* out, void* stream) {
  if (!c || !k || !out || k->n_files < 0 || min_lines < 1 || min_lines > 1024 || out->class_cap < 0 || out->member_cap < 0) return TSM_E_ARG;
  const int32_t nf = k->n_files;
  float* const ms = clear_ms(c, MS_CLONE);
  c->launches = 0;
  out->n_classes = out->n_members = 0;
  if (out->class_base) out->class_base[0] = 0;
  if (out->file_dup) memset(out->file_dup, 0, sizeof(uint32_t) * (size_t)nf);
  if (out->file_dup_assert) memset(out->file_dup_assert, 0, sizeof(uint32_t) * (size_t)nf);
  std::vector<int64_t> own_base;
  int64_t* line_base = out->line_base;
  if (!line_base) { own_base.resize((size_t)nf + 1); line_base = own_base.data(); }
  int64_t n_lines = 0;
  return line_records(c, k, true, line_base, INT64_MAX, &n_lines, stream, [&](const HostSide& S, unsigned long long total, cudaStream_t st) -> int {
    return clone_classes<true>(c, S.d.line_hash, S.d.line_base, (uint32_t)S.n, (uint32_t)total, S.d.line_flag, S.d.line_end, S.d.arena,
                               S.d.off, (uint32_t)min_lines, out, ms + 1, st);
  }, &ms[0]);
}

extern "C" int tsm_clones_last_ms(tsm_ctx* c, float* ms3) { return copy_ms(c, MS_CLONE, ms3, 3); }

// ------------------------------------------------------------------------------------- SPEC section 21 blind clones
// The lexer of section 21 over one side whose line records exist (S.total > 0), in the kernels of tsm_blind_kernels.cuh: line
// states, blind hashes and kept flags, an xscan of the kept flags (rank[l] = the kept lines before line l, rank[total] = all),
// the compaction of the kept lines (kline, khash, kflag) and per file its kept base and kept assertion lines.
struct BlindFront { DevBuf state, hash, kept, rank, bsum, kline, khash, kflag, kbase, kassert; };

static int blind_front(tsm_ctx* c, const HostSide& S, BlindFront& f, cudaStream_t st) {
  const unsigned long long total = S.total;
  const uint32_t T = (uint32_t)total, nfu = (uint32_t)S.n;
  const size_t L = (size_t)total;
  if (!f.state.alloc(L) || !f.hash.alloc(8 * L) || !f.kept.alloc(4 * L) || !f.rank.alloc(8 * (L + 1)) || !f.bsum.alloc(8 * (L / XS_TILE + 4)) ||
      !f.kline.alloc(8 * L) || !f.khash.alloc(8 * L) || !f.kflag.alloc(L) || !f.kbase.alloc(8 * ((size_t)nfu + 1)) ||
      !f.kassert.alloc(4 * (size_t)nfu)) {
    cudaGetLastError();
    return TSM_E_NOMEM;
  }
  const unsigned grid = (unsigned)((L + 255) / 256), fgrid = (unsigned)(((size_t)nfu * 32 + 255) / 256);
  unsigned long long* rank = f.rank.as<unsigned long long>();
  k_blind_state<<<grid, 256, 0, st>>>(S.d, nfu, total, f.state.as<uint8_t>());
  k_blind_scan<<<fgrid, 256, 0, st>>>(S.d.line_base, nfu, f.state.as<uint8_t>());
  k_blind_lines<<<grid, 256, 0, st>>>(S.d, nfu, total, f.state.as<uint8_t>(), f.hash.as<unsigned long long>(), f.kept.as<uint32_t>());
  xscan(f.kept.as<uint32_t>(), T, f.bsum.as<unsigned long long>(), rank, st);
  k_blind_compact<<<grid, 256, 0, st>>>(f.kept.as<uint32_t>(), rank, f.hash.as<unsigned long long>(), S.d.line_flag, total,
                                        f.kline.as<unsigned long long>(), f.khash.as<unsigned long long>(), f.kflag.as<uint8_t>());
  k_blind_files<<<(unsigned)(((size_t)nfu * 32 + 32 + 255) / 256), 256, 0, st>>>(S.d.line_base, nfu, rank, f.kflag.as<uint8_t>(),
                                                                                  f.kbase.as<unsigned long long>(), f.kassert.as<uint32_t>());
  CU(cudaGetLastError());
  c->launches += 8;                                      // state, scan, lines, xscan (3), compact, files
  return TSM_OK;
}

// The section-21 classes over one side whose line records exist (S, total lines > 0): blind_front, one synchronisation that reads the kept count, then clone_classes over
// the kept lines, with then, class_out and member_out as there (CloneDev::unit_line = the kept lines' lines).  A short kept_cap
// still runs the grouping, so that every count is set when it returns TSM_E_CAPACITY.  ms[0]: lexing + compaction, ms[1] / ms[2]:
// those of clone_classes.
template <typename Then = NoThen>
static int blind_classes(tsm_ctx* c, const HostSide& S, unsigned long long total, uint32_t min_lines, tsm_blind_result* b,
                         tsm_clone_result* out, float* ms, cudaStream_t st, Then then = {}, bool class_out = false, bool member_out = false) {
  const uint32_t nfu = (uint32_t)S.n;
  const size_t L = (size_t)total;
  BlindFront bf;
  CU(cudaEventRecord(c->diff_ev[EV_BLIND_LEX], st));
  int rc = blind_front(c, S, bf, st);
  if (rc != TSM_OK) return rc;
  CU(cudaEventRecord(c->diff_ev[EV_BLIND_LEX_END], st));
  unsigned long long* pin = c->h_rb->u64;
  CU(cudaMemcpyAsync(pin + 3, bf.rank.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
  if (b->kept_base) CU(cudaMemcpyAsync(b->kept_base, bf.kbase.p, 8 * ((size_t)nfu + 1), cudaMemcpyDeviceToHost, st));
  if (b->file_kept_assert) CU(cudaMemcpyAsync(b->file_kept_assert, bf.kassert.p, 4 * (size_t)nfu, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const unsigned long long nk = pin[3];
  b->n_kept = (int64_t)nk;
  ms[0] = elapsed_ms(c->diff_ev[EV_BLIND_LEX], c->diff_ev[EV_BLIND_LEX_END]);
  const bool kept_short = b->kept_cap < (int64_t)nk && (b->kept_line || b->blind_hash);
  if (!kept_short) {
    if (b->kept_line) CU(cudaMemcpyAsync(b->kept_line, bf.kline.p, 8 * nk, cudaMemcpyDeviceToHost, st));
    if (b->blind_hash) CU(cudaMemcpyAsync(b->blind_hash, bf.khash.p, 8 * nk, cudaMemcpyDeviceToHost, st));
  }
  const unsigned long long* kline = bf.kline.as<unsigned long long>();
  if (nk) rc = clone_classes<false>(c, bf.khash.as<unsigned long long>(), bf.kbase.as<unsigned long long>(), nfu, (uint32_t)nk,
                                    bf.kflag.as<uint8_t>(), nullptr, nullptr, nullptr, min_lines, out, ms + 1, st,
                                    [&](CloneDev d, cudaStream_t s2) { d.unit_line = kline; return then(d, s2); }, class_out, member_out);
  CU(cudaStreamSynchronize(st));
  return rc == TSM_OK && kept_short ? TSM_E_CAPACITY : rc;
}

// The line records of the corpus (line_records), then blind_classes over them.
extern "C" int tsm_clones_blind(tsm_ctx* c, const tsm_corpus* k, int32_t min_lines, tsm_blind_result* blind, tsm_clone_result* out,
                                void* stream) {
  if (!c || !k || !out || k->n_files < 0 || min_lines < 1 || min_lines > 1024 || out->class_cap < 0 || out->member_cap < 0 ||
      (blind && blind->kept_cap < 0))
    return TSM_E_ARG;
  const int32_t nf = k->n_files;
  float* const ms = clear_ms(c, MS_BLIND);
  c->launches = 0;
  out->n_classes = out->n_members = 0;
  if (out->class_base) out->class_base[0] = 0;
  if (out->file_dup) memset(out->file_dup, 0, sizeof(uint32_t) * (size_t)nf);
  if (out->file_dup_assert) memset(out->file_dup_assert, 0, sizeof(uint32_t) * (size_t)nf);
  tsm_blind_result none{nullptr, nullptr, nullptr, nullptr, 0, 0};
  tsm_blind_result* const b = blind ? blind : &none;
  b->n_kept = 0;
  if (b->kept_base) memset(b->kept_base, 0, sizeof(int64_t) * ((size_t)nf + 1));
  if (b->file_kept_assert) memset(b->file_kept_assert, 0, sizeof(uint32_t) * (size_t)nf);
  std::vector<int64_t> own_base;
  int64_t* line_base = out->line_base;
  if (!line_base) { own_base.resize((size_t)nf + 1); line_base = own_base.data(); }
  int64_t n_lines = 0;
  return line_records(c, k, true, line_base, INT64_MAX, &n_lines, stream, [&](const HostSide& S, unsigned long long total, cudaStream_t st) -> int {
    return blind_classes(c, S, total, (uint32_t)min_lines, b, out, ms + 1, st);
  }, &ms[0]);
}

extern "C" int tsm_clones_blind_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_BLIND, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 22 clone churn
// The edit marks of the pairs, on the lines of both revisions (S[i]: line records with line_base on the host; rmark[i]: one
// zeroed byte per line).  Each pair side is a view of its revision: its line_base from the files' line counts, its hashes and
// flags gathered from the revision's records (k_churn_gather), so that diff_core runs over the pairs without a second upload or
// scan.  k_churn_marks then puts every marked view line onto its revision line.  ms[2] += gather + diff, ms[3] += k_churn_marks.
static int churn_marks(tsm_ctx* c, HostSide* S, const int32_t* const pf[2], int32_t n, DevBuf* rmark, float* ms, cudaStream_t st) {
  HostSide V[2];
  DevBuf d_pf[2];
  CU(cudaEventRecord(c->diff_ev[EV_CCHURN.from], st));
  for (int i = 0; i < 2; ++i) {
    HostSide& v = V[i];
    v.n = n;
    v.base.assign((size_t)n + 1, 0);
    for (int32_t k = 0; k < n; ++k) {
      const int32_t f = pf[i][k];
      v.base[(size_t)k + 1] = v.base[(size_t)k] + (f >= 0 ? S[i].base[(size_t)f + 1] - S[i].base[(size_t)f] : 0);
    }
    v.total = v.base[(size_t)n];
    if (!v.line_base.alloc(8 * ((size_t)n + 1)) || !v.line_hash.alloc(8 * (size_t)v.total) || !v.line_flag.alloc((size_t)v.total) ||
        !d_pf[i].alloc(4 * (size_t)n))
      return TSM_E_CUDA;
    CU(cudaMemcpyAsync(v.line_base.p, v.base.data(), 8 * ((size_t)n + 1), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_pf[i].p, pf[i], 4 * (size_t)n, cudaMemcpyHostToDevice, st));
    if (v.total) {
      k_churn_gather<<<(unsigned)((v.total + 255) / 256), 256, 0, st>>>(v.line_base.as<unsigned long long>(), (uint32_t)n, d_pf[i].as<int32_t>(),
                                                                        S[i].d.line_base, S[i].d.line_hash, S[i].d.line_flag, v.total,
                                                                        v.line_hash.as<unsigned long long>(), v.line_flag.as<uint8_t>());
      c->launches++;
    }
    v.d.line_base = v.line_base.as<unsigned long long>();
    v.d.line_hash = v.line_hash.as<unsigned long long>();
    v.d.line_flag = v.line_flag.as<uint8_t>();
  }
  CU(cudaEventRecord(c->diff_ev[EV_CCHURN.to], st));
  CU(cudaGetLastError());
  const int launches = c->launches;
  std::vector<int64_t> added((size_t)n), removed((size_t)n);
  int rc = diff_core<DIFF_MARKS>(c, V[0], V[1], n, added.data(), removed.data(), nullptr, st);   // (synchronises st)
  c->launches += launches;
  if (rc != TSM_OK) return rc;
  ms[2] += span_ms(c, EV_CCHURN) + c->last_ms[MS_DIFF][1] + c->last_ms[MS_DIFF][2];
  CU(cudaEventRecord(c->diff_ev[EV_CCHURN.from], st));
  for (int i = 0; i < 2; ++i)
    if (V[i].total) {
      k_churn_marks<<<(unsigned)((V[i].total + 255) / 256), 256, 0, st>>>(V[i].d.line_base, (uint32_t)n, d_pf[i].as<int32_t>(), S[i].d.line_base,
                                                                          V[i].line_mark.as<uint8_t>(), V[i].total, rmark[i].as<uint8_t>());
      c->launches++;
    }
  CU(cudaEventRecord(c->diff_ev[EV_CCHURN.to], st));
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(st));
  ms[3] += span_ms(c, EV_CCHURN);
  return TSM_OK;
}

// The churn of one side's classes (CloneDev of clone_classes) under its revision's marks: per unit marked / marked assertion line
// (k_churn_units), their prefix sums, then k_churn_frags and k_churn_classes, copied into o's churn outputs.  ms[3] += their time.
static int churn_side(tsm_ctx* c, const CloneDev& d, const uint8_t* rmark, bool new_side, tsm_clone_churn_side* o, float* ms,
                      cudaStream_t st) {
  const uint32_t U = d.n_units, nc = d.nc;
  const unsigned long long nm = d.nm;
  DevBuf d_mk, d_mka, d_P, d_PA, d_bsum, d_ch, d_cha, d_state, d_counts, d_status;
  if (!d_mk.alloc(4 * (size_t)U) || !d_mka.alloc(4 * (size_t)U) || !d_P.alloc(8 * ((size_t)U + 1)) || !d_PA.alloc(8 * ((size_t)U + 1)) ||
      !d_bsum.alloc(8 * ((size_t)U / XS_TILE + 4)) || !d_ch.alloc(4 * nm) || !d_cha.alloc(4 * nm) || !d_state.alloc(nm) ||
      !d_counts.alloc(12 * (size_t)nc) || !d_status.alloc(nc)) {
    cudaGetLastError();
    return TSM_E_NOMEM;
  }
  const unsigned long long* P = d_P.as<unsigned long long>();
  const unsigned long long* PA = d_PA.as<unsigned long long>();
  CU(cudaEventRecord(c->diff_ev[EV_CCHURN.from], st));
  k_churn_units<<<(U + 255) / 256, 256, 0, st>>>(rmark, d.unit_line, d.unit_flag, U, d_mk.as<uint32_t>(), d_mka.as<uint32_t>());
  xscan(d_mk.as<uint32_t>(), U, d_bsum.as<unsigned long long>(), d_P.as<unsigned long long>(), st);
  xscan(d_mka.as<uint32_t>(), U, d_bsum.as<unsigned long long>(), d_PA.as<unsigned long long>(), st);
  k_churn_frags<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(d.class_base, d.class_len, nc, d.member, nm, P, PA, d_ch.as<uint32_t>(),
                                                               d_cha.as<uint32_t>(), d_state.as<uint8_t>());
  k_churn_classes<<<std::min<unsigned>((unsigned)c->sms * 8, (unsigned)(((size_t)nc * 32 + 255) / 256)), 256, 0, st>>>(
      d.class_base, nc, d_state.as<uint8_t>(), new_side, d_counts.as<uint32_t>(), d_status.as<uint8_t>());
  CU(cudaEventRecord(c->diff_ev[EV_CCHURN.to], st));
  CU(cudaGetLastError());
  c->launches += 9;                                        // units, 2 x xscan (3 each), frags, classes
  if (o->changed) CU(cudaMemcpyAsync(o->changed, d_ch.p, 4 * nm, cudaMemcpyDeviceToHost, st));
  if (o->changed_assert) CU(cudaMemcpyAsync(o->changed_assert, d_cha.p, 4 * nm, cudaMemcpyDeviceToHost, st));
  if (o->state) CU(cudaMemcpyAsync(o->state, d_state.p, nm, cudaMemcpyDeviceToHost, st));
  if (o->class_counts) CU(cudaMemcpyAsync(o->class_counts, d_counts.p, 12 * (size_t)nc, cudaMemcpyDeviceToHost, st));
  if (o->status) CU(cudaMemcpyAsync(o->status, d_status.p, nc, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  ms[3] += span_ms(c, EV_CCHURN);
  return TSM_OK;
}

// Both revisions to the device and their line records (one k_scan pass each, one synchronisation), the marks of the pairs
// (churn_marks), then per revision its classes - clone_classes over the line records, or blind_classes - whose continuation
// runs churn_side on the device arrays of the classes.  Both sides run also when one is short of a cap, so that every count is set.
extern "C" int tsm_clone_churn(tsm_ctx* c, const tsm_corpus* old_rev, const tsm_corpus* new_rev, const int32_t* pair_old,
                               const int32_t* pair_new, int64_t n_pairs, int32_t min_lines, int32_t blind, tsm_clone_churn_side* old_side,
                               tsm_clone_churn_side* new_side, void* stream) {
  if (!c || !old_rev || !new_rev || !old_side || !new_side || n_pairs < 0 || n_pairs > INT32_MAX || (n_pairs && (!pair_old || !pair_new)) ||
      min_lines < 1 || min_lines > 1024)
    return TSM_E_ARG;
  const tsm_corpus* rev[2] = {old_rev, new_rev};
  tsm_clone_churn_side* side[2] = {old_side, new_side};
  const int32_t* pf[2] = {pair_old, pair_new};
  const int32_t n = (int32_t)n_pairs;
  for (int i = 0; i < 2; ++i) {
    const tsm_clone_churn_side* o = side[i];
    if (rev[i]->n_files < 0 || o->clones.class_cap < 0 || o->clones.member_cap < 0 || (blind && o->blind.kept_cap < 0)) return TSM_E_ARG;
    std::vector<uint8_t> used((size_t)rev[i]->n_files, 0);
    for (int32_t k = 0; k < n; ++k) {
      const int32_t f = pf[i][k];
      if (f < -1 || f >= rev[i]->n_files || (f >= 0 && used[(size_t)f]++) || (pair_old[k] < 0 && pair_new[k] < 0)) return TSM_E_ARG;
    }
  }
  float* const ms = clear_ms(c, MS_CCHURN);
  c->launches = 0;
  for (int i = 0; i < 2; ++i) {
    tsm_clone_result& out = side[i]->clones;
    tsm_blind_result& b = side[i]->blind;
    const size_t nf = (size_t)rev[i]->n_files;
    out.n_classes = out.n_members = 0;
    if (out.line_base) memset(out.line_base, 0, sizeof(int64_t) * (nf + 1));
    if (out.class_base) out.class_base[0] = 0;
    if (out.file_dup) memset(out.file_dup, 0, sizeof(uint32_t) * nf);
    if (out.file_dup_assert) memset(out.file_dup_assert, 0, sizeof(uint32_t) * nf);
    if (blind) {
      b.n_kept = 0;
      if (b.kept_base) memset(b.kept_base, 0, sizeof(int64_t) * (nf + 1));
      if (b.file_kept_assert) memset(b.file_kept_assert, 0, sizeof(uint32_t) * nf);
    }
  }
  HostSide* scan[2];
  int ns = 0;
  for (int i = 0; i < 2; ++i)
    if (rev[i]->n_files > 0) {
      const int rc = check_sides({rev[i]}, true);
      if (rc != TSM_OK) return rc;
    }
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  HostSide S[2];
  DevBuf rmark[2];
  SyncGuard guard(st);
  for (int i = 0; i < 2; ++i)
    if (rev[i]->n_files > 0) {
      const int rc = side_upload(rev[i], S[i], st);
      if (rc != TSM_OK) return rc;
      scan[ns++] = &S[i];
    }
  if (ns) {
    const int rc = sides_records(c, scan, ns, st, &ms[0], true);
    if (rc != TSM_OK) return rc;
  }
  for (int i = 0; i < 2; ++i) {
    c->launches += S[i].launches;
    if (side[i]->clones.line_base)
      for (size_t f = 0; f < S[i].base.size(); ++f) side[i]->clones.line_base[f] = (int64_t)S[i].base[f];
    if (!rmark[i].alloc((size_t)S[i].total)) return TSM_E_CUDA;
    CU(cudaMemsetAsync(rmark[i].p, 0, (size_t)S[i].total, st));
  }
  if (n) {
    const int rc = churn_marks(c, S, pf, n, rmark, ms, st);
    if (rc != TSM_OK) return rc;
  }
  int rc_all = TSM_OK;
  for (int i = 0; i < 2; ++i) {
    if (S[i].total == 0) continue;
    tsm_clone_churn_side* o = side[i];
    const bool class_out = o->class_counts || o->status, member_out = o->changed || o->changed_assert || o->state;
    const uint8_t* mark = rmark[i].as<uint8_t>();
    auto then = [&](const CloneDev& d, cudaStream_t s2) { return churn_side(c, d, mark, i == 1, o, ms, s2); };
    float cms[3] = {0, 0, 0};
    int rc;
    if (blind)
      rc = blind_classes(c, S[i], S[i].total, (uint32_t)min_lines, &o->blind, &o->clones, cms, st, then, class_out, member_out);
    else
      rc = clone_classes<true>(c, S[i].d.line_hash, S[i].d.line_base, (uint32_t)S[i].n, (uint32_t)S[i].total, S[i].d.line_flag,
                               S[i].d.line_end, S[i].d.arena, S[i].d.off, (uint32_t)min_lines, &o->clones, cms + 1, st, then, class_out,
                               member_out);
    ms[1] += cms[0] + cms[1] + cms[2];
    if (rc == TSM_E_CAPACITY) rc_all = rc;
    else if (rc != TSM_OK) return rc;
  }
  return rc_all;
}

extern "C" int tsm_clone_churn_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_CCHURN, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 18 test smells
// The smell stage over one side whose line records (with header events) and case spans exist: the section-10 kinds
// (k_line_parens, k_stmt_kinds), k_smell_lines (with the test flag of every case), xscan of the test flags (dense test numbers;
// the test count lands at tidx[n_cases]) and k_smell_tests.  Events EV_SMELL_LINES, EV_SMELL_TESTS and EV_SMELL_END mark its
// parts.  bsum holds total / XS_TILE + 4 u64.
struct SmellBufs { DevBuf delta, kind, tflag, tidx, lines, hash, aline, smell, tests; };

static int smell_stage(tsm_ctx* c, const HostSide& S, const CaseSpans& sp, DevBuf& bsum, SmellBufs& m, int& launches, cudaStream_t st) {
  const unsigned long long total = S.total;
  const size_t L = (size_t)total;
  const uint32_t ne = sp.n_cases;
  if (!m.delta.alloc(4 * L) || !m.kind.alloc(L) || !m.tflag.alloc(4 * ((size_t)ne + 1)) || !m.tidx.alloc(8 * ((size_t)ne + 1)) ||
      !m.lines.alloc(sizeof(SmellLine) * L) || !m.hash.alloc(8 * L) || !m.aline.alloc(4 * L) || !m.smell.alloc(2 * L) ||
      !m.tests.alloc(sizeof(tsm_smell_test) * ((size_t)ne + 1)))
    return TSM_E_CUDA;
  const unsigned grid = (unsigned)((L + 255) / 256);
  CU(cudaMemsetAsync(m.smell.p, 0, 2 * L, st));
  if (L) {
    k_line_parens<<<grid, 256, 0, st>>>(S.d, S.n, total, m.delta.as<int32_t>(), m.kind.as<uint8_t>());
    k_stmt_kinds<<<(S.n * 32 + 127) / 128, 128, 0, st>>>(S.d, S.n, m.delta.as<int32_t>(), m.kind.as<uint8_t>());
  }
  CU(cudaEventRecord(c->diff_ev[EV_SMELL_LINES], st));
  if (L)
    k_smell_lines<<<grid, 256, 0, st>>>(S.d, S.n, total, sp.head.as<uint32_t>(), sp.case_of.as<unsigned long long>(), m.lines.as<SmellLine>(),
                                        m.tflag.as<uint32_t>());
  CU(cudaEventRecord(c->diff_ev[EV_SMELL_TESTS], st));
  xscan(m.tflag.as<uint32_t>(), ne, bsum.as<unsigned long long>(), m.tidx.as<unsigned long long>(), st);
  if (ne) {
    const SmellArgs a{S.d.line_base, (uint32_t)S.n, S.d.ext, m.kind.as<uint8_t>(), sp.head.as<uint32_t>(), sp.first.as<uint32_t>(), ne,
                      m.tflag.as<uint32_t>(), m.tidx.as<unsigned long long>(), m.lines.as<SmellLine>(), m.hash.as<unsigned long long>(),
                      m.aline.as<uint32_t>(), m.smell.as<uint16_t>(), m.tests.as<tsm_smell_test>()};
    k_smell_tests<<<std::min((ne + 7) / 8, (uint32_t)c->sms * 8), 256, 0, st>>>(a);
  }
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->diff_ev[EV_SMELL_END], st));
  launches += (L ? 6 : 3) + (ne ? 1 : 0);                 // parens, kinds, smell lines, xscan (3); tests
  return TSM_OK;
}

// The line records of the corpus with its header events (line_records), then the case spans and the smell stage.  One
// synchronisation at the end reads the test count; the outputs are copied when they fit.
extern "C" int tsm_smells(tsm_ctx* c, const tsm_corpus* k, int64_t* line_base, uint16_t* line_smell, int64_t line_cap, int64_t* n_lines,
                          tsm_smell_test* tests, int64_t test_cap, int64_t* n_tests, void* stream) {
  if (!c || !k || !n_lines || !n_tests || line_cap < 0 || test_cap < 0 || k->n_files < 0) return TSM_E_ARG;
  const int32_t nf = k->n_files;
  float* const ms = clear_ms(c, MS_SMELL);
  c->launches = 0;
  *n_tests = 0;
  std::vector<int64_t> own_base;
  if (!line_base) { own_base.resize((size_t)nf + 1); line_base = own_base.data(); }
  return line_records(c, k, true, line_base, INT64_MAX, n_lines, stream, [&](const HostSide& S, unsigned long long total, cudaStream_t st) -> int {
    const size_t L = (size_t)total;
    CaseSpans sp;
    SmellBufs m;
    DevBuf d_bsum;
    if (!d_bsum.alloc(8 * (L / XS_TILE + 4))) return TSM_E_CUDA;
    int launches = 0;
    CU(cudaEventRecord(c->diff_ev[EV_SMELL_KINDS], st));
    int rc = case_spans(S, sp, d_bsum, launches, st);
    if (rc == TSM_OK) rc = smell_stage(c, S, sp, d_bsum, m, launches, st);
    if (rc != TSM_OK) return rc;
    unsigned long long* pin = c->h_rb->u64;
    CU(cudaMemcpyAsync(pin, m.tidx.as<unsigned long long>() + sp.n_cases, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += launches;
    const unsigned long long nt = *pin;
    *n_tests = (int64_t)nt;
    ms[1] = elapsed_ms(c->diff_ev[EV_SMELL_KINDS], c->diff_ev[EV_SMELL_LINES]);
    ms[2] = elapsed_ms(c->diff_ev[EV_SMELL_LINES], c->diff_ev[EV_SMELL_TESTS]);
    ms[3] = elapsed_ms(c->diff_ev[EV_SMELL_TESTS], c->diff_ev[EV_SMELL_END]);
    if ((line_smell && line_cap < (int64_t)total) || (tests && test_cap < (int64_t)nt)) return TSM_E_CAPACITY;
    if (line_smell) CU(cudaMemcpyAsync(line_smell, m.smell.p, 2 * L, cudaMemcpyDeviceToHost, st));
    if (tests && nt) CU(cudaMemcpyAsync(tests, m.tests.p, sizeof(tsm_smell_test) * nt, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return TSM_OK;
  }, &ms[0], TSM_SCAN_HEADER_EVENTS);
}

extern "C" int tsm_smells_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_SMELL, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 25 lexical test smells
// The lexical stage of ns sides whose smell stage has run (nt[s] tests each): per side the line start states of the section-21
// lexer (k_blind_state, k_blind_scan), then for a side with tests k_lex_body, the count pass of k_lex_lines and an xscan of its
// name counts; one synchronisation reads the name totals of every side; then per side the write pass and k_lex_tests.  at_tests,
// when not NULL, is recorded before the k_lex_tests launches.  bsum holds total / XS_TILE + 4 u64 of the longest side; lsmell
// (every line) and lex (nt + 1 records) are the outputs.
struct LexBufs { DevBuf state, lxflag, lxend, lflag, ncnt, nbase, names, gset, lsmell, lex; };

static int lex_stage(tsm_ctx* c, const HostSide* const* S, const SmellBufs* m, const uint32_t* nt, int ns, DevBuf& bsum, LexBufs* x,
                     cudaEvent_t at_tests, int& launches, cudaStream_t st) {
  unsigned long long* const pin = c->h_rb->u64 + 2;        // the name total of each side (u64[0, 2) hold the callers' test counts)
  for (int s = 0; s < ns; ++s) {
    const HostSide& h = *S[s];
    LexBufs& b = x[s];
    const unsigned long long total = h.total;
    const size_t L = (size_t)total;
    const uint32_t nfu = (uint32_t)h.n;
    if (!b.state.alloc(L) || !b.lxflag.alloc(L) || !b.lxend.alloc(4 * L) || !b.lflag.alloc(L) || !b.ncnt.alloc(4 * L) ||
        !b.nbase.alloc(8 * (L + 1)) || !b.lsmell.alloc(L) || !b.lex.alloc(sizeof(tsm_lex_test) * ((size_t)nt[s] + 1)))
      return TSM_E_CUDA;
    const unsigned grid = (unsigned)((L + 255) / 256);
    if (L) {                                               // (a side of a revision pair may have no line)
      k_blind_state<<<grid, 256, 0, st>>>(h.d, nfu, total, b.state.as<uint8_t>());
      k_blind_scan<<<(unsigned)(((size_t)nfu * 32 + 255) / 256), 256, 0, st>>>(h.d.line_base, nfu, b.state.as<uint8_t>());
      launches += 2;
    }
    CU(cudaMemsetAsync(b.lxflag.p, 0, L, st));
    CU(cudaMemsetAsync(b.lsmell.p, 0, L, st));
    if (!nt[s]) continue;
    const unsigned tgrid = std::min((unsigned)((nt[s] + 7) / 8), (unsigned)c->sms * 8);
    k_lex_body<<<tgrid, 256, 0, st>>>(LexBody{m[s].tests.as<tsm_smell_test>(), nt[s], h.d.line_base, h.d.ext, m[s].kind.as<uint8_t>(),
                                              m[s].lines.as<SmellLine>(), b.lxflag.as<uint8_t>(), b.lxend.as<uint32_t>()});
    k_lex_lines<false><<<grid, 256, 0, st>>>(h.d, nfu, total, b.state.as<uint8_t>(), b.lxflag.as<uint8_t>(), b.lxend.as<uint32_t>(),
                                             b.lflag.as<uint8_t>(), b.ncnt.as<uint32_t>(), nullptr, nullptr);
    xscan(b.ncnt.as<uint32_t>(), (uint32_t)total, bsum.as<unsigned long long>(), b.nbase.as<unsigned long long>(), st);
    CU(cudaMemcpyAsync(pin + s, b.nbase.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
    launches += 5;                                         // body, lines, xscan (3)
  }
  CU(cudaStreamSynchronize(st));
  for (int s = 0; s < ns; ++s) {
    if (!nt[s]) continue;
    const HostSide& h = *S[s];
    LexBufs& b = x[s];
    const unsigned long long total = h.total;
    if (!b.names.alloc(8 * (size_t)pin[s]) || !b.gset.alloc(16 * (size_t)pin[s])) return TSM_E_CUDA;
    CU(cudaMemsetAsync(b.gset.p, 0xFF, 16 * (size_t)pin[s], st));
    k_lex_lines<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(h.d, (uint32_t)h.n, total, b.state.as<uint8_t>(), b.lxflag.as<uint8_t>(),
                                                                       b.lxend.as<uint32_t>(), b.lflag.as<uint8_t>(), b.ncnt.as<uint32_t>(),
                                                                       b.nbase.as<unsigned long long>(), b.names.as<unsigned long long>());
    ++launches;
  }
  if (at_tests) CU(cudaEventRecord(at_tests, st));
  for (int s = 0; s < ns; ++s) {
    if (!nt[s]) continue;
    const HostSide& h = *S[s];
    LexBufs& b = x[s];
    k_lex_tests<<<std::min((unsigned)((nt[s] + 7) / 8), (unsigned)c->sms * 8), 256, 0, st>>>(
        LexTests{m[s].tests.as<tsm_smell_test>(), nt[s], h.d.line_base, b.lflag.as<uint8_t>(), b.nbase.as<unsigned long long>(),
                 b.names.as<unsigned long long>(), b.gset.as<unsigned long long>(), b.lsmell.as<uint8_t>(), b.lex.as<tsm_lex_test>()});
    ++launches;
  }
  CU(cudaGetLastError());
  return TSM_OK;
}

// The line records with header events (line_records), the case spans and smell stage of tsm_smells, one synchronisation for the
// test count, then the lexical stage (lex_stage).  The outputs are copied when they fit.
extern "C" int tsm_smells_lexical(tsm_ctx* c, const tsm_corpus* k, int64_t* line_base, uint16_t* line_smell, uint8_t* line_lsmell,
                                  int64_t line_cap, int64_t* n_lines, tsm_smell_test* tests, tsm_lex_test* lex, int64_t test_cap,
                                  int64_t* n_tests, void* stream) {
  if (!c || !k || !n_lines || !n_tests || line_cap < 0 || test_cap < 0 || k->n_files < 0) return TSM_E_ARG;
  const int32_t nf = k->n_files;
  float* const ms = clear_ms(c, MS_LEXSMELL);
  c->launches = 0;
  *n_tests = 0;
  std::vector<int64_t> own_base;
  if (!line_base) { own_base.resize((size_t)nf + 1); line_base = own_base.data(); }
  return line_records(c, k, true, line_base, INT64_MAX, n_lines, stream, [&](const HostSide& S, unsigned long long total, cudaStream_t st) -> int {
    const size_t L = (size_t)total;
    CaseSpans sp;
    SmellBufs m;
    LexBufs x;
    DevBuf d_bsum;
    if (!d_bsum.alloc(8 * (L / XS_TILE + 4))) return TSM_E_CUDA;
    int launches = 0;
    CU(cudaEventRecord(c->diff_ev[EV_LX_FRONT], st));
    int rc = case_spans(S, sp, d_bsum, launches, st);
    if (rc == TSM_OK) rc = smell_stage(c, S, sp, d_bsum, m, launches, st);
    if (rc != TSM_OK) return rc;
    CU(cudaEventRecord(c->diff_ev[EV_LX_LINES], st));
    unsigned long long* pin = c->h_rb->u64;
    CU(cudaMemcpyAsync(pin, m.tidx.as<unsigned long long>() + sp.n_cases, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t nt = (uint32_t)*pin;
    *n_tests = (int64_t)nt;
    ms[1] = elapsed_ms(c->diff_ev[EV_LX_FRONT], c->diff_ev[EV_LX_LINES]);
    const HostSide* side = &S;
    rc = lex_stage(c, &side, &m, &nt, 1, d_bsum, &x, c->diff_ev[EV_LX_TESTS], launches, st);
    if (rc != TSM_OK) return rc;
    CU(cudaEventRecord(c->diff_ev[EV_LX_END], st));
    CU(cudaStreamSynchronize(st));
    c->launches += launches;
    ms[2] = elapsed_ms(c->diff_ev[EV_LX_LINES], c->diff_ev[EV_LX_TESTS]);
    ms[3] = elapsed_ms(c->diff_ev[EV_LX_TESTS], c->diff_ev[EV_LX_END]);
    if (((line_smell || line_lsmell) && line_cap < (int64_t)total) || ((tests || lex) && test_cap < (int64_t)nt)) return TSM_E_CAPACITY;
    if (line_smell) CU(cudaMemcpyAsync(line_smell, m.smell.p, 2 * L, cudaMemcpyDeviceToHost, st));
    if (line_lsmell) CU(cudaMemcpyAsync(line_lsmell, x.lsmell.p, L, cudaMemcpyDeviceToHost, st));
    if (tests && nt) CU(cudaMemcpyAsync(tests, m.tests.p, sizeof(tsm_smell_test) * nt, cudaMemcpyDeviceToHost, st));
    if (lex && nt) CU(cudaMemcpyAsync(lex, x.lex.p, sizeof(tsm_lex_test) * nt, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return TSM_OK;
  }, &ms[0], TSM_SCAN_HEADER_EVENTS);
}

extern "C" int tsm_smells_lexical_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_LEXSMELL, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 27 test-to-code links
// The line records with header events (line_records), the case spans and smell stage of tsm_smells and the line start states of
// the section-21 lexer; the tests of the test files (k_link_pick, xscan, k_link_gather), their code lines (k_lex_body,
// k_link_mark); one synchronisation for the test count, one for the definition and call totals, one for the link count; the
// outputs are copied when they fit.
constexpr unsigned long long kLinkMaxEntries = 1ull << 28;   // definitions or calls: 2^30 slots of the link table at most
static uint32_t link_slots(unsigned long long keys) {     // a power of two at least twice keys (and 1 024); keys <= 2^29
  unsigned long long s = 1024;
  while (s < 2 * keys) s <<= 1;
  return (uint32_t)s;
}

// One revision's link state, resident while the caller needs it: the tests of its test files (tests), the LinkDef and LinkCall
// arrays, both tables, the links with their first-call slots, and the records of tsm_test_links (out_tests, links, out_defs).
struct LinkStage {
  CaseSpans sp; SmellBufs m;
  DevBuf bsum, state, role, stem, grp, tflag, tpos, tests, lxflag, lxend, ltest, dcnt, ccnt, dbase, cbase;
  DevBuf defs, calls, name, ndefs, kmask, first, ntests, link, lcalls, lfirst, dslot, cslot, cflag, cpos, tlinks, lbase, dtests, dcalls, jbsum;
  DevBuf links, lbits, out_tests, out_defs;
  uint32_t na = 0, nt = 0, nd = 0, nc = 0, ns = 0;         // tests, link tests, definitions, calls, slots of the name table
  unsigned long long nk = 0;                               // links
};

// The link stage over one side whose line records (with header events) exist: the front (case spans, smell stage, lexer
// states, the tests of the test files and their code lines), k_link_lines, then the join to the records.  grp NULL: all 0.
// ms3 = { front, k_link_lines, join }.
static int link_stage(tsm_ctx* c, const HostSide& S, const uint8_t* role, const int32_t* stem, const uint16_t* grp, LinkStage& K,
                      float* ms3, int& launches, cudaStream_t st) {
  const unsigned long long total = S.total;
  const size_t L = (size_t)total;
  const uint32_t nfu = (uint32_t)S.n;
  const size_t nf = (size_t)S.n;
  CaseSpans& sp = K.sp;
  SmellBufs& m = K.m;
  if (!K.bsum.alloc(8 * (L / XS_TILE + 4)) || !K.state.alloc(L) || !K.role.alloc(nf) || !K.stem.alloc(4 * nf) ||
      !K.grp.alloc(2 * nf) || !K.lxflag.alloc(L) || !K.lxend.alloc(4 * L) || !K.ltest.alloc(4 * L) || !K.dcnt.alloc(4 * L) ||
      !K.ccnt.alloc(4 * L) || !K.dbase.alloc(8 * (L + 1)) || !K.cbase.alloc(8 * (L + 1)))
    return TSM_E_CUDA;
  CU(cudaMemcpyAsync(K.role.p, role, nf, cudaMemcpyHostToDevice, st));
  if (stem) CU(cudaMemcpyAsync(K.stem.p, stem, 4 * nf, cudaMemcpyHostToDevice, st));
  else CU(cudaMemsetAsync(K.stem.p, 0xFF, 4 * nf, st));
  if (grp) CU(cudaMemcpyAsync(K.grp.p, grp, 2 * nf, cudaMemcpyHostToDevice, st));
  else CU(cudaMemsetAsync(K.grp.p, 0, 2 * nf, st));
  CU(cudaEventRecord(c->diff_ev[EV_LK_FRONT], st));
  int rc = case_spans(S, sp, K.bsum, launches, st);
  if (rc == TSM_OK) rc = smell_stage(c, S, sp, K.bsum, m, launches, st);
  if (rc != TSM_OK) return rc;
  const unsigned grid = (unsigned)((L + 255) / 256);
  k_blind_state<<<grid, 256, 0, st>>>(S.d, nfu, total, K.state.as<uint8_t>());
  k_blind_scan<<<(unsigned)(((size_t)nfu * 32 + 255) / 256), 256, 0, st>>>(S.d.line_base, nfu, K.state.as<uint8_t>());
  launches += 2;
  unsigned long long* pin = c->h_rb->u64;
  CU(cudaMemcpyAsync(pin, m.tidx.as<unsigned long long>() + sp.n_cases, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const uint32_t na = (uint32_t)*pin;                      // the tests of every file
  K.na = na;
  if (!K.tflag.alloc(4 * ((size_t)na + 1)) || !K.tpos.alloc(8 * ((size_t)na + 1)) || !K.tests.alloc(sizeof(tsm_smell_test) * ((size_t)na + 1)))
    return TSM_E_CUDA;
  const unsigned agrid = (unsigned)((na + 255) / 256);
  if (na) k_link_pick<<<agrid, 256, 0, st>>>(m.tests.as<tsm_smell_test>(), na, K.role.as<uint8_t>(), K.tflag.as<uint32_t>());
  xscan(K.tflag.as<uint32_t>(), na, K.bsum.as<unsigned long long>(), K.tpos.as<unsigned long long>(), st);
  if (na) k_link_gather<<<agrid, 256, 0, st>>>(m.tests.as<tsm_smell_test>(), na, K.tflag.as<uint32_t>(), K.tpos.as<unsigned long long>(),
                                               K.tests.as<tsm_smell_test>());
  CU(cudaMemcpyAsync(pin, K.tpos.as<unsigned long long>() + na, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemsetAsync(K.lxflag.p, 0, L, st));
  CU(cudaMemsetAsync(K.ltest.p, 0xFF, 4 * L, st));
  CU(cudaStreamSynchronize(st));
  const uint32_t nt = (uint32_t)*pin;                      // the tests of the test files
  K.nt = nt;
  launches += na ? 5 : 3;
  const tsm_smell_test* dt = K.tests.as<tsm_smell_test>();
  const unsigned tgrid = std::min((unsigned)((nt + 7) / 8), (unsigned)c->sms * 8);
  if (nt) {
    k_lex_body<<<tgrid, 256, 0, st>>>(LexBody{dt, nt, S.d.line_base, S.d.ext, m.kind.as<uint8_t>(), m.lines.as<SmellLine>(),
                                              K.lxflag.as<uint8_t>(), K.lxend.as<uint32_t>()});
    k_link_mark<<<tgrid, 256, 0, st>>>(dt, nt, S.d.line_base, K.lxflag.as<uint8_t>(), K.ltest.as<uint32_t>());
    launches += 2;
  }
  CU(cudaEventRecord(c->diff_ev[EV_LK_LINES], st));
  k_link_lines<false><<<grid, 256, 0, st>>>(S.d, nfu, total, K.state.as<uint8_t>(), K.role.as<uint8_t>(), K.ltest.as<uint32_t>(),
                                            K.dcnt.as<uint32_t>(), K.ccnt.as<uint32_t>(), nullptr, nullptr, nullptr, nullptr);
  xscan(K.dcnt.as<uint32_t>(), (uint32_t)total, K.bsum.as<unsigned long long>(), K.dbase.as<unsigned long long>(), st);
  xscan(K.ccnt.as<uint32_t>(), (uint32_t)total, K.bsum.as<unsigned long long>(), K.cbase.as<unsigned long long>(), st);
  CU(cudaMemcpyAsync(pin, K.dbase.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(pin + 1, K.cbase.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const unsigned long long nd64 = pin[0], nc64 = pin[1];
  if (nd64 > kLinkMaxEntries || nc64 > kLinkMaxEntries) return TSM_E_NOMEM;   // (tables of more than 16 GiB)
  const uint32_t nd = (uint32_t)nd64, nc = (uint32_t)nc64;
  const uint32_t ns = link_slots(2ull * nd), nl = link_slots(2ull * nc);
  K.nd = nd; K.nc = nc; K.ns = ns;
  if (!K.jbsum.alloc(8 * ((size_t)std::max(nc, nt) / XS_TILE + 4)) || !K.defs.alloc(sizeof(LinkDef) * ((size_t)nd + 1)) || !K.calls.alloc(sizeof(LinkCall) * ((size_t)nc + 1)) ||
      !K.name.alloc(16 * (size_t)ns) || !K.ndefs.alloc(4 * (size_t)ns) || !K.kmask.alloc(4 * (size_t)ns) || !K.first.alloc(4 * (size_t)ns) ||
      !K.ntests.alloc(4 * (size_t)ns) || !K.link.alloc(16 * (size_t)nl) || !K.lcalls.alloc(4 * (size_t)nl) ||
      !K.lfirst.alloc(4 * (size_t)nl) || !K.dslot.alloc(4 * ((size_t)nd + 1)) || !K.cslot.alloc(4 * ((size_t)nc + 1)) ||
      !K.cflag.alloc(4 * ((size_t)nc + 1)) || !K.cpos.alloc(8 * ((size_t)nc + 1)) || !K.tlinks.alloc(4 * ((size_t)nt + 1)) ||
      !K.lbase.alloc(8 * ((size_t)nt + 1)) || !K.dtests.alloc(4 * ((size_t)nd + 1)) || !K.dcalls.alloc(4 * ((size_t)nd + 1)))
    return TSM_E_CUDA;
  k_link_lines<true><<<grid, 256, 0, st>>>(S.d, nfu, total, K.state.as<uint8_t>(), K.role.as<uint8_t>(), K.ltest.as<uint32_t>(),
                                           K.dcnt.as<uint32_t>(), K.ccnt.as<uint32_t>(), K.dbase.as<unsigned long long>(),
                                           K.cbase.as<unsigned long long>(), K.defs.as<LinkDef>(), K.calls.as<LinkCall>());
  launches += 8;                                           // lines (count), two xscans (3 each), lines (write)
  CU(cudaEventRecord(c->diff_ev[EV_LK_JOIN], st));
  CU(cudaMemsetAsync(K.name.p, 0, 16 * (size_t)ns, st));
  CU(cudaMemsetAsync(K.ndefs.p, 0, 4 * (size_t)ns, st));
  CU(cudaMemsetAsync(K.kmask.p, 0, 4 * (size_t)ns, st));
  CU(cudaMemsetAsync(K.first.p, 0xFF, 4 * (size_t)ns, st));
  CU(cudaMemsetAsync(K.ntests.p, 0, 4 * (size_t)ns, st));
  CU(cudaMemsetAsync(K.link.p, 0, 16 * (size_t)nl, st));
  CU(cudaMemsetAsync(K.lcalls.p, 0, 4 * (size_t)nl, st));
  CU(cudaMemsetAsync(K.lfirst.p, 0xFF, 4 * (size_t)nl, st));
  CU(cudaMemsetAsync(K.tlinks.p, 0, 4 * ((size_t)nt + 1), st));
  CU(cudaMemsetAsync(K.dtests.p, 0, 4 * ((size_t)nd + 1), st));
  CU(cudaMemsetAsync(K.dcalls.p, 0, 4 * ((size_t)nd + 1), st));
  const LinkTables T{K.name.as<LinkKey>(), ns - 1, K.ndefs.as<uint32_t>(), K.kmask.as<uint32_t>(), K.first.as<uint32_t>(),
                     K.ntests.as<uint32_t>(), K.link.as<LinkKey>(), nl - 1, K.lcalls.as<uint32_t>(), K.lfirst.as<uint32_t>()};
  const unsigned dgrid = (unsigned)((nd + 255) / 256), cgrid = (unsigned)((nc + 255) / 256);
  if (nd) k_link_defs<<<dgrid, 256, 0, st>>>(K.defs.as<LinkDef>(), nd, K.grp.as<uint16_t>(), K.stem.as<int32_t>(), T, K.dslot.as<uint32_t>());
  if (nc) {
    k_link_calls<<<cgrid, 256, 0, st>>>(K.calls.as<LinkCall>(), nc, K.ltest.as<uint32_t>(), dt, K.grp.as<uint16_t>(), T,
                                        K.cslot.as<uint32_t>(), K.tlinks.as<uint32_t>());
    k_link_first<<<cgrid, 256, 0, st>>>(K.cslot.as<uint32_t>(), nc, T, K.cflag.as<uint32_t>());
  }
  xscan(K.cflag.as<uint32_t>(), nc, K.jbsum.as<unsigned long long>(), K.cpos.as<unsigned long long>(), st);   // (nc may exceed the
  xscan(K.tlinks.as<uint32_t>(), nt, K.jbsum.as<unsigned long long>(), K.lbase.as<unsigned long long>(), st); //  lines: own sums)
  CU(cudaMemcpyAsync(pin, K.cpos.as<unsigned long long>() + nc, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const unsigned long long nk = *pin;                      // the links
  K.nk = nk;
  if (!K.links.alloc(sizeof(tsm_link) * ((size_t)nk + 1)) || !K.lbits.alloc((size_t)nk + 1) ||
      !K.out_tests.alloc(sizeof(tsm_link_test) * ((size_t)nt + 1)) || !K.out_defs.alloc(sizeof(tsm_link_def) * ((size_t)nd + 1)))
    return TSM_E_CUDA;
  if (nc)
    k_link_emit<<<cgrid, 256, 0, st>>>(LinkEmit{K.calls.as<LinkCall>(), nc, K.cslot.as<uint32_t>(), K.cflag.as<uint32_t>(),
                                                K.cpos.as<unsigned long long>(), K.ltest.as<uint32_t>(), dt, K.grp.as<uint16_t>(),
                                                K.stem.as<int32_t>(), S.d.line_base, K.defs.as<LinkDef>(), T, K.links.as<tsm_link>(),
                                                K.lbits.as<uint8_t>(), K.dtests.as<uint32_t>(), K.dcalls.as<uint32_t>()});
  if (nt)
    k_link_tests<<<tgrid, 256, 0, st>>>(LinkTests{dt, nt, S.d.line_base, K.cbase.as<unsigned long long>(), K.lbase.as<unsigned long long>(),
                                                  K.links.as<tsm_link>(), K.lbits.as<uint8_t>(), K.out_tests.as<tsm_link_test>()});
  if (nd) k_link_out<<<dgrid, 256, 0, st>>>(K.defs.as<LinkDef>(), nd, K.dslot.as<uint32_t>(), S.d.line_base, T, K.dtests.as<uint32_t>(),
                                            K.dcalls.as<uint32_t>(), K.out_defs.as<tsm_link_def>());
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->diff_ev[EV_LK_END], st));
  CU(cudaStreamSynchronize(st));
  launches += (nd ? 2 : 0) + (nc ? 3 : 0) + 6 + (nt ? 1 : 0);   // defs + out, calls + first + emit, two xscans, tests
  ms3[0] = elapsed_ms(c->diff_ev[EV_LK_FRONT], c->diff_ev[EV_LK_LINES]);
  ms3[1] = elapsed_ms(c->diff_ev[EV_LK_LINES], c->diff_ev[EV_LK_JOIN]);
  ms3[2] = elapsed_ms(c->diff_ev[EV_LK_JOIN], c->diff_ev[EV_LK_END]);
  return TSM_OK;
}

// The records of a link stage into out, when they fit (TSM_E_CAPACITY otherwise); the counts are always set.
static int link_copy(const LinkStage& K, tsm_links_result* out, cudaStream_t st) {
  const uint32_t nt = K.nt, nd = K.nd;
  const unsigned long long nk = K.nk;
  out->n_tests = nt; out->n_links = (int64_t)nk; out->n_defs = nd;
  if ((out->tests && out->test_cap < (int64_t)nt) || (out->links && out->link_cap < (int64_t)nk) || (out->defs && out->def_cap < (int64_t)nd))
    return TSM_E_CAPACITY;
  if (out->tests && nt) CU(cudaMemcpyAsync(out->tests, K.out_tests.p, sizeof(tsm_link_test) * nt, cudaMemcpyDeviceToHost, st));
  if (out->links && nk) CU(cudaMemcpyAsync(out->links, K.links.p, sizeof(tsm_link) * nk, cudaMemcpyDeviceToHost, st));
  if (out->defs && nd) CU(cudaMemcpyAsync(out->defs, K.out_defs.p, sizeof(tsm_link_def) * nd, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TSM_OK;
}

extern "C" int tsm_test_links(tsm_ctx* c, const tsm_corpus* k, const uint8_t* role, const int32_t* stem, tsm_links_result* out,
                              void* stream) {
  if (!c || !k || !role || !out || k->n_files < 0 || out->test_cap < 0 || out->link_cap < 0 || out->def_cap < 0) return TSM_E_ARG;
  const int32_t nf = k->n_files;
  for (int32_t f = 0; stem && f < nf; ++f)
    if (stem[f] < -1) return TSM_E_ARG;
  if (check_groups(k, 0, nf) != TSM_OK) return TSM_E_LAYOUT;
  float* const ms = clear_ms(c, MS_LINKS);
  c->launches = 0;
  out->n_tests = out->n_links = out->n_defs = 0;
  std::vector<int64_t> base((size_t)nf + 1);
  int64_t n_lines = 0;
  return line_records(c, k, true, base.data(), INT64_MAX, &n_lines, stream, [&](const HostSide& S, unsigned long long, cudaStream_t st) -> int {
    LinkStage K;
    int launches = 0;
    const int rc = link_stage(c, S, role, stem, k->grp, K, &ms[1], launches, st);
    if (rc != TSM_OK) return rc;
    c->launches += launches;
    return link_copy(K, out, st);
  }, &ms[0], TSM_SCAN_HEADER_EVENTS);
}

extern "C" int tsm_test_links_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_LINKS, ms4, 4); }

// The naming convention of section 27: the one place it lives (the CLI and the Python package call it).
extern "C" int tsm_focal_stems(const char* const* paths, const uint8_t* role, int32_t n, int32_t* stem) {
  if (n < 0 || (n && (!paths || !role || !stem))) return TSM_E_ARG;
  std::unordered_map<std::string, int32_t> ids;
  for (int32_t i = 0; i < n; ++i) {
    if (!paths[i]) return TSM_E_ARG;
    std::string b = paths[i];
    const size_t sl = b.find_last_of('/');
    if (sl != std::string::npos) b = b.substr(sl + 1);
    const size_t dot = b.find_last_of('.');
    if (dot != std::string::npos && dot > 0) b.resize(dot);
    if (role[i]) {
      static const char* const suffixes[] = {"_test", "_tests", "_unittest", "Test", "Tests"};
      static const char* const prefixes[] = {"test_", "test"};
      bool cut = false;
      for (const char* x : suffixes) {
        const size_t m = strlen(x);
        if (b.size() >= m && b.compare(b.size() - m, m, x) == 0) { b.resize(b.size() - m); cut = true; break; }
      }
      for (size_t p = 0; !cut && p < 2; ++p) {
        const size_t m = strlen(prefixes[p]);
        if (b.compare(0, m, prefixes[p]) == 0) { b = b.substr(m); cut = true; }
      }
      if (b.empty()) { stem[i] = -1; continue; }
    }
    stem[i] = ids.emplace(b, (int32_t)ids.size()).first->second;
  }
  return TSM_OK;
}

// ------------------------------------------------------------------------------------- SPEC section 23 similar tests
// One revision's section-23 state on the device, resident while the call needs it: the front (case spans, smell stage and
// blind_front; nt tests, nk kept lines) and the tokens, prefixes and posting lists of its compared tests.
struct StSide {
  CaseSpans sp; SmellBufs m; BlindFront bf; DevBuf bsum;
  DevBuf kbeg, kk, q, ktest, ctr, key, cnt, eord, pbase, tbsum, pkey, pcnt, tok, ptest, mbase, cursor, mem, cbase, cbsum, surv, pairs;
  unsigned long long nt = 0, nk = 0;
  uint32_t nl = 0, nb = 0;
  StEnum enum_args(uint32_t P) const {
    return StEnum{cbase.as<unsigned long long>(), nl, mbase.as<unsigned long long>(), mem.as<uint32_t>(), kk.as<uint32_t>(),
                  q.as<uint32_t>(), pbase.as<unsigned long long>(), tok.as<StToken>(), P, surv.as<uint2>(), ctr.as<uint32_t>() + 1};
  }
};

// The front of one side whose line records (with header events) exist: the case spans and smell stage of tsm_smells and
// blind_front, then one synchronisation for the test and kept counts.  ms[1] = its device time.
static int st_front(tsm_ctx* c, const HostSide& S, StSide& f, float* ms, cudaStream_t st) {
  const size_t L = (size_t)S.total;
  if (!f.bsum.alloc(8 * (L / XS_TILE + 4))) return TSM_E_CUDA;
  int launches = 0;
  CU(cudaEventRecord(c->diff_ev[EV_ST_FRONT], st));
  int rc = case_spans(S, f.sp, f.bsum, launches, st);
  if (rc == TSM_OK) rc = smell_stage(c, S, f.sp, f.bsum, f.m, launches, st);
  if (rc == TSM_OK) rc = blind_front(c, S, f.bf, st);
  if (rc != TSM_OK) return rc;
  CU(cudaEventRecord(c->diff_ev[EV_ST_LEXED], st));
  unsigned long long* pin = c->h_rb->u64;
  CU(cudaMemcpyAsync(pin, f.m.tidx.as<unsigned long long>() + f.sp.n_cases, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(pin + 1, f.bf.rank.as<unsigned long long>() + L, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  c->launches += launches;
  f.nt = pin[0];
  f.nk = pin[1];
  ms[1] += elapsed_ms(c->diff_ev[EV_ST_FRONT], c->diff_ev[EV_ST_LEXED]);
  return TSM_OK;
}

// The tokens of a side with nt > 0 behind st_front: k_st_tests (kbeg, kk, q, ktest; kmax at ctr[0]), the count table, the
// prefix tokens (k_st_prefix) and the scan of the lists' lengths into mbase.  Queued only: the posting lists come next.
static int st_tokens(const HostSide& S, StSide& f, uint32_t min_lines, uint32_t P, cudaStream_t st) {
  const unsigned long long nt = f.nt, nk = f.nk;
  if (nk >= (1ull << 30)) return TSM_E_NOMEM;              // the token tables are indexed by u32 with a spare slot
  const size_t NT = (size_t)nt, NK = (size_t)nk;
  size_t slots = 1;                                        // a power of two, at least 2 x the kept lines
  while (slots < 2 * NK) slots <<= 1;
  const uint32_t mask = (uint32_t)(slots - 1), nl = (uint32_t)slots + 1;   // + the slot of key ST_EMPTY
  f.nl = nl;
  f.nb = (nl + XS_TILE - 1) / XS_TILE;
  if (!f.kbeg.alloc(4 * NT) || !f.kk.alloc(4 * NT) || !f.q.alloc(4 * NT) || !f.ktest.alloc(4 * NK) || !f.ctr.alloc(16) ||
      !f.key.alloc(8 * (size_t)nl) || !f.cnt.alloc(4 * (size_t)nl) || !f.eord.alloc(8 * NK) || !f.pbase.alloc(8 * (NT + 1)) ||
      !f.tbsum.alloc(8 * (NT / XS_TILE + 4)) || !f.pkey.alloc(8 * (size_t)nl) || !f.pcnt.alloc(4 * (size_t)nl) ||
      !f.tok.alloc(sizeof(StToken) * NK) || !f.ptest.alloc(4 * NK) || !f.mbase.alloc(8 * ((size_t)nl + 1)) ||
      !f.cursor.alloc(4 * (size_t)nl) || !f.mem.alloc(4 * NK) || !f.cbase.alloc(8 * ((size_t)nl + 1)) ||
      !f.cbsum.alloc(8 * ((size_t)f.nb + 4)) || !f.surv.alloc(sizeof(uint2) * ST_CHUNK) || !f.pairs.alloc(sizeof(tsm_similar_pair) * ST_CHUNK)) {
    cudaGetLastError();
    return TSM_E_NOMEM;
  }
  uint32_t* ctr = f.ctr.as<uint32_t>();                   // kmax, survivors, pairs
  const uint32_t* ktest = f.ktest.as<uint32_t>();
  const unsigned long long* khash = f.bf.khash.as<unsigned long long>();
  CU(cudaMemsetAsync(f.ktest.p, 0xFF, 4 * NK, st));
  CU(cudaMemsetAsync(f.ctr.p, 0, 16, st));
  CU(cudaMemsetAsync(f.key.p, 0xFF, 8 * (size_t)nl, st));
  CU(cudaMemsetAsync(f.cnt.p, 0, 4 * (size_t)nl, st));
  CU(cudaMemsetAsync(f.pkey.p, 0xFF, 8 * (size_t)nl, st));
  CU(cudaMemsetAsync(f.pcnt.p, 0, 4 * (size_t)nl, st));
  CU(cudaMemsetAsync(f.cursor.p, 0, 4 * (size_t)nl, st));
  const unsigned kgrid = (unsigned)((NK + 255) / 256);
  k_st_tests<<<(unsigned)((NT + 255) / 256), 256, 0, st>>>(f.m.tests.as<tsm_smell_test>(), (uint32_t)nt, S.d.line_base,
                                                           f.bf.rank.as<unsigned long long>(), min_lines, P, f.kbeg.as<uint32_t>(),
                                                           f.kk.as<uint32_t>(), f.q.as<uint32_t>(), f.ktest.as<uint32_t>(), ctr);
  if (NK) {
    k_st_count<<<kgrid, 256, 0, st>>>(khash, ktest, (uint32_t)nk, f.key.as<unsigned long long>(), mask, f.cnt.as<uint32_t>(), f.eord.as<uint2>());
    k_st_order<<<kgrid, 256, 0, st>>>(ktest, (uint32_t)nk, f.cnt.as<uint32_t>(), f.eord.as<uint2>());
  }
  xscan(f.q.as<uint32_t>(), (uint32_t)nt, f.tbsum.as<unsigned long long>(), f.pbase.as<unsigned long long>(), st);
  if (NK)
    k_st_prefix<<<kgrid, 256, 0, st>>>(ktest, (uint32_t)nk, f.eord.as<uint2>(), f.kbeg.as<uint32_t>(), f.kk.as<uint32_t>(), f.q.as<uint32_t>(),
                                       f.pbase.as<unsigned long long>(), f.pkey.as<unsigned long long>(), mask, f.pcnt.as<uint32_t>(),
                                       f.tok.as<StToken>(), f.ptest.as<uint32_t>());
  xscan(f.pcnt.as<uint32_t>(), nl, f.cbsum.as<unsigned long long>(), f.mbase.as<unsigned long long>(), st);
  CU(cudaGetLastError());
  return TSM_OK;
}

// The warps and scratch of k_st_verify for patterns of up to kmax kept lines: V of a pattern of more than 2048 kept lines
// lives in a scratch slot of each warp, within 1 GiB.
struct StVerifyShape { uint32_t slot_words; unsigned blocks; };
static int st_verify_shape(const tsm_ctx* c, uint32_t kmax, DevBuf& scratch, StVerifyShape& v) {
  const uint32_t W = (kmax + 63) / 64, nbk = (W + 31) / 32;
  v.slot_words = nbk > 1 ? nbk * 32 : 0;
  v.blocks = (unsigned)c->sms * 4;
  if (v.slot_words) {
    v.blocks = (unsigned)std::max<size_t>(1, std::min<size_t>(v.blocks, ((size_t)1 << 27) / ((size_t)v.slot_words * 8)));
    if (!scratch.alloc(8 * (size_t)v.slot_words * v.blocks * 8)) { cudaGetLastError(); return TSM_E_NOMEM; }
  }
  return TSM_OK;
}

// Behind the posting lists and the scan of their candidate counts into cbase (queued by the caller): one synchronisation
// for the candidate total and kmax, then per chunk of ST_CHUNK virtual candidates the enumeration (enumerate(c0, n, st)
// queues it) and k_st_verify, and one synchronisation that copies the chunk's pairs out.  ms[2] += lists + enumeration,
// ms[3] += verification.
template <typename Enumerate>
static int st_verify_all(tsm_ctx* c, StSide& f, uint32_t P, Enumerate enumerate, std::vector<tsm_similar_pair>& pairs,
                         int64_t* n_candidates, float* ms, cudaStream_t st) {
  unsigned long long* pin = c->h_rb->u64;
  uint32_t* ctr = f.ctr.as<uint32_t>();
  pin[3] = 0;
  CU(cudaMemcpyAsync(pin + 2, f.cbase.as<unsigned long long>() + f.nl, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(pin + 3, ctr, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const unsigned long long n_virtual = pin[2];
  const uint32_t kmax = (uint32_t)pin[3];
  ms[2] += elapsed_ms(c->diff_ev[EV_ST_LEXED], c->diff_ev[EV_ST_LISTS]);
  DevBuf d_scratch;
  StVerifyShape vs;
  const int rc = st_verify_shape(c, kmax, d_scratch, vs);
  if (rc != TSM_OK) return rc;
  int64_t ncand = 0;
  uint32_t* cnt2 = reinterpret_cast<uint32_t*>(pin + 2);
  for (unsigned long long c0 = 0; c0 < n_virtual; c0 += ST_CHUNK) {
    const unsigned long long n = std::min<unsigned long long>(ST_CHUNK, n_virtual - c0);
    CU(cudaMemsetAsync(ctr + 1, 0, 8, st));
    CU(cudaEventRecord(c->diff_ev[EV_ST_ENUM], st));
    enumerate(c0, n, st);
    CU(cudaEventRecord(c->diff_ev[EV_ST_VERIFY], st));
    k_st_verify<<<vs.blocks, 256, 0, st>>>(f.surv.as<uint2>(), ctr + 1, f.kbeg.as<uint32_t>(), f.kk.as<uint32_t>(),
                                           f.bf.khash.as<unsigned long long>(), P,
                                           vs.slot_words ? d_scratch.as<unsigned long long>() : nullptr, vs.slot_words,
                                           f.pairs.as<tsm_similar_pair>(), ctr + 2);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_ST_END], st));
    CU(cudaMemcpyAsync(cnt2, ctr + 1, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += 2;
    ncand += cnt2[0];
    const uint32_t np = cnt2[1];
    ms[2] += elapsed_ms(c->diff_ev[EV_ST_ENUM], c->diff_ev[EV_ST_VERIFY]);
    ms[3] += elapsed_ms(c->diff_ev[EV_ST_VERIFY], c->diff_ev[EV_ST_END]);
    if (np) {
      const size_t had = pairs.size();
      pairs.resize(had + np);
      CU(cudaMemcpyAsync(pairs.data() + had, f.pairs.p, sizeof(tsm_similar_pair) * np, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
    }
  }
  *n_candidates = ncand;
  return TSM_OK;
}

// The tests and their kept blind lines of one side whose line records (with header events) exist: st_front; the prefix
// tokens, their posting lists and the scan of the lists' candidate counts; then st_verify_all over every pair of each list.
// tests / kept / pairs: host copies of the tests, their kept lines and the pairs (unordered).  ms[1..3] as
// tsm_similar_tests_last_ms.
static int similar_pairs(tsm_ctx* c, const HostSide& S, uint32_t min_lines, uint32_t P, std::vector<tsm_smell_test>& tests,
                         std::vector<uint32_t>& kept, std::vector<tsm_similar_pair>& pairs, int64_t* n_candidates, float* ms,
                         cudaStream_t st) {
  StSide f;
  int rc = st_front(c, S, f, ms, st);
  if (rc != TSM_OK) return rc;
  const size_t NT = (size_t)f.nt, NK = (size_t)f.nk;
  tests.resize(NT);
  kept.resize(NT);
  if (NT == 0) return TSM_OK;
  rc = st_tokens(S, f, min_lines, P, st);
  if (rc != TSM_OK) return rc;
  const unsigned kgrid = (unsigned)((NK + 255) / 256);
  if (NK)
    k_st_lists<<<kgrid, 256, 0, st>>>(f.tok.as<StToken>(), f.ptest.as<uint32_t>(), f.pbase.as<unsigned long long>() + NT,
                                      f.mbase.as<unsigned long long>(), f.cursor.as<uint32_t>(), f.mem.as<uint32_t>());
  k_st_csums<<<f.nb, 256, 0, st>>>(f.pcnt.as<uint32_t>(), f.nl, f.cbsum.as<unsigned long long>());
  k_xscan_top<<<1, 256, 0, st>>>(f.cbsum.as<unsigned long long>(), f.nb);
  k_st_capply<<<f.nb, 256, 0, st>>>(f.pcnt.as<uint32_t>(), f.nl, f.cbsum.as<unsigned long long>(), f.cbase.as<unsigned long long>());
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->diff_ev[EV_ST_LISTS], st));
  c->launches += 10 + (NK ? 4 : 0);                       // tests, 2 x xscan (3 each), the candidate scan (3); count, order, prefix, lists
  const StEnum ea = f.enum_args(P);
  rc = st_verify_all(c, f, P, [&](unsigned long long c0, unsigned long long n, cudaStream_t s2) {
    k_st_enum<<<(unsigned)std::min<unsigned long long>((n + 255) / 256, (unsigned long long)c->sms * 16), 256, 0, s2>>>(ea, c0, n);
  }, pairs, n_candidates, ms, st);
  if (rc != TSM_OK) return rc;
  CU(cudaMemcpyAsync(tests.data(), f.m.tests.p, sizeof(tsm_smell_test) * NT, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(kept.data(), f.kk.p, 4 * NT, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TSM_OK;
}

// The line records of the corpus with its header events (line_records), then similar_pairs; on the host the pairs are sorted
// and the classes formed by a union-find whose roots are the smallest tests of their components.
extern "C" int tsm_similar_tests(tsm_ctx* c, const tsm_corpus* k, int32_t min_lines, int32_t min_similarity, tsm_similar_result* out,
                                 void* stream) {
  if (!c || !k || !out || k->n_files < 0 || min_lines < 1 || min_similarity < 1 || min_similarity > 100 || out->test_cap < 0 ||
      out->pair_cap < 0 || out->class_cap < 0 || out->member_cap < 0)
    return TSM_E_ARG;
  float* const ms = clear_ms(c, MS_SIMTEST);
  c->launches = 0;
  out->n_tests = out->n_pairs = out->n_classes = out->n_members = out->n_candidates = 0;
  if (out->class_base) out->class_base[0] = 0;
  std::vector<int64_t> line_base((size_t)k->n_files + 1);
  std::vector<tsm_smell_test> tests;
  std::vector<uint32_t> kept;
  std::vector<tsm_similar_pair> pairs;
  int64_t n_lines = 0, n_candidates = 0;
  int rc = line_records(c, k, true, line_base.data(), INT64_MAX, &n_lines, stream, [&](const HostSide& S, unsigned long long, cudaStream_t st) -> int {
    return similar_pairs(c, S, (uint32_t)min_lines, (uint32_t)min_similarity, tests, kept, pairs, &n_candidates, ms, st);
  }, &ms[0], TSM_SCAN_HEADER_EVENTS);
  if (rc != TSM_OK) return rc;
  std::sort(pairs.begin(), pairs.end(), [](const tsm_similar_pair& x, const tsm_similar_pair& y) { return x.a != y.a ? x.a < y.a : x.b < y.b; });
  const size_t nt = tests.size();
  std::vector<int32_t> root(nt);
  std::vector<uint8_t> linked(nt, 0);
  for (size_t t = 0; t < nt; ++t) root[t] = (int32_t)t;
  auto find = [&](int32_t x) { while (root[(size_t)x] != x) x = root[(size_t)x] = root[(size_t)root[(size_t)x]]; return x; };
  for (const tsm_similar_pair& p : pairs) {
    const int32_t ra = find(p.a), rb = find(p.b);
    if (ra != rb) root[(size_t)std::max(ra, rb)] = std::min(ra, rb);
    linked[(size_t)p.a] = linked[(size_t)p.b] = 1;
  }
  std::vector<int64_t> class_of(nt, -1), base(1, 0);      // classes in order of their roots, the smallest members
  for (size_t t = 0; t < nt; ++t)
    if (linked[t] && find((int32_t)t) == (int32_t)t) { class_of[t] = (int64_t)base.size() - 1; base.push_back(0); }
  for (size_t t = 0; t < nt; ++t) if (linked[t]) ++base[(size_t)class_of[(size_t)find((int32_t)t)] + 1];
  for (size_t i = 1; i < base.size(); ++i) base[i] += base[i - 1];
  const int64_t nc = (int64_t)base.size() - 1, nm = base.back();
  out->n_tests = (int64_t)nt;
  out->n_pairs = (int64_t)pairs.size();
  out->n_classes = nc;
  out->n_members = nm;
  out->n_candidates = n_candidates;
  if (((out->tests || out->test_kept) && out->test_cap < (int64_t)nt) || (out->pairs && out->pair_cap < out->n_pairs) ||
      (out->class_base && out->class_cap < nc) || (out->member && out->member_cap < nm))
    return TSM_E_CAPACITY;
  if (out->tests) std::copy(tests.begin(), tests.end(), out->tests);
  if (out->test_kept) std::copy(kept.begin(), kept.end(), out->test_kept);
  if (out->pairs) std::copy(pairs.begin(), pairs.end(), out->pairs);
  if (out->class_base) std::copy(base.begin(), base.end(), out->class_base);
  if (out->member) {
    std::vector<int64_t> cur(base.begin(), base.end() - 1);
    for (size_t t = 0; t < nt; ++t) if (linked[t]) out->member[cur[(size_t)class_of[(size_t)find((int32_t)t)]]++] = (int32_t)t;
  }
  return TSM_OK;
}

extern "C" int tsm_similar_tests_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_SIMTEST, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 24 similar-test churn
namespace {
// The host view of one revision behind its front: its tests, the header line of each case, its marks and its files.
struct ScRev {
  const tsm_corpus* k = nullptr;
  std::vector<unsigned long long> base;                    // line_base
  std::vector<tsm_smell_test> tests;
  std::vector<uint32_t> head, kept;                        // the header line (global) of every case; kept lines per test
  std::vector<uint8_t> mark;
  std::vector<size_t> tfile, cfile;                        // first test / case of every file [n_files + 1]
  std::vector<int32_t> match;
  std::vector<uint8_t> change;
  void index() {
    const size_t nf = (size_t)k->n_files;
    tfile.assign(nf + 1, 0);
    cfile.assign(nf + 1, 0);
    for (const tsm_smell_test& t : tests) ++tfile[(size_t)t.file + 1];
    for (uint32_t h : head) ++cfile[(size_t)(std::upper_bound(base.begin(), base.end(), (unsigned long long)h) - base.begin())];
    for (size_t f = 0; f < nf; ++f) { tfile[f + 1] += tfile[f]; cfile[f + 1] += cfile[f]; }
  }
  // The case names (section 10) of the cases of file f.
  std::vector<std::string> names(int32_t f) const {
    std::vector<std::string> out;
    const uint8_t* p = k->arena + k->off[f];
    const int32_t size = k->len[f];
    int32_t line = 0, pos = 0;
    for (size_t c = cfile[(size_t)f]; c < cfile[(size_t)f + 1]; ++c) {
      for (const int32_t h = (int32_t)(head[c] - base[(size_t)f]); line < h; ++line)
        pos = (int32_t)((const uint8_t*)memchr(p + pos, '\n', (size_t)(size - pos)) - p) + 1;
      const uint8_t* lf = (const uint8_t*)memchr(p + pos, '\n', (size_t)(size - pos));
      out.push_back(tsm_names::case_name(k->ext ? k->ext[f] : 0, p + pos, (uint32_t)((lf ? (int32_t)(lf - p) : size) - pos)));
    }
    return out;
  }
};

// Section 24's test identity within the changed pair (fo, fn): the section-16 matching of their cases (step 1 through the
// kept-line correspondence of the marks, step 2 by tsm_names::match_by_name), then matched cases that are tests on both
// sides.  Appends (old test, new test) to `both`.
void sc_match_pair(ScRev& O, ScRev& N, int32_t fo, int32_t fn, std::vector<uint2>& both) {
  const size_t co = O.cfile[(size_t)fo], no = O.cfile[(size_t)fo + 1] - co, cn = N.cfile[(size_t)fn], nn = N.cfile[(size_t)fn + 1] - cn;
  const unsigned long long bo = O.base[(size_t)fo], bn = N.base[(size_t)fn];
  std::vector<uint32_t> okept;                             // the kept old lines, in order (local)
  for (unsigned long long l = bo; l < O.base[(size_t)fo + 1]; ++l) if (!O.mark[l]) okept.push_back((uint32_t)(l - bo));
  std::unordered_map<uint32_t, int64_t> old_case;          // local header line -> old case (within the file)
  for (size_t k = 0; k < no; ++k) old_case[(uint32_t)(O.head[co + k] - bo)] = (int64_t)k;
  std::vector<int64_t> match(nn, -1);
  std::vector<char> used(no, 0);
  size_t r = 0, j = 0;
  for (unsigned long long l = bn; l < N.base[(size_t)fn + 1] && j < nn; ++l) {
    if (N.head[cn + j] == l) {
      if (!N.mark[l] && r < okept.size()) {
        const auto it = old_case.find(okept[r]);
        if (it != old_case.end()) { match[j] = it->second; used[(size_t)it->second] = 1; }
      }
      ++j;
    }
    r += !N.mark[l];
  }
  if (std::find(match.begin(), match.end(), -1) != match.end() && std::find(used.begin(), used.end(), 0) != used.end())
    tsm_names::match_by_name(O.names(fo), N.names(fn), match, used);
  std::unordered_map<uint32_t, size_t> old_test;           // local header line -> old test
  for (size_t t = O.tfile[(size_t)fo]; t < O.tfile[(size_t)fo + 1]; ++t) old_test[(uint32_t)O.tests[t].line] = t;
  std::unordered_map<uint32_t, size_t> new_case;
  for (size_t k = 0; k < nn; ++k) new_case[(uint32_t)(N.head[cn + k] - bn)] = k;
  for (size_t t = N.tfile[(size_t)fn]; t < N.tfile[(size_t)fn + 1]; ++t) {
    const int64_t k = match[new_case.at((uint32_t)N.tests[t].line)];
    if (k < 0) continue;
    const auto it = old_test.find((uint32_t)(O.head[co + (size_t)k] - bo));
    if (it == old_test.end()) continue;
    both.push_back(make_uint2((uint32_t)it->second, (uint32_t)t));
  }
}
}  // namespace

// The section-23 score of explicit pairs of one side's tests: k_st_verify at P = 0 over the side's resident front, in
// chunks of ST_CHUNK, its scratch sized from the longest test of the pairs.  out[i] = {a, b, lcs, score} of pairs[i].
static int sc_cross(tsm_ctx* c, StSide& f, const std::vector<uint2>& pairs, const std::vector<uint32_t>& kept,
                    std::vector<tsm_similar_pair>& out, float* ms, cudaStream_t st) {
  out.assign(pairs.size(), tsm_similar_pair{});
  if (pairs.empty()) return TSM_OK;
  uint32_t kmax = 0;
  for (const uint2& p : pairs) kmax = std::max(kmax, std::max(kept[p.x], kept[p.y]));
  DevBuf d_scratch;
  StVerifyShape vs;
  int rc = st_verify_shape(c, kmax, d_scratch, vs);
  if (rc != TSM_OK) return rc;
  std::unordered_map<unsigned long long, size_t> at;
  for (size_t i = 0; i < pairs.size(); ++i) at[(unsigned long long)pairs[i].x << 32 | pairs[i].y] = i;
  uint32_t* ctr = f.ctr.as<uint32_t>();
  std::vector<tsm_similar_pair> got;
  for (size_t c0 = 0; c0 < pairs.size(); c0 += ST_CHUNK) {
    const uint32_t n = (uint32_t)std::min<size_t>(ST_CHUNK, pairs.size() - c0);
    const uint32_t cnt[2] = {n, 0};
    CU(cudaMemcpyAsync(f.surv.p, pairs.data() + c0, sizeof(uint2) * n, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(ctr + 1, cnt, 8, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(c->diff_ev[EV_ST_VERIFY], st));
    k_st_verify<<<vs.blocks, 256, 0, st>>>(f.surv.as<uint2>(), ctr + 1, f.kbeg.as<uint32_t>(), f.kk.as<uint32_t>(),
                                           f.bf.khash.as<unsigned long long>(), 0, vs.slot_words ? d_scratch.as<unsigned long long>() : nullptr,
                                           vs.slot_words, f.pairs.as<tsm_similar_pair>(), ctr + 2);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_ST_END], st));
    got.resize(n);
    CU(cudaMemcpyAsync(got.data(), f.pairs.p, sizeof(tsm_similar_pair) * n, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches++;
    ms[3] += elapsed_ms(c->diff_ev[EV_ST_VERIFY], c->diff_ev[EV_ST_END]);
    for (const tsm_similar_pair& p : got) out[at.at((unsigned long long)(uint32_t)p.a << 32 | (uint32_t)p.b)] = p;
  }
  return TSM_OK;
}

// Both revisions to the device and their line records with header events (one k_scan pass each), the marks of the pairs
// (churn_marks), per revision the front of tsm_similar_tests (st_front); on the host the test identity (unchanged files in
// order, sc_match_pair for the changed pairs); k_sc_change for the matched tests of changed pairs; per revision the tokens
// (st_tokens), posting lists with the dirty tests first and the restricted enumeration (st_verify_all over k_sc_enum); then
// the events on the host, with the cross scores of sc_cross.  Both fronts stay resident to the end.
extern "C" int tsm_similar_churn(tsm_ctx* c, const tsm_corpus* old_rev, const tsm_corpus* new_rev, const int32_t* pair_old,
                                 const int32_t* pair_new, int64_t n_pairs, int32_t min_lines, int32_t min_similarity,
                                 tsm_similar_churn_side* old_side, tsm_similar_churn_side* new_side, tsm_similar_event* events,
                                 int64_t event_cap, int64_t* n_events, void* stream) {
  if (!c || !old_rev || !new_rev || !old_side || !new_side || !n_events || n_pairs < 0 || n_pairs > INT32_MAX ||
      (n_pairs && (!pair_old || !pair_new)) || min_lines < 1 || min_similarity < 1 || min_similarity > 100 || event_cap < 0)
    return TSM_E_ARG;
  const tsm_corpus* rev[2] = {old_rev, new_rev};
  tsm_similar_churn_side* side[2] = {old_side, new_side};
  const int32_t* pf[2] = {pair_old, pair_new};
  const int32_t n = (int32_t)n_pairs;
  std::vector<int32_t> unpaired[2];
  for (int i = 0; i < 2; ++i) {
    if (rev[i]->n_files < 0 || side[i]->test_cap < 0) return TSM_E_ARG;
    std::vector<uint8_t> used((size_t)rev[i]->n_files, 0);
    for (int32_t k = 0; k < n; ++k) {
      const int32_t f = pf[i][k];
      if (f < -1 || f >= rev[i]->n_files || (f >= 0 && used[(size_t)f]++) || (pair_old[k] < 0 && pair_new[k] < 0)) return TSM_E_ARG;
    }
    for (int32_t f = 0; f < rev[i]->n_files; ++f) if (!used[(size_t)f]) unpaired[i].push_back(f);
  }
  if (unpaired[0].size() != unpaired[1].size()) return TSM_E_ARG;
  for (int i = 0; i < 2; ++i)
    if (rev[i]->n_files > 0) {
      const int rc = check_sides({rev[i]}, true);
      if (rc != TSM_OK) return rc;
    }
  for (size_t k = 0; k < unpaired[0].size(); ++k)
    if (old_rev->len[unpaired[0][k]] != new_rev->len[unpaired[1][k]]) return TSM_E_ARG;
  float* const ms = clear_ms(c, MS_SCHURN);
  c->launches = 0;
  *n_events = 0;
  for (int i = 0; i < 2; ++i) side[i]->n_tests = side[i]->n_candidates = 0;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  HostSide S[2];
  DevBuf rmark[2], d_both, d_same, d_dirty[2], d_dcnt[2], d_ccur[2];
  StSide F[2];
  SyncGuard guard(st);
  HostSide* scan[2];
  int ns = 0;
  for (int i = 0; i < 2; ++i)
    if (rev[i]->n_files > 0) {
      const int rc = side_upload(rev[i], S[i], st);
      if (rc != TSM_OK) return rc;
      scan[ns++] = &S[i];
    }
  if (ns) {
    const int rc = sides_records(c, scan, ns, st, &ms[0], true, TSM_SCAN_HEADER_EVENTS);
    if (rc != TSM_OK) return rc;
  }
  for (int i = 0; i < 2; ++i) {
    c->launches += S[i].launches;
    if (!rmark[i].alloc((size_t)S[i].total)) return TSM_E_CUDA;
    CU(cudaMemsetAsync(rmark[i].p, 0, (size_t)S[i].total, st));
  }
  float mms[4] = {0, 0, 0, 0};
  if (n) {
    const int rc = churn_marks(c, S, pf, n, rmark, mms, st);
    if (rc != TSM_OK) return rc;
  }
  ms[1] += mms[2] + mms[3];
  ScRev R[2];
  for (int i = 0; i < 2; ++i) {
    ScRev& r = R[i];
    r.k = rev[i];
    r.base = S[i].base;
    if (r.base.empty()) r.base.assign((size_t)rev[i]->n_files + 1, 0);
    if (S[i].total == 0) { r.index(); continue; }
    const int rc = st_front(c, S[i], F[i], ms, st);
    if (rc != TSM_OK) return rc;
    r.tests.resize((size_t)F[i].nt);
    r.head.resize(F[i].sp.n_cases);
    r.mark.resize((size_t)S[i].total);
    if (F[i].nt) CU(cudaMemcpyAsync(r.tests.data(), F[i].m.tests.p, sizeof(tsm_smell_test) * (size_t)F[i].nt, cudaMemcpyDeviceToHost, st));
    if (F[i].sp.n_cases) CU(cudaMemcpyAsync(r.head.data(), F[i].sp.first.p, 4 * (size_t)F[i].sp.n_cases, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(r.mark.data(), rmark[i].p, (size_t)S[i].total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    r.index();
  }
  ScRev &O = R[0], &N = R[1];
  O.match.assign(O.tests.size(), -1);
  N.match.assign(N.tests.size(), -1);
  O.change.assign(O.tests.size(), 'D');
  N.change.assign(N.tests.size(), 'A');
  for (size_t k = 0; k < unpaired[0].size(); ++k) {       // an unchanged file: test i is test i
    const int32_t fo = unpaired[0][k], fn = unpaired[1][k];
    const size_t to = O.tfile[(size_t)fo], tn = N.tfile[(size_t)fn], m = O.tfile[(size_t)fo + 1] - to;
    if (m != N.tfile[(size_t)fn + 1] - tn) return TSM_E_ARG;
    for (size_t t = 0; t < m; ++t) {
      O.match[to + t] = (int32_t)(tn + t); N.match[tn + t] = (int32_t)(to + t);
      O.change[to + t] = N.change[tn + t] = '=';
    }
  }
  std::vector<uint2> both;
  for (int32_t k = 0; k < n; ++k)
    if (pair_old[k] >= 0 && pair_new[k] >= 0) sc_match_pair(O, N, pair_old[k], pair_new[k], both);
  if (!both.empty()) {
    const uint32_t nm = (uint32_t)both.size();
    if (!d_both.alloc(sizeof(uint2) * nm) || !d_same.alloc(nm)) return TSM_E_CUDA;
    std::vector<uint8_t> same(nm);
    CU(cudaEventRecord(c->diff_ev[EV_ST_FRONT], st));
    CU(cudaMemcpyAsync(d_both.p, both.data(), sizeof(uint2) * nm, cudaMemcpyHostToDevice, st));
    ScChangeSide cs[2];
    for (int i = 0; i < 2; ++i)
      cs[i] = ScChangeSide{F[i].m.tests.as<tsm_smell_test>(), S[i].d.line_base, rmark[i].as<uint8_t>(), F[i].bf.rank.as<unsigned long long>(),
                           F[i].bf.khash.as<unsigned long long>()};
    k_sc_change<<<std::min((nm + 7) / 8, (uint32_t)c->sms * 8), 256, 0, st>>>(cs[0], cs[1], d_both.as<uint2>(), nm, d_same.as<uint8_t>());
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_ST_END], st));
    CU(cudaMemcpyAsync(same.data(), d_same.p, nm, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches++;
    ms[1] += elapsed_ms(c->diff_ev[EV_ST_FRONT], c->diff_ev[EV_ST_END]);
    for (uint32_t k = 0; k < nm; ++k) {
      const uint2 m = both[k];
      O.match[m.x] = (int32_t)m.y; N.match[m.y] = (int32_t)m.x;
      O.change[m.x] = N.change[m.y] = same[k] ? '=' : 'M';
    }
  }
  // Per side: the tokens, the posting lists with their dirty tests first, and the pairs with a dirty test.
  std::vector<tsm_similar_pair> pairs[2];
  for (int i = 0; i < 2; ++i) {
    StSide& f = F[i];
    ScRev& r = R[i];
    const size_t NT = r.tests.size(), NK = (size_t)f.nk;
    if (NT == 0) continue;
    CU(cudaEventRecord(c->diff_ev[EV_ST_LEXED], st));
    int rc = st_tokens(S[i], f, (uint32_t)min_lines, (uint32_t)min_similarity, st);
    if (rc != TSM_OK) return rc;
    std::vector<uint8_t> dirty(NT);
    for (size_t t = 0; t < NT; ++t) dirty[t] = r.change[t] != '=';
    if (!d_dirty[i].alloc(NT) || !d_dcnt[i].alloc(4 * (size_t)f.nl) || !d_ccur[i].alloc(4 * (size_t)f.nl)) return TSM_E_CUDA;
    CU(cudaMemcpyAsync(d_dirty[i].p, dirty.data(), NT, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(d_dcnt[i].p, 0, 4 * (size_t)f.nl, st));
    CU(cudaMemsetAsync(d_ccur[i].p, 0, 4 * (size_t)f.nl, st));
    const unsigned kgrid = (unsigned)((NK + 255) / 256);
    const unsigned long long* np = f.pbase.as<unsigned long long>() + NT;
    if (NK) {
      k_sc_dirty<<<kgrid, 256, 0, st>>>(f.tok.as<StToken>(), f.ptest.as<uint32_t>(), np, d_dirty[i].as<uint8_t>(), d_dcnt[i].as<uint32_t>());
      k_sc_lists<<<kgrid, 256, 0, st>>>(f.tok.as<StToken>(), f.ptest.as<uint32_t>(), np, f.mbase.as<unsigned long long>(),
                                        d_dirty[i].as<uint8_t>(), d_dcnt[i].as<uint32_t>(), f.cursor.as<uint32_t>(),
                                        d_ccur[i].as<uint32_t>(), f.mem.as<uint32_t>());
    }
    k_sc_csums<<<f.nb, 256, 0, st>>>(f.pcnt.as<uint32_t>(), d_dcnt[i].as<uint32_t>(), f.nl, f.cbsum.as<unsigned long long>());
    k_xscan_top<<<1, 256, 0, st>>>(f.cbsum.as<unsigned long long>(), f.nb);
    k_sc_capply<<<f.nb, 256, 0, st>>>(f.pcnt.as<uint32_t>(), d_dcnt[i].as<uint32_t>(), f.nl, f.cbsum.as<unsigned long long>(),
                                      f.cbase.as<unsigned long long>());
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_ST_LISTS], st));
    c->launches += 10 + (NK ? 5 : 0);                     // tests, 2 x xscan (3 each), the candidate scan (3); count, order, prefix, dirty, lists
    const StEnum ea = f.enum_args((uint32_t)min_similarity);
    const uint32_t* pcnt = f.pcnt.as<uint32_t>();
    const uint32_t* dcnt = d_dcnt[i].as<uint32_t>();
    rc = st_verify_all(c, f, (uint32_t)min_similarity, [&](unsigned long long c0, unsigned long long cn, cudaStream_t s2) {
      k_sc_enum<<<(unsigned)std::min<unsigned long long>((cn + 255) / 256, (unsigned long long)c->sms * 16), 256, 0, s2>>>(ea, pcnt, dcnt, c0, cn);
    }, pairs[i], &side[i]->n_candidates, ms, st);
    if (rc != TSM_OK) return rc;
    r.kept.resize(NT);
    CU(cudaMemcpyAsync(r.kept.data(), f.kk.p, 4 * NT, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  // The events: each side's pairs mapped through match, then the cross scores of the pairs seen on one side only.
  const auto key = [](int32_t a, int32_t b) { return (unsigned long long)(uint32_t)a << 32 | (uint32_t)b; };
  std::unordered_map<unsigned long long, size_t> new_at, old_image;
  for (size_t k = 0; k < pairs[1].size(); ++k) new_at[key(pairs[1][k].a, pairs[1][k].b)] = k;
  std::vector<tsm_similar_event> ev_old, ev_new;
  std::vector<uint2> cross[2];                             // pairs of each side whose score is wanted, in event order
  const uint32_t NONE = 0xFFFFFFFFu;
  for (const tsm_similar_pair& p : pairs[0]) {
    const int32_t ma = O.match[(size_t)p.a], mb = O.match[(size_t)p.b];
    tsm_similar_event e{0, p.a, p.b, ma, mb, p.lcs, p.score, NONE, NONE};
    if (ma >= 0 && mb >= 0) {
      const int32_t a = std::min(ma, mb), b = std::max(ma, mb);
      const auto it = new_at.find(key(a, b));
      if (it != new_at.end()) { old_image[key(a, b)] = (size_t)p.a << 32 | (uint32_t)p.b; continue; }   // changed: new side
      e.status = TSM_SIMILAR_DIVERGED;
      cross[1].push_back(make_uint2((uint32_t)a, (uint32_t)b));
    } else {
      e.status = ma < 0 && mb < 0 ? TSM_SIMILAR_REMOVED : TSM_SIMILAR_DROPPED;
    }
    ev_old.push_back(e);
  }
  std::unordered_map<unsigned long long, tsm_similar_pair> old_pair;
  for (const tsm_similar_pair& p : pairs[0]) old_pair[key(p.a, p.b)] = p;
  for (const tsm_similar_pair& p : pairs[1]) {
    const int32_t ma = N.match[(size_t)p.a], mb = N.match[(size_t)p.b];
    tsm_similar_event e{0, ma, mb, p.a, p.b, NONE, NONE, p.lcs, p.score};
    const auto img = old_image.find(key(p.a, p.b));
    if (img != old_image.end()) {
      const tsm_similar_pair& q = old_pair.at(key((int32_t)(img->second >> 32), (int32_t)(uint32_t)img->second));
      e.status = TSM_SIMILAR_CHANGED;
      e.old_lcs = q.lcs; e.old_score = q.score;
    } else if (ma >= 0 && mb >= 0) {
      e.status = TSM_SIMILAR_CONVERGED;
      cross[0].push_back(make_uint2((uint32_t)std::min(ma, mb), (uint32_t)std::max(ma, mb)));
    } else {
      e.status = ma < 0 && mb < 0 ? TSM_SIMILAR_CREATED : TSM_SIMILAR_COPIED;
    }
    ev_new.push_back(e);
  }
  std::vector<tsm_similar_pair> scored[2];
  for (int i = 0; i < 2; ++i) {
    const int rc = sc_cross(c, F[i], cross[i], R[i].kept, scored[i], ms, st);
    if (rc != TSM_OK) return rc;
  }
  for (size_t k = 0, x = 0; k < ev_old.size(); ++k)
    if (ev_old[k].status == TSM_SIMILAR_DIVERGED) { ev_old[k].lcs = scored[1][x].lcs; ev_old[k].score = scored[1][x].score; ++x; }
  for (size_t k = 0, x = 0; k < ev_new.size(); ++k)
    if (ev_new[k].status == TSM_SIMILAR_CONVERGED) { ev_new[k].old_lcs = scored[0][x].lcs; ev_new[k].old_score = scored[0][x].score; ++x; }
  std::sort(ev_old.begin(), ev_old.end(), [](const tsm_similar_event& x, const tsm_similar_event& y) {
    return x.old_a != y.old_a ? x.old_a < y.old_a : x.old_b < y.old_b; });
  std::sort(ev_new.begin(), ev_new.end(), [](const tsm_similar_event& x, const tsm_similar_event& y) { return x.a != y.a ? x.a < y.a : x.b < y.b; });
  *n_events = (int64_t)(ev_old.size() + ev_new.size());
  for (int i = 0; i < 2; ++i) side[i]->n_tests = (int64_t)R[i].tests.size();
  bool is_short = events && event_cap < *n_events;
  for (int i = 0; i < 2; ++i) {
    const tsm_similar_churn_side* o = side[i];
    is_short |= (o->tests || o->test_kept || o->match || o->change) && o->test_cap < o->n_tests;
  }
  if (is_short) return TSM_E_CAPACITY;
  if (events) {
    std::copy(ev_old.begin(), ev_old.end(), events);
    std::copy(ev_new.begin(), ev_new.end(), events + ev_old.size());
  }
  for (int i = 0; i < 2; ++i) {
    tsm_similar_churn_side* o = side[i];
    const ScRev& r = R[i];
    if (o->tests) std::copy(r.tests.begin(), r.tests.end(), o->tests);
    if (o->test_kept) std::copy(r.kept.begin(), r.kept.end(), o->test_kept);
    if (o->match) std::copy(r.match.begin(), r.match.end(), o->match);
    if (o->change) std::copy(r.change.begin(), r.change.end(), o->change);
  }
  return TSM_OK;
}

extern "C" int tsm_similar_churn_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_SCHURN, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 28 link churn
// Both revisions to the device and their line records with header events (one k_scan pass each), the marks of the pairs
// (churn_marks), per revision the link stage of tsm_test_links (link_stage, resident to the end); on the host the test identity
// (unchanged files in order, sc_match_pair for the changed pairs, restricted to the link tests); k_lc_change for the matched
// tests of changed pairs; then the join: k_lc_calls and k_lc_links over both sides into one table of (identity, name) keys, the
// kept ranks of both sides, k_lc_by_rank and k_lc_defmap, and k_lc_events counting, an xscan placing and k_lc_events writing the
// rows.  One synchronisation reads the row count.
extern "C" int tsm_link_churn(tsm_ctx* c, const tsm_corpus* old_rev, const tsm_corpus* new_rev, const uint8_t* old_role,
                              const int32_t* old_stem, const uint8_t* new_role, const int32_t* new_stem, const int32_t* pair_old,
                              const int32_t* pair_new, int64_t n_pairs, tsm_link_churn_side* old_side, tsm_link_churn_side* new_side,
                              tsm_link_event* events, int64_t event_cap, int64_t* n_events, void* stream) {
  if (!c || !old_rev || !new_rev || !old_role || !new_role || !old_side || !new_side || !n_events || n_pairs < 0 ||
      n_pairs > INT32_MAX || (n_pairs && (!pair_old || !pair_new)) || event_cap < 0)
    return TSM_E_ARG;
  const tsm_corpus* rev[2] = {old_rev, new_rev};
  const uint8_t* role[2] = {old_role, new_role};
  const int32_t* stem[2] = {old_stem, new_stem};
  tsm_link_churn_side* side[2] = {old_side, new_side};
  const int32_t* pf[2] = {pair_old, pair_new};
  const int32_t n = (int32_t)n_pairs;
  std::vector<int32_t> unpaired[2];
  for (int i = 0; i < 2; ++i) {
    const tsm_links_result& o = side[i]->links;
    if (rev[i]->n_files < 0 || o.test_cap < 0 || o.link_cap < 0 || o.def_cap < 0) return TSM_E_ARG;
    for (int32_t f = 0; stem[i] && f < rev[i]->n_files; ++f)
      if (stem[i][f] < -1) return TSM_E_ARG;
    std::vector<uint8_t> used((size_t)rev[i]->n_files, 0);
    for (int32_t k = 0; k < n; ++k) {
      const int32_t f = pf[i][k];
      if (f < -1 || f >= rev[i]->n_files || (f >= 0 && used[(size_t)f]++) || (pair_old[k] < 0 && pair_new[k] < 0)) return TSM_E_ARG;
    }
    for (int32_t f = 0; f < rev[i]->n_files; ++f) if (!used[(size_t)f]) unpaired[i].push_back(f);
  }
  if (unpaired[0].size() != unpaired[1].size()) return TSM_E_ARG;
  for (int i = 0; i < 2; ++i)
    if (rev[i]->n_files > 0) {
      const int rc = check_sides({rev[i]}, true);
      if (rc != TSM_OK) return rc;
    }
  for (size_t k = 0; k < unpaired[0].size(); ++k) {
    const int32_t fo = unpaired[0][k], fn = unpaired[1][k];
    if (old_rev->len[fo] != new_rev->len[fn] || (old_role[fo] != 0) != (new_role[fn] != 0)) return TSM_E_ARG;
  }
  float* const ms = clear_ms(c, MS_LCHURN);
  c->launches = 0;
  *n_events = 0;
  for (int i = 0; i < 2; ++i) side[i]->links.n_tests = side[i]->links.n_links = side[i]->links.n_defs = 0;
  cudaStream_t st = (cudaStream_t)stream;
  CallScope call(c, st);
  CU(call.status);
  HostSide S[2];
  LinkStage K[2];
  DevBuf rmark[2], kept[2], rank[2], d_bsum, d_both, d_same, d_omatch, d_tab, d_slot, d_byrank, d_cfile, d_dline, d_otest, d_cnt, d_pos, d_ev;
  SyncGuard guard(st);
  HostSide* scan[2];
  int ns = 0;
  for (int i = 0; i < 2; ++i)
    if (rev[i]->n_files > 0) {
      const int rc = side_upload(rev[i], S[i], st);
      if (rc != TSM_OK) return rc;
      scan[ns++] = &S[i];
    }
  if (ns) {
    const int rc = sides_records(c, scan, ns, st, &ms[0], true, TSM_SCAN_HEADER_EVENTS);
    if (rc != TSM_OK) return rc;
  }
  for (size_t k = 0; k < unpaired[0].size(); ++k) {       // (the definitions' kept ranks assume equal line counts)
    const size_t fo = (size_t)unpaired[0][k], fn = (size_t)unpaired[1][k];
    if (S[0].base[fo + 1] - S[0].base[fo] != S[1].base[fn + 1] - S[1].base[fn]) return TSM_E_ARG;
  }
  for (int i = 0; i < 2; ++i) {
    c->launches += S[i].launches;
    if (!rmark[i].alloc((size_t)S[i].total)) return TSM_E_CUDA;
    CU(cudaMemsetAsync(rmark[i].p, 0, (size_t)S[i].total, st));
  }
  float mms[4] = {0, 0, 0, 0};
  if (n) {
    const int rc = churn_marks(c, S, pf, n, rmark, mms, st);
    if (rc != TSM_OK) return rc;
  }
  ms[1] += mms[2] + mms[3];
  ScRev R[2];
  std::vector<int32_t> lidx[2];                            // per test of the revision: its link test, or -1
  for (int i = 0; i < 2; ++i) {
    ScRev& r = R[i];
    r.k = rev[i];
    r.base = S[i].base;
    if (r.base.empty()) r.base.assign((size_t)rev[i]->n_files + 1, 0);
    if (S[i].total == 0) { r.index(); continue; }
    float lms[3];
    int launches = 0;
    const int rc = link_stage(c, S[i], role[i], stem[i], nullptr, K[i], lms, launches, st);
    if (rc != TSM_OK) return rc;
    c->launches += launches;
    ms[1] += lms[0] + lms[1];
    ms[2] += lms[2];
    r.tests.resize(K[i].na);
    r.head.resize(K[i].sp.n_cases);
    r.mark.resize((size_t)S[i].total);
    if (K[i].na) CU(cudaMemcpyAsync(r.tests.data(), K[i].m.tests.p, sizeof(tsm_smell_test) * K[i].na, cudaMemcpyDeviceToHost, st));
    if (K[i].sp.n_cases) CU(cudaMemcpyAsync(r.head.data(), K[i].sp.first.p, 4 * (size_t)K[i].sp.n_cases, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(r.mark.data(), rmark[i].p, (size_t)S[i].total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    r.index();
  }
  for (int i = 0; i < 2; ++i) {
    int32_t next = 0;
    lidx[i].resize(R[i].tests.size());
    for (size_t t = 0; t < R[i].tests.size(); ++t) lidx[i][t] = role[i][R[i].tests[t].file] ? next++ : -1;
  }
  const uint32_t n_old = K[0].nt, n_new = K[1].nt;
  std::vector<int32_t> match[2] = {std::vector<int32_t>(n_old, -1), std::vector<int32_t>(n_new, -1)};
  std::vector<uint8_t> change[2] = {std::vector<uint8_t>(n_old, 'D'), std::vector<uint8_t>(n_new, 'A')};
  for (size_t k = 0; k < unpaired[0].size(); ++k) {       // an unchanged file: test i is test i
    const int32_t fo = unpaired[0][k], fn = unpaired[1][k];
    const size_t to = R[0].tfile[(size_t)fo], tn = R[1].tfile[(size_t)fn], m = R[0].tfile[(size_t)fo + 1] - to;
    if (m != R[1].tfile[(size_t)fn + 1] - tn) return TSM_E_ARG;
    for (size_t t = 0; t < m; ++t) {
      const int32_t a = lidx[0][to + t], b = lidx[1][tn + t];
      if (a < 0) continue;                                 // (the roles are equal: b is a link test too)
      match[0][(size_t)a] = b; match[1][(size_t)b] = a;
      change[0][(size_t)a] = change[1][(size_t)b] = '=';
    }
  }
  std::vector<uint2> all, both;
  for (int32_t k = 0; k < n; ++k)
    if (pair_old[k] >= 0 && pair_new[k] >= 0) sc_match_pair(R[0], R[1], pair_old[k], pair_new[k], all);
  for (const uint2& m : all)
    if (lidx[0][m.x] >= 0 && lidx[1][m.y] >= 0) both.push_back(make_uint2((uint32_t)lidx[0][m.x], (uint32_t)lidx[1][m.y]));
  if (!both.empty()) {
    const uint32_t nm = (uint32_t)both.size();
    if (!d_both.alloc(sizeof(uint2) * nm) || !d_same.alloc(nm)) return TSM_E_CUDA;
    std::vector<uint8_t> same(nm);
    CU(cudaEventRecord(c->diff_ev[EV_LC_FROM], st));
    CU(cudaMemcpyAsync(d_both.p, both.data(), sizeof(uint2) * nm, cudaMemcpyHostToDevice, st));
    k_lc_change<<<std::min((nm + 7) / 8, (uint32_t)c->sms * 8), 256, 0, st>>>(K[0].tests.as<tsm_smell_test>(), K[1].tests.as<tsm_smell_test>(),
                                                                              S[0].d.line_base, S[1].d.line_base, rmark[0].as<uint8_t>(),
                                                                              rmark[1].as<uint8_t>(), d_both.as<uint2>(), nm, d_same.as<uint8_t>());
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_LC_TO], st));
    CU(cudaMemcpyAsync(same.data(), d_same.p, nm, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches++;
    ms[1] += elapsed_ms(c->diff_ev[EV_LC_FROM], c->diff_ev[EV_LC_TO]);
    for (uint32_t k = 0; k < nm; ++k) {
      const uint2 m = both[k];
      match[0][m.x] = (int32_t)m.y; match[1][m.y] = (int32_t)m.x;
      change[0][m.x] = change[1][m.y] = same[k] ? '=' : 'M';
    }
  }
  // The join: one table of (identity, name) keys over the calls of both sides, the old definitions' corresponding lines, the rows.
  std::vector<uint2> otest;                                // per output test (old test, new test)
  for (uint32_t a = 0; a < n_old; ++a) if (match[0][a] < 0) otest.push_back(make_uint2(a, LK_NONE));
  for (uint32_t b = 0; b < n_new; ++b) otest.push_back(make_uint2(match[1][b] >= 0 ? (uint32_t)match[1][b] : LK_NONE, b));
  const uint32_t n_out = (uint32_t)otest.size(), nd_old = K[0].nd;
  const uint32_t slots = link_slots((unsigned long long)K[0].nc + K[1].nc);
  std::vector<int32_t> cfile((size_t)rev[0]->n_files + 1, -1);
  for (size_t k = 0; k < unpaired[0].size(); ++k) cfile[(size_t)unpaired[0][k]] = unpaired[1][k];
  for (int32_t k = 0; k < n; ++k) if (pair_old[k] >= 0) cfile[(size_t)pair_old[k]] = pair_new[k];
  const size_t maxL = (size_t)std::max(S[0].total, S[1].total);
  if (!d_bsum.alloc(8 * (std::max(maxL, (size_t)n_out) / XS_TILE + 4)) || !d_omatch.alloc(4 * ((size_t)n_old + 1)) ||
      !d_tab.alloc(16 * (size_t)slots) || !d_slot.alloc(sizeof(LcSlot) * slots) || !d_byrank.alloc(4 * ((size_t)S[1].total + 1)) ||
      !d_cfile.alloc(4 * cfile.size()) || !d_dline.alloc(4 * ((size_t)nd_old + 1)) || !d_otest.alloc(sizeof(uint2) * ((size_t)n_out + 1)) ||
      !d_cnt.alloc(4 * ((size_t)n_out + 1)) || !d_pos.alloc(8 * ((size_t)n_out + 1)))
    return TSM_E_CUDA;
  for (int i = 0; i < 2; ++i)
    if (!kept[i].alloc(4 * ((size_t)S[i].total + 1)) || !rank[i].alloc(8 * ((size_t)S[i].total + 1))) return TSM_E_CUDA;
  CU(cudaEventRecord(c->diff_ev[EV_LC_FROM], st));
  CU(cudaMemcpyAsync(d_omatch.p, match[0].data(), 4 * (size_t)n_old, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_cfile.p, cfile.data(), 4 * cfile.size(), cudaMemcpyHostToDevice, st));
  if (n_out) CU(cudaMemcpyAsync(d_otest.p, otest.data(), sizeof(uint2) * n_out, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(d_tab.p, 0, 16 * (size_t)slots, st));
  CU(cudaMemset2DAsync(d_slot.p, sizeof(LcSlot), 0, 8, slots, st));                             // the calls
  CU(cudaMemset2DAsync(d_slot.as<uint8_t>() + 8, sizeof(LcSlot), 0xFF, 8, slots, st));          // the links: none
  const int32_t* om = d_omatch.as<int32_t>();
  for (int i = 0; i < 2; ++i) {
    const LinkStage& k = K[i];
    if (k.nc) {
      k_lc_calls<<<(k.nc + 255) / 256, 256, 0, st>>>(k.calls.as<LinkCall>(), k.nc, k.ltest.as<uint32_t>(), (uint32_t)i, om, n_new,
                                                     d_tab.as<LinkKey>(), slots - 1, d_slot.as<LcSlot>());
      c->launches++;
    }
  }
  for (int i = 0; i < 2; ++i) {
    const LinkStage& k = K[i];
    if (k.nk) {
      k_lc_links<<<(unsigned)((k.nk + 255) / 256), 256, 0, st>>>(k.links.as<tsm_link>(), (uint32_t)k.nk, k.defs.as<LinkDef>(), (uint32_t)i, om,
                                                                 n_new, d_tab.as<LinkKey>(), slots - 1, d_slot.as<LcSlot>());
      c->launches++;
    }
  }
  for (int i = 0; i < 2; ++i) {
    const uint32_t total = (uint32_t)S[i].total;
    if (total) k_case_kept<<<(total + 255) / 256, 256, 0, st>>>(rmark[i].as<uint8_t>(), total, kept[i].as<uint32_t>());
    xscan(kept[i].as<uint32_t>(), total, d_bsum.as<unsigned long long>(), rank[i].as<unsigned long long>(), st);
    c->launches += total ? 4 : 0;
  }
  if (S[1].total)
    k_lc_by_rank<<<(unsigned)((S[1].total + 255) / 256), 256, 0, st>>>(kept[1].as<uint32_t>(), rank[1].as<unsigned long long>(),
                                                                       (uint32_t)S[1].total, d_byrank.as<uint32_t>());
  if (nd_old)
    k_lc_defmap<<<(nd_old + 255) / 256, 256, 0, st>>>(K[0].defs.as<LinkDef>(), nd_old, d_cfile.as<int32_t>(), S[0].d.line_base,
                                                      S[1].d.line_base, rmark[0].as<uint8_t>(), rank[0].as<unsigned long long>(),
                                                      rank[1].as<unsigned long long>(), d_byrank.as<uint32_t>(), d_dline.as<uint32_t>());
  c->launches += (S[1].total ? 1 : 0) + (nd_old ? 1 : 0);
  LcRev lr[2];
  for (int i = 0; i < 2; ++i) {
    const LinkStage& k = K[i];
    lr[i] = LcRev{k.links.as<tsm_link>(), k.lbase.as<unsigned long long>(), k.out_tests.as<tsm_link_test>(), k.defs.as<LinkDef>(),
                  k.name.as<LinkKey>(), k.ns ? k.ns - 1 : 0, k.ndefs.as<uint32_t>()};
  }
  LcEvents ea{lr[0], lr[1], d_otest.as<uint2>(), n_out, n_new, om, d_tab.as<LinkKey>(), slots - 1, d_slot.as<LcSlot>(),
              d_cfile.as<int32_t>(), d_dline.as<uint32_t>(), d_cnt.as<uint32_t>(), d_pos.as<unsigned long long>(), nullptr};
  const unsigned egrid = std::min((n_out + 7) / 8, (uint32_t)c->sms * 8);
  if (n_out) k_lc_events<false><<<egrid, 256, 0, st>>>(ea);
  xscan(d_cnt.as<uint32_t>(), n_out, d_bsum.as<unsigned long long>(), d_pos.as<unsigned long long>(), st);
  unsigned long long* pin = c->h_rb->u64;
  CU(cudaMemcpyAsync(pin, d_pos.as<unsigned long long>() + n_out, 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const unsigned long long ne = *pin;
  if (!d_ev.alloc(sizeof(tsm_link_event) * ((size_t)ne + 1))) return TSM_E_CUDA;
  ea.out = d_ev.as<tsm_link_event>();
  if (n_out) k_lc_events<true><<<egrid, 256, 0, st>>>(ea);
  CU(cudaGetLastError());
  CU(cudaEventRecord(c->diff_ev[EV_LC_TO], st));
  CU(cudaStreamSynchronize(st));
  c->launches += (n_out ? 5 : 3);                          // count, xscan (3), write
  ms[3] = elapsed_ms(c->diff_ev[EV_LC_FROM], c->diff_ev[EV_LC_TO]);
  *n_events = (int64_t)ne;
  bool is_short = events && event_cap < (int64_t)ne;
  for (int i = 0; i < 2; ++i) {
    tsm_links_result& o = side[i]->links;
    o.n_tests = K[i].nt; o.n_links = (int64_t)K[i].nk; o.n_defs = K[i].nd;
    is_short |= (o.tests && o.test_cap < o.n_tests) || (o.links && o.link_cap < o.n_links) || (o.defs && o.def_cap < o.n_defs) ||
                ((side[i]->match || side[i]->change) && o.test_cap < o.n_tests);
  }
  if (is_short) return TSM_E_CAPACITY;
  if (events && ne) CU(cudaMemcpyAsync(events, d_ev.p, sizeof(tsm_link_event) * ne, cudaMemcpyDeviceToHost, st));
  for (int i = 0; i < 2; ++i) {
    const int rc = link_copy(K[i], &side[i]->links, st);    // (synchronises st)
    if (rc != TSM_OK) return rc;
    if (side[i]->match) std::copy(match[i].begin(), match[i].end(), side[i]->match);
    if (side[i]->change) std::copy(change[i].begin(), change[i].end(), side[i]->change);
  }
  return TSM_OK;
}

extern "C" int tsm_link_churn_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_LCHURN, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 19 test-smell churn
// The line records of both sides with their header events, per side the case spans and the smell stage, one synchronisation
// for the case and test counts (the capacity check comes before the diff), with lex (section 26) the lexical stage of both sides
// (lex_stage), the marks diff, the case records (with the new side's by_rank) and k_smell_churn per side (<true> with lex).
// EV_CHURN_SMELLS times the smell stages, EV_CHURN_LEX the lexical stages, and EV_CHURN_CASES, the first slots again once
// read, the case records and churn behind the diff.
static int diff_smells(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                       tsm_diff_detail* detail, tsm_diff_smells* out, tsm_diff_lex_smells* lex, void* stream) {
  if (!c || !olds || !news || !added || !removed || !out || olds->n_files != news->n_files || out->cases.old_cap < 0 ||
      out->cases.new_cap < 0 || out->old_test_cap < 0 || out->new_test_cap < 0)
    return TSM_E_ARG;
  const int32_t n = olds->n_files;
  float* const ms = clear_ms(c, lex ? MS_LEXCHURN : MS_CHURN);
  out->cases.n_old = out->cases.n_new = out->n_old_tests = out->n_new_tests = 0;
  if (n == 0) return TSM_OK;
  float* const dm = c->last_ms[MS_DIFF];
  return pair_call(c, olds, news, TSM_SCAN_HEADER_EVENTS, &dm[0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    ms[0] = dm[0];
    const HostSide* side[2] = {&P.A, &P.B};
    PairCases pc;
    SmellBufs sb[2];
    LexBufs lb[2];
    DevBuf d_churn[2], d_lchurn[2];
    int launches = 0;
    CU(cudaEventRecord(c->diff_ev[EV_CHURN_SMELLS.from], st));
    int rc = pair_case_spans(P, pc, launches, st);
    for (int s = 0; s < 2 && rc == TSM_OK; ++s) rc = smell_stage(c, *side[s], pc.sp[s], pc.bsum, sb[s], launches, st);
    if (rc != TSM_OK) return rc;
    CU(cudaEventRecord(c->diff_ev[EV_CHURN_SMELLS.to], st));
    unsigned long long* pin = c->h_rb->u64;
    for (int s = 0; s < 2; ++s)
      CU(cudaMemcpyAsync(pin + s, sb[s].tidx.as<unsigned long long>() + pc.sp[s].n_cases, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    ms[1] = span_ms(c, EV_CHURN_SMELLS);
    const uint32_t nt[2] = {(uint32_t)pin[0], (uint32_t)pin[1]};
    out->cases.n_old = pc.sp[0].n_cases; out->cases.n_new = pc.sp[1].n_cases;
    out->n_old_tests = nt[0]; out->n_new_tests = nt[1];
    if ((out->cases.old_cases && out->cases.old_cap < out->cases.n_old) || (out->cases.new_cases && out->cases.new_cap < out->cases.n_new) ||
        ((out->old_tests || out->old_churn) && out->old_test_cap < (int64_t)nt[0]) ||
        ((out->new_tests || out->new_churn) && out->new_test_cap < (int64_t)nt[1]) ||
        (lex && (lex->old_lex || lex->old_churn) && out->old_test_cap < (int64_t)nt[0]) ||
        (lex && (lex->new_lex || lex->new_churn) && out->new_test_cap < (int64_t)nt[1]))
      return TSM_E_CAPACITY;
    if (lex) {
      CU(cudaEventRecord(c->diff_ev[EV_CHURN_LEX.from], st));
      rc = lex_stage(c, side, sb, nt, 2, pc.bsum, lb, nullptr, launches, st);
      if (rc != TSM_OK) return rc;
      CU(cudaEventRecord(c->diff_ev[EV_CHURN_LEX.to], st));
    }
    rc = diff_core<DIFF_MARKS>(c, P.A, P.B, n, added, removed, detail, st);
    if (rc != TSM_OK) return rc;
    ms[2] = dm[1] + dm[2];
    CU(cudaEventRecord(c->diff_ev[EV_CHURN_CASES.from], st));
    rc = case_records(c, P, pc, true, launches, st);
    if (rc != TSM_OK) return rc;
    for (int s = 0; s < 2; ++s) {
      if (!d_churn[s].alloc(sizeof(tsm_test_churn) * (size_t)nt[s])) return TSM_E_CUDA;
      if (lex && !d_lchurn[s].alloc(sizeof(tsm_lex_churn) * (size_t)nt[s])) return TSM_E_CUDA;
      if (!nt[s]) continue;
      const int o = 1 - s;
      const ChurnSide cs{side[s]->d.line_base, sb[s].tests.as<tsm_smell_test>(), nt[s], sb[s].smell.as<uint16_t>(),
                         side[s]->line_mark.as<uint8_t>(), pc.rank[s].as<unsigned long long>(), pc.sp[s].case_of.as<unsigned long long>(),
                         sb[o].smell.as<uint16_t>(), pc.by_rank[o].as<uint32_t>(), d_churn[s].as<tsm_test_churn>()};
      const unsigned grid = std::min((nt[s] + 7) / 8, (uint32_t)c->sms * 8);
      if (lex)
        k_smell_churn<true><<<grid, 256, 0, st>>>(cs, LexChurnSide{lb[s].lsmell.as<uint8_t>(), lb[o].lsmell.as<uint8_t>(),
                                                                   d_lchurn[s].as<tsm_lex_churn>()});
      else
        k_smell_churn<false><<<grid, 256, 0, st>>>(cs, LexChurnSide{});
      ++launches;
    }
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_CHURN_CASES.to], st));
    tsm_case* const h_cases[2] = {out->cases.old_cases, out->cases.new_cases};
    tsm_smell_test* const h_tests[2] = {out->old_tests, out->new_tests};
    tsm_test_churn* const h_churn[2] = {out->old_churn, out->new_churn};
    for (int s = 0; s < 2; ++s) {
      if (h_cases[s] && pc.sp[s].n_cases)
        CU(cudaMemcpyAsync(h_cases[s], pc.cases[s].p, sizeof(tsm_case) * pc.sp[s].n_cases, cudaMemcpyDeviceToHost, st));
      if (h_tests[s] && nt[s]) CU(cudaMemcpyAsync(h_tests[s], sb[s].tests.p, sizeof(tsm_smell_test) * nt[s], cudaMemcpyDeviceToHost, st));
      if (h_churn[s] && nt[s]) CU(cudaMemcpyAsync(h_churn[s], d_churn[s].p, sizeof(tsm_test_churn) * nt[s], cudaMemcpyDeviceToHost, st));
    }
    if (lex) {
      tsm_lex_test* const h_lex[2] = {lex->old_lex, lex->new_lex};
      tsm_lex_churn* const h_lchurn[2] = {lex->old_churn, lex->new_churn};
      for (int s = 0; s < 2; ++s) {
        if (h_lex[s] && nt[s]) CU(cudaMemcpyAsync(h_lex[s], lb[s].lex.p, sizeof(tsm_lex_test) * nt[s], cudaMemcpyDeviceToHost, st));
        if (h_lchurn[s] && nt[s])
          CU(cudaMemcpyAsync(h_lchurn[s], d_lchurn[s].p, sizeof(tsm_lex_churn) * nt[s], cudaMemcpyDeviceToHost, st));
      }
    }
    CU(cudaStreamSynchronize(st));
    if (lex) ms[1] += span_ms(c, EV_CHURN_LEX);
    ms[3] = span_ms(c, EV_CHURN_CASES);
    c->launches += launches;
    return TSM_OK;
  });
}

extern "C" int tsm_diff_pairs_smells(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                     tsm_diff_detail* detail, tsm_diff_smells* out, void* stream) {
  return diff_smells(c, olds, news, added, removed, detail, out, nullptr, stream);
}

extern "C" int tsm_diff_smells_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_CHURN, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 26 lexical test-smell churn
extern "C" int tsm_diff_pairs_smells_lexical(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                             tsm_diff_detail* detail, tsm_diff_smells* out, tsm_diff_lex_smells* lex, void* stream) {
  if (!lex) return TSM_E_ARG;
  return diff_smells(c, olds, news, added, removed, detail, out, lex, stream);
}

extern "C" int tsm_diff_smells_lexical_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_LEXCHURN, ms4, 4); }

// ------------------------------------------------------------------------------------- SPEC section 20 moved code
// The line records of both sides, the marks diff, then per side k_move_lines and three exclusive scans (alnum prefix, entry and
// run numbers); one synchronisation reads the entry and run counts, which size the join.  k_move_compact, the (step, hash) table
// (k_move_insert, xscan of each side's slot counts, k_move_scatter) and k_move_reach; per side the list of block starts
// (k_move_starts twice around an xscan) and k_move_runs twice around an xscan of the block counts; a second synchronisation
// reads the block counts for k_move_mark.  EV_MOVE_FLAGS and EV_MOVE_JOIN time the flags and the join with the reach,
// EV_MOVE_RUNS and EV_MOVE_MARK the runs and the marks: every slot again, the diff's own having been read by then.
struct MoveBufs { DevBuf flag, alnum, chg, head, apre, eidx, ridx, best, ent, run_first, run_end, cnt, base, cursor, slot_of, seg, seg_slot,
                  start, sidx, starts, rcnt, rbase, blocks; };

extern "C" int tsm_diff_pairs_moves(tsm_ctx* c, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                    tsm_diff_detail* detail, tsm_diff_moves* out, void* stream) {
  if (!c || !olds || !news || !added || !removed || !out || olds->n_files != news->n_files || out->marks.del_cap < 0 ||
      out->marks.ins_cap < 0 || out->old_cap < 0 || out->new_cap < 0)
    return TSM_E_ARG;
  const int32_t n = olds->n_files;
  for (int32_t i = 0; i < n; ++i) {                        // a pair's step: the same grp on both sides, below n_groups
    const uint16_t go = olds->grp ? olds->grp[i] : 0, gn = news->grp ? news->grp[i] : 0;
    if (go != gn || go >= olds->n_groups || gn >= news->n_groups) return TSM_E_ARG;
  }
  float* const mt = clear_ms(c, MS_MOVE);
  tsm_line_marks& mk = out->marks;
  mk.n_old = mk.n_new = 0;
  out->n_old_blocks = out->n_new_blocks = 0;
  if (n == 0) {
    if (mk.line_base_old) mk.line_base_old[0] = 0;
    if (mk.line_base_new) mk.line_base_new[0] = 0;
    return TSM_OK;
  }
  float* const dm = c->last_ms[MS_DIFF];
  return pair_call(c, olds, news, PAIR_GRP | PAIR_HOST_BASE, &dm[0], stream, [&](HostSidePair& P, cudaStream_t st) -> int {
    mt[0] = dm[0];
    const int rc = diff_core<DIFF_MARKS>(c, P.A, P.B, n, added, removed, detail, st);
    if (rc != TSM_OK) return rc;
    mt[1] = dm[1] + dm[2];
    MoveBufs mb[2];
    DevBuf d_bsum, d_slot_bsum, d_table;
    HostSide* const side[2] = {&P.A, &P.B};
    const uint32_t T[2] = {(uint32_t)P.A.total, (uint32_t)P.B.total};
    int launches = 0;
    if (!d_bsum.alloc(8 * ((size_t)std::max(T[0], T[1]) / XS_TILE + 4))) return TSM_E_CUDA;
    unsigned long long* const bsum = d_bsum.as<unsigned long long>();
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_FLAGS.from], st));
    for (int s = 0; s < 2; ++s) {
      MoveBufs& m = mb[s];
      const size_t L = T[s];
      if (!m.flag.alloc(L) || !m.alnum.alloc(4 * L) || !m.chg.alloc(4 * L) || !m.head.alloc(4 * L) || !m.apre.alloc(8 * (L + 1)) ||
          !m.eidx.alloc(8 * (L + 1)) || !m.ridx.alloc(8 * (L + 1)) || !m.best.alloc(8 * L))
        return TSM_E_CUDA;
      CU(cudaMemsetAsync(m.best.p, 0, 8 * L, st));
      if (L) k_move_lines<<<(unsigned)((L + 255) / 256), 256, 0, st>>>(side[s]->d, n, T[s], side[s]->line_mark.as<uint8_t>(), m.flag.as<uint8_t>(),
                                                                        m.alnum.as<uint32_t>(), m.chg.as<uint32_t>(), m.head.as<uint32_t>());
      xscan(m.alnum.as<uint32_t>(), T[s], bsum, m.apre.as<unsigned long long>(), st);
      xscan(m.chg.as<uint32_t>(), T[s], bsum, m.eidx.as<unsigned long long>(), st);
      xscan(m.head.as<uint32_t>(), T[s], bsum, m.ridx.as<unsigned long long>(), st);
      launches += (L ? 1 : 0) + 9;
    }
    CU(cudaGetLastError());
    unsigned long long* pin = c->h_rb->u64;
    for (int s = 0; s < 2; ++s) {
      CU(cudaMemcpyAsync(pin + 2 * s, mb[s].eidx.as<unsigned long long>() + T[s], 8, cudaMemcpyDeviceToHost, st));
      CU(cudaMemcpyAsync(pin + 2 * s + 1, mb[s].ridx.as<unsigned long long>() + T[s], 8, cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    const uint32_t ne[2] = {(uint32_t)pin[0], (uint32_t)pin[2]}, nr[2] = {(uint32_t)pin[1], (uint32_t)pin[3]};
    for (int s = 0; s < 2; ++s) {
      MoveBufs& m = mb[s];
      if (!m.ent.alloc(4 * (size_t)ne[s]) || !m.run_first.alloc(4 * (size_t)nr[s]) || !m.run_end.alloc(4 * (size_t)nr[s])) return TSM_E_CUDA;
      if (T[s])
        k_move_compact<<<(T[s] + 255) / 256, 256, 0, st>>>(m.flag.as<uint8_t>(), T[s], m.eidx.as<unsigned long long>(), m.ridx.as<unsigned long long>(),
                                                            m.ent.as<uint32_t>(), m.run_first.as<uint32_t>(), m.run_end.as<uint32_t>());
    }
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_FLAGS.to], st));
    // ---- the join: one table over the entries of both sides, at most half full
    const unsigned long long tot = (unsigned long long)ne[0] + ne[1];
    unsigned long long cap = 1024;
    while (cap < 2 * tot) cap <<= 1;
    if (cap > (1ull << 31)) return TSM_E_NOMEM;
    const uint32_t mask = (uint32_t)cap - 1;
    if (!d_table.alloc(sizeof(MoveKey) * cap)) return TSM_E_CUDA;
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_JOIN.from], st));
    CU(cudaMemsetAsync(d_table.p, 0, sizeof(MoveKey) * cap, st));
    for (int s = 0; s < 2; ++s) {
      MoveBufs& m = mb[s];
      if (!m.cnt.alloc(4 * cap) || !m.cursor.alloc(4 * cap) || !m.base.alloc(8 * (cap + 1)) || !m.slot_of.alloc(4 * (size_t)ne[s]) ||
          !m.seg.alloc(4 * (size_t)ne[s]) || (s == 0 && !m.seg_slot.alloc(4 * (size_t)ne[s])))
        return TSM_E_CUDA;
      CU(cudaMemsetAsync(m.cnt.p, 0, 4 * cap, st));
      CU(cudaMemsetAsync(m.cursor.p, 0, 4 * cap, st));
      if (ne[s])
        k_move_insert<<<(ne[s] + 255) / 256, 256, 0, st>>>(m.ent.as<uint32_t>(), ne[s], side[s]->d.line_hash, side[s]->d.line_base, n,
                                                            side[s]->grp.as<uint16_t>(), d_table.as<MoveKey>(), mask, m.cnt.as<uint32_t>(),
                                                            m.slot_of.as<uint32_t>());
    }
    if (!d_slot_bsum.alloc(8 * (cap / XS_TILE + 4))) return TSM_E_CUDA;
    for (int s = 0; s < 2; ++s) {
      MoveBufs& m = mb[s];
      xscan(m.cnt.as<uint32_t>(), (uint32_t)cap, d_slot_bsum.as<unsigned long long>(), m.base.as<unsigned long long>(), st);
      if (ne[s])
        k_move_scatter<<<(ne[s] + 255) / 256, 256, 0, st>>>(m.ent.as<uint32_t>(), m.slot_of.as<uint32_t>(), ne[s], m.base.as<unsigned long long>(),
                                                             m.cursor.as<uint32_t>(), m.seg.as<uint32_t>(), s == 0 ? m.seg_slot.as<uint32_t>() : nullptr);
      launches += 3 + (ne[s] ? 2 : 0);
    }
    MoveSide ms[2];
    for (int s = 0; s < 2; ++s)
      ms[s] = MoveSide{side[s]->d.line_hash, mb[s].flag.as<uint8_t>(), mb[s].ridx.as<unsigned long long>(), mb[s].run_end.as<uint32_t>(),
                       mb[s].best.as<unsigned long long>()};
    if (ne[0] && ne[1]) {
      k_move_reach<<<std::min((ne[0] + 7) / 8, (uint32_t)c->sms * 8), 256, 0, st>>>(ms[0], ms[1], mb[0].seg.as<uint32_t>(), mb[0].seg_slot.as<uint32_t>(),
                                                                                 ne[0], mb[1].seg.as<uint32_t>(), mb[1].base.as<unsigned long long>());
      ++launches;
    }
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_JOIN.to], st));
    // ---- the blocks of every run, in line order
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_RUNS.from], st));
    for (int s = 0; s < 2; ++s) {
      MoveBufs& m = mb[s];
      if (!m.start.alloc(4 * (size_t)ne[s]) || !m.sidx.alloc(8 * ((size_t)ne[s] + 1)) || !m.starts.alloc(4 * (size_t)ne[s]) ||
          !m.rcnt.alloc(4 * (size_t)nr[s]) || !m.rbase.alloc(8 * ((size_t)nr[s] + 1)) || !m.blocks.alloc(sizeof(tsm_move_block) * (size_t)ne[s]))
        return TSM_E_CUDA;
      const unsigned ge = (ne[s] + 255) / 256, g = (nr[s] + 255) / 256;
      const uint32_t* ent = m.ent.as<uint32_t>();
      const unsigned long long* best = m.best.as<unsigned long long>();
      if (ne[s])
        k_move_starts<0><<<ge, 256, 0, st>>>(ent, ne[s], best, m.apre.as<unsigned long long>(), m.start.as<uint32_t>(), nullptr, nullptr);
      xscan(m.start.as<uint32_t>(), ne[s], bsum, m.sidx.as<unsigned long long>(), st);
      if (ne[s])
        k_move_starts<1><<<ge, 256, 0, st>>>(ent, ne[s], best, nullptr, m.start.as<uint32_t>(), m.sidx.as<unsigned long long>(),
                                             m.starts.as<uint32_t>());
      if (nr[s])
        k_move_runs<0><<<g, 256, 0, st>>>(m.run_first.as<uint32_t>(), m.run_end.as<uint32_t>(), nr[s], best, m.eidx.as<unsigned long long>(),
                                          m.sidx.as<unsigned long long>(), ne[s], m.starts.as<uint32_t>(), m.rcnt.as<uint32_t>(), nullptr, nullptr);
      xscan(m.rcnt.as<uint32_t>(), nr[s], bsum, m.rbase.as<unsigned long long>(), st);
      if (nr[s])
        k_move_runs<1><<<g, 256, 0, st>>>(m.run_first.as<uint32_t>(), m.run_end.as<uint32_t>(), nr[s], best, m.eidx.as<unsigned long long>(),
                                          m.sidx.as<unsigned long long>(), ne[s], m.starts.as<uint32_t>(), nullptr,
                                          m.rbase.as<unsigned long long>(), m.blocks.as<tsm_move_block>());
      CU(cudaMemcpyAsync(pin + s, m.rbase.as<unsigned long long>() + nr[s], 8, cudaMemcpyDeviceToHost, st));
      launches += 6 + (ne[s] ? 2 : 0) + (nr[s] ? 2 : 0);
    }
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_RUNS.to], st));
    CU(cudaStreamSynchronize(st));
    const uint32_t nb[2] = {(uint32_t)pin[0], (uint32_t)pin[1]};
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_MARK.from], st));
    for (int s = 0; s < 2; ++s)
      if (nb[s]) {
        k_move_mark<<<(ne[s] + 255) / 256, 256, 0, st>>>(mb[s].ent.as<uint32_t>(), ne[s], mb[s].blocks.as<tsm_move_block>(), nb[s],
                                                          side[s]->d.line_flag, side[s]->line_mark.as<uint8_t>());
        ++launches;
      }
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->diff_ev[EV_MOVE_MARK.to], st));
    mk.n_old = (int64_t)T[0]; mk.n_new = (int64_t)T[1];
    out->n_old_blocks = nb[0]; out->n_new_blocks = nb[1];
    if (mk.line_base_old) memcpy(mk.line_base_old, P.A.base.data(), sizeof(int64_t) * ((size_t)n + 1));
    if (mk.line_base_new) memcpy(mk.line_base_new, P.B.base.data(), sizeof(int64_t) * ((size_t)n + 1));
    CU(cudaStreamSynchronize(st));
    mt[2] = span_ms(c, EV_MOVE_FLAGS) + span_ms(c, EV_MOVE_JOIN);
    mt[3] = span_ms(c, EV_MOVE_RUNS) + span_ms(c, EV_MOVE_MARK);
    c->launches += launches;
    if ((mk.del && mk.del_cap < mk.n_old) || (mk.ins && mk.ins_cap < mk.n_new) || (out->old_blocks && out->old_cap < (int64_t)nb[0]) ||
        (out->new_blocks && out->new_cap < (int64_t)nb[1]))
      return TSM_E_CAPACITY;
    uint8_t* const h_mark[2] = {mk.del, mk.ins};
    tsm_move_block* const h_blocks[2] = {out->old_blocks, out->new_blocks};
    for (int s = 0; s < 2; ++s) {
      if (h_mark[s] && T[s]) CU(cudaMemcpyAsync(h_mark[s], side[s]->line_mark.p, T[s], cudaMemcpyDeviceToHost, st));
      if (h_blocks[s] && nb[s]) CU(cudaMemcpyAsync(h_blocks[s], mb[s].blocks.p, sizeof(tsm_move_block) * nb[s], cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    return TSM_OK;
  });
}

extern "C" int tsm_moves_last_ms(tsm_ctx* c, float* ms4) { return copy_ms(c, MS_MOVE, ms4, 4); }
