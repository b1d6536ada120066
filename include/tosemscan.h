/* tosemscan.h - C ABI of libtosemscan.so, the H100-native corpus-scan hot path.
 *
 * Drop-in boundary.  The reference package (openjamoses/TOSEM-2021-Replication) ships NO code, hence
 * no plugin / operator / FFI interface to mirror (SURVEY.md section 8b): the only observable contract is
 * its file formats.  Each entry point below therefore cites the reference ARTEFACT whose
 * producing stage it replaces; docs/SPEC.md gives the byte-level rules, INTEGRATION.md the
 * bindings (ctypes / C++ CLI) a maintainer would add.
 *
 * Conventions: plain pointers and sizes, no exceptions, no global state; every call returns
 * TSM_OK (0) or a negative tsm_status; caller owns all host memory; a tsm_ctx owns device memory
 * and is bound to one CUDA device; calls on one ctx must be serialised by the caller (one host thread
 * at a time), calls on different ctxs are independent, also from different host threads on one device.
 * There is no CPU fallback: without a usable CUDA device tsm_create() fails with TSM_E_CUDA.
 *
 * Streams: `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).  Calls on one
 * ctx may use different streams: each call's device work is ordered after all earlier device work of
 * that ctx, whatever stream it was queued on, and tsm_create returns with the device initialised.
 * tsm_upload and tsm_scan_resident return with their work in flight on `stream`, so the corpus' host
 * arrays must stay unchanged until that work has run (a synchronisation of `stream`, or any later call
 * that synchronises); every other call that takes a stream synchronises it before it returns.  A call
 * that grows the ctx's scratch buffers or event lists frees device memory, which synchronises the device;
 * a call that allocates nothing waits for no device work other than the ctx's own.
 */
#ifndef TOSEMSCAN_H
#define TOSEMSCAN_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define TSM_ABI_VERSION 1
#define TSM_NUM_CATEGORIES 128   /* K of docs/SPEC.md section 6 */
#define TSM_ALIGN 128            /* file start alignment inside the arena */

typedef enum {
  TSM_OK = 0,
  TSM_E_ARG = -1,        /* null / negative / inconsistent argument */
  TSM_E_LAYOUT = -2,     /* corpus violates SPEC section 1 (alignment, bounds, grp >= n_groups) */
  TSM_E_CAPACITY = -3,   /* corpus exceeds what the ctx was created for (arena bytes, files, groups), a list would
                            need more than 2^32 - 16 entries, or caller-supplied output arrays are too small */
  TSM_E_CUDA = -4,       /* CUDA runtime error (no device, launch failure, ...) */
  TSM_E_NOMEM = -5,
  TSM_E_STATE = -6       /* call order (e.g. scan_resident before upload) */
} tsm_status;

/* ext tags (S1: value census of the `extension` column, Important-files/ML-Testing-v1.xlsx) */
enum { TSM_EXT_OTHER = 0, TSM_EXT_PY = 1, TSM_EXT_CC = 2, TSM_EXT_CPP = 3, TSM_EXT_JAVA = 4, TSM_EXT_C = 5, TSM_EXT_H = 6 };

/* scan flags */
#define TSM_SCAN_ASSERT_EVENTS 1u  /* produce assertion events (raw scan rows need them) */
#define TSM_SCAN_HEADER_EVENTS 2u  /* produce header events (method column needs them) */
#define TSM_SCAN_REV_B 8u          /* the later revision of the lost tool (docs/SPEC.md section 4b; golden G1: ML-Testing-v1.xlsx!DeepSpeech):
                                      also triggers on _CHECK / TESTEQUAL / FAIL, full statements for BOOST_CHECK( / NTA_CHECK( / Java */
#define TSM_SCAN_LINE_HASHES 4u    /* internal to tsm_line_hashes / tsm_diff_pairs*: per-line records; ignored by tsm_scan* */

/* Per-file record; replaces the per-file summary stage (S6: `total assert` of
 * selection/completed-labels/Release-Meta-tpot.csv:1-2). */
typedef struct tsm_file_stat {
  uint32_t n_lines, n_assert, n_headers, n_fixture;
  uint64_t digest;
} tsm_file_stat;

/* One assertion line; the raw-row stage (fileName,extension,test_name,method,statement,counts,
 * category: Important-files/ML-Testing-v1.xlsx!apollo_tests:R1) groups these. Offsets are
 * relative to the file start. */
typedef struct tsm_assert_event {
  uint32_t file, line_off, stmt_off;
  uint16_t stmt_len, cat;
  uint32_t ident_off;
  uint16_t ident_len, pad;
  uint64_t stmt_hash;
} tsm_assert_event;

typedef struct tsm_header_event { uint32_t file, line_off, line_len, kind; } tsm_header_event; /* kind bit0 = TEST_F */

/* Packed corpus (SPEC section 1). All pointers host memory for the host-path calls. */
typedef struct tsm_corpus {
  const uint8_t* arena;   /* off[n_files] bytes */
  const int32_t* off;     /* [n_files+1], multiples of TSM_ALIGN, ascending */
  const int32_t* len;     /* [n_files], off[i]+len[i] <= off[i+1] */
  const uint8_t* ext;     /* [n_files] TSM_EXT_* */
  const uint16_t* grp;    /* [n_files] < n_groups; NULL = all 0 */
  int32_t n_files;
  int32_t n_groups;       /* >= 1 */
} tsm_corpus;

/* Host-side result buffers. Any pointer may be NULL (that output is skipped). */
typedef struct tsm_result {
  tsm_file_stat* stats;          /* [n_files] */
  int64_t* group_counts;         /* [n_groups][TSM_NUM_CATEGORIES] */
  int64_t* global_counts;        /* [TSM_NUM_CATEGORIES] */
  tsm_assert_event* aev; int64_t aev_cap; int64_t n_aev;   /* canonical order (file, line_off) */
  tsm_header_event* hev; int64_t hev_cap; int64_t n_hev;
  int64_t totals[4];             /* lines, assertion lines, headers, fixture headers */
} tsm_result;

typedef struct tsm_ctx tsm_ctx;

int tsm_abi_version(void);
const char* tsm_strerror(int status);
const char* tsm_category_name(int id);   /* "" for 0/reserved, "<other>" for 127 */

/* Context sized for corpora up to (max_arena_bytes, max_files, max_groups).  max_events is the initial size of the
 * device candidate and event lists (0 = max_arena_bytes / 32 + max_files).  It is not a limit: when a scan finds more
 * assertion lines or headers than the lists hold, tsm_download (and so tsm_scan) grows them to the counts the scan
 * reached and scans the resident arena once more, and later scans keep the larger lists. */
int tsm_create(tsm_ctx** out, int device, int64_t max_arena_bytes, int32_t max_files,
               int32_t max_groups, int64_t max_events);
void tsm_destroy(tsm_ctx* ctx);

/* Host path, end to end: H2D of the corpus (overlapped slab by slab with the scan), the scan and
 * classify/aggregate kernels, D2H of the requested results, stream-synchronised on return.
 * Replaces stage (C) "corpus scan" of SURVEY.md section 1 for one packed batch. */
int tsm_scan(tsm_ctx* ctx, const tsm_corpus* corpus, tsm_result* result, uint32_t flags, void* stream);

/* Resident path (what bench.py's `value` times): upload once, scan many times, fetch once. */
int tsm_upload(tsm_ctx* ctx, const tsm_corpus* corpus, void* stream);
int tsm_scan_resident(tsm_ctx* ctx, uint32_t flags, void* stream);       /* kernels only, async */
/* Synchronises.  If aev_cap or hev_cap is smaller than the number of events of that kind, the call returns
 * TSM_E_CAPACITY with n_aev and n_hev set to both counts (everything else is filled): size the arrays and call
 * tsm_download again, the scan is not repeated. */
int tsm_download(tsm_ctx* ctx, tsm_result* result, void* stream);
/* Device address of the [n_groups+1][K] int64 count table of the last scan (row n_groups = global),
 * for the single multi-GPU allreduce (SURVEY.md section 8e); valid until the next scan.  When the scan's lists did
 * not overflow, the table is complete in `stream` order behind tsm_scan_resident: work queued on that stream after
 * the call reads the final table, and a consumer on another stream orders itself with an event recorded there.  It
 * is complete in any case once tsm_download has returned: a scan whose candidate list overflowed is redone there. */
int tsm_device_counts(tsm_ctx* ctx, void** dptr, int64_t* n_int64);
/* Kernel launches issued by the last tsm_scan / tsm_scan_resident call. */
int tsm_last_launch_count(tsm_ctx* ctx);
/* Device time (CUDA events on the launching stream) of the kernels of the last scan, in launch
 * order: k_plan, k_scan, k_classify (+ a 4th slot that is 0: the totals are fused into k_classify).
 * Synchronises on the last of them. */
int tsm_last_kernel_ms(tsm_ctx* ctx, float* ms4);
/* Per-kernel device time summed over every scan since the last reset (event ring, no host sync
 * inside a back-to-back series); waits for scans still in flight. */
int tsm_kernel_ms_stats(tsm_ctx* ctx, double* sum_ms4, int64_t* n_scans, int reset);

/* S8 revision-pair churn (Important-files/ML-Testing-v1.xlsx!projects:R1 `cloc, added, removed`):
 * pair i = (olds file i, news file i); added/removed [n_pairs] host arrays. */
int tsm_diff_pairs(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news,
                   int64_t* added, int64_t* removed, void* stream);

/* The same plus, per pair, the hunks of the canonical edit script (docs/SPEC.md section 8) classified as
 * add / del / mod, and how many inserted / deleted lines are assertion lines (BASELINE config C5,
 * "per-hunk diff + classify").  `ext` of both corpora is used for the assertion rule. */
typedef struct tsm_diff_detail { int64_t hunks_add, hunks_del, hunks_mod, added_assert, removed_assert; } tsm_diff_detail;
int tsm_diff_pairs_detail(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news,
                          int64_t* added, int64_t* removed, tsm_diff_detail* detail, void* stream);

/* A pair whose edit distance D is larger than 23 168 lines needs more than 2^28 trace entries ((D+1)(D+2)/2 ints, 1 GiB)
 * for its backtrack: tsm_diff_pairs_detail does not trace it - added / removed are exact, the detail reports ONE hunk
 * (add, del or mod by the counts) and added_assert = removed_assert = -1.  Every other pair of the call is unaffected.
 * A pure insertion or deletion (after the common prefix and suffix) needs no backtrack: its detail is exact at any D.
 *
 * Resident variant (bench.py's `value` for config C5): tsm_diff_upload copies both sides to HBM once and keeps them in
 * the ctx; every tsm_diff_resident call runs the kernels over them (k_scan over both sides for the line records,
 * k_diff_small - search, rows of V and backtrack of a pair in shared memory, four launches for four sizes of pairs - then
 * k_myers and, when detail != NULL, k_myers_trace for the pairs they leave over: distances above 127 lines, changed
 * regions of more than 4 096 lines) and copies the
 * per-pair results back.  tsm_diff_last_ms: device time (CUDA events on the launching stream) of the last diff call:
 * ms3 = { k_scan over both sides, k_diff_small, k_myers + k_myers_trace of the left-over pairs }. */
int tsm_diff_upload(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, void* stream);
int tsm_diff_resident(tsm_ctx* ctx, int64_t* added, int64_t* removed, tsm_diff_detail* detail, void* stream);
int tsm_diff_last_ms(tsm_ctx* ctx, float* ms3);

/* Changed assertion lines (docs/SPEC.md section 8): the lines the canonical edit script deletes from old or inserts into new
 * that are assertion lines (Rev A), each classified as a scan classifies it.  Deleted lines count under olds->grp, inserted
 * lines under news->grp; both corpora must have the same n_groups (else TSM_E_ARG).  An event is the scan's event of that
 * line (tsm_assert_event) with file = pair index and offsets relative to that side's file.  A pair the detail does not
 * trace (added_assert = removed_assert = -1) contributes nothing.  added / removed / detail are those of
 * tsm_diff_pairs_detail (detail may be NULL).  Any pointer of tsm_diff_asserts may be NULL (that output is skipped); n_aev and
 * n_rev are always set.  If aev_cap or rev_cap is smaller than its count, the call returns TSM_E_CAPACITY with both counts
 * set and everything else filled: size the arrays and call again. */
typedef struct tsm_diff_asserts {
  int64_t* added_counts;     /* [n_groups][TSM_NUM_CATEGORIES], inserted lines by news->grp */
  int64_t* removed_counts;   /* [n_groups][TSM_NUM_CATEGORIES], deleted lines by olds->grp */
  tsm_assert_event* aev; int64_t aev_cap; int64_t n_aev;   /* inserted lines, new side, canonical (file, line_off) order */
  tsm_assert_event* rev; int64_t rev_cap; int64_t n_rev;   /* deleted lines, old side, same order */
} tsm_diff_asserts;
int tsm_diff_pairs_asserts(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                           tsm_diff_detail* detail, tsm_diff_asserts* out, void* stream);
/* The same over the sides of the last tsm_diff_upload (whose grp it keeps); TSM_E_LAYOUT if a grp there was >= n_groups. */
int tsm_diff_resident_asserts(tsm_ctx* ctx, int64_t* added, int64_t* removed, tsm_diff_detail* detail, tsm_diff_asserts* out,
                              void* stream);

/* Rename similarity (docs/SPEC.md section 13): common[c] = sum over the line hashes h (section 3) shared by file cand_old[c] of
 * olds and file cand_new[c] of news of min(W_old(h), W_new(h)), where W_x(h) is the total weight of the lines of x with
 * hash h and a line weighs its bytes, plus 1 for its LF, minus 1 for the CR of a CRLF (git's diffcore-delta count).  The
 * host turns it into git's score floor(common * 60000 / max(size_old, size_new)).  The two corpora may have different file
 * counts; their ext and grp are not used.  An index out of range is TSM_E_ARG; the device needs about 16 B per candidate,
 * and TSM_E_NOMEM is returned when that does not fit.  n_cand = 0 is legal.  One k_scan pass per side gives the line
 * records; then per file the sorted distinct (hash, weight) list (shared memory up to 4 096 lines, a tiled sort through
 * global memory above) and one warp per candidate (persistent warps, binary search of the longer list).
 * tsm_similarity_last_ms: device time of the last call, ms3 = { k_scan over both sides, sort / merge, k_similarity }. */
int tsm_similarity(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, const int32_t* cand_old, const int32_t* cand_new,
                   int64_t n_cand, int64_t* common, void* stream);
int tsm_similarity_last_ms(tsm_ctx* ctx, float* ms3);

/* Edit marks (docs/SPEC.md section 14): the lines the canonical edit script of each pair deletes from olds and inserts into
 * news, one byte per line (1 = deleted / inserted, else 0) in the global line order of each side (line_base: files in order,
 * SPEC sections 2-3).  A pair tsm_diff_pairs_detail does not trace has its whole middle marked (every line between the common
 * prefix and suffix), the one hunk its detail reports.  added / removed / detail are those of tsm_diff_pairs_detail (detail
 * may be NULL).  line_base_old / line_base_new [n_pairs+1] and n_old / n_new are always set; if del_cap < n_old or
 * ins_cap < n_new the call returns TSM_E_CAPACITY with them set (and no diff run): size the arrays and call again.
 * Kernels: the DIFF_MARKS variants of k_diff_small (all four sizes) and k_myers_trace. */
typedef struct tsm_line_marks {
  int64_t* line_base_old; int64_t* line_base_new;   /* [n_pairs+1] */
  uint8_t* del; int64_t del_cap; int64_t n_old;     /* [lines of olds] */
  uint8_t* ins; int64_t ins_cap; int64_t n_new;     /* [lines of news] */
} tsm_line_marks;
int tsm_diff_pairs_marks(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                         tsm_diff_detail* detail, tsm_line_marks* marks, void* stream);

/* Test-case churn (docs/SPEC.md section 16): the cases of every old and every new side in global line order (files in order).
 * A case starts at a header line (section 5, by the side's ext) and runs to the next header line of its file or to the file's
 * end.  pair = the pair index; line = the 0-based header line in that file; n_lines; n_assert = its assertion lines (section 4,
 * Rev A); n_changed = its lines that the canonical script of section 8 deletes (old side) or inserts (new side) - every line of
 * the middle for a pair tsm_diff_pairs_detail does not trace; n_changed_assert = those that are assertion lines.  match (new
 * cases only, else -1): when the case's header line is not inserted and the old line it corresponds to (the k-th line of new
 * that is not inserted corresponds to the k-th line of old that is not deleted, section 14) is a header line, the index of the
 * old case that starts there; else -1.  Matching by case name is left to the host.  n_old and n_new are always set; if
 * old_cap < n_old or new_cap < n_new the call returns TSM_E_CAPACITY with both set (and no diff run): size the arrays and call
 * again.  added / removed / detail are those of tsm_diff_pairs_detail (detail may be NULL).
 * Kernels: k_scan with header events, the diff of tsm_diff_pairs_marks, then per side k_case_heads, k_case_kept, two
 * exclusive scans, k_case_lines and k_case_reduce (csrc/tsm_case_kernels.cuh). */
typedef struct tsm_case { int32_t pair, line, n_lines, n_assert, n_changed, n_changed_assert, match; } tsm_case;
typedef struct tsm_diff_cases {
  tsm_case* old_cases; int64_t old_cap; int64_t n_old;
  tsm_case* new_cases; int64_t new_cap; int64_t n_new;
} tsm_diff_cases;
int tsm_diff_pairs_cases(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                         tsm_diff_detail* detail, tsm_diff_cases* out, void* stream);

/* Assertion edits (docs/SPEC.md section 17): which deleted assertion line of a pair became which inserted one.  chg is filled
 * exactly as tsm_diff_pairs_asserts fills it (same tables, same events in the same order, same capacity rule), except that
 * both event arrays are required here (else TSM_E_ARG).  An edit pairs deleted line chg->rev[rev] with inserted line
 * chg->aev[aev] of the same hunk (both changed assertion lines of a traced pair with the same number of kept lines before
 * them); score = floor(120000 * lcs / (|a| + |b|)) over the stripped lines a, b (section 2), lcs = the length of their longest
 * common byte subsequence.  Per hunk, the candidates with score >= 30000 are taken greedily by score (descending), then rev,
 * then aev (ascending), each line in at most one edit.  Edits are ordered by aev; n_edits <= min(n_aev, n_rev).  n_aev,
 * n_rev and n_edits are always set; if an event cap or edit_cap is smaller than its count, the call returns TSM_E_CAPACITY
 * with all three set: size the arrays and call again.  added / removed / detail are those of tsm_diff_pairs_detail (detail
 * may be NULL).  n_files = 0 is legal.
 * Kernels: the diff of tsm_diff_pairs_marks, then per side k_case_kept, k_edit_flag, two exclusive scans and k_edit_compact,
 * k_classify over the compacted lines, k_edit_ranges, k_edit_score (patterns up to 256 bytes) and k_edit_score_long
 * (csrc/tsm_edit_kernels.cuh); the pairing runs on the host.  tsm_assert_edits_last_ms: ms3 = { k_scan over both sides (device),
 * the diff kernels (device), compact to pairing (host clock, k_classify and the copies included) } of the last call. */
typedef struct tsm_assert_edit { int64_t rev, aev; int32_t score, _pad; } tsm_assert_edit;   /* indices into chg->rev / chg->aev */
int tsm_diff_pairs_assert_edits(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                                tsm_diff_detail* detail, tsm_diff_asserts* chg, tsm_assert_edit* edits, int64_t edit_cap,
                                int64_t* n_edits, void* stream);
int tsm_assert_edits_last_ms(tsm_ctx* ctx, float* ms3);

/* Line provenance (docs/SPEC.md section 14, `tosem-scan blame`): the origin of every line of every new side.  The pairs form
 * chains: prev[i] is the pair whose new side is pair i's old side (prev[i] < i; each pair is the prev of at most one pair), or
 * -1 for a chain head, whose old side's origins are origin_in[in_base[i] .. in_base[i+1]) (in_base [n_pairs+1], ascending;
 * only the heads' ranges are read).  The k-th line of new that the script does not insert takes the origin of the k-th line of
 * old that it does not delete; inserted line j (0-based) of pair i gets {label[i], j + 1}.  TSM_E_ARG for a bad prev, or for
 * a pair whose old side has another line count than its prev's new side or its head range.  line_base_old / line_base_new
 * [n_pairs+1] (may be NULL) and *n_lines (lines of news) are always set; if cap < *n_lines the call returns TSM_E_CAPACITY
 * (no diff run): size origin_out and call again.  added / removed / detail as tsm_diff_pairs_detail (detail may be NULL).
 * Kernels: the diff of tsm_diff_pairs_marks, then k_blame (a warp per chain, longest chains first).
 * tsm_diff_last_ms after this call: ms3 = { k_scan over both sides, k_diff_small, k_myers + k_myers_trace }; tsm_blame_last_ms:
 * the k_blame launch. */
typedef struct tsm_origin { int32_t change, line; } tsm_origin;
int tsm_blame_pairs(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                    tsm_diff_detail* detail, const int32_t* prev, const int32_t* label, const tsm_origin* origin_in,
                    const int64_t* in_base, int64_t* line_base_old, int64_t* line_base_new, tsm_origin* origin_out,
                    int64_t cap, int64_t* n_lines, void* stream);
int tsm_blame_last_ms(tsm_ctx* ctx, float* ms);

/* S9 line / n-gram hashes (docs/SPEC.md section 3; SURVEY.md section 8a S9 - a design choice of the north star, attested by no
 * artefact of the package): the records of every line of every file, files in order, from ONE pass of the scan
 * kernel over the source.  line_base[n_files+1] and *n_lines are always filled; line_hash (SPEC section 3), line_end
 * (file-relative position of the line's LF, or the file size), line_flag (1 = assertion line, SPEC section 4, by the
 * file's ext) and ngram_hash hold `cap` lines each and may be NULL; if cap < *n_lines the call returns TSM_E_CAPACITY
 * so that the caller can size the arrays and call again.  ngram_hash[i] = hash of the window of up to ngram_n
 * consecutive lines of the same file that starts at line i.  tsm_diff_pairs* and tsm_statements use the same pass. */
int tsm_line_hashes(tsm_ctx* ctx, const tsm_corpus* corpus, int64_t* line_base, uint64_t* line_hash, uint32_t* line_end,
                    uint8_t* line_flag, int64_t cap, int64_t* n_lines, int32_t ngram_n, uint64_t* ngram_hash, void* stream);

/* Duplicated test code (docs/SPEC.md section 15, `tosem-scan clones`): the maximal classes of windows of min_lines lines (1 to
 * 1024, else TSM_E_ARG) whose n-gram keys (section 3) are equal, in the global line order of section 3 (files in order).  A class
 * is its fragments [member[j], member[j] + class_len[c]) for class_base[c] <= j < class_base[c+1]; classes are in ascending
 * order of their first fragment, fragments in ascending order of start.  file_dup[f] / file_dup_assert[f]: the lines of file f
 * inside some fragment, and those of them that are assertion lines (section 4, Rev A, by the file's ext).  Any pointer of the
 * result may be NULL (that output is skipped); n_classes and n_members are always set.  class_base holds class_cap + 1
 * entries, class_len class_cap, member member_cap: if class_cap < n_classes or member_cap < n_members the call returns
 * TSM_E_CAPACITY with both counts set: size the arrays and call again (the call is redone).  n_files = 0 is legal.  The
 * grouping table has 28 B per slot and two to four slots per line of the corpus; TSM_E_NOMEM is returned when it does not fit
 * the device's free memory.
 * Kernels: k_scan for the line records, k_ngrams for the keys, then grouping through one open-addressing hash table, the
 * class lengths by warp ballots, a sort of every class' fragments and the coverage (csrc/tsm_clone_kernels.cuh).
 * tsm_clones_last_ms: device time of the last call, ms3 = { k_scan, grouping + classes, members + coverage }. */
typedef struct tsm_clone_result {
  int64_t* line_base;                                    /* [n_files+1] */
  uint32_t* file_dup; uint32_t* file_dup_assert;         /* [n_files] */
  int64_t* class_base; uint32_t* class_len; int64_t class_cap; int64_t n_classes;
  int64_t* member; int64_t member_cap; int64_t n_members;   /* global first line of each fragment */
} tsm_clone_result;
int tsm_clones(tsm_ctx* ctx, const tsm_corpus* corpus, int32_t min_lines, tsm_clone_result* out, void* stream);
int tsm_clones_last_ms(tsm_ctx* ctx, float* ms3);

/* Near-miss duplicated test code (docs/SPEC.md section 21, `tosem-scan clones --blind`): the classes of section 15 over the kept
 * lines of the corpus, whose windows are compared by the blind form of their lines - identifiers, numbers and literals
 * replaced by placeholders, keywords and punctuation kept, whitespace and comments dropped, by a lexer that knows where
 * comments and strings (also those spanning lines) begin and end.  A line is kept when its blind form is not empty; kept lines
 * are numbered globally, files in order.  `out` means what it means for tsm_clones, over kept lines: member and class_len are in
 * kept numbering, file_dup / file_dup_assert count kept lines, and out->line_base is the line_base of section 3.  `blind`
 * (may be NULL): kept_base[f] = the kept lines before file f, kept_line / blind_hash the original global line and the
 * bytes_hash of the blind form of each kept line (kept_cap entries each), file_kept_assert[f] = the kept assertion lines of
 * file f; n_kept is always set.  Any pointer may be NULL; a short kept_cap (with kept_line or blind_hash given), class_cap or
 * member_cap returns TSM_E_CAPACITY with all counts set.  Arguments, streams and memory errors as for tsm_clones.
 * Kernels: k_scan for the line records; k_blind_state (per-line transfer functions of the cross-line lexer states),
 * k_blind_scan (per-file scan of them), k_blind_lines (the blind hash of every line), the compaction of the kept lines
 * (csrc/tsm_blind_kernels.cuh); then the kernels of tsm_clones over the kept lines.
 * tsm_clones_blind_last_ms: device time of the last call, ms4 = { k_scan, lexing + compaction, grouping + classes, members +
 * coverage }. */
typedef struct tsm_blind_result {
  int64_t* kept_base;                                    /* [n_files+1] kept lines before each file (global kept numbering) */
  int64_t* kept_line;                                    /* [kept_cap]  original global line (section 3) of each kept line */
  uint64_t* blind_hash;                                  /* [kept_cap]  bytes_hash of each kept line's blind form */
  uint32_t* file_kept_assert;                            /* [n_files]   kept lines of the file that are assertion lines */
  int64_t kept_cap; int64_t n_kept;
} tsm_blind_result;
int tsm_clones_blind(tsm_ctx* ctx, const tsm_corpus* corpus, int32_t min_lines, tsm_blind_result* blind, tsm_clone_result* out,
                     void* stream);
int tsm_clones_blind_last_ms(tsm_ctx* ctx, float* ms4);

/* Clone churn along a revision history (docs/SPEC.md section 22): which fragments of the clone classes of two revisions a step
 * edits.  old_rev / new_rev are the two revisions (n_files = 0 is legal); pair k pairs file pair_old[k] of old_rev with file
 * pair_new[k] of new_rev, either -1 for none (a deletion or an addition).  A file in no pair is unchanged.  The pairs' edit
 * marks are those of tsm_diff_pairs_marks.  Per side (old_side: old_rev, new_side: new_rev):
 *   clones, blind    what tsm_clones (blind = 0) or tsm_clones_blind (blind != 0; `blind` is read only then) gives for that
 *                    revision alone at min_lines, with the same pointer and capacity rules
 *   changed          [member_cap] per fragment, its marked units (lines, or kept lines with blind): deleted lines on the old
 *                    side, inserted lines on the new side; changed_assert those of them that are assertion lines
 *   state            [member_cap] TSM_FRAG_KEPT (changed = 0), TSM_FRAG_WHOLE (changed = class_len) or TSM_FRAG_EDITED
 *   class_counts     [class_cap][3] per class its kept, edited and whole fragments
 *   status           [class_cap] TSM_CLONE_UNTOUCHED when every fragment is kept, else the first rule that holds:
 *                    old side  REMOVED (every fragment whole), DIVERGED (a kept and an edited one), DROPPED (a kept one), CHANGED
 *                    new side  CREATED (every fragment whole), COPIED (a kept and a whole one), JOINED (a kept one), CHANGED
 * Any output pointer may be NULL (it is skipped); the counts of both sides are always set.  A short class_cap, member_cap or
 * kept_cap (for a given output sized by it) returns TSM_E_CAPACITY with all counts set: size the arrays and call again.
 * TSM_E_ARG for min_lines outside 1..1024, a file index out of range, a file in two pairs of one side or a pair (-1, -1);
 * n_pairs = 0 is legal (nothing is touched).  Memory errors as for tsm_clones.
 * Kernels: k_scan over both revisions; per pair side a view of its revision's line records (k_churn_gather) and the diff of
 * tsm_diff_pairs_marks over the views; k_churn_marks onto the revision lines; per revision the kernels of tsm_clones (or
 * tsm_clones_blind), then k_churn_units, two exclusive scans, k_churn_frags and k_churn_classes
 * (csrc/tsm_clone_churn_kernels.cuh).
 * tsm_clone_churn_last_ms: device time of the last call, ms4 = { k_scan over both revisions, classes of both (lexing included),
 * k_churn_gather + the marks diff, k_churn_marks + the churn kernels of both sides }. */
enum { TSM_FRAG_KEPT = 0, TSM_FRAG_EDITED = 1, TSM_FRAG_WHOLE = 2 };
enum { TSM_CLONE_UNTOUCHED = 0, TSM_CLONE_CHANGED = 1, TSM_CLONE_REMOVED = 2, TSM_CLONE_DIVERGED = 3, TSM_CLONE_DROPPED = 4,
       TSM_CLONE_CREATED = 5, TSM_CLONE_COPIED = 6, TSM_CLONE_JOINED = 7 };
typedef struct tsm_clone_churn_side {
  tsm_clone_result clones;
  tsm_blind_result blind;
  uint32_t* changed; uint32_t* changed_assert; uint8_t* state;   /* [clones.member_cap] */
  uint32_t* class_counts; uint8_t* status;                       /* [clones.class_cap][3], [clones.class_cap] */
} tsm_clone_churn_side;
int tsm_clone_churn(tsm_ctx* ctx, const tsm_corpus* old_rev, const tsm_corpus* new_rev, const int32_t* pair_old,
                    const int32_t* pair_new, int64_t n_pairs, int32_t min_lines, int32_t blind, tsm_clone_churn_side* old_side,
                    tsm_clone_churn_side* new_side, void* stream);
int tsm_clone_churn_last_ms(tsm_ctx* ctx, float* ms4);

/* Test smells (docs/SPEC.md section 18, `tosem-scan smells`): the tests of every file (section-16 cases whose header opens a test
 * by the rule of its family), their bodies and the nine smells below, as one record per test in global line order (files in
 * order, then header line) and the smell bits of every line (its instances; 0 outside test bodies).  Bit k of `smells` and of
 * line_smell[l] is smell k of the TSM_SMELL_* list.  The test-level smells `empty` and `assertion_free`, and `ignored` found on
 * the decorators or the header, are instances on the header line.
 *   file          index of the file in the corpus
 *   line          0-based header line inside the file
 *   body_lines    lines of the body, header line included (section 18's body end)
 *   n_assert      assertion lines of the test (header statement and code lines only: no comment or docstring line)
 *   smells        OR of the smell bits of the test
 *   n_instances   instance lines of the test, one per (line, smell) pair: the sum of popcount(line_smell) over its body
 * line_base[n_files+1] and line_smell hold the lines of every file (line_cap of them), tests test_cap records.  Any output
 * pointer may be NULL (it is skipped); *n_lines and *n_tests are always set.  If line_smell is given with line_cap < *n_lines,
 * or tests with test_cap < *n_tests, the call returns TSM_E_CAPACITY: size the arrays and call again.  n_files = 0 is legal.
 * Kernels: k_scan with the header events, k_line_parens + k_stmt_kinds (section 10), k_case_heads + xscan + k_case_lines (the
 * case spans), k_smell_lines and k_smell_tests (csrc/tsm_smell_kernels.cuh).
 * tsm_smells_last_ms: device time of the last call, ms4 = { k_scan, kinds + case spans, k_smell_lines, k_smell_tests }. */
enum { TSM_SMELL_EMPTY = 0, TSM_SMELL_ASSERTION_FREE = 1, TSM_SMELL_DUPLICATE_ASSERT = 2, TSM_SMELL_REDUNDANT_ASSERT = 3,
       TSM_SMELL_CONDITIONAL_LOGIC = 4, TSM_SMELL_EXCEPTION_HANDLING = 5, TSM_SMELL_SLEEPY = 6, TSM_SMELL_PRINT = 7,
       TSM_SMELL_IGNORED = 8, TSM_N_SMELLS = 9 };
typedef struct tsm_smell_test { int32_t file, line, body_lines, n_assert; uint32_t smells; int32_t n_instances; } tsm_smell_test;
int tsm_smells(tsm_ctx* ctx, const tsm_corpus* corpus, int64_t* line_base, uint16_t* line_smell, int64_t line_cap, int64_t* n_lines,
               tsm_smell_test* tests, int64_t test_cap, int64_t* n_tests, void* stream);
int tsm_smells_last_ms(tsm_ctx* ctx, float* ms4);

/* Similar tests (docs/SPEC.md section 23, `tosem-scan similar-tests`): the pairs of tests of section 18 whose sequences of kept
 * blind lines (section 21, header line included) are at least min_similarity % alike, and the classes they link.  A test is
 * compared when it has at least min_lines kept lines (min_lines >= 1, else TSM_E_ARG).  Tests a < b form a pair when both are
 * compared and 200 * lcs >= P * (k(a) + k(b)), lcs being the longest common subsequence of their sequences (two kept lines are
 * equal when their blind hashes are), k their lengths and P = min_similarity in 1..100 (else TSM_E_ARG).
 *   tests, test_kept   every test, exactly as tsm_smells returns them (global line order), and its kept lines k (test_cap each)
 *   pairs              every pair {a, b, lcs, score}, score = floor(120000 * lcs / (k(a) + k(b))), ascending (a, b) (pair_cap)
 *   class_base/member  the connected components of at least two tests of the graph of the pairs (single linkage), ordered by
 *                      their smallest test, members ascending: class c is member[class_base[c] .. class_base[c+1])
 *                      (class_base holds class_cap + 1 entries, member member_cap)
 *   n_candidates       the candidate pairs whose LCS was computed (those that pass the exact prefix and size filters)
 *                      (a count of work, not of the answer: lines of equal counts are ordered by their slot in a hash table
 *                      filled by atomics, so the prefixes, and with them this count, may differ from call to call; the
 *                      pairs do not)
 * Any output pointer may be NULL (it is skipped); every count is always set.  A short cap for a given output returns
 * TSM_E_CAPACITY with every count set: size the arrays and call again.  n_files = 0 is legal.  Memory errors as for tsm_clones.
 * Kernels: k_scan with the header events, the case spans and smell stage of tsm_smells, the lexer of tsm_clones_blind; then
 * k_st_tests, a count table of the blind hashes (k_st_count, k_st_order), the prefix tokens and their posting lists (k_st_prefix,
 * k_st_lists), a scan of the lists' candidate counts (k_st_csums, k_st_capply), and per chunk of that virtual candidate space
 * k_st_enum (filters) and k_st_verify (bit-parallel LCS, one warp per candidate) (csrc/tsm_simtest_kernels.cuh).  The classes are
 * formed on the host from the pairs.
 * tsm_similar_tests_last_ms: device time of the last call, ms4 = { k_scan, case spans + smell stage + lexer, token table +
 * prefixes + posting lists + enumeration, verification }. */
typedef struct tsm_similar_pair { int32_t a, b; uint32_t lcs, score; } tsm_similar_pair;
typedef struct tsm_similar_result {
  tsm_smell_test* tests; uint32_t* test_kept; int64_t test_cap; int64_t n_tests;
  tsm_similar_pair* pairs; int64_t pair_cap; int64_t n_pairs;
  int64_t* class_base; int64_t class_cap; int64_t n_classes;
  int32_t* member; int64_t member_cap; int64_t n_members;
  int64_t n_candidates;
} tsm_similar_result;
int tsm_similar_tests(tsm_ctx* ctx, const tsm_corpus* corpus, int32_t min_lines, int32_t min_similarity, tsm_similar_result* out,
                      void* stream);
int tsm_similar_tests_last_ms(tsm_ctx* ctx, float* ms4);

/* Test-smell churn (docs/SPEC.md section 19): the section-16 cases and the section-18 tests of both sides of every revision pair,
 * and per test how many of its smell instances the revision adds (new side) or removes (old side).  cases is filled exactly as
 * tsm_diff_pairs_cases fills it.  old_tests / new_tests are the tsm_smell_test records of tsm_smells over each side's corpus
 * alone, with file = the pair index; old_churn / new_churn hold one tsm_test_churn per test, in the same order:
 *   case_idx      index of the test's case among the cases of its side (the case that starts at its header line)
 *   instances[k]  body lines of the test with smell bit k (their sum is n_instances)
 *   churned[k]    those of them that are added instances (new side) or removed instances (old side): the line is inserted
 *                 (deleted), or it is kept and the corresponding line of the other side (section 14) lacks bit k.
 * Any output pointer may be NULL (it is skipped).  cases.n_old / n_new, n_old_tests and n_new_tests are always set; if a given
 * output's cap is smaller than its count, the call returns TSM_E_CAPACITY with all four set (and no diff run): size the arrays
 * and call again.  added / removed / detail are those of tsm_diff_pairs_detail (detail may be NULL).  n_files = 0 is legal.
 * Kernels: k_scan with header events, per side the case spans and the smell stage of tsm_smells, the diff of
 * tsm_diff_pairs_marks, the case kernels of tsm_diff_pairs_cases and k_smell_churn per side (csrc/tsm_smell_kernels.cuh).
 * tsm_diff_smells_last_ms: device time of the last call, ms4 = { k_scan over both sides, the smell stage of both sides (case
 * spans included), k_diff_small + k_myers + k_myers_trace, case records + k_smell_churn }. */
typedef struct tsm_test_churn { int32_t case_idx; int32_t instances[TSM_N_SMELLS]; int32_t churned[TSM_N_SMELLS]; } tsm_test_churn;
typedef struct tsm_diff_smells {
  tsm_diff_cases cases;
  tsm_smell_test* old_tests; tsm_test_churn* old_churn; int64_t old_test_cap; int64_t n_old_tests;
  tsm_smell_test* new_tests; tsm_test_churn* new_churn; int64_t new_test_cap; int64_t n_new_tests;
} tsm_diff_smells;
int tsm_diff_pairs_smells(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                          tsm_diff_detail* detail, tsm_diff_smells* out, void* stream);
int tsm_diff_smells_last_ms(tsm_ctx* ctx, float* ms4);

/* Moved code (docs/SPEC.md section 20, git's `--color-moved=blocks`): the blocks of changed lines that a step moves.  A pair's
 * step is its grp; it must be the same on both sides and below olds->n_groups (grp NULL: every pair in step 0), else TSM_E_ARG.
 * Deleted and inserted lines of one step match when their line hashes (section 3) are equal; a block is a stretch of a run
 * (maximal changed lines of one file on one side) that follows one matching diagonal as far as both runs allow, with at least 20
 * alphanumeric bytes.  old_blocks / new_blocks hold the blocks of each side in ascending line order:
 *   line      global line of the block's first line on its side (marks.line_base_* give the files)
 *   partner   global line on the other side of the first line it matches (the smallest of the longest reach)
 *   n_lines   lines of the block
 *   n_assert  its assertion lines (section 4, Rev A, by the side's ext)
 * marks is filled as tsm_diff_pairs_marks fills it, except that a moved line has bit 1 set too (value 3).  Any output pointer may
 * be NULL (it is skipped); marks.n_old / n_new, n_old_blocks and n_new_blocks are always set.  If a given output's cap is smaller
 * than its count, the call returns TSM_E_CAPACITY with all four set: size the arrays and call again.  added / removed / detail
 * are those of tsm_diff_pairs_detail (detail may be NULL).  n_files = 0 is legal.
 * Kernels: the diff of tsm_diff_pairs_marks, then k_move_lines, k_move_compact, k_move_insert, k_move_scatter, k_move_reach,
 * k_move_starts, k_move_runs and k_move_mark (csrc/tsm_move_kernels.cuh).  The reach costs one comparison per matching (deleted, inserted)
 * pair of a step: quadratic in a line that repeats on both sides of one step.
 * tsm_moves_last_ms: device time of the last call, ms4 = { k_scan over both sides, k_diff_small + k_myers + k_myers_trace,
 * k_move_lines to k_move_reach (the join and the reach), k_move_starts + k_move_runs + k_move_mark (the blocks) }. */
typedef struct tsm_move_block { int64_t line, partner; int32_t n_lines, n_assert; } tsm_move_block;
typedef struct tsm_diff_moves {
  tsm_line_marks marks;
  tsm_move_block* old_blocks; int64_t old_cap; int64_t n_old_blocks;
  tsm_move_block* new_blocks; int64_t new_cap; int64_t n_new_blocks;
} tsm_diff_moves;
int tsm_diff_pairs_moves(tsm_ctx* ctx, const tsm_corpus* olds, const tsm_corpus* news, int64_t* added, int64_t* removed,
                         tsm_diff_detail* detail, tsm_diff_moves* out, void* stream);
int tsm_moves_last_ms(tsm_ctx* ctx, float* ms4);

/* Body statements (docs/SPEC.md section 10; Important-files/ML-Analysis-v4.xlsx!Apollo:R2-R26, golden G2): the
 * kind of every line of every file - 0 blank, 1 first line of a statement, 2 continuation (lines
 * are joined while the parentheses are open).  line_base[n_files+1] and *n_lines are always filled;
 * line_end (file-relative end of each line) and line_kind hold `cap` lines: if cap < *n_lines the call
 * returns TSM_E_CAPACITY so that the caller can size the arrays and call again. */
int tsm_statements(tsm_ctx* ctx, const tsm_corpus* corpus, int64_t* line_base, uint32_t* line_end,
                   uint8_t* line_kind, int64_t cap, int64_t* n_lines, void* stream);

/* S10 reduce (RQs/taxonomy_test2.csv -> RQs/RQ3/tests_strategy_rq32.csv, RQs/RQ4/
 * tests_methods_v2.csv): out[f*n_repos+r] = distinct case ids with flags[row*n_flags+f] != 0 in
 * repo r; cases_per_repo[r] = distinct case ids of repo r. Host arrays; integer work on device. */
int tsm_reduce(tsm_ctx* ctx, const uint8_t* flags, const int32_t* repo, const int32_t* case_id,
               int32_t n_rows, int32_t n_flags, int32_t n_repos, int32_t n_cases,
               int64_t* out, int64_t* cases_per_repo, void* stream);

/* ---- host-only helpers (no CUDA context needed) ------------------------------------------- */
/* Pinned host memory for arenas/results (cudaHostAlloc); returns NULL on failure. */
void* tsm_host_alloc(int64_t bytes);
void tsm_host_free(void* p);
/* Arena size (multiple of TSM_ALIGN) for files of the given sizes; fills off[n+1]. <0 on overflow. */
int64_t tsm_layout(const int32_t* len, int32_t n_files, int32_t* off);
/* Deterministic synthetic corpus (SURVEY.md section 8d; std::mt19937_64, one engine per file).
 * size_law 0: every file exactly fixed_size bytes; 1: truncated power law pdf ~ x^-1.5 on
 * [128 B, 1 MiB] rounded up to whole lines.  Slot i holds logical file first_index + i*index_stride,
 * so ranks generate disjoint round-robin shards of one logical corpus.  Two steps: tsm_gen_sizes
 * -> tsm_layout -> tsm_gen_fill. */
int tsm_gen_sizes(uint64_t seed, int32_t n_files, int size_law, int32_t fixed_size, int32_t first_index,
                  int32_t index_stride, int32_t* len, uint8_t* ext, uint16_t* grp, int32_t n_groups);
int tsm_gen_fill(uint64_t seed, int32_t n_files, int size_law, int32_t first_index, int32_t index_stride,
                 const int32_t* off, const int32_t* len, const uint8_t* ext, uint8_t* arena);
/* new = old with Poisson(lambda) line edits (insert/delete/replace of Geometric(0.4) runs). Returns
 * bytes written to dst (<= cap) or <0. */
int64_t tsm_gen_edit(uint64_t seed, const uint8_t* src, int32_t src_len, double lambda,
                     uint8_t* dst, int64_t cap);

/* BASELINE config C5: n (old, new) revision pairs; old ~ the size law 1 with the target clamped to cap bytes,
 * new = old with Poisson(lambda) line edits.  Slot i holds logical pair index[i], or first_index + i*index_stride
 * when index is NULL (ranks take size-balanced shares of one logical pair set through index lists).
 * tsm_gen_pair_sizes -> tsm_layout (twice) -> tsm_gen_pair_fill. */
int tsm_gen_pair_sizes(uint64_t seed, int32_t n_pairs, const int32_t* index, int32_t first_index, int32_t index_stride,
                       int32_t cap, double lambda, int32_t* len_old, int32_t* len_new, uint8_t* ext);
int tsm_gen_pair_fill(uint64_t seed, int32_t n_pairs, const int32_t* index, int32_t first_index, int32_t index_stride,
                      int32_t cap, double lambda, const uint8_t* ext, const int32_t* off_old, const int32_t* len_old,
                      uint8_t* arena_old, const int32_t* off_new, const int32_t* len_new, uint8_t* arena_new);

#ifdef __cplusplus
}
#endif
#endif
