// tosem_scan_cli.cpp - `tosem-scan`, the C++ host driver of the corpus-scan loop.
//
// The reference package ships no entry point to stay compatible with (SURVEY.md section 0, section 8b); what it
// ships are the loop's OUTPUT SCHEMAS, and this driver writes exactly those:
//   raw rows      fileName,extension,test_name,method,statement,counts,category
//                 (Important-files/ML-Testing-v1.xlsx!apollo_tests:R1)
//   per-file      Id,FileName,total assert,assertion   ("32:assertEqual, 15:assertIn, ...")
//                 (selection/completed-labels/Release-Meta-tpot.csv:1-2)
//   RQ tables     RQs/RQ3/tests_strategy_rq32.csv, RQs/RQ4/tests_methods_v2.csv from
//                 RQs/taxonomy_test2.csv
//   churn         cloc,added,removed  (Important-files/ML-Testing-v1.xlsx!projects:R1)
// All CSVs are CRLF, UTF-8, RFC-4180 quoted, like every CSV the package ships.
//
// Host work only: tree walk + test-file selection (S0), extension / test_name tags (S1, S2), packing
// into the pinned byte arena, method strings (S3, host side of SPEC section 5), CSV.  Every byte of the scan
// itself goes through libtosemscan.so (sm_90a kernels); there is no CPU fallback.
//
//   tosem-scan scan   <project-root>... [--rows F] [--summary F] [--gpus N] [--all-files] [--batch-bytes N]
//   tosem-scan reduce <taxonomy.csv> [--strategy F] [--methods F] [--properties F] [--correlate F] [--correlate-tex F] [--correlate-counts F] [--correlate-merged F]
//   tosem-scan diff   <old-root> <new-root> [--out F] [--asserts F] [--assert-churn F] [--cases F] [--assert-edits F] [--smells F]
//                     [--lexical] [--moves F] [--clones F] [--similar-tests F] [--min-lines N] [--similarity P] [--links F] [--find-renames N] [--batch-bytes N]
//   tosem-scan body   <project-root>... [--batch-bytes N] [--out F]
//   tosem-scan releases <snapshot-root>=<tag>... | --git <repository> [<revision>...]   [--batch-bytes N] [--out F]
//   tosem-scan history <git-repository> [--rev R] [--max-commits N] [--all-files] [--dry-run] [--out F] [--asserts F] [--assert-churn F] [--cases F]
//                      [--assert-edits F] [--smells F] [--lexical] [--moves F] [--clones F] [--similar-tests F] [--links F] [--find-renames N] [--batch-bytes N]
//   tosem-scan blame <git-repository> [--rev R] [--max-commits N] [--all-files] [--find-renames N] [--batch-bytes N] [--out F] [--asserts F]
//   tosem-scan clones <project-root>... | --git <repository> [--rev R]   [--min-lines N] [--blind] [--all-files] [--out F]
// Every command that scans files does it with scan_batches: batches of at most --batch-bytes of arena (clones: all files in one),
// one context, the next batch read while the current one is scanned.  Every command that diffs revision pairs (diff, history,
// blame) does it with pair_batches: batches of at most --batch-bytes per side (with --moves: whole steps), one context shared
// with the rename pairing.
#include <algorithm>
#include <atomic>
#include <cctype>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fcntl.h>
#include <unistd.h>
#include <filesystem>
#include <fstream>
#include <functional>
#include <future>
#include <map>
#include <memory>
#include <numeric>
#include <optional>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>
#include <nccl.h>

#include "../../include/tosemscan.h"
#include "git_store.hpp"
#include "tsm_names.hpp"

namespace fs = std::filesystem;
using tsm_names::case_name;
using tsm_names::is_w;
using tsm_names::method_string;

static bool die(const std::string& m) { fprintf(stderr, "tosem-scan: %s\n", m.c_str()); exit(2); return false; }
static void ck(int rc, const char* what) { if (rc != TSM_OK) die(std::string(what) + ": " + tsm_strerror(rc)); }

static std::string lower(std::string s) { for (char& c : s) if (c >= 'A' && c <= 'Z') c = (char)(c + 32); return s; }

// ---------------------------------------------------------------------------------- CSV (RFC 4180, CRLF)
static std::string csv_cell(const std::string& s) {
  if (s.find_first_of(",\"\r\n") == std::string::npos) return s;
  std::string o = "\"";
  for (char c : s) { if (c == '"') o += '"'; o += c; }
  return o + "\"";
}
static void csv_row(std::ostream& os, const std::vector<std::string>& cells) {
  for (size_t i = 0; i < cells.size(); ++i) { if (i) os << ','; os << csv_cell(cells[i]); }
  os << "\r\n";
}
static std::vector<std::vector<std::string>> csv_read(const std::string& path) {
  std::ifstream in(path, std::ios::binary);
  if (!in) die("cannot open " + path);
  std::string data((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  if (data.compare(0, 3, "\xEF\xBB\xBF") == 0) data.erase(0, 3);
  std::vector<std::vector<std::string>> rows;
  std::vector<std::string> row;
  std::string cell;
  bool q = false, any = false;
  for (size_t i = 0; i < data.size(); ++i) {
    const char c = data[i];
    if (q) {
      if (c == '"') { if (i + 1 < data.size() && data[i + 1] == '"') { cell += '"'; ++i; } else q = false; }
      else cell += c;
    } else if (c == '"') { q = true; any = true; }
    else if (c == ',') { row.push_back(cell); cell.clear(); any = true; }
    else if (c == '\n' || c == '\r') {
      if (c == '\r' && i + 1 < data.size() && data[i + 1] == '\n') ++i;
      if (any || !cell.empty()) { row.push_back(cell); rows.push_back(row); }
      row.clear(); cell.clear(); any = false;
    } else { cell += c; any = true; }
  }
  if (any || !cell.empty()) { row.push_back(cell); rows.push_back(row); }
  return rows;
}

// ---------------------------------------------------------------------------------- S0-S2: walk and tag
struct FileEntry {
  std::string rel, abs; int ext; int grp; int64_t size;
  std::shared_ptr<const std::vector<uint8_t>> blob;       // set instead of `abs` when the bytes come from a git object store
};

static int ext_tag(const std::string& rel) {               // S1
  const size_t d = rel.rfind('.');
  if (d == std::string::npos || rel.find('/', d) != std::string::npos) return TSM_EXT_OTHER;
  const std::string e = rel.substr(d + 1);
  if (e == "py") return TSM_EXT_PY;
  if (e == "cc") return TSM_EXT_CC;
  if (e == "cpp") return TSM_EXT_CPP;
  if (e == "java") return TSM_EXT_JAVA;
  if (e == "c") return TSM_EXT_C;
  if (e == "h") return TSM_EXT_H;
  return TSM_EXT_OTHER;
}
static const char* ext_name(int t) { static const char* n[] = {"", "py", "cc", "cpp", "java", "c", "h"}; return n[t]; }
static std::string base_name(const std::string& p) { const size_t s = p.rfind('/'); return s == std::string::npos ? p : p.substr(s + 1); }

static std::string test_name_tag(const std::string& rel, bool fixture) {   // S2 (mock / Module: parity unpinned, omitted)
  std::string t;
  if (rel.rfind("external/", 0) == 0) t = "external";
  else if (rel.find("integration") != std::string::npos) t = "integration";
  else if (rel.find("regression") != std::string::npos) t = "regression";
  else if (rel.find("swarming") != std::string::npos) t = "swarming";
  else t = "unit_test";
  bool proto = false, smoke = false;
  size_t p = 0;
  while (p < rel.size()) {
    size_t q = rel.find('/', p);
    if (q == std::string::npos) break;                     // last component is the file name
    const std::string comp = rel.substr(p, q - p);
    if (comp.rfind("protobuf-", 0) == 0) proto = true;
    if (comp == "smoke") smoke = true;
    p = q + 1;
  }
  if (proto) t += ", Protocol Buffers";
  if (smoke) t += ", smoke";
  if (fixture) t += ", Fixture";
  return t;
}

// Which files of a revision a step walk keeps: the study's selection (S0 / S1, or every file with --all-files) or that of the
// links (section 27: every file with a lexer family, under any path).
using Select = std::function<bool(const std::string&)>;
static bool study_file(const std::string& rel) { return lower(rel).find("test") != std::string::npos && ext_tag(rel) != TSM_EXT_OTHER; }
static bool link_file(const std::string& rel) { return ext_tag(rel) != TSM_EXT_OTHER; }
static Select selection(bool all_files) { return all_files ? Select([](const std::string&) { return true; }) : Select(study_file); }

static void walk(const std::string& root, int grp, bool all_files, std::vector<FileEntry>& out) {
  std::vector<fs::path> paths;
  for (auto it = fs::recursive_directory_iterator(root, fs::directory_options::skip_permission_denied);
       it != fs::recursive_directory_iterator(); ++it)
    if (it->is_regular_file() && !it->is_symlink()) paths.push_back(it->path());
  std::sort(paths.begin(), paths.end());
  for (const fs::path& p : paths) {
    const std::string rel = fs::relative(p, root).generic_string();
    const int ext = ext_tag(rel);
    if (!all_files) {
      if (lower(rel).find("test") == std::string::npos) continue;          // S0: path contains `test`
      if (ext == TSM_EXT_OTHER) continue;                                   // S1: no rows for other extensions
    }
    out.push_back({rel, p.string(), ext, grp, (int64_t)fs::file_size(p), nullptr});
  }
}

// ---------------------------------------------------------------------------------- scan
struct HostFree { void operator()(uint8_t* p) const { tsm_host_free(p); } };
struct CtxFree { void operator()(tsm_ctx* c) const { tsm_destroy(c); } };
// A context at the smallest size, for calls that grow it to what they need (reduce, rename pairing, the diffs of revision pairs).
static std::unique_ptr<tsm_ctx, CtxFree> small_context() {
  tsm_ctx* ctx = nullptr;
  ck(tsm_create(&ctx, 0, 1 << 20, 16, 1, 0), "tsm_create");
  return std::unique_ptr<tsm_ctx, CtxFree>(ctx);
}

struct Batch {                                             // one packed arena of files; move-only, it owns its pinned arena
  std::vector<uint32_t> idx;                               // indices into the walk's file list, ascending
  std::vector<int32_t> off, len;
  std::vector<uint8_t> ext;
  std::vector<uint16_t> grp;
  std::unique_ptr<uint8_t[], HostFree> arena;
  int64_t bytes = 0;                                       // arena bytes (padded file sizes)
  size_t count() const { return idx.size(); }
  tsm_corpus corpus(int32_t n_groups) const {
    return {arena.get(), off.data(), len.data(), ext.data(), grp.data(), (int32_t)len.size(), n_groups};
  }
};

// The files of lengths B.len laid out by tsm_layout (B.off, B.bytes) in a zeroed pinned arena, their ext / grp tags zero; the
// caller fills the bytes and the tags.
static void alloc_arena(Batch& B) {
  const size_t n = B.len.size();
  B.off.resize(n + 1); B.ext.assign(n, 0); B.grp.assign(n, 0);
  B.bytes = tsm_layout(B.len.data(), (int32_t)n, B.off.data());
  if (B.bytes < 0) die("batch does not fit an int32-indexed arena");
  B.arena.reset((uint8_t*)tsm_host_alloc(std::max<int64_t>(B.bytes, 128)));
  if (!B.arena) die("pinned arena allocation failed (no CUDA device? there is no CPU fallback)");
  memset(B.arena.get(), 0, (size_t)std::max<int64_t>(B.bytes, 128));
}

// Byte strings held in memory, packed into one arena in order (ext / grp tags zero).
static Batch pack(const std::vector<const std::vector<uint8_t>*>& bytes) {
  Batch B;
  for (const std::vector<uint8_t>* v : bytes) B.len.push_back((int32_t)v->size());
  alloc_arena(B);
  for (size_t i = 0; i < bytes.size(); ++i) if (B.len[i]) memcpy(B.arena.get() + B.off[i], bytes[i]->data(), bytes[i]->size());
  return B;
}

static bool read_file(const std::string& path, uint8_t* dst, int64_t size) {   // false on a short read
  const int fd = open(path.c_str(), O_RDONLY);
  int64_t got = 0;
  while (fd >= 0 && got < size) {
    const ssize_t r = read(fd, dst + got, (size_t)(size - got));
    if (r <= 0) break;
    got += r;
  }
  if (fd >= 0) close(fd);
  return got == size;
}

static void load_batch(const std::vector<FileEntry>& files, Batch& b) {
  const size_t n = b.count();
  b.len.resize(n);
  for (size_t i = 0; i < n; ++i) b.len[i] = (int32_t)files[b.idx[i]].size;
  alloc_arena(b);
  for (size_t i = 0; i < n; ++i) { b.ext[i] = (uint8_t)files[b.idx[i]].ext; b.grp[i] = (uint16_t)files[b.idx[i]].grp; }
  // the reads of a batch run on a few host threads (a source tree is many small files: latency-bound)
  const unsigned nt = std::max(1u, std::min({std::thread::hardware_concurrency(), 32u, (unsigned)((n + 63) / 64)}));
  std::atomic<long> bad{-1};
  auto reader = [&](unsigned t) {
    for (size_t i = t; i < n && bad.load(std::memory_order_relaxed) < 0; i += nt) {
      if (files[b.idx[i]].blob) { if (b.len[i]) memcpy(b.arena.get() + b.off[i], files[b.idx[i]].blob->data(), (size_t)b.len[i]); continue; }
      if (!read_file(files[b.idx[i]].abs, b.arena.get() + b.off[i], b.len[i])) bad.store((long)i);
    }
  };
  std::vector<std::thread> th;
  for (unsigned t = 1; t < nt; ++t) th.emplace_back(reader, t);
  reader(0);
  for (std::thread& x : th) x.join();
  if (bad.load() >= 0) die("short read: " + files[b.idx[(size_t)bad.load()]].abs);
}

// The files `indices` (ascending) cut in order into batches of at most max_bytes of arena (128-byte padded sizes) and max_files
// files; a file larger than max_bytes is a batch of its own.  Not loaded yet: Batch::bytes is the arena load_batch will lay out.
static std::vector<Batch> plan_batches(const std::vector<FileEntry>& files, const std::vector<uint32_t>& indices, int64_t max_bytes,
                                       size_t max_files) {
  std::vector<Batch> out;
  for (uint32_t i : indices) {
    const int64_t padded = (files[i].size + 127) / 128 * 128;
    if (out.empty() || out.back().bytes + padded > max_bytes || out.back().count() >= max_files) out.emplace_back();
    out.back().idx.push_back(i);
    out.back().bytes += padded;
  }
  return out;
}
static std::vector<uint32_t> all_of(const std::vector<FileEntry>& files) {
  std::vector<uint32_t> v(files.size());
  std::iota(v.begin(), v.end(), 0u);
  return v;
}
// Batches of every command but `scan`: --batch-bytes defaults to kBatch (bytes per side of a diff or of the tsm_similarity call
// of rename pairing, arena bytes of a scan), and a scan batch holds at most kBatchFiles files.
static const int64_t kBatch = 512ll << 20;
static const size_t kBatchFiles = 1u << 19;

static void cu_ck(cudaError_t e, const char* what) { if (e != cudaSuccess) die(std::string(what) + ": " + cudaGetErrorString(e)); }
static void nccl_ck(ncclResult_t r, const char* what) { if (r != ncclSuccess) die(std::string(what) + ": " + ncclGetErrorString(r)); }

// tsm_scan of one packed batch of `bytes` with the events `flags` asks for in aev / hev.  The host arrays start at bytes / 8 + 1024
// entries; a denser batch returns TSM_E_CAPACITY with both counts, and its events are downloaded again into arrays of that size.
static void scan_events(tsm_ctx* ctx, const tsm_corpus& c, int64_t bytes, tsm_result& r, uint32_t flags, cudaStream_t st,
                        std::vector<tsm_assert_event>& aev, std::vector<tsm_header_event>& hev) {
  const bool want_a = flags & TSM_SCAN_ASSERT_EVENTS, want_h = flags & TSM_SCAN_HEADER_EVENTS;
  auto size = [&](int64_t na, int64_t nh) {
    aev.resize(want_a ? (size_t)na : 0); hev.resize(want_h ? (size_t)nh : 0);
    r.aev = want_a ? aev.data() : nullptr; r.aev_cap = (int64_t)aev.size();
    r.hev = want_h ? hev.data() : nullptr; r.hev_cap = (int64_t)hev.size();
  };
  const int64_t cap = std::max<int64_t>(bytes / 8 + 1024, 1024);
  size(cap, cap);
  int rc = tsm_scan(ctx, &c, &r, flags, st);
  if (rc == TSM_E_CAPACITY && (r.n_aev > cap || r.n_hev > cap)) {
    size(std::max<int64_t>(r.n_aev, 1), std::max<int64_t>(r.n_hev, 1));
    rc = tsm_download(ctx, &r, st);
  }
  ck(rc, "tsm_scan");
  aev.resize(want_a ? (size_t)r.n_aev : 0); hev.resize(want_h ? (size_t)r.n_hev : 0);
}

// One scanned batch: per-file records, the count table ([n_groups][K] by group, [K] over the batch, then the 4 totals of
// tsm_result), the events `flags` asked for, and the context that holds the batch for more calls on it.
struct Scanned {
  const std::vector<tsm_file_stat>& stats;
  const std::vector<int64_t>& counts;
  const std::vector<tsm_assert_event>& aev;
  const std::vector<tsm_header_event>& hev;
  tsm_ctx* ctx;
};
using ScanFn = std::function<void(const Batch&, const Scanned&)>;

// Every batch of `batches` loaded, scanned with `flags` on one context of `device` (sized to the largest batch) and handed to
// `fn`.  Host pipeline: while the GPU scans batch b (tsm_scan overlaps its H2D slabs with the kernels), a background task
// already reads the files of batch b + 1 into its pinned arena.  At most two arenas are alive: a batch's arena is freed as soon
// as `fn` returns.  No batches: no context, `fn` never runs.
static void scan_batches(const std::vector<FileEntry>& files, std::vector<Batch>& batches, int device, int32_t n_groups, uint32_t flags,
                         const ScanFn& fn) {
  if (batches.empty()) return;
  cu_ck(cudaSetDevice(device), "cudaSetDevice");
  cudaStream_t st;
  cu_ck(cudaStreamCreate(&st), "cudaStreamCreate");
  int64_t max_arena = 1 << 20; int32_t max_files = 16;
  for (const Batch& b : batches) { max_arena = std::max(max_arena, b.bytes + 4096); max_files = std::max(max_files, (int32_t)b.count()); }
  tsm_ctx* ctx = nullptr;
  ck(tsm_create(&ctx, device, max_arena, max_files, n_groups, 0), "tsm_create");
  auto load = [&](size_t b) {
    return std::async(std::launch::async, [&files, &batches, b, device] { cudaSetDevice(device); load_batch(files, batches[b]); });
  };
  std::future<void> next = load(0);
  std::vector<tsm_file_stat> stats;
  std::vector<int64_t> counts;
  std::vector<tsm_assert_event> aev;
  std::vector<tsm_header_event> hev;
  const size_t K = TSM_NUM_CATEGORIES;
  for (size_t b = 0; b < batches.size(); ++b) {
    Batch& B = batches[b];
    next.get();
    if (b + 1 < batches.size()) next = load(b + 1);
    stats.resize(B.count());
    counts.assign((size_t)(n_groups + 1) * K + 4, 0);
    tsm_result r{};
    r.stats = stats.data(); r.group_counts = counts.data(); r.global_counts = counts.data() + (size_t)n_groups * K;
    scan_events(ctx, B.corpus(n_groups), B.bytes, r, flags, st, aev, hev);
    std::copy(r.totals, r.totals + 4, counts.end() - 4);
    fn(B, Scanned{stats, counts, aev, hev, ctx});
    B.arena.reset();
    std::vector<int32_t>().swap(B.off); std::vector<int32_t>().swap(B.len);
  }
  tsm_destroy(ctx);
  cudaStreamDestroy(st);
}

// The statement of an assertion event (the statement may be longer than the 16-bit event field: its end is re-derived on the
// host if saturated) and its category cell (the verbatim identifier for 127, docs/SPEC.md section 6).
static std::string event_statement(const uint8_t* base, int32_t size, const tsm_assert_event& ev) {
  uint32_t sl = ev.stmt_len;
  if (sl == 65535) { const uint8_t* p = base + ev.stmt_off; uint32_t e = 0, last = 0; while (ev.stmt_off + e < (uint32_t)size && p[e] != '\n' && p[e] != '(') { if (!is_w(p[e])) last = e + 1; ++e; } sl = last; }
  return std::string((const char*)base + ev.stmt_off, sl);
}
static std::string event_category(const uint8_t* base, const tsm_assert_event& ev) {
  return ev.cat == 127 ? std::string((const char*)base + ev.ident_off, ev.ident_len) : std::string(tsm_category_name(ev.cat));
}
// The assertion cell of a per-file row, "n:category, ...": the categories in first-seen order, stably sorted by count, descending.
struct CategoryHist {
  std::map<std::string, int64_t> n;
  std::vector<std::string> order;
  void add(const std::string& cat) { if (!n.count(cat)) order.push_back(cat); n[cat]++; }
  std::string cell() {
    std::stable_sort(order.begin(), order.end(), [&](const std::string& x, const std::string& y) { return n[x] > n[y]; });
    std::string a;
    for (const std::string& c : order) { if (!a.empty()) a += ", "; a += std::to_string(n[c]) + ":" + c; }
    return a;
  }
};

// The 1-based line numbers of ascending offsets into one file, counting the newlines from the previous offset on.
struct LineCounter {
  const uint8_t* base;
  uint32_t pos = 0;
  int64_t line = 1;
  int64_t at(uint32_t off) { for (; pos < off; ++pos) line += base[pos] == '\n'; return line; }
};

// The raw rows (fileName, extension, test_name, method, statement, counts, category: ML-Testing-v1.xlsx!apollo_tests:R1) and
// the summary row (Id, FileName, total assert, assertion: Release-Meta-tpot.csv:1-2) of one file, from its events.
static void render_file(const FileEntry& f, int64_t id, const uint8_t* base, int32_t size, uint32_t slot, const tsm_file_stat& st,
                        const std::vector<tsm_assert_event>& aev, size_t& ai, const std::vector<tsm_header_event>& hev, size_t& hi,
                        bool want_rows, bool want_sum, std::string& rows_txt, std::string& sum_txt) {
  struct Row { int64_t hdr; std::string stmt; int cat; std::string catname; int64_t count; bool fixture; std::string method; };
  std::vector<Row> rows;
  std::map<std::pair<int64_t, std::string>, size_t> index;
  CategoryHist hist;
  int64_t cur_hdr = -1; bool cur_fix = false; std::string cur_method = "xxxx";
  while (ai < aev.size() && aev[ai].file == slot) {
    const tsm_assert_event& ev = aev[ai++];
    while (hi < hev.size() && hev[hi].file == slot && hev[hi].line_off <= ev.line_off) {   // governing header
      const tsm_header_event& h = hev[hi++];
      cur_hdr = h.line_off; cur_fix = (h.kind & 1u) != 0;
      cur_method = method_string(f.ext, base + h.line_off, h.line_len);
    }
    const std::string stmt = event_statement(base, size, ev), cat = event_category(base, ev);
    auto key = std::make_pair(cur_hdr, stmt);
    auto it = index.find(key);
    if (it == index.end()) { index[key] = rows.size(); rows.push_back({cur_hdr, stmt, ev.cat, cat, 1, cur_fix, cur_method}); }
    else rows[it->second].count++;
    hist.add(cat);
  }
  while (hi < hev.size() && hev[hi].file == slot) ++hi;
  if (want_rows && !rows.empty()) {
    std::ostringstream os;
    for (const Row& r : rows)
      csv_row(os, {f.rel, ext_name(f.ext), test_name_tag(f.rel, r.fixture), r.method, r.stmt, std::to_string(r.count), r.catname});
    rows_txt = os.str();
  }
  if (want_sum) {
    std::ostringstream os;
    csv_row(os, {std::to_string(id), f.rel, std::to_string(st.n_assert), hist.cell()});
    sum_txt = os.str();
  }
}

static int cmd_scan(const std::vector<std::string>& roots, const std::string& rows_path, const std::string& summary_path,
                    int gpus, bool all_files, int64_t batch_bytes, bool rev_b) {
  std::vector<FileEntry> files;
  for (size_t g = 0; g < roots.size(); ++g) walk(roots[g], (int)g, all_files, files);
  const int n_groups = (int)std::max<size_t>(roots.size(), 1);
  fprintf(stderr, "tosem-scan: %zu files selected under %zu root(s)\n", files.size(), roots.size());
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) die("no CUDA device (there is no CPU fallback)");
  gpus = std::max(1, std::min(gpus, ndev));
  // ---- shares of the GPUs (SURVEY.md section 8e): files sorted by size, descending, each to the GPU with the least bytes
  //      so far (LPT), so that every GPU gets the same byte total whatever the size law is; then, per GPU, batches of at most
  //      --batch-bytes of arena (and 1M files) in walk order
  std::vector<std::vector<Batch>> share((size_t)gpus);
  {
    std::vector<uint32_t> order(files.size());
    for (size_t i = 0; i < files.size(); ++i) {
      if (files[i].size >= (1ll << 30)) die("file larger than 1 GiB: " + files[i].abs);
      order[i] = (uint32_t)i;
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return files[x].size > files[y].size; });
    std::vector<std::vector<uint32_t>> mine((size_t)gpus);
    std::vector<int64_t> load((size_t)gpus, 0);            // greedy LPT: the next largest file goes to the lightest GPU
    for (uint32_t i : order) {
      size_t g = 0;
      for (size_t k = 1; k < (size_t)gpus; ++k) if (load[k] < load[g]) g = k;
      mine[g].push_back(i);
      load[g] += files[i].size + 128;
    }
    for (int g = 0; g < gpus; ++g) {
      std::sort(mine[(size_t)g].begin(), mine[(size_t)g].end());
      share[(size_t)g] = plan_batches(files, mine[(size_t)g], batch_bytes, 1u << 20);
    }
  }
  // one host thread per GPU; one ncclAllReduce of the count table at the end
  std::vector<ncclComm_t> comms(gpus);
  std::vector<int> devs(gpus);
  for (int i = 0; i < gpus; ++i) devs[i] = i;
  if (gpus > 1) {
    // stdout carries the aggregate CSV: whatever NCCL prints while initialising (its version banner
    // under NCCL_DEBUG=VERSION) is routed to stderr
    fflush(stdout);
    const int saved = dup(1);
    dup2(2, 1);
    const ncclResult_t nr = ncclCommInitAll(comms.data(), gpus, devs.data());
    fflush(stdout);
    dup2(saved, 1);
    close(saved);
    nccl_ck(nr, "ncclCommInitAll");
  }
  const size_t table = (size_t)(n_groups + 1) * TSM_NUM_CATEGORIES + 4;
  std::vector<std::vector<int64_t>> totals(gpus, std::vector<int64_t>(table, 0));
  const bool want_rows = !rows_path.empty(), want_sum = !summary_path.empty();
  std::vector<std::string> rows_txt(want_rows ? files.size() : 0), sum_txt(want_sum ? files.size() : 0);   // per file, written in walk order at the end
  auto worker = [&](int g) {
    const uint32_t flags = TSM_SCAN_ASSERT_EVENTS | TSM_SCAN_HEADER_EVENTS | (rev_b ? TSM_SCAN_REV_B : 0u);
    scan_batches(files, share[(size_t)g], g, n_groups, flags, [&](const Batch& B, const Scanned& s) {
      for (size_t i = 0; i < table; ++i) totals[g][i] += s.counts[i];
      if (!want_rows && !want_sum) return;
      size_t ai = 0, hi = 0;
      std::string none;
      for (size_t i = 0; i < B.count(); ++i) {
        const uint32_t fi = B.idx[i];
        render_file(files[fi], (int64_t)fi + 1, B.arena.get() + B.off[i], B.len[i], (uint32_t)i, s.stats[i], s.aev, ai, s.hev, hi, want_rows,
                    want_sum, want_rows ? rows_txt[fi] : none, want_sum ? sum_txt[fi] : none);
      }
    });
    cu_ck(cudaSetDevice(g), "cudaSetDevice");
    cudaStream_t st;
    cu_ck(cudaStreamCreate(&st), "cudaStreamCreate");
    int64_t* d_acc = nullptr;                               // this GPU's count table, input and output of the allreduce
    cu_ck(cudaMalloc((void**)&d_acc, table * sizeof(int64_t)), "cudaMalloc");
    cu_ck(cudaMemcpyAsync(d_acc, totals[g].data(), table * sizeof(int64_t), cudaMemcpyHostToDevice, st), "cudaMemcpyAsync");
    if (gpus > 1)                                           // the single collective of the path (SURVEY.md section 8e)
      nccl_ck(ncclAllReduce(d_acc, d_acc, table, ncclInt64, ncclSum, comms[g], st), "ncclAllReduce");
    cu_ck(cudaMemcpyAsync(totals[g].data(), d_acc, table * sizeof(int64_t), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    cu_ck(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    cudaFree(d_acc);
    cudaStreamDestroy(st);
  };
  if (gpus == 1) worker(0);
  else {
    std::vector<std::thread> th;
    for (int g = 0; g < gpus; ++g) th.emplace_back(worker, g);
    for (auto& t : th) t.join();
    for (int g = 0; g < gpus; ++g) ncclCommDestroy(comms[g]);
  }
  // ---- rows + summary, in walk order
  if (want_rows) {
    std::ofstream os(rows_path, std::ios::binary);
    csv_row(os, {"fileName", "extension", "test_name", "method", "statement", "counts", "category"});
    for (const std::string& t : rows_txt) os << t;
  }
  if (want_sum) {
    std::ofstream os(summary_path, std::ios::binary);
    csv_row(os, {"Id", "FileName", "total assert", "assertion"});
    for (const std::string& t : sum_txt) os << t;
  }
  // ---- the aggregate table (global counts after the allreduce) to stdout
  const std::vector<int64_t>& T = totals[0];
  printf("category,count\r\n");
  for (int k = 0; k < TSM_NUM_CATEGORIES; ++k) {
    const int64_t v = T[(size_t)n_groups * TSM_NUM_CATEGORIES + k];
    if (v) printf("%s,%lld\r\n", k == 0 ? "" : tsm_category_name(k), (long long)v);
  }
  const size_t tot = (size_t)(n_groups + 1) * TSM_NUM_CATEGORIES;
  int64_t share_min = -1, share_max = 0;
  for (int g = 0; g < gpus; ++g) {
    int64_t bsum = 0;
    for (const Batch& b : share[(size_t)g]) for (uint32_t i : b.idx) bsum += files[i].size;
    share_min = share_min < 0 ? bsum : std::min(share_min, bsum); share_max = std::max(share_max, bsum);
  }
  fprintf(stderr, "tosem-scan: lines=%lld assertion_lines=%lld headers=%lld fixture_headers=%lld on %d GPU(s), shares %lld..%lld bytes\n",
          (long long)T[tot], (long long)T[tot + 1], (long long)T[tot + 2], (long long)T[tot + 3], gpus, (long long)std::max<int64_t>(share_min, 0), (long long)share_max);
  return 0;
}

// ---------------------------------------------------------------------------------- reduce (S10)
struct FlagDef { const char* name; const char* col; const char* val; const char* col2; };
// the column mapping of tools/make_golden.py: 171 / 171 cells of tests_strategy_rq32.csv reproduce.  `val` may list
// several values separated by '|': the error rows merge Error_Type values (the merge sets were recovered by
// exhaustive search over the value subsets against the nine shipped per-repository cells, tools/make_golden.py)
static const FlagDef kStrategy[] = {
    {"status_analysis", "status_test", "1", nullptr}, {"value_error", "Error_Type", "ValueError", nullptr},
    {"runtime_error", "Error_Type", "RuntimeError|Exception|NotImplementedError|StopIteration|TimeOut|Timeout|TimeoutError|Warning|nullptr", nullptr}, {"memory_error", "Error_Type", "MemoryError", nullptr},
    {"type_error", "Error_Type", "TypeError", nullptr}, {"import_error", "Error_Type", "ImportError", nullptr},
    {"key_error", "Error_Type", "KeyError", nullptr}, {"AssertionError", "Error_Type", "AssertionError|SyntaxError", nullptr},
    {"FileError", "Error_Type", "FileError|SchemaError", nullptr}, {"NotImplementedError", "Error_Type", "NotImplementedError", nullptr},
    {"negative_test", "negative_test", "1", nullptr}, {"logical_condition", "logical_statement", "1", "logical_expression"},
    {"Null_pointer", "null_pointer", "1", nullptr}, {"value_range", "value_range", "1", nullptr},
    {"absolute_relative_tolerence", "Approximation_Type", "absolute_relative_tolerence", nullptr},
    {"error_bounding", "Approximation_Type", "error_bounding", nullptr},
    {"rounding_tolence", "Approximation_Type", "rounding_tolence", nullptr},
    {"instance_check", "checks_type", "instance_check", nullptr}, {"sub_set_checks", "checks_type", "sub_set_checks", nullptr}};
static const FlagDef kMethods[] = {
    {"regression", "regression", nullptr, nullptr}, {"integration", "Integration", nullptr, nullptr},
    {"end_to_end", "end_to_end", nullptr, nullptr}, {"sanity", "sanity", nullptr, nullptr},
    {"mock_test", "mock_test", nullptr, nullptr}, {"periodic_validation", "periodic_validation", nullptr, nullptr},
    {"example_test", "example_test", nullptr, nullptr}, {"static_inspection", "static_inspection_test", nullptr, nullptr},
    {"robustness_test", "roboustness", nullptr, nullptr}, {"experimental", "Experimental_benchmark_test", nullptr, nullptr},
    {"api_test", "API", nullptr, nullptr}, {"threat", "ThreadTest", nullptr, nullptr}, {"blob", "blob_performance", nullptr, nullptr}};

// RQ3 property table (RQs/RQ3/tests_prop_rq3.csv): a case has a property when the `Data` or the `Model` label of
// one of its rows is in the property's label set.  The sets are not written down in the package; 17 of the 21 were
// recovered by search against the nine shipped per-repository cells (exact, tools/make_golden.py), the other four
// (Consistency, Features Importance, Concurrency, Anomaly) use the label of the same name.
struct PropDef { const char* name; const char* labels; };
static const PropDef kProperties[] = {
    {"Consistency", "Consistency"}, {"Data Distribution", "Distribution"},
    {"Data Validity", "Validity|Data Error|Data Error and Validity"}, {"Completeness", "Completeness"},
    {"Correctness", "Correctness|Accuracy & Precision|Statistical Evidence/ explainability"}, {"Robustness", "Robustness"},
    {"Efficiency", "Time behaviour|Resource Usage|Training Efficiency"},
    {"Data Relation", "Relation & Association|Closeness|Missing Data|Data Differencing|Data Quality"},
    {"Scalability", "Scalability"}, {"Features Importance", "Feature Importance"},
    {"Data Restoration and Recoverability", "Recoverability|Data Restoration"},
    {"Concurrency and Parallelism", "Parallel Processing|parallel"}, {"Uncertainty", "uncertainty"}, {"Anomaly", "Anomaly"},
    {"Data Migration Loss and Corruption", "Data Loss"}, {"Bias and Fairness", "Model Bias"},
    {"Security and Privacy", "Security|Data Encapsulation"}, {"Data Uniqueness", "Uniqueness"},
    {"Data Timeliness", "Timeliness"}, {"Data Integration Integrity", "Validate data integration and integrity"},
    {"Compatibility and Portability", "Compatibility"}};

// RQ3 strategy x property table (RQs/RQ3/tests_correlate_rq3.csv): 20 rows x 21 columns, one cell = the share of a
// repository's cases that have BOTH the strategy flag and the property, for the nine repositories in the order below.
// Row predicates are single taxonomy values (the strategy table above merges Error_Type values, this one does not);
// `decision` reads logical_statement and `logical_condition` reads logical_expression - recovered against the shipped
// cells, 394 of 420 bit-identical (tools/make_golden.py, tests/golden/ledger.json G3).
struct CorrRow { const char* name; const char* col; const char* val; };
static const CorrRow kCorrRows[] = {
    {"rounding_tolence", "Approximation_Type", "rounding_tolence"}, {"instance_check", "checks_type", "instance_check"},
    {"MemoryError", "Error_Type", "MemoryError"}, {"negative_test", "negative_test", "1"},
    {"status_analysis", "status_test", "1"}, {"value_range_analysis", "value_range", "1"},
    {"sub_set_checks", "checks_type", "sub_set_checks"}, {"ValueError", "Error_Type", "ValueError"},
    {"decision", "logical_statement", "1"}, {"error_bounding", "Approximation_Type", "error_bounding"},
    {"Null_pointer", "null_pointer", "1"}, {"boundary", "boundary", "1"},
    {"absolute_relative_tolerence", "Approximation_Type", "absolute_relative_tolerence"},
    {"ImportError", "Error_Type", "ImportError"}, {"pseaudo_oracle", "Pseaudo_Oracle", "1"},
    {"RuntimeError", "Error_Type", "RuntimeError"}, {"logical_condition", "logical_expression", "1"},
    {"TypeError", "Error_Type", "TypeError"}, {"KeyError", "Error_Type", "KeyError"},
    {"NotImplementedError", "Error_Type", "NotImplementedError"}};
struct CorrCol { const char* name; const char* prop; };        // column header of the shipped table -> name in kProperties
static const CorrCol kCorrCols[] = {
    {"Distribution", "Data Distribution"}, {"Validity", "Data Validity"}, {"Consistency", "Consistency"},
    {"Completeness", "Completeness"}, {"Correctness", "Correctness"}, {"Robustness", "Robustness"},
    {"Efficiency", "Efficiency"}, {"Relation", "Data Relation"}, {"Scalability", "Scalability"},
    {"Feature Importance", "Features Importance"}, {"Restoration", "Data Restoration and Recoverability"},
    {"Concurrency", "Concurrency and Parallelism"}, {"uncertainty", "Uncertainty"}, {"Anomaly", "Anomaly"},
    {"Data Loss", "Data Migration Loss and Corruption"}, {"Bias", "Bias and Fairness"},
    {"Security", "Security and Privacy"}, {"Uniqueness", "Data Uniqueness"}, {"Timeliness", "Data Timeliness"},
    {"integration", "Data Integration Integrity"}, {"Compatibility", "Compatibility and Portability"}};

// Four more one-row tables in the same layout for the MERGED rows of the strategy table
// (RQs/RQ3/tests_correlate_{FileError,RuntimeError,assertion,logical}.csv): row name -> row of kStrategy.
struct MergedRow { const char* name; const char* strategy; };
static const MergedRow kMergedRows[] = {{"FileError", "FileError"}, {"RuntimeError", "runtime_error"},
                                        {"AssertionError", "AssertionError"}, {"logical", "logical_condition"}};

static bool one_of(const std::string& have, const std::string& want) {   // `want` = '|'-separated values
  for (size_t a = 0; a <= want.size();) {
    const size_t b = std::min(want.find('|', a), want.size());
    if (have == want.substr(a, b - a)) return true;
    a = b + 1;
  }
  return false;
}

static std::string trim(const std::string& s) {
  size_t a = 0, b = s.size();
  while (a < b && (s[a] == ' ' || s[a] == '\t')) ++a;
  while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\t')) --b;
  return s.substr(a, b - a);
}
static std::string fmt_num(double v, int dec) {            // shipped cells drop trailing zeros ("0", "43.771")
  char buf[64];
  snprintf(buf, sizeof buf, "%.*f", dec, v);
  std::string s = buf;
  if (s.find('.') != std::string::npos) { while (!s.empty() && s.back() == '0') s.pop_back(); if (!s.empty() && s.back() == '.') s.pop_back(); }
  return s.empty() ? "0" : s;
}
static std::string fmt_pyfloat2(double v) {                 // repr(round(v, 2)) of the shipped correlate cells: "0.0", "1.22", "12.2"
  char buf[64];
  snprintf(buf, sizeof buf, "%.2f", v);
  std::string s = buf;
  while (s.size() > 1 && s.back() == '0' && s[s.size() - 2] != '.') s.pop_back();
  return s;
}
static double round_to(double v, int dec) { const double p = std::pow(10.0, dec); return std::round(v * p) / p; }

static int cmd_reduce(const std::string& path, const std::string& strategy_path, const std::string& methods_path,
                      const std::string& properties_path, const std::string& correlate_path, const std::string& correlate_tex_path,
                      const std::string& correlate_counts_path, const std::string& correlate_merged_path) {
  auto rows = csv_read(path);
  if (rows.size() < 2) die("empty taxonomy");
  std::map<std::string, int> col;
  for (size_t i = 0; i < rows[0].size(); ++i) col[rows[0][i]] = (int)i;
  for (const char* need : {"Cases", "Repo"}) if (!col.count(need)) die(std::string("taxonomy lacks column ") + need);
  // repo ids in the column order of tests_strategy_rq32.csv:1 when all nine are present, else first-seen order
  std::vector<std::string> repos = {"autokeras", "auto_sklearn", "tpot", "Ray", "DeepSpeech2", "google_automl", "nni", "Apollo", "Nupic"};
  std::map<std::string, int> rid, cid;
  for (size_t r = 1; r < rows.size(); ++r) if ((int)rows[r].size() > col["Repo"] && !std::count(repos.begin(), repos.end(), rows[r][col["Repo"]])) repos.push_back(rows[r][col["Repo"]]);
  for (size_t i = 0; i < repos.size(); ++i) rid[repos[i]] = (int)i;
  const int nS = sizeof(kStrategy) / sizeof(kStrategy[0]), nM = sizeof(kMethods) / sizeof(kMethods[0]);
  const int nP = sizeof(kProperties) / sizeof(kProperties[0]);
  const int nCR = sizeof(kCorrRows) / sizeof(kCorrRows[0]), nCC = sizeof(kCorrCols) / sizeof(kCorrCols[0]);
  const bool corr = !correlate_path.empty() || !correlate_tex_path.empty() || !correlate_counts_path.empty();
  const bool merged = !correlate_merged_path.empty();
  const int nMR = sizeof(kMergedRows) / sizeof(kMergedRows[0]);
  const int nF = nS + nM + nP + (corr ? nCR * nCC : 0) + (merged ? nMR * nCC : 0);   // the correlate tables are more flag columns of the same reduction
  int merged_row[sizeof(kMergedRows) / sizeof(kMergedRows[0])];
  for (int j = 0; j < nMR; ++j) {
    merged_row[j] = -1;
    for (int k = 0; k < nS; ++k) if (!strcmp(kMergedRows[j].strategy, kStrategy[k].name)) merged_row[j] = k;
    if (merged_row[j] < 0) die(std::string("no strategy row named ") + kMergedRows[j].strategy);
  }
  int corr_prop[sizeof(kCorrCols) / sizeof(kCorrCols[0])];
  for (int q = 0; q < nCC; ++q) {
    corr_prop[q] = -1;
    for (int j = 0; j < nP; ++j) if (!strcmp(kCorrCols[q].prop, kProperties[j].name)) corr_prop[q] = j;
    if (corr_prop[q] < 0) die(std::string("no property named ") + kCorrCols[q].prop);
  }
  std::vector<uint8_t> flags; std::vector<int32_t> repo, cas;
  auto cell = [&](const std::vector<std::string>& r, const char* c) -> std::string {
    auto it = col.find(c); return (it == col.end() || it->second >= (int)r.size()) ? std::string() : trim(r[it->second]); };
  for (size_t r = 1; r < rows.size(); ++r) {
    const auto& R = rows[r];
    if ((int)R.size() <= std::max(col["Cases"], col["Repo"])) continue;
    const std::string cs = R[col["Cases"]];
    if (!cid.count(cs)) { const int k = (int)cid.size(); cid[cs] = k; }
    repo.push_back(rid[R[col["Repo"]]]); cas.push_back(cid[cs]);
    const size_t s0 = flags.size();
    for (int j = 0; j < nS; ++j) {
      bool v = one_of(cell(R, kStrategy[j].col), kStrategy[j].val);
      if (kStrategy[j].col2) v = v || cell(R, kStrategy[j].col2) == "1";
      flags.push_back(v);
    }
    for (int j = 0; j < nM; ++j) { const std::string v = cell(R, kMethods[j].col); flags.push_back(!(v.empty() || v == "0")); }
    const std::string data = cell(R, "Data"), model = cell(R, "Model");
    const size_t p0 = flags.size();
    for (int j = 0; j < nP; ++j)
      flags.push_back((!data.empty() && one_of(data, kProperties[j].labels)) || (!model.empty() && one_of(model, kProperties[j].labels)));
    if (corr)
      for (int j = 0; j < nCR; ++j) {
        const bool s_on = cell(R, kCorrRows[j].col) == kCorrRows[j].val;
        for (int q = 0; q < nCC; ++q) flags.push_back(s_on && flags[p0 + (size_t)corr_prop[q]]);
      }
    if (merged)
      for (int j = 0; j < nMR; ++j) {
        const bool s_on = flags[s0 + (size_t)merged_row[j]] != 0;
        for (int q = 0; q < nCC; ++q) flags.push_back(s_on && flags[p0 + (size_t)corr_prop[q]]);
      }
  }
  const int n_rows = (int)repo.size(), n_repos = (int)repos.size(), n_cases = (int)cid.size();
  std::vector<int64_t> out((size_t)nF * n_repos), cpr((size_t)n_repos);
  ck(tsm_reduce(small_context().get(), flags.data(), repo.data(), cas.data(), n_rows, nF, n_repos, n_cases, out.data(), cpr.data(), nullptr),
     "tsm_reduce");
  int64_t all_cases = 0; for (int64_t c : cpr) all_cases += c;
  // row order of the property and correlate tables: the shipped one when all nine repositories are present, else that of `repos`
  std::vector<std::string> order = {"auto_sklearn", "google_automl", "tpot", "autokeras", "Nupic", "Apollo", "nni", "Ray", "DeepSpeech2"};
  for (auto& r : repos) if (!std::count(order.begin(), order.end(), r)) order.push_back(r);
  if (!strategy_path.empty()) {                             // layout of RQs/RQ3/tests_strategy_rq32.csv
    std::ofstream os(strategy_path, std::ios::binary);
    std::vector<std::string> h = {"Tests"};
    for (auto& r : repos) h.push_back(r);
    h.push_back("");
    for (auto& r : repos) h.push_back(r);
    csv_row(os, h);
    std::vector<std::vector<double>> v(nS, std::vector<double>(n_repos));
    std::vector<double> colsum(n_repos, 0.0);
    for (int j = 0; j < nS; ++j) for (int r = 0; r < n_repos; ++r) {
      // rounded twice, like the shipped cells (docs/SPEC.md section 9): 26/142 -> 18.3099 -> /1.1 -> 16.6454
      v[j][r] = cpr[r] ? round_to(round_to(100.0 * out[(size_t)j * n_repos + r] / cpr[r], 4) / 1.1, 4) : 0.0;
      colsum[r] += v[j][r];
    }
    for (int j = 0; j < nS; ++j) {
      std::vector<std::string> row = {kStrategy[j].name};
      for (int r = 0; r < n_repos; ++r) row.push_back(fmt_num(v[j][r], 4));
      row.push_back("");
      for (int r = 0; r < n_repos; ++r) row.push_back(fmt_num(colsum[r] > 0 ? round_to(v[j][r] / colsum[r] * 100.0, 2) : 0.0, 2));
      csv_row(os, row);
    }
    std::vector<std::string> last = {""};
    for (int r = 0; r < n_repos; ++r) last.push_back(fmt_num(colsum[r], 4));
    last.push_back("");
    for (int r = 0; r < n_repos; ++r) last.push_back("100");
    csv_row(os, last);
  }
  if (!methods_path.empty()) {                              // first three columns of RQs/RQ4/tests_methods_v2.csv
    std::ofstream os(methods_path, std::ios::binary);
    csv_row(os, {"Test_methods", "total_cases", "percentage"});
    for (int j = 0; j < nM; ++j) {
      int64_t t = 0;
      for (int r = 0; r < n_repos; ++r) t += out[(size_t)(nS + j) * n_repos + r];
      csv_row(os, {kMethods[j].name, std::to_string(t), fmt_num(all_cases ? round_to(100.0 * t / all_cases, 4) : 0.0, 4)});
    }
  }
  if (!properties_path.empty()) {                           // layout of RQs/RQ3/tests_prop_rq3.csv:1-10
    std::ofstream os(properties_path, std::ios::binary);
    std::vector<std::string> h = {"Repos"};
    for (int j = 0; j < nP; ++j) h.push_back(kProperties[j].name);
    csv_row(os, h);
    int64_t denom = 0;                                      // one denominator for every row: Apollo's case count (the 216 of
    if (rid.count("Apollo")) denom = cpr[(size_t)rid["Apollo"]];   // the shipped table), else the largest repository
    if (denom == 0) for (int64_t c : cpr) denom = std::max(denom, c);
    for (auto& name : order) {
      if (!rid.count(name) || cpr[(size_t)rid[name]] == 0) continue;
      const int r = rid[name];
      std::vector<std::string> row = {name};
      for (int j = 0; j < nP; ++j)
        row.push_back(fmt_num(denom ? round_to(100.0 * out[(size_t)(nS + nM + j) * n_repos + r] / denom, 4) : 0.0, 4));
      csv_row(os, row);
    }
  }
  // A table of the correlate layout: 21 property columns, one row per name, the row j counts in the flag columns c0 + j * nCC + q.
  // Three shipped layouts of the same counts: RQs/RQ3/tests_correlate_rq3.csv (0: "repo:(p%), " for every repository),
  // tests_correlate_rq4.csv (1: LaTeX cells "$repo:p\%$, " of the non-zero repositories) and tests_combined_correlate_rq3.csv
  // (2: the distinct cases of all repositories together).
  auto correlate = [&](const std::string& outp, int layout, size_t c0, const std::vector<std::string>& names) {
    if (outp.empty()) return;
    std::ofstream os(outp, std::ios::binary);
    std::vector<std::string> h = {"Tests"};
    for (int q = 0; q < nCC; ++q) h.push_back(kCorrCols[q].name);
    csv_row(os, h);
    for (size_t j = 0; j < names.size(); ++j) {
      std::vector<std::string> row = {names[j]};
      for (int q = 0; q < nCC; ++q) {
        const int64_t* d = &out[(c0 + j * nCC + q) * n_repos];
        int64_t all = 0;
        for (int r = 0; r < n_repos; ++r) all += d[r];
        std::string cellv = "0";                            // a pairing no case has is the bare string "0" in every layout
        if (layout == 2) cellv = std::to_string(all);
        else if (all) {
          cellv.clear();
          for (auto& name : order) {
            if (!rid.count(name) || cpr[(size_t)rid[name]] == 0) continue;
            const int r = rid[name];
            const std::string pct = fmt_pyfloat2(100.0 * (double)d[r] / (double)cpr[r]);
            if (layout == 0) cellv += name + ":(" + pct + "%), ";
            else if (d[r]) cellv += "$" + name + ":" + pct + "\\%$, ";
          }
        }
        row.push_back(cellv);
      }
      csv_row(os, row);
    }
  };
  const size_t c0 = (size_t)(nS + nM + nP);
  if (corr) {
    for (const CorrRow& cr : kCorrRows) if (!col.count(cr.col)) die(std::string("taxonomy lacks column ") + cr.col);
    std::vector<std::string> names;
    for (const CorrRow& cr : kCorrRows) names.push_back(cr.name);
    correlate(correlate_path, 0, c0, names);
    correlate(correlate_tex_path, 1, c0, names);
    correlate(correlate_counts_path, 2, c0, names);
  }
  if (merged) {                                             // the four one-row tables, as four rows of one file in layout 0
    std::vector<std::string> names;
    for (const MergedRow& mr : kMergedRows) names.push_back(mr.name);
    correlate(correlate_merged_path, 0, c0 + (corr ? (size_t)(nCR * nCC) : 0), names);
  }
  fprintf(stderr, "tosem-scan: reduce %d rows, %d cases, %d repos\n", n_rows, n_cases, n_repos);
  return 0;
}

// ---------------------------------------------------------------------------------- body statements (SPEC section 10)

static int cmd_body(const std::vector<std::string>& roots, const std::string& out_path, int64_t batch_bytes) {
  std::vector<FileEntry> files;
  for (size_t g = 0; g < roots.size(); ++g) walk(roots[g], (int)g, false, files);
  fprintf(stderr, "tosem-scan: %zu files selected under %zu root(s)\n", files.size(), roots.size());
  std::ofstream os;
  if (!out_path.empty()) { os.open(out_path, std::ios::binary); csv_row(os, {"Index", "text", "Category", "cases", "File_ID", "Component"}); }
  int64_t index = 0, cases = 0, file_id = 0, n_stmt = 0;   // carried across batches
  const int32_t n_groups = (int32_t)roots.size();
  std::vector<Batch> batches = plan_batches(files, all_of(files), batch_bytes, kBatchFiles);
  scan_batches(files, batches, 0, n_groups, TSM_SCAN_HEADER_EVENTS, [&](const Batch& B, const Scanned& s) {
    const tsm_corpus c = B.corpus(n_groups);
    const std::vector<tsm_header_event>& hev = s.hev;
    std::vector<int64_t> base(B.count() + 1);
    int64_t nl = 0;
    int rc = tsm_statements(s.ctx, &c, base.data(), nullptr, nullptr, 0, &nl, nullptr);
    if (rc != TSM_OK && rc != TSM_E_CAPACITY) ck(rc, "tsm_statements");
    std::vector<uint32_t> lend((size_t)std::max<int64_t>(nl, 1));
    std::vector<uint8_t> kind((size_t)std::max<int64_t>(nl, 1));
    ck(tsm_statements(s.ctx, &c, base.data(), lend.data(), kind.data(), nl, &nl, nullptr), "tsm_statements");
    size_t hi = 0;
    for (size_t i = 0; i < B.count(); ++i) {
      const FileEntry& f = files[B.idx[i]];
      const uint8_t* p = B.arena.get() + B.off[i];
      ++file_id;
      bool in_case = false;
      std::string cur_stmt; bool have = false, listed = false;
      auto flush = [&]() {
        if (have && listed && cur_stmt.find_first_not_of("{}(); \t\r\x0b\x0c") != std::string::npos) {
          ++n_stmt;
          if (os.is_open()) csv_row(os, {std::to_string(++index), cur_stmt, "", std::to_string(cases), std::to_string(file_id), ""});
        }
        have = false; cur_stmt.clear();
      };
      uint32_t pos = 0;
      for (int64_t l = base[i]; l < base[i + 1]; ++l) {
        const uint32_t e = lend[(size_t)l];
        const bool is_hdr = hi < hev.size() && hev[hi].file == i && hev[hi].line_off == pos;
        if (kind[(size_t)l] == 1) { flush(); listed = in_case && !is_hdr; have = true; }
        if (is_hdr) {                                       // a new test case starts here
          ++hi; in_case = true; ++cases;
          if (os.is_open()) csv_row(os, {std::to_string(++index), case_name(f.ext, p + pos, e - pos), "", std::to_string(cases), std::to_string(file_id), ""});
        }
        if (kind[(size_t)l] != 0 && have) {
          uint32_t b = pos, z = e;
          while (b < z && is_w(p[b])) ++b;
          while (z > b && is_w(p[z - 1])) --z;
          if (!cur_stmt.empty()) cur_stmt += ' ';
          cur_stmt.append((const char*)p + b, z - b);
        }
        pos = e + 1;
      }
      flush();
      while (hi < hev.size() && hev[hi].file == i) ++hi;
    }
  });
  printf("files,cases,statements\r\n%lld,%lld,%lld\r\n", (long long)file_id, (long long)cases, (long long)n_stmt);
  return 0;
}

// ---------------------------------------------------------------------------------- release presence matrix (S7, SPEC section 11)
struct SnapFile { std::string rel; uint64_t digest; int64_t size; uint32_t n_assert; std::string hist; };

// Scan one snapshot: per selected test file its digest, assertion total and "n:category, ..." histogram.
static std::vector<SnapFile> scan_snapshot(const std::vector<FileEntry>& files, int64_t batch_bytes) {
  std::vector<SnapFile> out;
  std::vector<Batch> batches = plan_batches(files, all_of(files), batch_bytes, kBatchFiles);
  scan_batches(files, batches, 0, 1, TSM_SCAN_ASSERT_EVENTS, [&](const Batch& B, const Scanned& s) {
    size_t ai = 0;
    for (size_t i = 0; i < B.count(); ++i) {
      CategoryHist hist;
      for (; ai < s.aev.size() && s.aev[ai].file == i; ++ai) hist.add(event_category(B.arena.get() + B.off[i], s.aev[ai]));
      out.push_back({files[B.idx[i]].rel, s.stats[i].digest, files[B.idx[i]].size, s.stats[i].n_assert, hist.cell()});
    }
  });
  return out;
}

// The selected test files (S0 + S1) of one tree of a git repository, in the order `walk` gives for a checkout of it
// (names sorted at every level, depth first); their bytes are inflated here and scanned like files read from disk.
static void walk_git(gitstore::Store& gs, const gitstore::Oid& tree, const std::string& prefix, bool all_files, std::vector<FileEntry>& out) {
  std::vector<gitstore::TreeEntry> es;
  if (!gs.tree(tree, es)) die("unreadable tree " + tree.hex());
  std::sort(es.begin(), es.end(), [](const gitstore::TreeEntry& a, const gitstore::TreeEntry& b) { return a.name < b.name; });
  for (const gitstore::TreeEntry& e : es) {
    const std::string rel = prefix + e.name;
    if (e.is_tree()) { walk_git(gs, e.oid, rel + "/", all_files, out); continue; }
    if (!e.is_blob()) continue;
    const int ext = ext_tag(rel);
    if (!all_files && (lower(rel).find("test") == std::string::npos || ext == TSM_EXT_OTHER)) continue;
    gitstore::Object o;
    if (!gs.read(e.oid, o) || o.type != gitstore::OBJ_BLOB) die("unreadable blob " + e.oid.hex());
    if (o.data.size() > 0x7fff0000u) die("blob too large: " + rel);
    FileEntry f{rel, "", ext, 0, (int64_t)o.data.size(), nullptr};
    f.blob = std::make_shared<const std::vector<uint8_t>>(std::move(o.data));
    out.push_back(std::move(f));
  }
}

// specs: <snapshot-root>=<tag>...; or, with --git <repository>, revisions (tags, branches, object names) in release
// order - none = every tag of the repository, oldest commit first.
static int cmd_releases(const std::vector<std::string>& specs_in, const std::string& out_path, const std::string& git_repo,
                        int64_t batch_bytes) {
  std::vector<std::string> specs = specs_in;
  gitstore::Store gs;
  if (!git_repo.empty()) {
    std::string err;
    if (!gs.open(git_repo, err)) die(err);
    if (specs.empty()) {
      std::vector<std::pair<long long, std::string>> byt;
      for (const std::string& t : gs.tag_names()) {
        gitstore::Oid id; gitstore::Commit c;
        if (gs.resolve("refs/tags/" + t, id) && gs.commit(id, c)) byt.push_back({c.time, t});
      }
      std::sort(byt.begin(), byt.end());
      for (auto& kv : byt) specs.push_back(kv.second);
      if (specs.empty()) die("the repository has no tags; name the revisions");
    }
  }
  struct Identity { std::string name; std::vector<std::string> path; uint64_t digest; int64_t size; uint32_t n_assert; std::string hist; std::string cur; };
  std::vector<std::string> tags;
  std::vector<Identity> ids;
  for (size_t t = 0; t < specs.size(); ++t) {
    std::vector<FileEntry> files;
    if (!git_repo.empty()) {
      gitstore::Oid id; gitstore::Commit c;
      if (!gs.resolve(specs[t], id) || !gs.commit(id, c)) die("cannot resolve revision " + specs[t]);
      tags.push_back(specs[t]);
      walk_git(gs, c.tree, "", false, files);
    } else {
      const size_t eq = specs[t].rfind('=');
      if (eq == std::string::npos) die("releases arguments are <snapshot-root>=<tag>");
      tags.push_back(specs[t].substr(eq + 1));
      walk(specs[t].substr(0, eq), 0, false, files);
    }
    const std::vector<SnapFile> snap = scan_snapshot(files, batch_bytes);
    std::vector<char> id_taken(ids.size(), 0), f_done(snap.size(), 0);
    auto bind = [&](size_t fi, size_t id) {
      const SnapFile& f = snap[fi];
      ids[id].path[t] = f.rel; ids[id].cur = f.rel; ids[id].digest = f.digest; ids[id].size = f.size;
      ids[id].n_assert = f.n_assert; ids[id].hist = f.hist; id_taken[id] = 1; f_done[fi] = 1;
    };
    for (Identity& I : ids) I.path.resize(t + 1);
    for (size_t fi = 0; fi < snap.size(); ++fi)                       // (1) same relative path
      for (size_t id = 0; id < id_taken.size(); ++id)
        if (!id_taken[id] && ids[id].cur == snap[fi].rel) { bind(fi, id); break; }
    for (size_t fi = 0; fi < snap.size(); ++fi)                       // (2) same content: a pure move
      if (!f_done[fi])
        for (size_t id = 0; id < id_taken.size(); ++id)
          if (!id_taken[id] && ids[id].size == snap[fi].size && ids[id].digest == snap[fi].digest) { bind(fi, id); break; }
    for (size_t fi = 0; fi < snap.size(); ++fi) {                     // (3) same base name, unambiguous
      if (f_done[fi]) continue;
      int hit = -1, n = 0;
      for (size_t id = 0; id < id_taken.size(); ++id)
        if (!id_taken[id] && base_name(ids[id].cur) == base_name(snap[fi].rel)) { hit = (int)id; ++n; }
      if (n == 1) bind(fi, (size_t)hit);
    }
    for (size_t fi = 0; fi < snap.size(); ++fi)                       // new identities, in walk order
      if (!f_done[fi]) {
        Identity I; I.name = snap[fi].rel; I.path.assign(t + 1, "");
        ids.push_back(I); id_taken.push_back(0);
        bind(fi, ids.size() - 1);
      }
  }
  std::ofstream os;
  if (!out_path.empty()) {
    os.open(out_path, std::ios::binary);
    std::vector<std::string> h = {"Id", "FileName"};
    for (const std::string& g : tags) h.push_back(g);
    h.push_back("total assert"); h.push_back("assertion");
    csv_row(os, h);
    for (size_t i = 0; i < ids.size(); ++i) {
      std::vector<std::string> row = {std::to_string(i + 1), ids[i].name};
      for (size_t t = 0; t < tags.size(); ++t) row.push_back(t < ids[i].path.size() ? ids[i].path[t] : "");
      row.push_back(std::to_string(ids[i].n_assert)); row.push_back(ids[i].hist);
      csv_row(os, row);
    }
  }
  printf("identities,snapshots\r\n%zu,%zu\r\n", ids.size(), tags.size());
  return 0;
}

// ---------------------------------------------------------------------------------- renames (docs/SPEC.md section 13)
// One group = the deleted and the added files of one commit (history) or of one tree pair (diff), binary files already
// left out.  find_renames pairs them in three one-to-one steps - exact (identical bytes), base name, matrix - with the
// inexact scores of every group from ONE tsm_similarity call over the candidates that pass git's size filter.
struct RenameFile { std::string path; std::vector<uint8_t> bytes; };
struct RenamePair { size_t del, add; int similarity; bool exact; };
struct RenameGroup { std::vector<RenameFile> del, add; std::vector<RenamePair> pairs; };

static void find_renames(tsm_ctx* ctx, std::vector<RenameGroup>& groups, int min_pct) {
  const int64_t kMax = 60000, min_score = 600ll * min_pct, base_score = min_score + (kMax - min_score) / 2;
  struct Cand { size_t g, d, a; };
  std::vector<Cand> cands;
  std::vector<std::vector<size_t>> del_order(groups.size()), add_order(groups.size());   // path order of each side
  std::vector<std::vector<char>> del_used(groups.size()), add_used(groups.size());
  for (size_t g = 0; g < groups.size(); ++g) {
    RenameGroup& G = groups[g];
    G.pairs.clear();
    auto order = [](const std::vector<RenameFile>& v) {
      std::vector<size_t> o(v.size());
      for (size_t i = 0; i < o.size(); ++i) o[i] = i;
      std::sort(o.begin(), o.end(), [&](size_t x, size_t y) { return v[x].path < v[y].path; });
      return o;
    };
    del_order[g] = order(G.del); add_order[g] = order(G.add);
    del_used[g].assign(G.del.size(), 0); add_used[g].assign(G.add.size(), 0);
    // 1. exact: per added file in path order, the unpaired deleted file with the same bytes (same base name first)
    for (size_t a : add_order[g]) {
      long best = -1;
      for (size_t d : del_order[g]) {
        if (del_used[g][d] || G.del[d].bytes != G.add[a].bytes) continue;
        if (best < 0) best = (long)d;
        if (base_name(G.del[d].path) == base_name(G.add[a].path)) { best = (long)d; break; }
      }
      if (best < 0) continue;
      del_used[g][(size_t)best] = add_used[g][a] = 1;
      G.pairs.push_back({(size_t)best, a, 100, true});
    }
    // candidates of the inexact steps: git's size filter (a pair with 100 * min < N * max cannot reach the threshold)
    for (size_t d = 0; d < G.del.size(); ++d)
      for (size_t a = 0; a < G.add.size(); ++a) {
        if (del_used[g][d] || add_used[g][a]) continue;
        const int64_t x = (int64_t)G.del[d].bytes.size(), y = (int64_t)G.add[a].bytes.size();
        if (std::max(x, y) == 0 || 100 * std::min(x, y) < (int64_t)min_pct * std::max(x, y)) continue;
        cands.push_back({g, d, a});
      }
  }
  std::map<std::pair<size_t, size_t>, std::vector<int64_t>> score;   // (group, del) -> score per added file (-1: no candidate)
  if (!cands.empty()) {
    std::vector<const std::vector<uint8_t>*> so, sn;                // the files of the candidates, each once per side
    std::map<std::pair<size_t, size_t>, int32_t> io, in;
    std::vector<int32_t> co, cn;
    for (const Cand& c : cands) {
      auto o = io.emplace(std::make_pair(c.g, c.d), (int32_t)so.size());
      if (o.second) so.push_back(&groups[c.g].del[c.d].bytes);
      auto n = in.emplace(std::make_pair(c.g, c.a), (int32_t)sn.size());
      if (n.second) sn.push_back(&groups[c.g].add[c.a].bytes);
      co.push_back(o.first->second); cn.push_back(n.first->second);
    }
    std::vector<int64_t> common(cands.size());
    {
      const Batch PO = pack(so), PN = pack(sn);
      const tsm_corpus ko = PO.corpus(1), kn = PN.corpus(1);
      ck(tsm_similarity(ctx, &ko, &kn, co.data(), cn.data(), (int64_t)cands.size(), common.data(), nullptr), "tsm_similarity");
    }
    for (size_t k = 0; k < cands.size(); ++k) {
      const Cand& c = cands[k];
      std::vector<int64_t>& row = score[{c.g, c.d}];
      row.resize(groups[c.g].add.size(), -1);
      const int64_t m = (int64_t)std::max(groups[c.g].del[c.d].bytes.size(), groups[c.g].add[c.a].bytes.size());
      row[c.a] = common[k] * kMax / m;
    }
  }
  auto get = [&](size_t g, size_t d, size_t a) -> int64_t {
    auto it = score.find({g, d});
    return it == score.end() ? -1 : it->second[a];
  };
  for (size_t g = 0; g < groups.size(); ++g) {
    RenameGroup& G = groups[g];
    // 2. base name: a base name that occurs once among the remaining deleted files and once among the remaining added ones
    std::map<std::string, std::pair<int, size_t>> bd, ba;   // base name -> (count, file)
    for (size_t d = 0; d < G.del.size(); ++d) if (!del_used[g][d]) { auto& e = bd[base_name(G.del[d].path)]; e.first++; e.second = d; }
    for (size_t a = 0; a < G.add.size(); ++a) if (!add_used[g][a]) { auto& e = ba[base_name(G.add[a].path)]; e.first++; e.second = a; }
    for (size_t a : add_order[g]) {
      if (add_used[g][a]) continue;
      const auto& ea = ba[base_name(G.add[a].path)];
      auto it = bd.find(base_name(G.add[a].path));
      if (ea.first != 1 || it == bd.end() || it->second.first != 1) continue;
      const size_t d = it->second.second;
      const int64_t s = get(g, d, a);
      if (s < base_score) continue;
      del_used[g][d] = add_used[g][a] = 1;
      G.pairs.push_back({d, a, (int)(s / 600), false});
    }
    // 3. matrix: per added file its 4 best candidates (score, same base name, old path), then all of them greedily
    struct M { int64_t s; bool same; size_t d, a; };
    auto better = [&](const M& x, const M& y) {
      if (x.s != y.s) return x.s > y.s;
      if (x.same != y.same) return x.same;
      if (G.del[x.d].path != G.del[y.d].path) return G.del[x.d].path < G.del[y.d].path;
      return G.add[x.a].path < G.add[y.a].path;
    };
    std::vector<M> kept;
    for (size_t a : add_order[g]) {
      if (add_used[g][a]) continue;
      std::vector<M> mine;
      for (size_t d : del_order[g]) {
        if (del_used[g][d]) continue;
        const int64_t s = get(g, d, a);
        if (s >= min_score && s >= 0) mine.push_back({s, base_name(G.del[d].path) == base_name(G.add[a].path), d, a});
      }
      std::sort(mine.begin(), mine.end(), better);
      if (mine.size() > 4) mine.resize(4);
      kept.insert(kept.end(), mine.begin(), mine.end());
    }
    std::sort(kept.begin(), kept.end(), better);
    for (const M& m : kept) {
      if (del_used[g][m.d] || add_used[g][m.a]) continue;
      del_used[g][m.d] = add_used[g][m.a] = 1;
      G.pairs.push_back({m.d, m.a, (int)(m.s / 600), false});
    }
  }
}

// ---------------------------------------------------------------------------------- diff (S8)
// Changed assertion lines (docs/SPEC.md section 8) of one diff call: [n_groups][K] tables by group and the events of both
// sides (tsm_diff_pairs_asserts), event arrays grown to the counts the library reports when they are too small.
struct ChangedAsserts { std::vector<int64_t> added_counts, removed_counts; std::vector<tsm_assert_event> aev, rev; };
static void diff_asserts(tsm_ctx* ctx, const tsm_corpus& ca, const tsm_corpus& cn, int64_t* added, int64_t* removed,
                         tsm_diff_detail* det, ChangedAsserts& r) {
  const size_t table = (size_t)ca.n_groups * TSM_NUM_CATEGORIES;
  r.added_counts.assign(table, 0); r.removed_counts.assign(table, 0);
  int64_t cap = ((int64_t)ca.off[ca.n_files] + cn.off[cn.n_files]) / 64 + 1024;
  for (;;) {
    r.aev.resize((size_t)cap); r.rev.resize((size_t)cap);
    tsm_diff_asserts o{r.added_counts.data(), r.removed_counts.data(), r.aev.data(), cap, 0, r.rev.data(), cap, 0};
    const int rc = tsm_diff_pairs_asserts(ctx, &ca, &cn, added, removed, det, &o, nullptr);
    if (rc == TSM_E_CAPACITY && std::max(o.n_aev, o.n_rev) > cap) { cap = std::max(o.n_aev, o.n_rev); continue; }
    ck(rc, "tsm_diff_pairs_asserts");
    r.aev.resize((size_t)o.n_aev); r.rev.resize((size_t)o.n_rev);
    return;
  }
}
// The same with the assertion edits of docs/SPEC.md section 17 (tsm_diff_pairs_assert_edits, one call for both): `chg` is
// filled as diff_asserts fills it, `edits` pairs its events.  Event and edit arrays grow to the counts the library reports.
static void diff_assert_edits(tsm_ctx* ctx, const tsm_corpus& ca, const tsm_corpus& cn, int64_t* added, int64_t* removed,
                              tsm_diff_detail* det, ChangedAsserts& r, std::vector<tsm_assert_edit>& edits) {
  const size_t table = (size_t)ca.n_groups * TSM_NUM_CATEGORIES;
  r.added_counts.assign(table, 0); r.removed_counts.assign(table, 0);
  int64_t cap = ((int64_t)ca.off[ca.n_files] + cn.off[cn.n_files]) / 64 + 1024, ecap = cap;
  for (;;) {
    r.aev.resize((size_t)cap); r.rev.resize((size_t)cap); edits.resize((size_t)ecap);
    tsm_diff_asserts o{r.added_counts.data(), r.removed_counts.data(), r.aev.data(), cap, 0, r.rev.data(), cap, 0};
    int64_t ne = 0;
    const int rc = tsm_diff_pairs_assert_edits(ctx, &ca, &cn, added, removed, det, &o, edits.data(), ecap, &ne, nullptr);
    if (rc == TSM_E_CAPACITY && (std::max(o.n_aev, o.n_rev) > cap || ne > ecap)) {
      cap = std::max(cap, std::max(o.n_aev, o.n_rev)); ecap = std::max(ecap, ne);
      continue;
    }
    ck(rc, "tsm_diff_pairs_assert_edits");
    r.aev.resize((size_t)o.n_aev); r.rev.resize((size_t)o.n_rev); edits.resize((size_t)ne);
    return;
  }
}
// The --asserts rows of pair `pair` on one side: `lead` cells, fileName, change ('+' new side, '-' old side), 1-based line
// number in that side's file, statement, category.  `k` walks the side's events (canonical order) across calls.
static void assert_rows(std::ostream& os, const std::vector<std::string>& lead, const std::string& path, const uint8_t* base,
                        int32_t size, const std::vector<tsm_assert_event>& ev, size_t& k, uint32_t pair, const char* change) {
  LineCounter lc{base};
  for (; k < ev.size() && ev[k].file == pair; ++k) {
    const tsm_assert_event& e = ev[k];
    std::vector<std::string> row = lead;
    row.insert(row.end(), {path, change, std::to_string(lc.at(e.line_off)), event_statement(base, size, e), event_category(base, e)});
    csv_row(os, row);
  }
}
// The --assert-churn rows of one [K] pair of rows: every category with a changed line.
static void churn_rows(std::ostream& os, const std::vector<std::string>& lead, const int64_t* added, const int64_t* removed) {
  for (int k = 0; k < TSM_NUM_CATEGORIES; ++k)
    if (added[k] || removed[k]) {
      std::vector<std::string> row = lead;
      row.insert(row.end(), {tsm_category_name(k), std::to_string(added[k]), std::to_string(removed[k])});
      csv_row(os, row);
    }
}

// Test-case churn (docs/SPEC.md section 16) of one diff call: the case records of both sides (tsm_diff_pairs_cases), arrays
// grown to the counts the library reports when they are too small.
struct CaseLists { std::vector<tsm_case> olds, news; };
static void diff_cases(tsm_ctx* ctx, const tsm_corpus& ca, const tsm_corpus& cn, int64_t* added, int64_t* removed,
                       tsm_diff_detail* det, CaseLists& r) {
  int64_t co = (int64_t)ca.off[ca.n_files] / 512 + 64, cc = (int64_t)cn.off[cn.n_files] / 512 + 64;
  for (;;) {
    r.olds.resize((size_t)co); r.news.resize((size_t)cc);
    tsm_diff_cases o{r.olds.data(), co, 0, r.news.data(), cc, 0};
    const int rc = tsm_diff_pairs_cases(ctx, &ca, &cn, added, removed, det, &o, nullptr);
    if (rc == TSM_E_CAPACITY && (o.n_old > co || o.n_new > cc)) { co = std::max(co, o.n_old); cc = std::max(cc, o.n_new); continue; }
    ck(rc, "tsm_diff_pairs_cases");
    r.olds.resize((size_t)o.n_old); r.news.resize((size_t)o.n_new);
    return;
  }
}

// Test-smell churn (docs/SPEC.md section 19) of one diff call: the case records (as diff_cases), the tests of both sides and their
// churn records (tsm_diff_pairs_smells), arrays grown to the counts the library reports when they are too small.  lexical: one
// tsm_diff_pairs_smells_lexical call instead, which adds the lexical records of every test (section 26); without it they stay empty.
struct SmellLists {
  std::vector<tsm_smell_test> olds, news; std::vector<tsm_test_churn> old_churn, new_churn;
  std::vector<tsm_lex_test> old_lex, new_lex; std::vector<tsm_lex_churn> old_lchurn, new_lchurn;
};
static void diff_smells(tsm_ctx* ctx, const tsm_corpus& ca, const tsm_corpus& cn, int64_t* added, int64_t* removed,
                        tsm_diff_detail* det, CaseLists& c, SmellLists& r, bool lexical) {
  int64_t co = (int64_t)ca.off[ca.n_files] / 512 + 64, cc = (int64_t)cn.off[cn.n_files] / 512 + 64, to = co, tn = cc;
  for (;;) {
    c.olds.resize((size_t)co); c.news.resize((size_t)cc);
    r.olds.resize((size_t)to); r.old_churn.resize((size_t)to); r.news.resize((size_t)tn); r.new_churn.resize((size_t)tn);
    tsm_diff_smells o{{c.olds.data(), co, 0, c.news.data(), cc, 0}, r.olds.data(), r.old_churn.data(), to, 0,
                      r.news.data(), r.new_churn.data(), tn, 0};
    int rc;
    if (lexical) {
      r.old_lex.resize((size_t)to); r.old_lchurn.resize((size_t)to); r.new_lex.resize((size_t)tn); r.new_lchurn.resize((size_t)tn);
      tsm_diff_lex_smells x{r.old_lex.data(), r.old_lchurn.data(), r.new_lex.data(), r.new_lchurn.data()};
      rc = tsm_diff_pairs_smells_lexical(ctx, &ca, &cn, added, removed, det, &o, &x, nullptr);
    } else {
      rc = tsm_diff_pairs_smells(ctx, &ca, &cn, added, removed, det, &o, nullptr);
    }
    if (rc == TSM_E_CAPACITY && (o.cases.n_old > co || o.cases.n_new > cc || o.n_old_tests > to || o.n_new_tests > tn)) {
      co = std::max(co, o.cases.n_old); cc = std::max(cc, o.cases.n_new); to = std::max(to, o.n_old_tests); tn = std::max(tn, o.n_new_tests);
      continue;
    }
    ck(rc, lexical ? "tsm_diff_pairs_smells_lexical" : "tsm_diff_pairs_smells");
    c.olds.resize((size_t)o.cases.n_old); c.news.resize((size_t)o.cases.n_new);
    r.olds.resize((size_t)o.n_old_tests); r.old_churn.resize((size_t)o.n_old_tests);
    r.news.resize((size_t)o.n_new_tests); r.new_churn.resize((size_t)o.n_new_tests);
    if (lexical) {
      r.old_lex.resize((size_t)o.n_old_tests); r.old_lchurn.resize((size_t)o.n_old_tests);
      r.new_lex.resize((size_t)o.n_new_tests); r.new_lchurn.resize((size_t)o.n_new_tests);
    }
    return;
  }
}

static const char* const kSmellNames[TSM_N_SMELLS] = {"empty", "assertion_free", "duplicate_assert", "redundant_assert",
                                                      "conditional_logic", "exception_handling", "sleepy", "print", "ignored"};
static const char* const kLexSmellNames[TSM_N_LSMELLS] = {"assertion_roulette", "magic_number", "suboptimal_assert", "mystery_guest",
                                                         "obscure_setup"};

// The case name (docs/SPEC.md section 10) of every case of one side of a pair, from the header lines of the side's bytes.
static std::vector<std::string> case_names(const uint8_t* base, int32_t size, int ext, const tsm_case* cs, size_t n) {
  std::vector<std::string> out;
  int32_t line = 0, pos = 0;
  for (size_t k = 0; k < n; ++k) {                          // cases in line order: one walk over the bytes
    for (; line < cs[k].line; ++line) pos = (int32_t)((const uint8_t*)memchr(base + pos, '\n', (size_t)(size - pos)) - base) + 1;
    const uint8_t* lf = (const uint8_t*)memchr(base + pos, '\n', (size_t)(size - pos));
    out.push_back(case_name(ext, base + pos, (uint32_t)((lf ? (int32_t)(lf - base) : size) - pos)));
  }
  return out;
}

// The cases of one pair (docs/SPEC.md section 16): its old cases oc[0, no) and new cases nc[0, nn), old case index o_first being
// oc[0], their names, and per new case the old case it matches (-1: none) and per old case whether one matches it.  Matches by
// kept header line come with the records, matches by name (once among the unmatched cases of each side) are made here.
struct CaseSide { const uint8_t* base; int32_t size; int ext; const std::string* path; };
struct PairCaseMatch {
  std::vector<std::string> na, nb; std::vector<int64_t> match; std::vector<char> used;
  PairCaseMatch(const CaseSide& o, const CaseSide& nw, const tsm_case* oc, size_t no, const tsm_case* nc, size_t nn, size_t o_first)
      : na(case_names(o.base, o.size, o.ext, oc, no)), nb(case_names(nw.base, nw.size, nw.ext, nc, nn)), match(nn, -1), used(no, 0) {
    for (size_t j = 0; j < nn; ++j)
      if (nc[j].match >= 0) { match[j] = nc[j].match - (int64_t)o_first; used[(size_t)match[j]] = 1; }
    tsm_names::match_by_name(na, nb, match, used);
  }
};

// The --cases rows of one pair (docs/SPEC.md section 16): the D rows in old line order, then the A and M rows in new line order.
static void case_rows(std::ostream& os, std::vector<std::string> lead, const CaseSide& o, const CaseSide& nw, const std::string* old_path,
                      const tsm_case* oc, size_t no, const tsm_case* nc, size_t nn, size_t o_first) {
  const PairCaseMatch pm(o, nw, oc, no, nc, nn, o_first);
  const std::vector<std::string>&na = pm.na, &nb = pm.nb;
  const std::vector<int64_t>& match = pm.match;
  const std::vector<char>& used = pm.used;
  auto num = [](int64_t v) { return std::to_string(v); };
  auto row = [&](const std::string& path, std::vector<std::string> cells) {
    std::vector<std::string> r = lead;
    r.push_back(path);
    r.insert(r.end(), cells.begin(), cells.end());
    if (old_path) r.push_back(*old_path);
    csv_row(os, r);
  };
  for (size_t k = 0; k < no; ++k) {
    if (used[k]) continue;
    const tsm_case& c = oc[k];
    row(*o.path, {na[k], "D", "", num(c.line + 1), "", num(c.n_lines), "", num(c.n_assert), "", num(c.n_changed), "", num(c.n_changed_assert)});
  }
  for (size_t j = 0; j < nn; ++j) {
    const tsm_case& c = nc[j];
    if (match[j] < 0) {
      row(*nw.path, {nb[j], "A", num(c.line + 1), "", num(c.n_lines), "", num(c.n_assert), "", num(c.n_changed), "", num(c.n_changed_assert), ""});
      continue;
    }
    const tsm_case& d = oc[(size_t)match[j]];
    if (c.n_changed || d.n_changed || c.n_lines != d.n_lines)
      row(*nw.path, {nb[j], "M", num(c.line + 1), num(d.line + 1), num(c.n_lines), num(d.n_lines), num(c.n_assert), num(d.n_assert),
                     num(c.n_changed), num(d.n_changed), num(c.n_changed_assert), num(d.n_changed_assert)});
  }
}

// The lexical records of one side's tests (docs/SPEC.md section 26), or none (lex NULL).
struct LexSide { const tsm_lex_test* lex; const tsm_lex_churn* churn; };

// The --smells rows of one pair (docs/SPEC.md section 19) from its cases (as case_rows, new case index n_first being nc[0]) and
// its tests ot / nt with their churn records och / nch: two tests match when their cases do.  D tests in old line order, then A
// and M tests in new line order, each test's rows in smell order: the nine, then with lexical records (ol / nl) the five of
// section 26, whose smells, instances and churn those records give.
static void smell_rows(std::ostream& os, const std::vector<std::string>& lead, const CaseSide& o, const CaseSide& nw, const std::string* old_path,
                       const tsm_case* oc, size_t no, const tsm_case* nc, size_t nn, size_t o_first, size_t n_first,
                       const tsm_smell_test* ot, const tsm_test_churn* och, size_t nto, const tsm_smell_test* nt, const tsm_test_churn* nch,
                       size_t ntn, LexSide ol, LexSide nl) {
  const int nk = TSM_N_SMELLS + (ol.lex || nl.lex ? TSM_N_LSMELLS : 0);   // (a side without tests has no records)
  auto name_of = [](int k) { return k < TSM_N_SMELLS ? kSmellNames[k] : kLexSmellNames[k - TSM_N_SMELLS]; };
  auto smells = [](const tsm_smell_test& x, LexSide l, size_t t) {   // the nine bits, then the five
    return (uint32_t)x.smells | (l.lex ? l.lex[t].smells << TSM_N_SMELLS : 0u);
  };
  auto inst = [](const tsm_test_churn& c, LexSide l, size_t t, int k) {
    return (int64_t)(k < TSM_N_SMELLS ? c.instances[k] : l.churn[t].instances[k - TSM_N_SMELLS]);
  };
  auto churned = [](const tsm_test_churn& c, LexSide l, size_t t, int k) {
    return (int64_t)(k < TSM_N_SMELLS ? c.churned[k] : l.churn[t].churned[k - TSM_N_SMELLS]);
  };
  const PairCaseMatch pm(o, nw, oc, no, nc, nn, o_first);
  std::vector<int64_t> test_of_case(no, -1), pair_of(ntn, -1);   // old test of each old case; matched old test of each new test
  std::vector<char> old_matched(nto, 0);
  for (size_t t = 0; t < nto; ++t) test_of_case[(size_t)och[t].case_idx - o_first] = (int64_t)t;
  for (size_t t = 0; t < ntn; ++t) {
    const int64_t m = pm.match[(size_t)nch[t].case_idx - n_first];
    if (m >= 0 && test_of_case[(size_t)m] >= 0) { pair_of[t] = test_of_case[(size_t)m]; old_matched[(size_t)pair_of[t]] = 1; }
  }
  auto num = [](int64_t v) { return std::to_string(v); };
  auto row = [&](const std::string& path, const std::string& test, std::vector<std::string> cells) {
    std::vector<std::string> r = lead;
    r.insert(r.end(), {path, test});
    r.insert(r.end(), cells.begin(), cells.end());
    if (old_path) r.push_back(*old_path);
    csv_row(os, r);
  };
  for (size_t t = 0; t < nto; ++t) {
    if (old_matched[t]) continue;
    const std::string& name = pm.na[(size_t)och[t].case_idx - o_first];
    const uint32_t sm = smells(ot[t], ol, t);
    for (int k = 0; k < nk; ++k)
      if (sm >> k & 1u)
        row(*o.path, name, {"D", "", num(ot[t].line + 1), name_of(k), "removed", "", num(inst(och[t], ol, t, k)), "",
                            num(churned(och[t], ol, t, k))});
  }
  for (size_t t = 0; t < ntn; ++t) {
    const std::string& name = pm.nb[(size_t)nch[t].case_idx - n_first];
    const tsm_smell_test& x = nt[t];
    const tsm_test_churn& c = nch[t];
    const uint32_t sn = smells(x, nl, t);
    if (pair_of[t] < 0) {
      for (int k = 0; k < nk; ++k)
        if (sn >> k & 1u)
          row(*nw.path, name, {"A", num(x.line + 1), "", name_of(k), "introduced", num(inst(c, nl, t, k)), "", num(churned(c, nl, t, k)), ""});
      continue;
    }
    const size_t u = (size_t)pair_of[t];
    const tsm_smell_test& y = ot[u];
    const tsm_test_churn& d = och[u];
    const uint32_t so = smells(y, ol, u);
    for (int k = 0; k < nk; ++k) {
      const bool hn = sn >> k & 1u, ho = so >> k & 1u;
      const int64_t cn = churned(c, nl, t, k), co = churned(d, ol, u, k);
      const char* ev = hn && !ho ? "introduced" : ho && !hn ? "removed" : hn && ho && (cn || co) ? "changed" : nullptr;
      if (ev)
        row(*nw.path, name, {"M", num(x.line + 1), num(y.line + 1), name_of(k), ev, num(inst(c, nl, t, k)), num(inst(d, ol, u, k)),
                             num(cn), num(co)});
    }
  }
}

// The --assert-edits rows of pair `pair` (docs/SPEC.md section 17), in new line order: `lead` cells, fileName (the new path),
// 1-based oldLine and line, similarity in %, statement and category of both lines, then oldFileName when old_path is given.
// `ke` walks the edits (aev order) and `kr` the deleted-line events across calls.
static void edit_rows(std::ostream& os, const std::vector<std::string>& lead, const CaseSide& o, const CaseSide& nw, const std::string* old_path,
                      const ChangedAsserts& chg, const std::vector<tsm_assert_edit>& ed, size_t& ke, size_t& kr, uint32_t pair) {
  const size_t r0 = kr;
  LineCounter lo{o.base}, ln{nw.base};
  std::vector<int64_t> old_line;                           // line of each deleted-line event of the pair (events in line order)
  for (; kr < chg.rev.size() && chg.rev[kr].file == pair; ++kr) old_line.push_back(lo.at(chg.rev[kr].line_off));
  for (; ke < ed.size() && chg.aev[(size_t)ed[ke].aev].file == pair; ++ke) {
    const tsm_assert_edit& e = ed[ke];
    const tsm_assert_event &a = chg.rev[(size_t)e.rev], &b = chg.aev[(size_t)e.aev];
    std::vector<std::string> row = lead;
    row.insert(row.end(), {*nw.path, std::to_string(old_line[(size_t)e.rev - r0]), std::to_string(ln.at(b.line_off)), std::to_string(e.score / 600),
                           event_statement(o.base, o.size, a), event_statement(nw.base, nw.size, b), event_category(o.base, a),
                           event_category(nw.base, b)});
    if (old_path) row.push_back(*old_path);
    csv_row(os, row);
  }
}

// Moved code (docs/SPEC.md section 20) of one diff call: the first global line of every pair on each side and the moved blocks of
// both sides (tsm_diff_pairs_moves, the batch's groups being its steps), block arrays grown to the counts the library reports.
struct MoveLists { std::vector<int64_t> base[2]; std::vector<tsm_move_block> blocks[2]; };
static void diff_moves(tsm_ctx* ctx, const tsm_corpus& ca, const tsm_corpus& cn, MoveLists& r) {
  const size_t n = (size_t)ca.n_files;
  std::vector<int64_t> added(n), removed(n);
  for (std::vector<int64_t>& b : r.base) b.assign(n + 1, 0);
  int64_t cap[2] = {1024, 1024};
  for (;;) {
    for (int s = 0; s < 2; ++s) r.blocks[s].resize((size_t)cap[s]);
    tsm_diff_moves o{{r.base[0].data(), r.base[1].data(), nullptr, 0, 0, nullptr, 0, 0}, r.blocks[0].data(), cap[0], 0, r.blocks[1].data(), cap[1], 0};
    const int rc = tsm_diff_pairs_moves(ctx, &ca, &cn, added.data(), removed.data(), nullptr, &o, nullptr);
    if (rc == TSM_E_CAPACITY && (o.n_old_blocks > cap[0] || o.n_new_blocks > cap[1])) {
      cap[0] = std::max(cap[0], o.n_old_blocks); cap[1] = std::max(cap[1], o.n_new_blocks);
      continue;
    }
    ck(rc, "tsm_diff_pairs_moves");
    r.blocks[0].resize((size_t)o.n_old_blocks); r.blocks[1].resize((size_t)o.n_new_blocks);
    return;
  }
}

// The --moves rows of pair i (docs/SPEC.md section 20): `lead` cells, fileName, change ('-' a block moved away, old side; '+' a
// block moved here, new side), 1-based line, lines, asserts, then otherFileName and the 1-based otherLine of the block's partner
// on the other side.  The '-' rows in old line order, then the '+' rows in new line order.  k[s] walks the blocks of side s
// across calls; path(s, j) is the path of pair j on side s.
static void move_rows(std::ostream& os, const std::vector<std::string>& lead, const MoveLists& m, size_t i, size_t k[2],
                      const std::function<const std::string&(int, size_t)>& path) {
  for (int s = 0; s < 2; ++s) {
    const std::vector<int64_t>&here = m.base[s], &there = m.base[1 - s];
    for (; k[s] < m.blocks[s].size() && m.blocks[s][k[s]].line < here[i + 1]; ++k[s]) {
      const tsm_move_block& b = m.blocks[s][k[s]];
      const size_t j = (size_t)(std::upper_bound(there.begin(), there.end(), b.partner) - there.begin()) - 1;
      std::vector<std::string> row = lead;
      row.insert(row.end(), {path(s, i), s ? "+" : "-", std::to_string(b.line - here[i] + 1), std::to_string(b.n_lines),
                             std::to_string(b.n_assert), path(1 - s, j), std::to_string(b.partner - there[j] + 1)});
      csv_row(os, row);
    }
  }
}

// One changed file of a revision pair.  `step` is its commit (history) or 0 (diff); `o` and `n` name the bytes of the old and
// the new side for the caller's loader, -1 where that side does not exist.  A rename (--find-renames) moves the deleted file's
// `o` onto the added file and keeps the deleted file's path and the score in %.
struct Change { size_t step; std::string path; int64_t o, n; std::string old_path; int similarity; };
using Loader = std::function<std::vector<uint8_t>(int64_t)>;

// Per step: lines added and removed, files diffed.  Over all steps: binary files skipped, files diffed, renames.
struct ChangeTotals {
  std::vector<int64_t> added, removed, files;
  int64_t binaries = 0, diffed = 0, renames = 0, renames_exact = 0;
  explicit ChangeTotals(size_t n_steps) : added(n_steps, 0), removed(n_steps, 0), files(n_steps, 0) {}
};

// Like git's numstat, no line counts for a binary file: one with a NUL byte in its first 8000.
static bool binary(const std::vector<uint8_t>& v) { return !v.empty() && memchr(v.data(), 0, std::min<size_t>(v.size(), 8000)) != nullptr; }

// --find-renames: the deleted and the added files of a step (binary ones left out) form a group; groups are paired together
// until a side holds batch_bytes bytes (a group is never split, so the pairs do not depend on where that is), then every pair's
// two changes become one (old side of the deleted file, new side of the added one) at the added file's place.
static void pair_renames(tsm_ctx* ctx, std::vector<Change>& changes, const Loader& load, int pct, int64_t batch_bytes, ChangeTotals& t) {
  struct Move { size_t del, add; int similarity; };
  std::vector<Move> moves;
  std::vector<RenameGroup> groups;
  std::vector<std::vector<size_t>> at_del, at_add;        // change of each file of each group
  int64_t bytes_d = 0, bytes_a = 0;
  auto flush = [&]() {
    find_renames(ctx, groups, pct);
    for (size_t g = 0; g < groups.size(); ++g)
      for (const RenamePair& rp : groups[g].pairs) {
        moves.push_back({at_del[g][rp.del], at_add[g][rp.add], rp.similarity});
        t.renames_exact += rp.exact;
      }
    groups.clear(); at_del.clear(); at_add.clear();
    bytes_d = bytes_a = 0;
  };
  for (size_t c0 = 0, c1 = 0; c0 < changes.size(); c0 = c1) {
    std::vector<size_t> del, add;
    for (c1 = c0; c1 < changes.size() && changes[c1].step == changes[c0].step; ++c1) {
      if (changes[c1].o >= 0 && changes[c1].n < 0) del.push_back(c1);
      if (changes[c1].o < 0 && changes[c1].n >= 0) add.push_back(c1);
    }
    if (del.empty() || add.empty()) continue;
    RenameGroup G;
    std::vector<size_t> gd, ga;
    for (size_t c : del) {
      std::vector<uint8_t> x = load(changes[c].o);
      if (!binary(x)) { bytes_d += (int64_t)x.size() + 256; G.del.push_back({changes[c].path, std::move(x)}); gd.push_back(c); }
    }
    for (size_t c : add) {
      std::vector<uint8_t> x = load(changes[c].n);
      if (!binary(x)) { bytes_a += (int64_t)x.size() + 256; G.add.push_back({changes[c].path, std::move(x)}); ga.push_back(c); }
    }
    if (G.del.empty() || G.add.empty()) continue;
    groups.push_back(std::move(G)); at_del.push_back(gd); at_add.push_back(ga);
    if (bytes_d >= batch_bytes || bytes_a >= batch_bytes) flush();
  }
  if (!groups.empty()) flush();
  std::vector<char> drop(changes.size(), 0);
  for (const Move& m : moves) {
    Change& a = changes[m.add];
    a.o = changes[m.del].o; a.old_path = changes[m.del].path; a.similarity = m.similarity;
    drop[m.del] = 1;
  }
  t.renames = (int64_t)moves.size();
  std::vector<Change> kept;
  for (size_t c = 0; c < changes.size(); ++c) if (!drop[c]) kept.push_back(std::move(changes[c]));
  changes.swap(kept);
}

// One batch of revision pairs: the changes [r0, r1), of which those at `idx` (ascending) are packed into the two sides, pair i
// being change idx[i]; the others are binary on a side and skipped.  With grouped steps, group g of both sides is step
// group_step[g]; else every pair is in group 0.
struct PairBatch {
  size_t r0, r1;
  std::vector<size_t> idx;
  Batch olds, news;
  std::vector<size_t> group_step;
  tsm_ctx* ctx;
  int32_t n_groups() const { return group_step.empty() ? 1 : (int32_t)group_step.size(); }
};

// The changes cut in order into batches, each handed to `fn`, one whose changes are all binary too (with an empty idx).  Both
// sides are loaded until one holds batch_bytes bytes; with group_steps (the assertion tables and the moves: a group is a u16) a
// batch also holds at most 65 535 steps, binary-only steps counted.  With whole_steps (the moves, which cross the files of a
// step) a batch takes whole steps: a step joins it only while both sides stay within batch_bytes and the int32-indexed arena, so
// a step larger than that is a batch of its own (and one larger than the arena is refused).  A step loaded but not taken is kept
// for the next batch.  t.binaries and t.diffed count the skipped and the packed changes.
static void pair_batches(tsm_ctx* ctx, const std::vector<Change>& changes, const Loader& load, int64_t batch_bytes, bool group_steps,
                         bool whole_steps, ChangeTotals& t, const std::function<void(const PairBatch&)>& fn) {
  struct StepLoad { size_t s1 = 0; std::vector<size_t> idx; std::vector<std::vector<uint8_t>> x, y; int64_t so = 0, sn = 0, binaries = 0; };
  auto load_pair = [&](size_t r, std::vector<uint8_t>& x, std::vector<uint8_t>& y) {   // false: binary on a side
    const Change& c = changes[r];
    x = c.o >= 0 ? load(c.o) : std::vector<uint8_t>(); y = c.n >= 0 ? load(c.n) : std::vector<uint8_t>();
    if (binary(x) || binary(y)) return false;
    if (x.size() > 0x7fff0000u || y.size() > 0x7fff0000u) die("blob too large: " + c.path);
    return true;
  };
  auto load_step = [&](size_t r1) {                        // the changes of the step that starts at r1
    StepLoad S;
    for (S.s1 = r1; S.s1 < changes.size() && changes[S.s1].step == changes[r1].step; ++S.s1) {
      std::vector<uint8_t> x, y;
      if (!load_pair(S.s1, x, y)) { ++S.binaries; continue; }
      S.so += (int64_t)x.size() + 256; S.sn += (int64_t)y.size() + 256;
      S.x.push_back(std::move(x)); S.y.push_back(std::move(y)); S.idx.push_back(S.s1);
    }
    return S;
  };
  const int64_t arena_max = (1ll << 31) - 4097;
  std::optional<StepLoad> carry;                           // whole_steps: the loaded step the previous batch did not take
  for (size_t r0 = 0, r1 = 0; r0 < changes.size(); r0 = r1) {
    PairBatch b{r0, r0, {}, {}, {}, {}, ctx};
    std::vector<std::vector<uint8_t>> blobs[2];            // old, new
    int64_t so = 0, sn = 0;
    size_t steps = 0;
    if (whole_steps) {
      const int64_t limit = std::min(batch_bytes, arena_max);
      for (r1 = r0; r1 < changes.size();) {
        StepLoad S = carry ? std::move(*carry) : load_step(r1);
        carry.reset();
        if (r1 > r0 && (so + S.so > limit || sn + S.sn > limit || (group_steps && steps + 1 > 65535))) { carry = std::move(S); break; }
        ++steps;
        t.binaries += S.binaries;
        for (size_t k = 0; k < S.idx.size(); ++k) {
          blobs[0].push_back(std::move(S.x[k])); blobs[1].push_back(std::move(S.y[k])); b.idx.push_back(S.idx[k]);
        }
        so += S.so; sn += S.sn;
        r1 = S.s1;
      }
      if (std::max(so, sn) > arena_max)
        die("--moves keeps every step in one batch, and a side of step " + std::to_string(changes[r0].step) +
            " does not fit an int32-indexed arena (2 GiB)");
    } else {
      for (r1 = r0; r1 < changes.size() && so < batch_bytes && sn < batch_bytes; ++r1) {
        const Change& c = changes[r1];
        if (group_steps && (r1 == r0 || c.step != changes[r1 - 1].step) && ++steps > 65535) break;
        std::vector<uint8_t> x, y;
        if (!load_pair(r1, x, y)) { ++t.binaries; continue; }
        so += (int64_t)x.size() + 256; sn += (int64_t)y.size() + 256;
        blobs[0].push_back(std::move(x)); blobs[1].push_back(std::move(y)); b.idx.push_back(r1);
      }
    }
    b.r1 = r1;
    std::vector<const std::vector<uint8_t>*> sides[2];
    for (int s = 0; s < 2; ++s) for (const std::vector<uint8_t>& v : blobs[s]) sides[s].push_back(&v);
    b.olds = pack(sides[0]); b.news = pack(sides[1]);
    // ext tags of both sides feed the assertion-line classification of the changed lines
    for (size_t i = 0; i < b.idx.size(); ++i) {
      const Change& c = changes[b.idx[i]];
      b.news.ext[i] = (uint8_t)ext_tag(c.path);
      b.olds.ext[i] = c.old_path.empty() ? b.news.ext[i] : (uint8_t)ext_tag(c.old_path);
      if (!group_steps) continue;
      if (b.group_step.empty() || b.group_step.back() != c.step) b.group_step.push_back(c.step);
      b.olds.grp[i] = b.news.grp[i] = (uint16_t)(b.group_step.size() - 1);
    }
    t.diffed += (int64_t)b.idx.size();
    fn(b);
  }
}

// What `diff` and `history` write.  Every row starts with the `lead(step)` cells named `lead_head`; the --assert-churn rows with
// the first `churn_lead` of them.  --out has a row for every diffed change when `zero_rows`, else only for those that change a
// line or pair a rename.  An empty path is an output not asked for; rename_pct -1 is no rename pairing.
struct DiffOptions {
  int rename_pct = -1;
  int64_t batch_bytes = kBatch;
  std::string out, asserts, churn, cases, edits, smells, moves;
  bool smell_lexical = false;                              // --lexical, read only with --smells
  std::string clones;                                      // --clones F, with its --min-lines, --blind and the file selection
  int clone_min_lines = 5; bool clone_blind = false, all_files = false;
  std::string links;                                       // --links F (docs/SPEC.md section 28)
  std::string similar;                                     // --similar-tests F, with --min-lines (shared with --clones) and --similarity
  int similar_min_lines = 5, similar_pct = 70;
  bool zero_rows = false;
  std::vector<std::string> lead_head;
  size_t churn_lead = 0;
  std::function<std::vector<std::string>(size_t)> lead = [](size_t) { return std::vector<std::string>(); };
};

// The diff of one batch: per pair the lines added and removed and the detail; with `asserts` the changed assertion lines and
// the [group][K] tables, with `edits` also the assertion edits (the same call), with `cases` the case records, with `smells`
// the case records, the tests and their smell churn (one call, which also serves `cases`; with `lexical` also the lexical smells),
// with `moves` the moved blocks (a call of its own).
struct PairDiff {
  std::vector<int64_t> added, removed; std::vector<tsm_diff_detail> det; ChangedAsserts chg; CaseLists cases; std::vector<tsm_assert_edit> edits;
  SmellLists smells; MoveLists moves;
};
static PairDiff diff_batch(const PairBatch& b, bool asserts, bool cases, bool edits, bool smells, bool lexical, bool moves) {
  const size_t n = b.idx.size();
  PairDiff d{std::vector<int64_t>(n), std::vector<int64_t>(n), std::vector<tsm_diff_detail>(n), {}, {}, {}, {}, {}};
  const tsm_corpus ca = b.olds.corpus(b.n_groups()), cn = b.news.corpus(b.n_groups());
  if (edits) diff_assert_edits(b.ctx, ca, cn, d.added.data(), d.removed.data(), d.det.data(), d.chg, d.edits);
  else if (asserts) diff_asserts(b.ctx, ca, cn, d.added.data(), d.removed.data(), d.det.data(), d.chg);
  else if (smells) diff_smells(b.ctx, ca, cn, d.added.data(), d.removed.data(), d.det.data(), d.cases, d.smells, lexical);
  else if (cases) diff_cases(b.ctx, ca, cn, d.added.data(), d.removed.data(), d.det.data(), d.cases);
  else ck(tsm_diff_pairs_detail(b.ctx, &ca, &cn, d.added.data(), d.removed.data(), d.det.data(), nullptr), "tsm_diff_pairs_detail");
  if (asserts && (cases || smells)) {                      // a second call: the assertion tables and the cases are separate diffs
    std::vector<int64_t> a2(n), r2(n);
    if (smells) diff_smells(b.ctx, ca, cn, a2.data(), r2.data(), nullptr, d.cases, d.smells, lexical);
    else diff_cases(b.ctx, ca, cn, a2.data(), r2.data(), nullptr, d.cases);
  }
  if (moves) diff_moves(b.ctx, ca, cn, d.moves);
  return d;
}

// The diff of an ordered list of changes of `n_steps` steps, after --find-renames pairing: one diff_batch per batch of
// pair_batches, its steps grouped when the assertion tables are asked for, then the rows.
static ChangeTotals diff_changes(std::vector<Change>& changes, size_t n_steps, const Loader& load, const DiffOptions& o) {
  ChangeTotals t(n_steps);
  const bool renames = o.rename_pct >= 0;
  const auto ctx = small_context();
  if (renames) pair_renames(ctx.get(), changes, load, o.rename_pct, o.batch_bytes, t);
  std::ofstream os, as, cs, ch, es, ss, ms;                // --out, --asserts, --cases, --assert-churn, --assert-edits, --smells, --moves
  auto open = [&](std::ofstream& f, const std::string& path, size_t n_lead, std::vector<std::string> head) {
    if (path.empty()) return;
    f.open(path, std::ios::binary);
    head.insert(head.begin(), o.lead_head.begin(), o.lead_head.begin() + (long)n_lead);
    csv_row(f, head);
  };
  std::vector<std::string> out_head = {"fileName", "cloc", "added", "removed", "hunks_add", "hunks_del", "hunks_mod", "added_assert", "removed_assert"};
  std::vector<std::string> case_head = {"fileName", "case", "change", "line", "oldLine", "lines", "oldLines", "asserts", "oldAsserts",
                                        "insertedLines", "deletedLines", "insertedAsserts", "deletedAsserts"};
  if (renames) out_head.insert(out_head.end(), {"oldFileName", "similarity"});
  if (renames) case_head.push_back("oldFileName");
  std::vector<std::string> edit_head = {"fileName", "oldLine", "line", "similarity", "oldStatement", "statement", "oldCategory", "category"};
  if (renames) edit_head.push_back("oldFileName");
  std::vector<std::string> smell_head = {"fileName", "test", "change", "line", "oldLine", "smell", "event", "instances", "oldInstances",
                                         "addedInstances", "removedInstances"};
  if (renames) smell_head.push_back("oldFileName");
  open(os, o.out, o.lead_head.size(), out_head);
  open(as, o.asserts, o.lead_head.size(), {"fileName", "change", "line", "statement", "category"});
  open(cs, o.cases, o.lead_head.size(), case_head);
  open(ch, o.churn, o.churn_lead, {"category", "added", "removed"});
  open(es, o.edits, o.lead_head.size(), edit_head);
  open(ss, o.smells, o.lead_head.size(), smell_head);
  open(ms, o.moves, o.lead_head.size(), {"fileName", "change", "line", "lines", "asserts", "otherFileName", "otherLine"});
  const bool want_asserts = !o.asserts.empty() || !o.churn.empty() || es.is_open();
  std::map<size_t, std::vector<int64_t>> churn;            // per step with changed assertion lines: its [K] added and removed rows
  pair_batches(ctx.get(), changes, load, o.batch_bytes, want_asserts || ms.is_open(), ms.is_open(), t, [&](const PairBatch& b) {
    const size_t n = b.idx.size();
    if (!n) return;
    const PairDiff d = diff_batch(b, want_asserts, cs.is_open(), es.is_open(), ss.is_open(), o.smell_lexical, ms.is_open());
    auto path = [&](int s, size_t j) -> const std::string& {  // the path of pair j on side s (0 old, 1 new)
      const Change& c = changes[b.idx[j]];
      return s == 0 && !c.old_path.empty() ? c.old_path : c.path;
    };
    size_t km[2] = {0, 0};                                 // the first block of each side of pair i
    for (size_t g = 0; ch.is_open() && g < b.group_step.size(); ++g) {   // a step's files may span two batches
      const int64_t* ad = d.chg.added_counts.data() + g * TSM_NUM_CATEGORIES;
      const int64_t* rm = d.chg.removed_counts.data() + g * TSM_NUM_CATEGORIES;
      if (std::all_of(ad, ad + TSM_NUM_CATEGORIES, [](int64_t v) { return v == 0; }) &&
          std::all_of(rm, rm + TSM_NUM_CATEGORIES, [](int64_t v) { return v == 0; })) continue;
      std::vector<int64_t>& tab = churn[b.group_step[g]];
      tab.resize(2 * TSM_NUM_CATEGORIES, 0);
      for (int k = 0; k < TSM_NUM_CATEGORIES; ++k) { tab[(size_t)k] += ad[k]; tab[(size_t)(TSM_NUM_CATEGORIES + k)] += rm[k]; }
    }
    // ka, kr, ko, kn, to, tn: pair i's first event, case and test of each side; ke, ker: its first edit and the deleted-line event
    // edit_rows is at
    for (size_t i = 0, ka = 0, kr = 0, ko = 0, kn = 0, to = 0, tn = 0, ke = 0, ker = 0; i < n; ++i) {
      const Change& c = changes[b.idx[i]];
      const std::string& old_path = c.old_path.empty() ? c.path : c.old_path;
      const CaseSide olds{b.olds.arena.get() + b.olds.off[i], b.olds.len[i], b.olds.ext[i], &old_path};
      const CaseSide news{b.news.arena.get() + b.news.off[i], b.news.len[i], b.news.ext[i], &c.path};
      if (as.is_open()) {
        assert_rows(as, o.lead(c.step), old_path, olds.base, olds.size, d.chg.rev, kr, (uint32_t)i, "-");
        assert_rows(as, o.lead(c.step), c.path, news.base, news.size, d.chg.aev, ka, (uint32_t)i, "+");
      }
      if (es.is_open()) edit_rows(es, o.lead(c.step), olds, news, renames ? &c.old_path : nullptr, d.chg, d.edits, ke, ker, (uint32_t)i);
      const size_t o0 = ko, n0 = kn;
      while (ko < d.cases.olds.size() && d.cases.olds[ko].pair == (int32_t)i) ++ko;
      while (kn < d.cases.news.size() && d.cases.news[kn].pair == (int32_t)i) ++kn;
      if (cs.is_open() && (ko > o0 || kn > n0))
        case_rows(cs, o.lead(c.step), olds, news, renames ? &c.old_path : nullptr, d.cases.olds.data() + o0, ko - o0, d.cases.news.data() + n0,
                  kn - n0, o0);
      const size_t to0 = to, tn0 = tn;
      auto lex_side = [](const std::vector<tsm_lex_test>& l, const std::vector<tsm_lex_churn>& c, size_t t0) {
        return l.empty() ? LexSide{nullptr, nullptr} : LexSide{l.data() + t0, c.data() + t0};
      };
      while (to < d.smells.olds.size() && d.smells.olds[to].file == (int32_t)i) ++to;
      while (tn < d.smells.news.size() && d.smells.news[tn].file == (int32_t)i) ++tn;
      if (to > to0 || tn > tn0)
        smell_rows(ss, o.lead(c.step), olds, news, renames ? &c.old_path : nullptr, d.cases.olds.data() + o0, ko - o0, d.cases.news.data() + n0,
                   kn - n0, o0, n0, d.smells.olds.data() + to0, d.smells.old_churn.data() + to0, to - to0, d.smells.news.data() + tn0,
                   d.smells.new_churn.data() + tn0, tn - tn0, lex_side(d.smells.old_lex, d.smells.old_lchurn, to0),
                   lex_side(d.smells.new_lex, d.smells.new_lchurn, tn0));
      if (ms.is_open()) move_rows(ms, o.lead(c.step), d.moves, i, km, path);
      t.added[c.step] += d.added[i]; t.removed[c.step] += d.removed[i]; t.files[c.step]++;
      if (!os.is_open() || !(o.zero_rows || d.added[i] || d.removed[i] || c.similarity >= 0)) continue;
      std::vector<std::string> row = o.lead(c.step);
      row.insert(row.end(), {c.path, std::to_string(d.added[i] + d.removed[i]), std::to_string(d.added[i]), std::to_string(d.removed[i]),
                             std::to_string(d.det[i].hunks_add), std::to_string(d.det[i].hunks_del), std::to_string(d.det[i].hunks_mod),
                             std::to_string(d.det[i].added_assert), std::to_string(d.det[i].removed_assert)});
      if (renames) row.insert(row.end(), {c.old_path, c.similarity >= 0 ? std::to_string(c.similarity) : ""});
      csv_row(os, row);
    }
  });
  for (const auto& kv : churn) {
    const std::vector<std::string> l = o.lead(kv.first);
    churn_rows(ch, {l.begin(), l.begin() + (long)o.churn_lead}, kv.second.data(), kv.second.data() + TSM_NUM_CATEGORIES);
  }
  return t;
}

// ---------------------------------------------------------------------------------- clone churn (docs/SPEC.md section 22)
// A revision of the clone churn: its selected files in the order of `clones --git --rev` (walk_git: path components compared
// one by one) with their bytes, and those bytes packed once into a pinned arena.
static bool path_less(const std::string& a, const std::string& b) {
  for (size_t i = 0, j = 0;;) {
    size_t ei = a.find('/', i), ej = b.find('/', j);
    if (ei == std::string::npos) ei = a.size();
    if (ej == std::string::npos) ej = b.size();
    const int c = a.compare(i, ei - i, b, j, ej - j);
    if (c) return c < 0;
    if (ei == a.size() || ej == b.size()) return ei == a.size() && ej != b.size();
    i = ei + 1; j = ej + 1;
  }
}
struct PathLess { bool operator()(const std::string& a, const std::string& b) const { return path_less(a, b); } };
using Blob = std::shared_ptr<const std::vector<uint8_t>>;
struct Revision {
  std::vector<std::string> paths;
  std::vector<Blob> blobs;
  Batch b;
  std::map<std::string, int32_t> index;                    // path -> file index
};
static Revision make_revision(const std::map<std::string, Blob, PathLess>& files) {
  Revision r;
  std::vector<const std::vector<uint8_t>*> bytes;
  std::vector<int32_t> len, off(files.size() + 1);
  for (const auto& kv : files) {
    r.index[kv.first] = (int32_t)r.paths.size();
    r.paths.push_back(kv.first); r.blobs.push_back(kv.second); bytes.push_back(kv.second.get());
    len.push_back((int32_t)kv.second->size());
  }
  const int64_t need = tsm_layout(len.data(), (int32_t)len.size(), off.data());
  if (need < 0 || need + 4096 >= (1ll << 31))
    die("the selected files (" + std::to_string(need < 0 ? INT64_MAX : need + 4096) + " bytes of arena) do not fit one int32-indexed "
        "arena; clones are found across all files at once, so select fewer files");
  r.b = pack(bytes);
  for (size_t i = 0; i < r.paths.size(); ++i) r.b.ext[i] = (uint8_t)ext_tag(r.paths[i]);
  return r;
}

static const char* const kCloneStatus[] = {"untouched", "changed", "removed", "diverged", "dropped", "created", "copied", "joined"};
static const char* const kFragState[] = {"kept", "edited", "whole"};

// The file pairs of one step: the step's changes (after --find-renames; `old_path` names the old side of a rename) as file
// indices of the two revisions.  A change binary on a side (a NUL byte in its first 8000) is a deletion plus an addition.
struct StepPairs { std::vector<int32_t> po, pn; };
static StepPairs step_pairs(const Revision& ro, const Revision& rn, const Change* c0, const Change* c1,
                            const std::function<bool(const Change&)>& is_binary) {
  StepPairs sp;
  for (const Change* c = c0; c != c1; ++c) {
    const int32_t a = c->o >= 0 ? ro.index.at(c->old_path.empty() ? c->path : c->old_path) : -1;
    const int32_t b = c->n >= 0 ? rn.index.at(c->path) : -1;
    if (a >= 0 && b >= 0 && is_binary(*c)) { sp.po.push_back(a); sp.pn.push_back(-1); sp.po.push_back(-1); sp.pn.push_back(b); }
    else { sp.po.push_back(a); sp.pn.push_back(b); }
  }
  return sp;
}

// What the step driver hands each step to: the two revisions, the step's pairs and the lead cells of its rows.
using StepSink = std::function<void(tsm_ctx*, const Revision&, const Revision&, const StepPairs&, const std::vector<std::string>&)>;

// One step of --clones: tsm_clone_churn over the two revisions and the step's pairs, then one row per fragment of every touched
// class, the old side first.
static void clone_churn_step(tsm_ctx* ctx, const Revision& ro, const Revision& rn, const StepPairs& sp, const DiffOptions& d,
                             const std::vector<std::string>& lead, std::ostream& os) {
  const std::vector<int32_t>&po = sp.po, &pn = sp.pn;
  const Revision* rev[2] = {&ro, &rn};
  struct Side { std::vector<int64_t> base, cbase, member, kbase, kline; std::vector<uint32_t> clen, changed, changed_a, counts; std::vector<uint8_t> state, status; };
  Side S[2];
  tsm_clone_churn_side cs[2] = {};
  const tsm_corpus co = ro.b.corpus(1), cn = rn.b.corpus(1);
  auto call = [&] {
    ck(tsm_clone_churn(ctx, &co, &cn, po.data(), pn.data(), (int64_t)po.size(), d.clone_min_lines, d.clone_blind, &cs[0], &cs[1], nullptr),
       "tsm_clone_churn");
  };
  for (int s = 0; s < 2; ++s) {
    S[s].base.resize(rev[s]->paths.size() + 1); S[s].kbase.resize(rev[s]->paths.size() + 1);
    cs[s].clones.line_base = S[s].base.data(); cs[s].blind.kept_base = S[s].kbase.data();
  }
  call();                                                  // the counts; the second call fills arrays of that size
  for (int s = 0; s < 2; ++s) {
    Side& x = S[s];
    tsm_clone_churn_side& c = cs[s];
    const size_t nc = (size_t)c.clones.n_classes, nm = (size_t)c.clones.n_members, nk = (size_t)c.blind.n_kept;
    x.cbase.resize(nc + 1); x.clen.resize(std::max<size_t>(nc, 1)); x.counts.resize(3 * std::max<size_t>(nc, 1)); x.status.resize(std::max<size_t>(nc, 1));
    x.member.resize(std::max<size_t>(nm, 1)); x.changed.resize(std::max<size_t>(nm, 1)); x.changed_a.resize(std::max<size_t>(nm, 1));
    x.state.resize(std::max<size_t>(nm, 1)); x.kline.resize(std::max<size_t>(nk, 1));
    c.clones.class_base = x.cbase.data(); c.clones.class_len = x.clen.data(); c.clones.class_cap = (int64_t)nc;
    c.clones.member = x.member.data(); c.clones.member_cap = (int64_t)nm;
    c.blind.kept_line = x.kline.data(); c.blind.kept_cap = (int64_t)nk;
    c.changed = x.changed.data(); c.changed_assert = x.changed_a.data(); c.state = x.state.data();
    c.class_counts = x.counts.data(); c.status = x.status.data();
  }
  call();
  for (int s = 0; s < 2; ++s) {
    const Side& x = S[s];
    const std::vector<int64_t>& fbase = d.clone_blind ? x.kbase : x.base;   // the numbering of member
    for (int64_t k = 0; k < cs[s].clones.n_classes; ++k) {
      if (!x.status[(size_t)k]) continue;
      const int64_t b0 = x.cbase[(size_t)k], b1 = x.cbase[(size_t)k + 1];
      for (int64_t j = b0; j < b1; ++j) {
        const int64_t at = x.member[(size_t)j], last = at + x.clen[(size_t)k] - 1;
        const size_t f = (size_t)(std::upper_bound(fbase.begin(), fbase.end(), at) - fbase.begin() - 1);
        const int64_t first = (d.clone_blind ? x.kline[(size_t)at] : at) - x.base[f] + 1;
        const int64_t end = (d.clone_blind ? x.kline[(size_t)last] : last) - x.base[f] + 1;
        std::vector<std::string> row = lead;
        row.insert(row.end(), {s ? "+" : "-", std::to_string(k + 1), kCloneStatus[x.status[(size_t)k]], std::to_string(b1 - b0),
                               rev[s]->paths[f], std::to_string(first), std::to_string(end), kFragState[x.state[(size_t)j]],
                               std::to_string(x.changed[(size_t)j]), std::to_string(x.changed_a[(size_t)j])});
        csv_row(os, row);
      }
    }
  }
}

static std::vector<std::string> clone_churn_head(std::vector<std::string> lead) {
  lead.insert(lead.end(), {"side", "class", "status", "fragments", "fileName", "first_line", "last_line", "state", "changed_lines",
                           "changed_assert_lines"});
  return lead;
}

// `diff --clones` / `--similar-tests` / `--links`: the files of each root that `sel` keeps are the two revisions; a file
// whose bytes differ, or that one root lacks, is a change (then --find-renames); one step, handed to every sink.
static void diff_steps(const std::string& old_root, const std::string& new_root, const DiffOptions& o, const std::vector<StepSink>& sinks,
                       const Select& sel) {
  std::vector<FileEntry> fa, fb;
  for (int s = 0; s < 2; ++s) {
    std::vector<FileEntry> all;
    walk(s ? new_root : old_root, 0, true, all);
    for (FileEntry& f : all) if (sel(f.rel)) (s ? fb : fa).push_back(std::move(f));
  }
  std::vector<Blob> blobs;                                 // the loader's names: the files of fa, then those of fb
  std::map<std::string, Blob, PathLess> ra, rb;
  std::map<std::string, int64_t> name_a, name_b;
  for (int s = 0; s < 2; ++s)
    for (const FileEntry& f : s ? fb : fa) {
      auto v = std::make_shared<std::vector<uint8_t>>((size_t)f.size);
      if (!read_file(f.abs, v->data(), f.size)) die("short read: " + f.abs);
      if (v->size() > 0x7fff0000u) die("blob too large: " + f.rel);
      (s ? name_b : name_a)[f.rel] = (int64_t)blobs.size();
      (s ? rb : ra)[f.rel] = v;
      blobs.push_back(v);
    }
  std::vector<Change> changes;
  for (const auto& kv : ra) {
    auto it = name_b.find(kv.first);
    if (it != name_b.end() && *blobs[(size_t)it->second] == *kv.second) continue;
    changes.push_back({0, kv.first, name_a[kv.first], it == name_b.end() ? -1 : it->second, "", -1});
  }
  for (const auto& kv : rb) if (!name_a.count(kv.first)) changes.push_back({0, kv.first, -1, name_b[kv.first], "", -1});
  const Loader load = [&](int64_t s) { return *blobs[(size_t)s]; };
  const auto ctx = small_context();
  ChangeTotals t(1);
  if (o.rename_pct >= 0) pair_renames(ctx.get(), changes, load, o.rename_pct, o.batch_bytes, t);
  const Revision ro = make_revision(ra), rn = make_revision(rb);
  const StepPairs sp = step_pairs(ro, rn, changes.data(), changes.data() + changes.size(),
                                  [&](const Change& c) { return binary(*blobs[(size_t)c.o]) || binary(*blobs[(size_t)c.n]); });
  for (const StepSink& sink : sinks) sink(ctx.get(), ro, rn, sp, {});
}

// ---------------------------------------------------------------------------------- similar-test churn (docs/SPEC.md section 24)
static const char* const kSimilarStatus[] = {"changed", "removed", "dropped", "diverged", "created", "copied", "converged"};

// The 1-based header line and the case name (section 10) of every test of a revision, from the files' bytes.
struct TestNames { std::vector<std::string> name; };
static TestNames test_names(const Revision& r, const std::vector<tsm_smell_test>& tests) {
  TestNames out;
  int32_t f = -1, line = 0;
  size_t pos = 0;
  for (const tsm_smell_test& t : tests) {                  // tests in global line order: one walk per file
    const std::vector<uint8_t>& b = *r.blobs[(size_t)t.file];
    if (t.file != f) { f = t.file; line = 0; pos = 0; }
    for (; line < t.line; ++line) pos = (size_t)((const uint8_t*)memchr(b.data() + pos, '\n', b.size() - pos) - b.data()) + 1;
    const uint8_t* lf = (const uint8_t*)memchr(b.data() + pos, '\n', b.size() - pos);
    out.name.push_back(case_name(ext_tag(r.paths[(size_t)f]), b.data() + pos, (uint32_t)((lf ? (size_t)(lf - b.data()) : b.size()) - pos)));
  }
  return out;
}

// One step of --similar-tests: tsm_similar_churn over the two revisions and the step's pairs (counts first, then the arrays), then
// one row per event.  A row names its test and the other test of the pair, each on both sides (empty cells for a side without it).
static void similar_churn_step(tsm_ctx* ctx, const Revision& ro, const Revision& rn, const StepPairs& sp, const DiffOptions& d,
                               const std::vector<std::string>& lead, std::ostream& os) {
  const tsm_corpus co = ro.b.corpus(1), cn = rn.b.corpus(1);
  tsm_similar_churn_side cs[2] = {};
  int64_t n_ev = 0;
  auto call = [&](tsm_similar_event* ev) {
    ck(tsm_similar_churn(ctx, &co, &cn, sp.po.data(), sp.pn.data(), (int64_t)sp.po.size(), d.similar_min_lines, d.similar_pct, &cs[0],
                         &cs[1], ev, n_ev, &n_ev, nullptr), "tsm_similar_churn");
  };
  call(nullptr);
  std::vector<tsm_smell_test> tests[2];
  std::vector<int32_t> match[2];
  std::vector<uint8_t> change[2];
  for (int s = 0; s < 2; ++s) {
    const size_t nt = (size_t)cs[s].n_tests;
    tests[s].resize(std::max<size_t>(nt, 1)); match[s].resize(std::max<size_t>(nt, 1)); change[s].resize(std::max<size_t>(nt, 1));
    cs[s].tests = tests[s].data(); cs[s].match = match[s].data(); cs[s].change = change[s].data(); cs[s].test_cap = (int64_t)nt;
    tests[s].resize(nt);
  }
  std::vector<tsm_similar_event> ev(std::max<int64_t>(n_ev, 1));
  call(ev.data());
  const Revision* rev[2] = {&ro, &rn};
  const TestNames names[2] = {test_names(ro, tests[0]), test_names(rn, tests[1])};
  auto num = [](int64_t v) { return std::to_string(v); };
  // The cells of one test given by its index on each side (-1: absent): fileName, test, oldLine, line, change, and its old path.
  auto cells = [&](int32_t o, int32_t n, std::vector<std::string>& row, std::string& old_path) {
    const int s = n >= 0 ? 1 : 0;
    const int32_t t = s ? n : o;
    const tsm_smell_test& x = tests[s][(size_t)t];
    row.insert(row.end(), {rev[s]->paths[(size_t)x.file], names[s].name[(size_t)t], o >= 0 ? num(tests[0][(size_t)o].line + 1) : "",
                           n >= 0 ? num(tests[1][(size_t)n].line + 1) : "", std::string(1, (char)change[s][(size_t)t])});
    old_path = o >= 0 ? ro.paths[(size_t)tests[0][(size_t)o].file] : "";
  };
  const uint32_t NONE = 0xFFFFFFFFu;
  auto pct = [&](uint32_t v) { return v == NONE ? std::string() : num(v / 600); };
  auto lcs = [&](uint32_t v) { return v == NONE ? std::string() : num(v); };
  for (int64_t k = 0; k < n_ev; ++k) {
    const tsm_similar_event& e = ev[(size_t)k];
    std::vector<std::string> row = lead;
    row.push_back(kSimilarStatus[e.status]);
    std::string op_a, op_b;
    cells(e.old_a, e.a, row, op_a);
    cells(e.old_b, e.b, row, op_b);
    row.insert(row.end(), {lcs(e.old_lcs), pct(e.old_score), lcs(e.lcs), pct(e.score)});
    if (d.rename_pct >= 0) row.insert(row.end(), {op_a, op_b});
    csv_row(os, row);
  }
}

static std::vector<std::string> similar_churn_head(std::vector<std::string> lead, bool renames) {
  lead.insert(lead.end(), {"status", "fileName", "test", "oldLine", "line", "change", "otherFileName", "otherTest", "otherOldLine",
                           "otherLine", "otherChange", "oldLcs", "oldSimilarity", "lcs", "similarity"});
  if (renames) lead.insert(lead.end(), {"oldFileName", "otherOldFileName"});
  return lead;
}

// ---------------------------------------------------------------------------------- link churn (docs/SPEC.md section 28)
static const char* const kLinkEvents[] = {"added", "removed", "retargeted", "redefined", "eager_introduced", "eager_removed",
                                          "lazy_introduced", "lazy_removed"};
static const char* const kLinkCauses[] = {"test", "call", "definition"};

// One step of --links: per revision the roles (S0) and stems (tsm_focal_stems), tsm_link_churn over the two revisions and the step's
// pairs (counts first, then the arrays), then one row per event in its order.
static void link_churn_step(tsm_ctx* ctx, const Revision& ro, const Revision& rn, const StepPairs& sp, const DiffOptions& d,
                            const std::vector<std::string>& lead, std::ostream& os) {
  const Revision* rev[2] = {&ro, &rn};
  const tsm_corpus co = ro.b.corpus(1), cn = rn.b.corpus(1);
  struct Side {
    std::vector<uint8_t> role; std::vector<int32_t> stem;
    std::vector<tsm_link_test> tests; std::vector<tsm_link> links; std::vector<tsm_link_def> defs;
    std::vector<int32_t> match; std::vector<uint8_t> change;
  } S[2];
  tsm_link_churn_side cs[2] = {};
  for (int s = 0; s < 2; ++s) {
    const size_t nf = rev[s]->paths.size();
    std::vector<const char*> paths(nf);
    S[s].role.resize(std::max<size_t>(nf, 1)); S[s].stem.resize(std::max<size_t>(nf, 1));
    for (size_t i = 0; i < nf; ++i) {
      paths[i] = rev[s]->paths[i].c_str();
      S[s].role[i] = lower(rev[s]->paths[i]).find("test") != std::string::npos;   // S0
    }
    ck(tsm_focal_stems(paths.data(), S[s].role.data(), (int32_t)nf, S[s].stem.data()), "tsm_focal_stems");
  }
  int64_t n_ev = 0;
  auto call = [&](tsm_link_event* ev) {
    ck(tsm_link_churn(ctx, &co, &cn, S[0].role.data(), S[0].stem.data(), S[1].role.data(), S[1].stem.data(), sp.po.data(), sp.pn.data(),
                      (int64_t)sp.po.size(), &cs[0], &cs[1], ev, n_ev, &n_ev, nullptr), "tsm_link_churn");
  };
  call(nullptr);                                           // the counts; the second call fills arrays of that size
  for (int s = 0; s < 2; ++s) {
    tsm_links_result& r = cs[s].links;
    const size_t nt = (size_t)r.n_tests, nk = (size_t)r.n_links, nd = (size_t)r.n_defs;
    S[s].tests.resize(std::max<size_t>(nt, 1)); S[s].links.resize(std::max<size_t>(nk, 1)); S[s].defs.resize(std::max<size_t>(nd, 1));
    S[s].match.resize(std::max<size_t>(nt, 1)); S[s].change.resize(std::max<size_t>(nt, 1));
    r.tests = S[s].tests.data(); r.test_cap = (int64_t)nt; r.links = S[s].links.data(); r.link_cap = (int64_t)nk;
    r.defs = S[s].defs.data(); r.def_cap = (int64_t)nd;
    cs[s].match = S[s].match.data(); cs[s].change = S[s].change.data();
  }
  std::vector<tsm_link_event> ev((size_t)std::max<int64_t>(n_ev, 1));
  call(ev.data());
  TestNames names[2];
  for (int s = 0; s < 2; ++s) {
    std::vector<tsm_smell_test> at((size_t)cs[s].links.n_tests, tsm_smell_test{});
    for (size_t t = 0; t < at.size(); ++t) { at[t].file = S[s].tests[t].file; at[t].line = S[s].tests[t].line; }
    names[s] = test_names(*rev[s], at);
  }
  auto num = [](int64_t v) { return std::to_string(v); };
  auto opt = [&](int32_t v) { return v >= 0 ? num(v) : std::string(); };
  auto callee = [&](int s, int32_t j) {
    const tsm_link_def& df = S[s].defs[(size_t)S[s].links[(size_t)j].name_def];
    return std::string((const char*)rev[s]->blobs[(size_t)df.file]->data() + df.name_off, (size_t)df.name_len);
  };
  auto target = [&](int s, int32_t j, std::vector<std::string>& row) {   // defFile, defLine of side s's link j
    const int32_t t = j >= 0 ? S[s].links[(size_t)j].target : -1;
    if (t < 0) { row.insert(row.end(), {"", ""}); return; }
    const tsm_link_def& df = S[s].defs[(size_t)t];
    row.insert(row.end(), {rev[s]->paths[(size_t)df.file], num(df.line + 1)});
  };
  for (int64_t k = 0; k < n_ev; ++k) {
    const tsm_link_event& e = ev[(size_t)k];
    const int s = e.test >= 0 ? 1 : 0;
    const int32_t t = s ? e.test : e.old_test;
    std::vector<std::string> row = lead;
    row.insert(row.end(), {rev[s]->paths[(size_t)S[s].tests[(size_t)t].file], names[s].name[(size_t)t], std::string(1, (char)S[s].change[(size_t)t]),
                           e.test >= 0 ? num(S[1].tests[(size_t)e.test].line + 1) : "",
                           e.old_test >= 0 ? num(S[0].tests[(size_t)e.old_test].line + 1) : ""});
    if (e.event >= TSM_LINKEV_EAGER_INTRODUCED) {
      row.insert(row.end(), {"", kLinkEvents[e.event], "", "", "", "", "", "", "", "", ""});
    } else {
      row.insert(row.end(), {e.link >= 0 ? callee(1, e.link) : callee(0, e.old_link), kLinkEvents[e.event],
                             e.cause >= 0 ? kLinkCauses[e.cause] : "", opt(e.calls), opt(e.old_calls), num(e.defs), num(e.old_defs)});
      target(1, e.link, row);
      target(0, e.old_link, row);
    }
    if (d.rename_pct >= 0) row.push_back(e.old_test >= 0 ? ro.paths[(size_t)S[0].tests[(size_t)e.old_test].file] : "");
    csv_row(os, row);
  }
}

static std::vector<std::string> link_churn_head(std::vector<std::string> lead, bool renames) {
  lead.insert(lead.end(), {"fileName", "test", "change", "line", "oldLine", "callee", "event", "cause", "calls", "oldCalls", "definitions",
                           "oldDefinitions", "defFile", "defLine", "oldDefFile", "oldDefLine"});
  if (renames) lead.push_back("oldFileName");
  return lead;
}

// The outputs of --clones, --similar-tests and --links: their files with their header rows, and one sink each; `walk` runs the step
// driver once over the first two (nothing when neither is asked for) and once, with the links' selection, for --links.
static void step_outputs(const DiffOptions& o, const std::vector<std::string>& lead_head,
                         const std::function<void(const std::vector<StepSink>&, const Select&, bool)>& walk) {
  std::ofstream clones, similar, links;
  std::vector<StepSink> sinks;
  if (!o.clones.empty()) {
    clones.open(o.clones, std::ios::binary);
    csv_row(clones, clone_churn_head(lead_head));
    sinks.push_back([&](tsm_ctx* ctx, const Revision& ro, const Revision& rn, const StepPairs& sp, const std::vector<std::string>& lead) {
      clone_churn_step(ctx, ro, rn, sp, o, lead, clones);
    });
  }
  if (!o.similar.empty()) {
    similar.open(o.similar, std::ios::binary);
    csv_row(similar, similar_churn_head(lead_head, o.rename_pct >= 0));
    sinks.push_back([&](tsm_ctx* ctx, const Revision& ro, const Revision& rn, const StepPairs& sp, const std::vector<std::string>& lead) {
      similar_churn_step(ctx, ro, rn, sp, o, lead, similar);
    });
  }
  if (!sinks.empty()) walk(sinks, selection(o.all_files), false);
  if (!o.links.empty()) {                                  // (its own walk: the links need the production files)
    links.open(o.links, std::ios::binary);
    csv_row(links, link_churn_head(lead_head, o.rename_pct >= 0));
    walk({[&](tsm_ctx* ctx, const Revision& ro, const Revision& rn, const StepPairs& sp, const std::vector<std::string>& lead) {
      link_churn_step(ctx, ro, rn, sp, o, lead, links);
    }}, link_file, true);
  }
}

static int cmd_diff(const std::string& old_root, const std::string& new_root, const DiffOptions& o) {
  std::vector<FileEntry> a, b;
  walk(old_root, 0, true, a);
  walk(new_root, 0, true, b);
  // pairs by relative path; a file present on one side only is paired with the empty file.  The loader's names: the
  // files of `a`, then those of `b`.
  std::map<std::string, int64_t> in_a, in_b;
  for (size_t i = 0; i < a.size(); ++i) in_a[a[i].rel] = (int64_t)i;
  for (size_t j = 0; j < b.size(); ++j) in_b[b[j].rel] = (int64_t)(a.size() + j);
  std::vector<Change> changes;
  for (const FileEntry& f : a) { auto it = in_b.find(f.rel); changes.push_back({0, f.rel, in_a[f.rel], it == in_b.end() ? -1 : it->second, "", -1}); }
  for (const FileEntry& f : b) if (!in_a.count(f.rel)) changes.push_back({0, f.rel, -1, in_b[f.rel], "", -1});
  auto load = [&](int64_t s) {
    const FileEntry& f = s < (int64_t)a.size() ? a[(size_t)s] : b[(size_t)s - a.size()];
    std::vector<uint8_t> v((size_t)f.size);
    if (!read_file(f.abs, v.data(), f.size)) die("short read: " + f.abs);
    return v;
  };
  const ChangeTotals t = diff_changes(changes, 1, load, o);
  step_outputs(o, {}, [&](const std::vector<StepSink>& sinks, const Select& sel, bool) { diff_steps(old_root, new_root, o, sinks, sel); });
  if (t.binaries) fprintf(stderr, "tosem-scan: %lld binary file(s) skipped\n", (long long)t.binaries);
  if (o.rename_pct >= 0)
    fprintf(stderr, "tosem-scan: %lld rename(s) found (%lld exact, %lld inexact)\n", (long long)t.renames, (long long)t.renames_exact,
            (long long)(t.renames - t.renames_exact));
  printf("cloc,added,removed\r\n%lld,%lld,%lld\r\n", (long long)(t.added[0] + t.removed[0]), (long long)t.added[0], (long long)t.removed[0]);
  return 0;
}

// ---------------------------------------------------------------------------------- S8 on a real repository
// `tosem-scan history <repo>`: the churn of the test files along the first-parent history of a revision, read straight
// from the git object store (host/git_store.hpp: loose objects, packfiles, refs - no `git` process, no checkout).
// Host: commit chain, tree diff by object name (only entries whose blob changed are opened), blob inflation into the
// two pinned arenas.  GPU: diff_changes.  Rows: one per (commit, changed file).

// The changed blobs under two trees, as changes of `step`; their object names are appended to `objs` (the loader's names).
static void tree_diff(gitstore::Store& gs, const gitstore::Oid* a, const gitstore::Oid* b, const std::string& prefix, const Select& sel,
                      size_t step, std::vector<gitstore::Oid>& objs, std::vector<Change>& out) {
  std::vector<gitstore::TreeEntry> ea, eb;
  if (a && !gs.tree(*a, ea)) die("unreadable tree " + a->hex());
  if (b && !gs.tree(*b, eb)) die("unreadable tree " + b->hex());
  std::map<std::string, const gitstore::TreeEntry*> ma, mb;
  for (auto& e : ea) ma[e.name] = &e;
  for (auto& e : eb) mb[e.name] = &e;
  std::vector<std::string> names;
  for (auto& kv : ma) names.push_back(kv.first);
  for (auto& kv : mb) if (!ma.count(kv.first)) names.push_back(kv.first);
  std::sort(names.begin(), names.end());
  for (const std::string& nm : names) {
    const gitstore::TreeEntry* x = ma.count(nm) ? ma[nm] : nullptr;
    const gitstore::TreeEntry* y = mb.count(nm) ? mb[nm] : nullptr;
    if (x && y && x->oid == y->oid && x->is_tree() == y->is_tree()) continue;     // same object: nothing below it changed
    const std::string path = prefix + nm;
    const bool xt = x && x->is_tree(), yt = y && y->is_tree();
    if (xt || yt) tree_diff(gs, xt ? &x->oid : nullptr, yt ? &y->oid : nullptr, path + "/", sel, step, objs, out);
    const bool xb = x && x->is_blob(), yb = y && y->is_blob();                     // (symlinks and submodules are not files of the study)
    if (!xb && !yb) continue;
    if (!sel(path)) continue;
    Change c{step, path, -1, -1, "", -1};
    if (xb) { c.o = (int64_t)objs.size(); objs.push_back(x->oid); }
    if (yb) { c.n = (int64_t)objs.size(); objs.push_back(y->oid); }
    out.push_back(c);
  }
}

// The first-parent chain of `rev` in the repository at `repo` (at most max_commits commits; all when 0), oldest first, and the
// changed selected files of every commit against its parent, as changes of the commit's place in the chain; `load` reads the
// blobs of the changes, which `objs` names.
struct Step { gitstore::Oid id; gitstore::Commit c; };
struct History {
  gitstore::Store gs;
  std::vector<Step> chain;
  std::vector<gitstore::Oid> objs;
  std::vector<Change> changes;
  const Loader load = [this](int64_t s) {
    gitstore::Object x;
    if (!gs.read(objs[(size_t)s], x) || x.type != gitstore::OBJ_BLOB) die("unreadable blob " + objs[(size_t)s].hex());
    return std::move(x.data);
  };
  History(const std::string& repo, const std::string& rev, int64_t max_commits, const Select& sel) {
    std::string err;
    if (!gs.open(repo, err)) die(err);
    gitstore::Oid head;
    if (!gs.resolve(rev, head)) die("cannot resolve revision " + rev);
    for (gitstore::Oid id = head; max_commits <= 0 || (int64_t)chain.size() < max_commits;) {
      Step st{id, {}};
      if (!gs.commit(id, st.c)) die("unreadable commit " + id.hex());
      chain.push_back(st);
      if (st.c.parents.empty()) break;
      id = st.c.parents[0];
    }
    std::reverse(chain.begin(), chain.end());               // oldest first
    for (size_t i = 0; i < chain.size(); ++i) {
      gitstore::Commit parent;
      const bool has_parent = !chain[i].c.parents.empty();
      if (has_parent && !gs.commit(chain[i].c.parents[0], parent)) die("unreadable commit " + chain[i].c.parents[0].hex());
      if (has_parent && parent.tree == chain[i].c.tree) continue;
      tree_diff(gs, has_parent ? &parent.tree : nullptr, &chain[i].c.tree, "", sel, i, objs, changes);
    }
  }
};

// `history --clones` / `--similar-tests` / `--links`: the files `sel` keeps (h's selection) of the current revision kept as live paths, from the boundary commit's
// tree (the parent of the window's first commit; none for a root commit) and each commit's changes after --find-renames.  Blobs
// are read once while they are live (cached by object name), and a revision is packed once: the new side of one step is the old
// side of the next.  Every sink gets each commit that changes a selected file, from one walk.
static void selected_blobs(gitstore::Store& gs, const gitstore::Oid& tree, const std::string& prefix, const Select& sel,
                           std::map<std::string, gitstore::Oid, PathLess>& out) {
  std::vector<gitstore::TreeEntry> es;
  if (!gs.tree(tree, es)) die("unreadable tree " + tree.hex());
  for (const gitstore::TreeEntry& e : es) {
    const std::string rel = prefix + e.name;
    if (e.is_tree()) { selected_blobs(gs, e.oid, rel + "/", sel, out); continue; }
    if (!e.is_blob() || !sel(rel)) continue;
    out[rel] = e.oid;
  }
}

static void history_steps(History& h, const DiffOptions& o, const std::vector<StepSink>& sinks, const Select& sel) {
  std::vector<Change> changes = h.changes;
  const auto ctx = small_context();
  ChangeTotals t(h.chain.size());
  if (o.rename_pct >= 0) pair_renames(ctx.get(), changes, h.load, o.rename_pct, o.batch_bytes, t);
  std::map<std::string, gitstore::Oid, PathLess> live;
  if (!h.chain.empty() && !h.chain[0].c.parents.empty()) {
    gitstore::Commit p0;
    if (!h.gs.commit(h.chain[0].c.parents[0], p0)) die("unreadable commit " + h.chain[0].c.parents[0].hex());
    selected_blobs(h.gs, p0.tree, "", sel, live);
  }
  std::map<gitstore::Oid, Blob> cache;
  auto files_of = [&](const std::map<std::string, gitstore::Oid, PathLess>& paths) {
    std::map<std::string, Blob, PathLess> f;
    for (const auto& kv : paths) {
      Blob& b = cache[kv.second];
      if (!b) {
        gitstore::Object x;
        if (!h.gs.read(kv.second, x) || x.type != gitstore::OBJ_BLOB) die("unreadable blob " + kv.second.hex());
        if (x.data.size() > 0x7fff0000u) die("blob too large: " + kv.first);
        b = std::make_shared<const std::vector<uint8_t>>(std::move(x.data));
      }
      f[kv.first] = b;
    }
    return f;
  };
  std::unique_ptr<Revision> cur;
  for (size_t c0 = 0, c1 = 0; c0 < changes.size(); c0 = c1) {
    for (c1 = c0; c1 < changes.size() && changes[c1].step == changes[c0].step; ++c1) {}
    if (!cur) cur = std::make_unique<Revision>(make_revision(files_of(live)));
    std::map<std::string, gitstore::Oid, PathLess> next = live;
    for (size_t c = c0; c < c1; ++c)
      if (changes[c].o >= 0) next.erase(changes[c].old_path.empty() ? changes[c].path : changes[c].old_path);
    for (size_t c = c0; c < c1; ++c)
      if (changes[c].n >= 0) next[changes[c].path] = h.objs[(size_t)changes[c].n];
    auto rn = std::make_unique<Revision>(make_revision(files_of(next)));
    auto is_binary = [&](const Change& c) { return binary(*cache.at(h.objs[(size_t)c.o])) || binary(*cache.at(h.objs[(size_t)c.n])); };
    const StepPairs sp = step_pairs(*cur, *rn, changes.data() + c0, changes.data() + c1, is_binary);
    const std::vector<std::string> lead = o.lead(changes[c0].step);
    for (const StepSink& sink : sinks) sink(ctx.get(), *cur, *rn, sp, lead);
    cur = std::move(rn);
    live.swap(next);
    std::set<gitstore::Oid> keep;                          // the cache holds the live blobs only
    for (const auto& kv : live) keep.insert(kv.second);
    for (auto it = cache.begin(); it != cache.end();) it = keep.count(it->first) ? std::next(it) : cache.erase(it);
  }
}

// --dry-run: no GPU - the rows carry the object names, sizes and an FNV-1a checksum of both blobs instead of the counts
// (what the CPU tests compare with `git diff-tree` / `git cat-file`).
static int cmd_history(const std::string& repo, const std::string& rev, int64_t max_commits, bool all_files, bool dry_run, DiffOptions o) {
  History h(repo, rev, max_commits, selection(all_files));
  o.lead = [&](size_t step) {
    const Step& st = h.chain[step];
    return std::vector<std::string>{st.id.hex(), st.c.parents.empty() ? "" : st.c.parents[0].hex(), std::to_string(st.c.time)};
  };
  ChangeTotals t(h.chain.size());
  if (dry_run) {
    std::ofstream os;
    if (!o.out.empty()) {
      os.open(o.out, std::ios::binary);
      csv_row(os, {"commit", "parent", "time", "fileName", "old_blob", "new_blob", "old_size", "new_size", "old_fnv", "new_fnv"});
    }
    auto fnv = [](const std::vector<uint8_t>& v) { uint64_t h = 0xcbf29ce484222325ull; for (uint8_t b : v) h = (h ^ b) * 0x100000001b3ull; char buf[24]; snprintf(buf, sizeof buf, "%016llx", (unsigned long long)h); return std::string(buf); };
    for (const Change& c : h.changes) {
      const std::vector<uint8_t> x = c.o >= 0 ? h.load(c.o) : std::vector<uint8_t>(), y = c.n >= 0 ? h.load(c.n) : std::vector<uint8_t>();
      if (os.is_open()) {
        std::vector<std::string> row = o.lead(c.step);
        row.insert(row.end(), {c.path, c.o >= 0 ? h.objs[(size_t)c.o].hex() : "", c.n >= 0 ? h.objs[(size_t)c.n].hex() : "",
                               std::to_string(x.size()), std::to_string(y.size()), fnv(x), fnv(y)});
        csv_row(os, row);
      }
      t.files[c.step]++;
    }
  } else {
    o.zero_rows = true; o.lead_head = {"commit", "parent", "time"}; o.churn_lead = 1;
    step_outputs(o, o.lead_head, [&](const std::vector<StepSink>& sinks, const Select& sel, bool links) {   // (before diff_changes,
      if (!links) { history_steps(h, o, sinks, sel); return; }                                       //  which pairs the renames
      History hl(repo, rev, max_commits, sel);                                                       //  of h.changes in place)
      history_steps(hl, o, sinks, sel);
    });
    t = diff_changes(h.changes, h.chain.size(), h.load, o);
  }
  printf("commit,files,cloc,added,removed\r\n");
  int64_t ta = 0, tr = 0;
  for (size_t i = 0; i < h.chain.size(); ++i) {
    ta += t.added[i]; tr += t.removed[i];
    printf("%s,%lld,%lld,%lld,%lld\r\n", h.chain[i].id.hex().c_str(), (long long)t.files[i], (long long)(t.added[i] + t.removed[i]),
           (long long)t.added[i], (long long)t.removed[i]);
  }
  fprintf(stderr, "tosem-scan: history of %s: %zu commits, %lld changed files diffed on the GPU, %lld binary skipped, cloc %lld (+%lld -%lld)\n",
          rev.c_str(), h.chain.size(), (long long)t.diffed, (long long)t.binaries, (long long)(ta + tr), (long long)ta, (long long)tr);
  if (o.rename_pct >= 0)
    fprintf(stderr, "tosem-scan: %lld rename(s) found at %d%% (%lld exact, %lld inexact)\n", (long long)t.renames, o.rename_pct,
            (long long)t.renames_exact, (long long)(t.renames - t.renames_exact));
  return 0;
}

// ---------------------------------------------------------------------------------- line provenance (docs/SPEC.md section 14)
// `tosem-scan blame <repo>`: the commit, path and line that introduced every line of the selected files at a revision.  The
// walk, the tree diff, the rename pairing and the batch loop are those of `history`; each batch of changes goes through
// tsm_blame_pairs, a pair continuing the chain of the batch's last pair that wrote its old path, or starting from the origins
// the host keeps per live path between batches.  An origin's `change` is an index into `owners`: (commit of the window, or -1
// for the boundary commit P0, and the path in that commit).

static int64_t count_lines(const std::vector<uint8_t>& v) {                 // docs/SPEC.md section 2
  int64_t n = std::count(v.begin(), v.end(), (uint8_t)'\n');
  return n + (!v.empty() && v.back() != '\n');
}

// The origins of one live path: `org`, or (lazy) every line of blob `obj` with the origin (owner, line).
struct PathState { std::vector<tsm_origin> org; int32_t owner = -1; int64_t obj = -1; };

static int cmd_blame(const std::string& repo, const std::string& rev, int64_t max_commits, bool all_files, int rename_pct,
                     int64_t batch_bytes, const std::string& out_path, const std::string& asserts_path) {
  History h(repo, rev, max_commits, selection(all_files));
  const std::vector<Step>& chain = h.chain;
  const bool cut = !chain.empty() && !chain[0].c.parents.empty();          // the window does not reach the root
  Step p0{};
  if (cut) { p0.id = chain[0].c.parents[0]; if (!h.gs.commit(p0.id, p0.c)) die("unreadable commit " + p0.id.hex()); }
  struct Owner { int64_t step; std::string path; };
  std::vector<Owner> owners;
  std::map<std::pair<int64_t, std::string>, int32_t> owner_id;
  auto owner = [&](int64_t step, const std::string& path) {
    auto it = owner_id.find({step, path});
    if (it != owner_id.end()) return it->second;
    owners.push_back({step, path});
    return owner_id[{step, path}] = (int32_t)owners.size() - 1;
  };
  auto lazy = [&](const PathState& st, const std::vector<uint8_t>* bytes) {   // the origins of a lazy state
    std::vector<tsm_origin> v;
    const int64_t n = count_lines(bytes ? *bytes : h.load(st.obj));
    for (int64_t j = 0; j < n; ++j) v.push_back({st.owner, (int32_t)(j + 1)});
    return v;
  };
  std::map<std::string, PathState> live;                   // host state between batches
  ChangeTotals t(chain.size());
  auto ctx = small_context();
  if (rename_pct >= 0) pair_renames(ctx.get(), h.changes, h.load, rename_pct, batch_bytes, t);
  pair_batches(ctx.get(), h.changes, h.load, batch_bytes, false, false, t, [&](const PairBatch& b) {
    // the batch's view of every path it touches: the pair that last wrote it, a lazy state (binary change) or gone
    struct View { int kind; size_t pair; PathState st; };   // kind 0 pair, 1 state, 2 gone
    std::map<std::string, View> view;
    const size_t n = b.idx.size();
    std::vector<int32_t> prev(n, -1), label(n);
    std::vector<int64_t> in_base(n + 1, 0);
    std::vector<tsm_origin> origin_in;
    for (size_t r = b.r0, i = 0; r < b.r1; ++r) {
      const Change& c = h.changes[r];
      const std::string& src = c.old_path.empty() ? c.path : c.old_path;
      if (i < n && b.idx[i] == r) {
        if (c.o >= 0) {
          auto v = view.find(src);
          if (v != view.end() && v->second.kind == 0) prev[i] = (int32_t)v->second.pair;
          else {
            PathState st;
            if (v != view.end() && v->second.kind == 1) st = v->second.st;
            else if (live.count(src)) st = live[src];
            else if (cut) st.owner = owner(-1, src), st.obj = c.o;          // unchanged since P0: a boundary line
            else die("no origins for " + src);
            std::vector<tsm_origin> head = st.org.empty() && st.obj >= 0 ? lazy(st, nullptr) : st.org;
            origin_in.insert(origin_in.end(), head.begin(), head.end());
          }
        }
        in_base[i + 1] = (int64_t)origin_in.size();
        label[i] = owner((int64_t)c.step, c.path);
        if (src != c.path) view[src] = View{2, 0, {}};
        view[c.path] = c.n >= 0 ? View{0, i, {}} : View{2, 0, {}};
        ++i;
      } else {                                              // binary on a side: a text new side takes its lines from this commit
        if (src != c.path) view[src] = View{2, 0, {}};
        PathState st;
        st.owner = owner((int64_t)c.step, c.path); st.obj = c.n;
        view[c.path] = c.n >= 0 && !binary(h.load(c.n)) ? View{1, 0, st} : View{2, 0, {}};
      }
    }
    std::vector<tsm_origin> out;
    std::vector<int64_t> base_new(n + 1, 0);
    if (n) {
      const tsm_corpus ca = b.olds.corpus(1), cn = b.news.corpus(1);
      std::vector<int64_t> added(n), removed(n);
      std::vector<tsm_diff_detail> det(n);
      int64_t cap = 0, got = 0;
      if (origin_in.empty()) origin_in.push_back({0, 0});
      for (;;) {
        out.resize((size_t)std::max<int64_t>(cap, 1));
        const int rc = tsm_blame_pairs(b.ctx, &ca, &cn, added.data(), removed.data(), det.data(), prev.data(), label.data(), origin_in.data(),
                                       in_base.data(), nullptr, base_new.data(), out.data(), cap, &got, nullptr);
        if (rc == TSM_E_CAPACITY && got > cap) { cap = got; continue; }
        ck(rc, "tsm_blame_pairs");
        break;
      }
    }
    for (auto& kv : view) {
      if (kv.second.kind == 2) { live.erase(kv.first); continue; }
      if (kv.second.kind == 1) { live[kv.first] = kv.second.st; continue; }
      const size_t i = kv.second.pair;
      PathState st;
      st.org.assign(out.begin() + base_new[i], out.begin() + base_new[i + 1]);
      live[kv.first] = std::move(st);
    }
  });
  ctx.reset();                                             // the assertion scan below has a context of its own
  // the selected files at R, path order: their origins (a file untouched by the window is all boundary lines)
  std::vector<FileEntry> files;
  if (!chain.empty()) walk_git(h.gs, chain.back().c.tree, "", all_files, files);
  std::vector<std::vector<tsm_origin>> org(files.size());
  for (size_t f = 0; f < files.size(); ++f) {
    if (binary(*files[f].blob)) continue;
    auto it = live.find(files[f].rel);
    if (it != live.end()) org[f] = it->second.org.empty() && it->second.obj >= 0 ? lazy(it->second, files[f].blob.get()) : it->second.org;
    else if (cut) { PathState st; st.owner = owner(-1, files[f].rel); org[f] = lazy(st, files[f].blob.get()); }
    if ((int64_t)org[f].size() != count_lines(*files[f].blob)) die("blame: origins and lines of " + files[f].rel + " differ");
  }
  auto commit_of = [&](int32_t o) -> const Step& { return owners[(size_t)o].step < 0 ? p0 : chain[(size_t)owners[(size_t)o].step]; };
  auto cells = [&](const std::string& path, int64_t line, const tsm_origin& g) {
    const Step& st = commit_of(g.change);
    return std::vector<std::string>{path, std::to_string(line), st.id.hex(), std::to_string(st.c.time), owners[(size_t)g.change].path,
                                    std::to_string(g.line), owners[(size_t)g.change].step < 0 ? "1" : "0"};
  };
  std::ofstream os;
  if (!out_path.empty()) {
    os.open(out_path, std::ios::binary);
    csv_row(os, {"fileName", "line", "commit", "time", "origFileName", "origLine", "boundary"});
    for (size_t f = 0; f < files.size(); ++f)
      for (size_t j = 0; j < org[f].size(); ++j) csv_row(os, cells(files[f].rel, (int64_t)j + 1, org[f][j]));
  }
  // the assertion lines at R (SPEC section 4 Rev A, ext of the path at R): a scan with assertion events, in batches
  std::vector<int64_t> lines_of(owners.size(), 0), asserts_of(owners.size(), 0);
  for (size_t f = 0; f < files.size(); ++f) for (const tsm_origin& g : org[f]) lines_of[(size_t)g.change]++;
  int64_t n_asserts = 0;
  std::ofstream as;
  if (!asserts_path.empty() && !files.empty()) {
    as.open(asserts_path, std::ios::binary);
    csv_row(as, {"fileName", "line", "commit", "time", "origFileName", "origLine", "boundary", "statement", "category"});
  }
  std::vector<Batch> batches = plan_batches(files, all_of(files), batch_bytes, kBatchFiles);
  scan_batches(files, batches, 0, 1, TSM_SCAN_ASSERT_EVENTS, [&](const Batch& B, const Scanned& s) {
    size_t k = 0;
    for (size_t i = 0; i < B.count(); ++i) {
      const size_t f = B.idx[i];
      const uint8_t* base = B.arena.get() + B.off[i];
      LineCounter lc{base};
      for (; k < s.aev.size() && s.aev[k].file == i; ++k) {
        const int64_t line = lc.at(s.aev[k].line_off);
        if (org[f].empty()) continue;                        // (binary)
        const tsm_origin& g = org[f][(size_t)line - 1];
        asserts_of[(size_t)g.change]++; ++n_asserts;
        if (!as.is_open()) continue;
        std::vector<std::string> row = cells(files[f].rel, line, g);
        row.insert(row.end(), {event_statement(base, B.len[i], s.aev[k]), event_category(base, s.aev[k])});
        csv_row(as, row);
      }
    }
  });
  // survival counts per commit that owns a line at R, in window order (the boundary commit first)
  std::vector<int64_t> cl(chain.size() + 1, 0), ca(chain.size() + 1, 0);
  for (size_t o = 0; o < owners.size(); ++o) {
    const size_t s = (size_t)(owners[o].step + 1);
    cl[s] += lines_of[o]; ca[s] += asserts_of[o];
  }
  printf("commit,lines,asserts\r\n");
  int64_t total = 0;
  for (size_t s = 0; s <= chain.size(); ++s) {
    total += cl[s];
    if (cl[s]) printf("%s,%lld,%lld\r\n", (s ? chain[s - 1].id : p0.id).hex().c_str(), (long long)cl[s], (long long)ca[s]);
  }
  fprintf(stderr, "tosem-scan: blame of %s: %zu commits, %lld changed files on the GPU, %lld binary skipped, %zu files, %lld lines, %lld assertion lines\n",
          rev.c_str(), chain.size(), (long long)t.diffed, (long long)t.binaries, files.size(), (long long)total,
          (long long)n_asserts);
  if (cut) fprintf(stderr, "tosem-scan: boundary commit %s\n", p0.id.hex().c_str());
  if (rename_pct >= 0)
    fprintf(stderr, "tosem-scan: %lld rename(s) found at %d%% (%lld exact, %lld inexact)\n", (long long)t.renames, rename_pct,
            (long long)t.renames_exact, (long long)(t.renames - t.renames_exact));
  return 0;
}

// ---------------------------------------------------------------------------------- clones (docs/SPEC.md section 15)
static std::string repo_name(const std::string& path) {
  std::string s = fs::path(path).lexically_normal().generic_string();
  while (s.size() > 1 && s.back() == '/') s.pop_back();
  return base_name(s);
}

// One tsm_clones call over every selected file (classes cross roots and batches), plus one tsm_scan for the per-file line and
// assertion-line totals.  stdout: one row per root and an <all> row; --out: one row per fragment, classes numbered from 1 in
// SPEC order, lines 1-based.  --blind: one tsm_clones_blind call instead (docs/SPEC.md section 21); lines and assertion lines
// count kept lines, and a fragment's first / last line are those of its first and last kept line.
static int cmd_clones(const std::vector<std::string>& roots, const std::string& git_repo, const std::string& rev, int min_lines,
                      bool blind, bool all_files, const std::string& out_path) {
  std::vector<FileEntry> files;
  std::vector<std::string> names;
  if (!git_repo.empty()) {
    gitstore::Store gs;
    std::string err;
    if (!gs.open(git_repo, err)) die(err);
    gitstore::Oid id; gitstore::Commit cm;
    if (!gs.resolve(rev, id) || !gs.commit(id, cm)) die("cannot resolve revision " + rev);
    walk_git(gs, cm.tree, "", all_files, files);
    names.push_back(repo_name(git_repo));
  } else {
    for (size_t g = 0; g < roots.size(); ++g) { walk(roots[g], (int)g, all_files, files); names.push_back(repo_name(roots[g])); }
  }
  fprintf(stderr, "tosem-scan: %zu files selected under %zu root(s)\n", files.size(), names.size());
  std::vector<Batch> batches = plan_batches(files, all_of(files), (1ll << 31) - 4097, INT32_MAX);
  int64_t need = 4096;
  for (const Batch& b : batches) need += b.bytes;
  if (batches.size() > 1 || need >= (1ll << 31))           // (one batch over the limit: a single file that large)
    die("the selected files (" + std::to_string(need) + " bytes of arena) do not fit one int32-indexed arena; clones are found "
        "across all files at once, so select fewer files");
  const size_t ng = names.size();
  std::vector<std::vector<int64_t>> tot(ng + 1, std::vector<int64_t>(6, 0));   // files, lines, dup, asserts, dup asserts, classes
  std::ofstream os;
  if (!out_path.empty()) { os.open(out_path, std::ios::binary); csv_row(os, {"class", "repository", "fileName", "first_line", "last_line"}); }
  scan_batches(files, batches, 0, (int32_t)ng, 0, [&](const Batch& B, const Scanned& s) {
    const int32_t nf = (int32_t)B.count();
    const tsm_corpus c = B.corpus((int32_t)ng);
    std::vector<int64_t> base((size_t)nf + 1), cbase(1), member(1), kbase((size_t)nf + 1), kline(1);
    std::vector<uint32_t> dup((size_t)nf), dupa((size_t)nf), clen(1), kassert((size_t)nf);
    tsm_clone_result r{base.data(), dup.data(), dupa.data(), nullptr, nullptr, 0, 0, nullptr, 0, 0};
    tsm_blind_result kr{kbase.data(), nullptr, nullptr, kassert.data(), 0, 0};
    auto call = [&] {
      if (blind) ck(tsm_clones_blind(s.ctx, &c, min_lines, &kr, &r, nullptr), "tsm_clones_blind");
      else ck(tsm_clones(s.ctx, &c, min_lines, &r, nullptr), "tsm_clones");
    };
    call();                                                // the counts; the second call fills arrays of that size
    cbase.resize((size_t)r.n_classes + 1); clen.resize((size_t)std::max<int64_t>(r.n_classes, 1)); member.resize((size_t)std::max<int64_t>(r.n_members, 1));
    r.class_base = cbase.data(); r.class_len = clen.data(); r.class_cap = r.n_classes; r.member = member.data(); r.member_cap = r.n_members;
    kline.resize((size_t)std::max<int64_t>(kr.n_kept, 1));
    kr.kept_line = kline.data(); kr.kept_cap = kr.n_kept;
    call();
    const std::vector<int64_t>& fbase = blind ? kbase : base;   // the numbering of member
    for (int32_t i = 0; i < nf; ++i) {
      const size_t g = (size_t)files[B.idx[(size_t)i]].grp;
      const int64_t lines = blind ? kbase[(size_t)i + 1] - kbase[(size_t)i] : (int64_t)s.stats[(size_t)i].n_lines;
      const int64_t asserts = blind ? (int64_t)kassert[(size_t)i] : (int64_t)s.stats[(size_t)i].n_assert;
      const int64_t v[5] = {1, lines, dup[(size_t)i], asserts, dupa[(size_t)i]};
      for (int k = 0; k < 5; ++k) { tot[g][(size_t)k] += v[k]; tot[ng][(size_t)k] += v[k]; }
    }
    tot[ng][5] = r.n_classes;
    std::vector<int64_t> seen(ng, -1);                    // the last class counted for each root
    for (int64_t k = 0; k < r.n_classes; ++k)
      for (int64_t j = cbase[(size_t)k]; j < cbase[(size_t)k + 1]; ++j) {
        const int64_t at = member[(size_t)j];
        const size_t f = (size_t)(std::upper_bound(fbase.begin(), fbase.end(), at) - fbase.begin() - 1);
        const FileEntry& fe = files[B.idx[f]];
        if (seen[(size_t)fe.grp] != k) { seen[(size_t)fe.grp] = k; tot[(size_t)fe.grp][5]++; }
        if (os.is_open()) {
          const int64_t last = at + clen[(size_t)k] - 1;
          const int64_t first = (blind ? kline[(size_t)at] : at) - base[f] + 1, end = (blind ? kline[(size_t)last] : last) - base[f] + 1;
          csv_row(os, {std::to_string(k + 1), names[(size_t)fe.grp], fe.rel, std::to_string(first), std::to_string(end)});
        }
      }
  });
  std::ostringstream so;
  csv_row(so, {"repository", "files", "lines", "duplicated_lines", "assertion_lines", "duplicated_assertion_lines", "classes"});
  for (size_t g = 0; g <= ng; ++g) {
    std::vector<std::string> row = {g < ng ? names[g] : "<all>"};
    for (int64_t v : tot[g]) row.push_back(std::to_string(v));
    csv_row(so, row);
  }
  fputs(so.str().c_str(), stdout);
  return 0;
}

// Test smells (docs/SPEC.md section 18): tsm_smells per batch (tests never cross files, so batches are independent).  stdout: per
// root the files and the tests with each smell, and an <all> row; --out: one row per instance line, in file, header line, instance
// line and smell order, lines 1-based; the statement is the stripped instance line (empty for the test-level smells).
// --lexical: one tsm_smells_lexical call per batch instead, which adds the five smells of docs/SPEC.md section 25 after the nine,
// in the stdout columns and the --out rows.
static int cmd_smells(const std::vector<std::string>& roots, const std::string& git_repo, const std::string& rev, bool all_files,
                      const std::string& out_path, int64_t batch_bytes, bool lexical) {
  std::vector<FileEntry> files;
  std::vector<std::string> names;
  if (!git_repo.empty()) {
    gitstore::Store gs;
    std::string err;
    if (!gs.open(git_repo, err)) die(err);
    gitstore::Oid id; gitstore::Commit cm;
    if (!gs.resolve(rev, id) || !gs.commit(id, cm)) die("cannot resolve revision " + rev);
    walk_git(gs, cm.tree, "", all_files, files);
    names.push_back(repo_name(git_repo));
  } else {
    for (size_t g = 0; g < roots.size(); ++g) { walk(roots[g], (int)g, all_files, files); names.push_back(repo_name(roots[g])); }
  }
  fprintf(stderr, "tosem-scan: %zu files selected under %zu root(s)\n", files.size(), names.size());
  const size_t ng = names.size();
  const int nk = TSM_N_SMELLS + (lexical ? TSM_N_LSMELLS : 0);
  std::vector<std::vector<int64_t>> tot(ng + 1, std::vector<int64_t>(2 + (size_t)nk, 0));   // files, tests, tests per smell
  std::ofstream os;
  if (!out_path.empty()) { os.open(out_path, std::ios::binary); csv_row(os, {"repository", "fileName", "test", "line", "smell", "smellLine", "statement"}); }
  std::vector<Batch> batches = plan_batches(files, all_of(files), batch_bytes, kBatchFiles);
  scan_batches(files, batches, 0, (int32_t)ng, TSM_SCAN_HEADER_EVENTS, [&](const Batch& B, const Scanned& s) {
    const int32_t nf = (int32_t)B.count();
    const tsm_corpus c = B.corpus((int32_t)ng);
    std::vector<int64_t> base((size_t)nf + 1);
    int64_t lines = 0, nl = 0, nt = 0;                     // the batch's scan bounds both outputs: its lines, and its header
    for (int32_t i = 0; i < nf; ++i) lines += s.stats[(size_t)i].n_lines;   // lines (each test starts at one), so one call fills them
    std::vector<uint16_t> smell((size_t)std::max<int64_t>(lines, 1));
    std::vector<tsm_smell_test> tests(std::max<size_t>(s.hev.size(), 1));
    std::vector<uint8_t> lsmell(lexical ? smell.size() : 0);
    std::vector<tsm_lex_test> lex(lexical ? tests.size() : 0);
    if (lexical)
      ck(tsm_smells_lexical(s.ctx, &c, base.data(), smell.data(), lsmell.data(), lines, &nl, tests.data(), lex.data(),
                            (int64_t)s.hev.size(), &nt, nullptr), "tsm_smells_lexical");
    else
      ck(tsm_smells(s.ctx, &c, base.data(), smell.data(), lines, &nl, tests.data(), (int64_t)s.hev.size(), &nt, nullptr), "tsm_smells");
    for (int32_t i = 0; i < nf; ++i) { tot[(size_t)files[B.idx[(size_t)i]].grp][0]++; tot[ng][0]++; }
    int32_t at_file = -1;
    std::vector<uint32_t> start;                           // byte offset of every line of file at_file
    for (int64_t t = 0; t < nt; ++t) {
      const tsm_smell_test& r = tests[(size_t)t];
      const uint32_t lsm = lexical ? lex[(size_t)t].smells : 0u;
      const FileEntry& fe = files[B.idx[(size_t)r.file]];
      for (size_t g : {(size_t)fe.grp, ng}) {
        tot[g][1]++;
        for (int k = 0; k < TSM_N_SMELLS; ++k) tot[g][2 + (size_t)k] += (r.smells >> k) & 1;
        for (int k = 0; k < nk - TSM_N_SMELLS; ++k) tot[g][2 + TSM_N_SMELLS + (size_t)k] += (lsm >> k) & 1;
      }
      if (!os.is_open() || !(r.smells || lsm)) continue;
      const uint8_t* p = B.arena.get() + B.off[(size_t)r.file];
      const uint32_t len = (uint32_t)B.len[(size_t)r.file];
      if (at_file != r.file) {
        at_file = r.file; start.assign(1, 0);
        for (uint32_t q = 0; q < len; ++q) if (p[q] == '\n') start.push_back(q + 1);
      }
      auto line_end = [&](int64_t l) { return (size_t)l + 1 < start.size() ? start[(size_t)l + 1] - 1 : len; };
      auto stripped = [&](int64_t l) {
        uint32_t b = start[(size_t)l], z = line_end(l);
        while (b < z && is_w(p[b])) ++b;
        while (z > b && is_w(p[z - 1])) --z;
        return std::string((const char*)p + b, z - b);
      };
      const std::string name = case_name(fe.ext, p + start[(size_t)r.line], line_end(r.line) - start[(size_t)r.line]);
      const int64_t g0 = base[(size_t)r.file] + r.line;
      for (int64_t l = r.line; l < (int64_t)r.line + r.body_lines; ++l) {
        const uint16_t bits = smell[(size_t)(g0 + l - r.line)];
        for (int k = 0; k < TSM_N_SMELLS; ++k)
          if ((bits >> k) & 1) {
            const bool test_level = k == TSM_SMELL_EMPTY || k == TSM_SMELL_ASSERTION_FREE;
            csv_row(os, {names[(size_t)fe.grp], fe.rel, name, std::to_string(r.line + 1), kSmellNames[k], std::to_string(l + 1),
                         test_level ? std::string() : stripped(l)});
          }
        const uint8_t lbits = lexical ? lsmell[(size_t)(g0 + l - r.line)] : 0;
        for (int k = 0; k < TSM_N_LSMELLS; ++k)
          if ((lbits >> k) & 1)
            csv_row(os, {names[(size_t)fe.grp], fe.rel, name, std::to_string(r.line + 1), kLexSmellNames[k], std::to_string(l + 1),
                         k == TSM_LSMELL_OBSCURE_SETUP ? std::string() : stripped(l)});
      }
    }
  });
  std::ostringstream so;
  std::vector<std::string> head = {"repository", "files", "tests"};
  for (const char* n : kSmellNames) head.push_back(n);
  if (lexical)
    for (const char* n : kLexSmellNames) head.push_back(n);
  csv_row(so, head);
  for (size_t g = 0; g <= ng; ++g) {
    std::vector<std::string> row = {g < ng ? names[g] : "<all>"};
    for (int64_t v : tot[g]) row.push_back(std::to_string(v));
    csv_row(so, row);
  }
  fputs(so.str().c_str(), stdout);
  return 0;
}

// Similar tests (docs/SPEC.md section 23): ONE tsm_similar_tests call over every selected file (pairs cross roots).  stdout: per
// root its files, tests, compared tests, tests in a pair, and the pairs and classes with a member in it, and an <all> row;
// --out: one row per pair in (a, b) order; --classes: one row per class member.  Lines are 1-based header lines; a test is named
// by its section-10 case name.
static int cmd_similar_tests(const std::vector<std::string>& roots, const std::string& git_repo, const std::string& rev, int min_lines,
                             int similarity, bool all_files, const std::string& out_path, const std::string& classes_path) {
  std::vector<FileEntry> files;
  std::vector<std::string> names;
  if (!git_repo.empty()) {
    gitstore::Store gs;
    std::string err;
    if (!gs.open(git_repo, err)) die(err);
    gitstore::Oid id; gitstore::Commit cm;
    if (!gs.resolve(rev, id) || !gs.commit(id, cm)) die("cannot resolve revision " + rev);
    walk_git(gs, cm.tree, "", all_files, files);
    names.push_back(repo_name(git_repo));
  } else {
    for (size_t g = 0; g < roots.size(); ++g) { walk(roots[g], (int)g, all_files, files); names.push_back(repo_name(roots[g])); }
  }
  fprintf(stderr, "tosem-scan: %zu files selected under %zu root(s)\n", files.size(), names.size());
  std::vector<Batch> batches = plan_batches(files, all_of(files), (1ll << 31) - 4097, INT32_MAX);
  int64_t need = 4096;
  for (const Batch& b : batches) need += b.bytes;
  if (batches.size() > 1 || need >= (1ll << 31))
    die("the selected files (" + std::to_string(need) + " bytes of arena) do not fit one int32-indexed arena; similar tests are "
        "found across all files at once, so select fewer files");
  const size_t ng = names.size();
  std::vector<std::vector<int64_t>> tot(ng + 1, std::vector<int64_t>(6, 0));   // files, tests, compared, similar, pairs, classes
  std::ofstream os, oc;
  if (!out_path.empty()) {
    os.open(out_path, std::ios::binary);
    csv_row(os, {"repository", "fileName", "test", "line", "otherRepository", "otherFileName", "otherTest", "otherLine", "keptLines",
                 "otherKeptLines", "lcs", "similarity"});
  }
  if (!classes_path.empty()) {
    oc.open(classes_path, std::ios::binary);
    csv_row(oc, {"class", "repository", "fileName", "test", "line", "last_line", "keptLines"});
  }
  scan_batches(files, batches, 0, (int32_t)ng, TSM_SCAN_HEADER_EVENTS, [&](const Batch& B, const Scanned& s) {
    const int32_t nf = (int32_t)B.count();
    const tsm_corpus c = B.corpus((int32_t)ng);
    // A test starts at a header event, so the tests, the members (<= tests) and the classes (<= tests / 2) fit these arrays; the
    // pairs are a guess, and a second call (which redoes all the work) sizes them only when it is short.
    const int64_t cap_t = (int64_t)s.hev.size();
    std::vector<tsm_smell_test> tests((size_t)std::max<int64_t>(cap_t, 1));
    std::vector<uint32_t> kept(tests.size());
    std::vector<int64_t> cbase((size_t)cap_t + 1);
    std::vector<int32_t> member(tests.size());
    std::vector<tsm_similar_pair> pairs((size_t)std::max<int64_t>(4 * cap_t, 1 << 16));
    tsm_similar_result r{tests.data(), kept.data(), cap_t, 0, pairs.data(), (int64_t)pairs.size(), 0, cbase.data(), cap_t, 0,
                         member.data(), cap_t, 0, 0};
    int rc = tsm_similar_tests(s.ctx, &c, min_lines, similarity, &r, nullptr);
    if (rc == TSM_E_CAPACITY && r.n_pairs > r.pair_cap) {
      pairs.resize((size_t)r.n_pairs);
      r.pairs = pairs.data(); r.pair_cap = r.n_pairs;
      rc = tsm_similar_tests(s.ctx, &c, min_lines, similarity, &r, nullptr);
    }
    ck(rc, "tsm_similar_tests");
    const int64_t nt = r.n_tests;
    std::vector<std::string> tname((size_t)nt);             // the case name of every test
    int32_t at_file = -1;
    std::vector<uint32_t> start;
    for (int64_t t = 0; t < nt; ++t) {
      const tsm_smell_test& x = tests[(size_t)t];
      const uint8_t* p = B.arena.get() + B.off[(size_t)x.file];
      const uint32_t len = (uint32_t)B.len[(size_t)x.file];
      if (at_file != x.file) {
        at_file = x.file; start.assign(1, 0);
        for (uint32_t q = 0; q < len; ++q) if (p[q] == '\n') start.push_back(q + 1);
      }
      const uint32_t e = (size_t)x.line + 1 < start.size() ? start[(size_t)x.line + 1] - 1 : len;
      tname[(size_t)t] = case_name(files[B.idx[(size_t)x.file]].ext, p + start[(size_t)x.line], e - start[(size_t)x.line]);
    }
    auto grp = [&](int64_t t) { return (size_t)files[B.idx[(size_t)tests[(size_t)t].file]].grp; };
    for (int32_t i = 0; i < nf; ++i) { tot[(size_t)files[B.idx[(size_t)i]].grp][0]++; tot[ng][0]++; }
    std::vector<uint8_t> linked((size_t)nt, 0);
    for (int64_t j = 0; j < r.n_members; ++j) linked[(size_t)member[(size_t)j]] = 1;
    for (int64_t t = 0; t < nt; ++t)
      for (size_t g : {grp(t), ng}) {
        tot[g][1]++;
        tot[g][2] += kept[(size_t)t] >= (uint32_t)min_lines;
        tot[g][3] += linked[(size_t)t];
      }
    for (int64_t k = 0; k < r.n_pairs; ++k) {
      const tsm_similar_pair& q = pairs[(size_t)k];
      const size_t ga = grp(q.a), gb = grp(q.b);
      tot[ga][4]++;
      if (gb != ga) tot[gb][4]++;
      tot[ng][4]++;
      if (!os.is_open()) continue;
      const tsm_smell_test &ta = tests[(size_t)q.a], &tb = tests[(size_t)q.b];
      csv_row(os, {names[ga], files[B.idx[(size_t)ta.file]].rel, tname[(size_t)q.a], std::to_string(ta.line + 1), names[gb],
                   files[B.idx[(size_t)tb.file]].rel, tname[(size_t)q.b], std::to_string(tb.line + 1), std::to_string(kept[(size_t)q.a]),
                   std::to_string(kept[(size_t)q.b]), std::to_string(q.lcs), std::to_string(q.score / 600)});
    }
    tot[ng][5] = r.n_classes;
    for (int64_t k = 0; k < r.n_classes; ++k) {
      std::vector<uint8_t> seen(ng, 0);
      for (int64_t j = cbase[(size_t)k]; j < cbase[(size_t)k + 1]; ++j) {
        const int32_t t = member[(size_t)j];
        const size_t g = grp(t);
        if (!seen[g]) { seen[g] = 1; tot[g][5]++; }
        if (!oc.is_open()) continue;
        const tsm_smell_test& x = tests[(size_t)t];
        csv_row(oc, {std::to_string(k + 1), names[g], files[B.idx[(size_t)x.file]].rel, tname[(size_t)t], std::to_string(x.line + 1),
                     std::to_string(x.line + x.body_lines), std::to_string(kept[(size_t)t])});
      }
    }
  });
  std::ostringstream so;
  csv_row(so, {"repository", "files", "tests", "compared_tests", "similar_tests", "pairs", "classes"});
  for (size_t g = 0; g <= ng; ++g) {
    std::vector<std::string> row = {g < ng ? names[g] : "<all>"};
    for (int64_t v : tot[g]) row.push_back(std::to_string(v));
    csv_row(so, row);
  }
  fputs(so.str().c_str(), stdout);
  return 0;
}

// Test-to-code links (docs/SPEC.md section 27): ONE tsm_test_links call over every file with a lexer family under the roots (names
// resolve across files).  A file is a test file when its path contains `test` (S0); the stems of the naming convention come from
// tsm_focal_stems.  stdout: per root its test and production files, tests, tests with a link, definitions, definitions whose name
// some test links, links, ambiguous links, Eager and Lazy tests, and an <all> row; --out: one row per link in (test, first call)
// order; --defs: one row per definition in line order.  Lines are 1-based; a test is named by its section-10 case name.
static int cmd_links(const std::vector<std::string>& roots, const std::string& git_repo, const std::string& rev,
                     const std::string& out_path, const std::string& defs_path) {
  std::vector<FileEntry> all, files;
  std::vector<std::string> names;
  if (!git_repo.empty()) {
    gitstore::Store gs;
    std::string err;
    if (!gs.open(git_repo, err)) die(err);
    gitstore::Oid id; gitstore::Commit cm;
    if (!gs.resolve(rev, id) || !gs.commit(id, cm)) die("cannot resolve revision " + rev);
    walk_git(gs, cm.tree, "", true, all);
    names.push_back(repo_name(git_repo));
  } else {
    for (size_t g = 0; g < roots.size(); ++g) { walk(roots[g], (int)g, true, all); names.push_back(repo_name(roots[g])); }
  }
  for (FileEntry& f : all)
    if (f.ext != TSM_EXT_OTHER) files.push_back(std::move(f));
  fprintf(stderr, "tosem-scan: %zu files selected under %zu root(s)\n", files.size(), names.size());
  std::vector<Batch> batches = plan_batches(files, all_of(files), (1ll << 31) - 4097, INT32_MAX);
  int64_t need = 4096;
  for (const Batch& b : batches) need += b.bytes;
  if (batches.size() > 1 || need >= (1ll << 31))
    die("the selected files (" + std::to_string(need) + " bytes of arena) do not fit one int32-indexed arena; links are resolved "
        "across all files at once, so select fewer files");
  const size_t ng = names.size();
  std::vector<std::vector<int64_t>> tot(ng + 1, std::vector<int64_t>(10, 0));
  std::ofstream os, ds;
  if (!out_path.empty()) {
    os.open(out_path, std::ios::binary);
    csv_row(os, {"repository", "fileName", "test", "line", "callee", "kind", "calls", "definitions", "defFile", "defLine", "focal"});
  }
  if (!defs_path.empty()) {
    ds.open(defs_path, std::ios::binary);
    csv_row(ds, {"repository", "fileName", "line", "name", "kind", "tests", "tests_by_name", "calls"});
  }
  static const char* const kinds[] = {"", "function", "class"};
  scan_batches(files, batches, 0, (int32_t)ng, 0, [&](const Batch& B, const Scanned& s) {
    const int32_t nf = (int32_t)B.count();
    const tsm_corpus c = B.corpus((int32_t)ng);
    std::vector<const char*> paths((size_t)nf);
    std::vector<uint8_t> role((size_t)nf);
    std::vector<int32_t> stem((size_t)std::max(nf, 1));
    for (int32_t i = 0; i < nf; ++i) {
      const FileEntry& fe = files[B.idx[(size_t)i]];
      paths[(size_t)i] = fe.rel.c_str();
      role[(size_t)i] = lower(fe.rel).find("test") != std::string::npos;   // S0
    }
    ck(tsm_focal_stems(paths.data(), role.data(), nf, stem.data()), "tsm_focal_stems");
    tsm_links_result r{};
    ck(tsm_test_links(s.ctx, &c, role.data(), stem.data(), &r, nullptr), "tsm_test_links");   // the counts
    std::vector<tsm_link_test> tests((size_t)std::max<int64_t>(r.n_tests, 1));
    std::vector<tsm_link> links((size_t)std::max<int64_t>(r.n_links, 1));
    std::vector<tsm_link_def> defs((size_t)std::max<int64_t>(r.n_defs, 1));
    r.tests = tests.data(); r.test_cap = r.n_tests; r.links = links.data(); r.link_cap = r.n_links; r.defs = defs.data(); r.def_cap = r.n_defs;
    ck(tsm_test_links(s.ctx, &c, role.data(), stem.data(), &r, nullptr), "tsm_test_links");
    auto grp_of = [&](int32_t f) { return (size_t)files[B.idx[(size_t)f]].grp; };
    auto add = [&](size_t g, int k, int64_t v) { tot[g][(size_t)k] += v; tot[ng][(size_t)k] += v; };
    for (int32_t i = 0; i < nf; ++i) add(grp_of(i), role[(size_t)i] ? 0 : 1, 1);
    for (int64_t t = 0; t < r.n_tests; ++t) {
      const tsm_link_test& x = tests[(size_t)t];
      const size_t g = grp_of(x.file);
      add(g, 2, 1); add(g, 3, x.links > 0); add(g, 8, (x.flags & TSM_LINK_EAGER) != 0); add(g, 9, (x.flags & TSM_LINK_LAZY) != 0);
    }
    for (int64_t d = 0; d < r.n_defs; ++d) { add(grp_of(defs[(size_t)d].file), 4, 1); add(grp_of(defs[(size_t)d].file), 5, defs[(size_t)d].tests_by_name > 0); }
    for (int64_t k = 0; k < r.n_links; ++k) {
      const size_t g = grp_of(tests[(size_t)links[(size_t)k].test].file);
      add(g, 6, 1); add(g, 7, links[(size_t)k].target < 0);
    }
    auto name_of = [&](const tsm_link_def& d) { return std::string((const char*)B.arena.get() + B.off[(size_t)d.file] + d.name_off, (size_t)d.name_len); };
    if (os.is_open()) {
      int32_t at_test = -1;
      std::string tname;
      for (int64_t k = 0; k < r.n_links; ++k) {
        const tsm_link& l = links[(size_t)k];
        const tsm_link_test& x = tests[(size_t)l.test];
        const FileEntry& fe = files[B.idx[(size_t)x.file]];
        if (at_test != l.test) {                           // the test's case name, from its header line
          at_test = l.test;
          const uint8_t* p = B.arena.get() + B.off[(size_t)x.file];
          const uint32_t len = (uint32_t)B.len[(size_t)x.file];
          uint32_t b = 0;
          for (int32_t n = 0; n < x.line; ++b) if (p[b] == '\n') ++n;
          uint32_t e = b;
          while (e < len && p[e] != '\n') ++e;
          tname = case_name(fe.ext, p + b, e - b);
        }
        const tsm_link_def& nd = defs[(size_t)l.name_def];
        const tsm_link_def* td = l.target >= 0 ? &defs[(size_t)l.target] : nullptr;
        const bool focal = td && stem[(size_t)x.file] >= 0 && stem[(size_t)td->file] == stem[(size_t)x.file];
        csv_row(os, {names[(size_t)fe.grp], fe.rel, tname, std::to_string(l.line + 1), name_of(nd), kinds[(td ? td : &nd)->kind],
                     std::to_string(l.calls), std::to_string(l.n_defs), td ? files[B.idx[(size_t)td->file]].rel : std::string(),
                     td ? std::to_string(td->line + 1) : std::string(), focal ? "1" : "0"});
      }
    }
    if (ds.is_open())
      for (int64_t k = 0; k < r.n_defs; ++k) {
        const tsm_link_def& d = defs[(size_t)k];
        const FileEntry& fe = files[B.idx[(size_t)d.file]];
        csv_row(ds, {names[(size_t)fe.grp], fe.rel, std::to_string(d.line + 1), name_of(d), kinds[d.kind], std::to_string(d.tests),
                     std::to_string(d.tests_by_name), std::to_string(d.calls)});
      }
  });
  std::ostringstream so;
  csv_row(so, {"repository", "test_files", "production_files", "tests", "linked_tests", "definitions", "linked_definitions", "links",
               "ambiguous_links", "eager", "lazy"});
  for (size_t g = 0; g <= ng; ++g) {
    std::vector<std::string> row = {g < ng ? names[g] : "<all>"};
    for (int64_t v : tot[g]) row.push_back(std::to_string(v));
    csv_row(so, row);
  }
  fputs(so.str().c_str(), stdout);
  return 0;
}

static void usage() {
  fprintf(stderr,
          "usage: tosem-scan scan   <project-root>... [--rows F] [--summary F] [--gpus N] [--all-files] [--batch-bytes N] [--rev-b]\n"
          "       tosem-scan reduce <taxonomy.csv> [--strategy F] [--methods F] [--properties F] [--correlate F] [--correlate-tex F] [--correlate-counts F] [--correlate-merged F]\n"
          "       tosem-scan diff   <old-root> <new-root> [--out F] [--asserts F] [--assert-churn F] [--cases F] [--assert-edits F] [--smells F [--lexical]]\n"
          "                         [--moves F] [--clones F [--min-lines N] [--blind] [--all-files]] [--similar-tests F [--min-lines N] [--similarity P]] [--links F] [--find-renames N] [--batch-bytes N]\n"
          "       tosem-scan body   <project-root>... [--batch-bytes N] [--out F]\n"
          "       tosem-scan releases <snapshot-root>=<tag>... [--batch-bytes N] [--out F]\n"
          "       tosem-scan releases --git <repository> [<revision>...] [--batch-bytes N] [--out F]\n"
          "       tosem-scan history <git-repository> [--rev R] [--max-commits N] [--all-files] [--dry-run] [--out F] [--asserts F] [--assert-churn F]\n"
          "                          [--cases F] [--assert-edits F] [--smells F [--lexical]] [--moves F] [--clones F [--min-lines N] [--blind]] [--similar-tests F [--similarity P]] [--links F]\n"
          "                          [--find-renames N] [--batch-bytes N]\n"
          "       tosem-scan blame <git-repository> [--rev R] [--max-commits N] [--all-files] [--find-renames N] [--batch-bytes N] [--out F] [--asserts F]\n"
          "       tosem-scan clones <project-root>... [--min-lines N] [--blind] [--all-files] [--out F]\n"
          "       tosem-scan clones --git <repository> [--rev R] [--min-lines N] [--blind] [--all-files] [--out F]\n"
          "       tosem-scan smells <project-root>... [--lexical] [--all-files] [--batch-bytes N] [--out F]\n"
          "       tosem-scan smells --git <repository> [--rev R] [--lexical] [--all-files] [--batch-bytes N] [--out F]\n"
          "       tosem-scan similar-tests <project-root>... | --git <repository> [--rev R] [--min-lines N] [--similarity P] [--all-files]\n"
          "                                [--out F] [--classes F]\n"
          "       tosem-scan links <project-root>... | --git <repository> [--rev R] [--out F] [--defs F]\n"
          "smells: per root the tests with each of nine test smells; --out F: one row per instance line (docs/SPEC.md section 18).\n"
          "--lexical (smells): five more smells from the assertion calls' arguments, lexed with string awareness: assertion_roulette,\n"
          "  magic_number, suboptimal_assert, mystery_guest, obscure_setup (docs/SPEC.md section 25).\n"
          "similar-tests: pairs of tests whose kept blind lines are at least P %% alike (LCS, default 70) and their classes, over\n"
          "               tests of at least N kept lines (default 5); --out F: one row per pair; --classes F: one row per class member\n"
          "               (docs/SPEC.md section 23).\n"
          "links: per root the tests, the production definitions and the links between them, by called name and the naming\n"
          "       convention's focal files, with Eager and Lazy tests; --out F: one row per link; --defs F: one row per definition\n"
          "       (docs/SPEC.md section 27).\n"
          "--blind (clones): near-miss copies - lines compared with identifiers, literals, whitespace and comments blinded, over the\n"
          "                  lines that keep a token (docs/SPEC.md section 21).\n"
          "--find-renames N (0..100): pair deleted and added files at least N %% similar, as git -M<N>%% does (docs/SPEC.md section 13).\n"
          "--cases F: one row per test case that a revision adds (A), deletes (D) or modifies (M) (docs/SPEC.md section 16).\n"
          "--assert-edits F: one row per deleted assertion line that an inserted one of the same hunk replaces, with their similarity\n"
          "                  (docs/SPEC.md section 17).\n"
          "--smells F: one row per (test, smell) that a revision introduces, removes or changes, with the smell's instances and the\n"
          "            instance lines it adds and removes (docs/SPEC.md section 19); with --lexical also the five lexical smells\n"
          "            (docs/SPEC.md section 26).\n"
          "--moves F: one row per block of changed lines that a commit moves, within or across its files, as git diff\n"
          "           --color-moved=blocks finds them (docs/SPEC.md section 20); a commit is never split across batches, and one\n"
          "           larger than --batch-bytes is a batch of its own.\n"
          "--clones F: per commit, one row per fragment of every clone class of the parent (-) or the commit (+) that the commit\n"
          "            edits, with the class's status (copied, diverged, ...) and the fragment's changed lines (docs/SPEC.md section 22).\n"
          "--similar-tests F: per commit, one row per pair of similar tests (docs/SPEC.md section 23) that the commit creates, changes or\n"
          "            breaks up (copied, changed, diverged, ...), with both tests on both sides and their similarity before and after\n"
          "            (docs/SPEC.md section 24); --min-lines N (shared with --clones) and --similarity P as for similar-tests.\n"
          "--links F: per commit that changes a file with a lexer family (any path: production files too), one row per test-to-code\n"
          "            link that the commit adds, removes, retargets or redefines, and per Eager / Lazy Test flag it introduces or\n"
          "            removes, test by test (docs/SPEC.md section 28); not with --dry-run.\n"
          "--batch-bytes N: files go to the GPU in batches of at most N bytes (per side of a diff; a larger file alone); scan: 1 GiB, else 512 MiB.\n"
          "Scans run on the GPU through libtosemscan.so (sm_90a); there is no CPU fallback.\n");
}

int main(int argc, char** argv) {
  if (argc < 2 || !strcmp(argv[1], "-h") || !strcmp(argv[1], "--help")) { usage(); return argc < 2 ? 2 : 0; }
  const std::string cmd = argv[1];
  std::vector<std::string> pos;
  std::map<std::string, std::string> opt;
  bool all_files = false, rev_b = false, dry_run = false, blind = false, lexical = false;
  for (int i = 2; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--all-files") all_files = true;
    else if (a == "--rev-b") rev_b = true;
    else if (a == "--dry-run") dry_run = true;
    else if (a == "--blind") blind = true;
    else if (a == "--lexical") lexical = true;
    else if (a.rfind("--", 0) == 0) { if (i + 1 >= argc) die("missing value for " + a); opt[a] = argv[++i]; }
    else pos.push_back(a);
  }
  auto batch_bytes = [&](int64_t dflt, int64_t least) {
    return opt.count("--batch-bytes") ? std::max<int64_t>(least, atoll(opt["--batch-bytes"].c_str())) : dflt;
  };
  if (cmd == "scan") { if (pos.empty()) die("scan needs at least one project root"); return cmd_scan(pos, opt["--rows"], opt["--summary"], opt.count("--gpus") ? atoi(opt["--gpus"].c_str()) : 1, all_files,
                                        batch_bytes(1ll << 30, 4096), rev_b); }
  if (cmd == "reduce") { if (pos.size() != 1) die("reduce needs the taxonomy csv"); return cmd_reduce(pos[0], opt["--strategy"], opt["--methods"], opt["--properties"], opt["--correlate"], opt["--correlate-tex"], opt["--correlate-counts"], opt["--correlate-merged"]); }
  if (cmd == "releases") { if (pos.empty() && !opt.count("--git")) die("releases needs <root>=<tag>... or --git <repository>"); return cmd_releases(pos, opt["--out"], opt["--git"], batch_bytes(kBatch, 1)); }
  if (cmd == "clones") {
    if (pos.empty() == !opt.count("--git")) die("clones needs project roots or --git <repository>, not both");
    const long n = opt.count("--min-lines") ? strtol(opt["--min-lines"].c_str(), nullptr, 10) : 5;
    if (n < 1 || n > 1024) die("--min-lines needs a number of lines from 1 to 1024");
    return cmd_clones(pos, opt["--git"], opt.count("--rev") ? opt["--rev"] : "HEAD", (int)n, blind, all_files, opt["--out"]);
  }
  if (cmd == "smells") {
    if (pos.empty() == !opt.count("--git")) die("smells needs project roots or --git <repository>, not both");
    return cmd_smells(pos, opt["--git"], opt.count("--rev") ? opt["--rev"] : "HEAD", all_files, opt["--out"], batch_bytes(kBatch, 1), lexical);
  }
  if (cmd == "similar-tests") {
    if (pos.empty() == !opt.count("--git")) die("similar-tests needs project roots or --git <repository>, not both");
    const long n = opt.count("--min-lines") ? strtol(opt["--min-lines"].c_str(), nullptr, 10) : 5;
    if (n < 1 || n > INT32_MAX) die("--min-lines needs a number of lines of at least 1");
    const long p = opt.count("--similarity") ? strtol(opt["--similarity"].c_str(), nullptr, 10) : 70;
    if (p < 1 || p > 100) die("--similarity needs a percentage from 1 to 100");
    return cmd_similar_tests(pos, opt["--git"], opt.count("--rev") ? opt["--rev"] : "HEAD", (int)n, (int)p, all_files, opt["--out"],
                             opt["--classes"]);
  }
  if (cmd == "links") {
    if (pos.empty() == !opt.count("--git")) die("links needs project roots or --git <repository>, not both");
    return cmd_links(pos, opt["--git"], opt.count("--rev") ? opt["--rev"] : "HEAD", opt["--out"], opt["--defs"]);
  }
  if (cmd == "body") { if (pos.empty()) die("body needs at least one project root"); return cmd_body(pos, opt["--out"], batch_bytes(kBatch, 1)); }
  int rename_pct = -1;                                     // --find-renames N (docs/SPEC.md section 13); -1 = off
  if (opt.count("--find-renames")) {
    std::string v = opt["--find-renames"];
    if (!v.empty() && v.back() == '%') v.pop_back();
    char* end = nullptr;
    const long pct = v.empty() ? -1 : strtol(v.c_str(), &end, 10);
    if (pct < 0 || pct > 100 || *end) die("--find-renames needs a similarity from 0 to 100");
    rename_pct = (int)pct;
  }
  DiffOptions d;                                           // diff and history
  d.rename_pct = rename_pct; d.batch_bytes = batch_bytes(kBatch, 1);
  d.out = opt["--out"]; d.asserts = opt["--asserts"]; d.churn = opt["--assert-churn"]; d.cases = opt["--cases"];
  d.edits = opt["--assert-edits"]; d.smells = opt["--smells"]; d.moves = opt["--moves"];
  d.smell_lexical = lexical && opt.count("--smells");      // (--lexical is read only with --smells)
  if (opt.count("--clones")) {                             // (--min-lines and --blind are read only with --clones)
    d.clones = opt["--clones"]; d.clone_blind = blind; d.all_files = all_files;
    const long n = opt.count("--min-lines") ? strtol(opt["--min-lines"].c_str(), nullptr, 10) : 5;
    if (n < 1 || n > 1024) die("--min-lines needs a number of lines from 1 to 1024");
    d.clone_min_lines = (int)n;
    if (dry_run) die("--dry-run and --clones cannot be combined (clone churn needs the GPU)");
  }
  if (opt.count("--similar-tests")) {                      // (--similarity is read only with --similar-tests)
    d.similar = opt["--similar-tests"]; d.all_files = all_files;
    const long n = opt.count("--min-lines") ? strtol(opt["--min-lines"].c_str(), nullptr, 10) : 5;
    if (n < 1 || n > INT32_MAX) die("--min-lines needs a number of lines of at least 1");
    const long p = opt.count("--similarity") ? strtol(opt["--similarity"].c_str(), nullptr, 10) : 70;
    if (p < 1 || p > 100) die("--similarity needs a percentage from 1 to 100");
    d.similar_min_lines = (int)n; d.similar_pct = (int)p;
    if (dry_run) die("--dry-run and --similar-tests cannot be combined (similar-test churn needs the GPU)");
  }
  if (opt.count("--links")) {
    d.links = opt["--links"];
    if (dry_run) die("--dry-run and --links cannot be combined (link churn needs the GPU)");
  }
  const std::string rev = opt.count("--rev") ? opt["--rev"] : "HEAD";
  const int64_t max_commits = opt.count("--max-commits") ? atoll(opt["--max-commits"].c_str()) : 0;
  if (cmd == "history") { if (pos.size() != 1) die("history needs the repository");
                          if (dry_run && rename_pct >= 0) die("--dry-run and --find-renames cannot be combined (renames need the GPU)");
                          return cmd_history(pos[0], rev, max_commits, all_files, dry_run, d); }
  if (cmd == "blame") { if (pos.size() != 1) die("blame needs the repository");
                        return cmd_blame(pos[0], rev, max_commits, all_files, rename_pct, d.batch_bytes, d.out, d.asserts); }
  if (cmd == "diff") { if (pos.size() != 2) die("diff needs <old-root> <new-root>"); return cmd_diff(pos[0], pos[1], d); }
  usage();
  return 2;
}
