#!/usr/bin/env python3
"""Cost of the clone churn (docs/SPEC.md section 22) against the composition it replaces, one GPU:

    python tools/bench_clone_churn.py [--min-lines 5] [--steps 10] [--warmup 3] [--c4-files 100000]

Two synthetic steps.  C5: 4 000 files of BASELINE config C5's old-side law plus 20 planted copies (30 lines of a file pasted into a
file of their own) as R_old; R_new = R_old with tsm_gen_edit (lambda = 6) of 40 files, a one-line fix in the middle of each planted
copy (an edit to one copy of a clone class) and 20 new pasted tests.  C4: --c4-files files of config C4's size law with the same
kind of step.  Per step, tsm_clone_churn (exact) alternates
with the composition it replaces on the same inputs: tsm_clones of each revision plus tsm_diff_pairs_marks over the pairs (the pair
sides packed as corpora of their own).  Reported per workload: the median whole-call time on the host clock (every call
synchronises before it returns) over --steps rounds after --warmup, the median phases of tsm_clone_churn_last_ms, the counts,
whether the churn's classes equal tsm_clones' (every array), and the card's name and power limit.  Prints one JSON line per
workload; writes nothing."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import orc_clones as ocl  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402


def paste(data, rng):
    """30 consecutive lines of a file (from a random line), LF-terminated: a pasted test."""
    lines = data.split(b"\n")
    k = int(rng.integers(0, max(len(lines) - 30, 1)))
    return b"\n".join(lines[k:k + 30]) + b"\n"


def planted_step(files, exts, seed, n_edit=40, n_fix=20, n_paste=20):
    """(old_files, old_exts, new_files, new_exts, pair_old, pair_new): R_old is `files` plus n_fix planted copies (30 lines of a
    file pasted into a file of their own); R_new edits n_edit files (gen_edit, lambda = 6), changes one line in the middle of each
    planted copy (a one-copy fix inside a duplicated window) and adds n_paste new pasted tests."""
    rng = np.random.default_rng(seed)
    idx = rng.permutation(len(files))
    old, old_exts = list(files), list(exts)
    for i in idx[n_edit:n_edit + n_fix]:
        old.append(paste(files[i], rng)); old_exts.append(exts[i])
    new, new_exts = list(old), list(old_exts)
    po, pn = [], []
    for i in idx[:n_edit]:
        new[i] = ts.gen_edit(seed + int(i), files[i], 6.0)
        po.append(int(i)); pn.append(int(i))
    for j in range(len(files), len(old)):
        lines = old[j].split(b"\n")
        lines[len(lines) // 2] += b"  # fixed"
        new[j] = b"\n".join(lines)
        po.append(j); pn.append(j)
    for i in idx[-n_paste:]:
        new.append(paste(files[i], rng)); new_exts.append(exts[i])
        po.append(-1); pn.append(len(new) - 1)
    return old, np.array(old_exts, np.uint8), new, np.array(new_exts, np.uint8), po, pn


def run(sc, name, files, exts, args):
    files, exts, new, new_exts, po, pn = planted_step(files, exts, 0x22)
    ro, rn = ts.pack(files, exts, pinned=True), ts.pack(new, new_exts, pinned=True)
    pair_o = ts.pack([files[i] if i >= 0 else b"" for i in po], np.array([exts[i] if i >= 0 else 1 for i in po], np.uint8), pinned=True)
    pair_n = ts.pack([new[i] for i in pn], np.array([new_exts[i] for i in pn], np.uint8), pinned=True)
    cap = None
    for _ in range(args.warmup):
        r = sc.clone_churn(ro, rn, po, pn, args.min_lines, cap=cap)
        cap = max(len(r[s][k]) for s in ("old", "new") for k in ("class_len", "member"))
        sc.clones(ro, args.min_lines, cap=cap), sc.clones(rn, args.min_lines, cap=cap), sc.diff_marks(pair_o, pair_n)
    t, tc, ms = [], [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        r = sc.clone_churn(ro, rn, po, pn, args.min_lines, cap=cap)
        t.append(1e3 * (time.perf_counter() - t0))
        ms.append(sc.clone_churn_last_ms())
        t0 = time.perf_counter()
        co, cn = sc.clones(ro, args.min_lines, cap=cap), sc.clones(rn, args.min_lines, cap=cap)
        sc.diff_marks(pair_o, pair_n)
        tc.append(1e3 * (time.perf_counter() - t0))
    equal = all(np.array_equal(r[s][k], c[k]) for s, c in (("old", co), ("new", cn)) for k in ocl.KEYS)
    print(json.dumps({"metric": "tsm_clone_churn against 2 x tsm_clones + tsm_diff_pairs_marks, " + name, "unit": "ms",
                      "files_old": ro.n_files, "files_new": rn.n_files, "bytes_old": ro.source_bytes, "pairs": len(po),
                      "lines_old": int(r["old"]["line_base"][-1]), "min_lines": args.min_lines, "steps": args.steps, "warmup": args.warmup,
                      "clone_churn": {"ms_median": float(np.median(t)), "ms_min": float(min(t)),
                                      "device_ms_median": dict(zip(("k_scan", "classes", "gather_marks_diff", "churn_kernels"),
                                                                   (float(x) for x in np.median(np.array(ms), axis=0))))},
                      "composition": {"ms_median": float(np.median(tc)), "ms_min": float(min(tc))},
                      "classes": [len(r[s]["class_len"]) for s in ("old", "new")],
                      "touched_classes": [int((r[s]["status"] > 0).sum()) for s in ("old", "new")],
                      "classes_equal_to_tsm_clones": equal, "gpu": card()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-lines", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--c4-files", type=int, default=100000)
    args = ap.parse_args()
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, _ = ts.gen_pairs(0x7053454D0005, 4000, pinned=False)
    run(sc, "4 000 C5-law files", [a.file_bytes(i) for i in range(a.n_files)], a.ext.copy(), args)
    c = ts.gen_corpus(0x7053454D0C22, args.c4_files, size_law=1, pinned=False)
    run(sc, "%d C4-law files" % args.c4_files, [c.file_bytes(i) for i in range(c.n_files)], c.ext.copy(), args)
    sc.close()


if __name__ == "__main__":
    main()
