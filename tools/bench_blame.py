"""Device time of line provenance (docs/SPEC.md section 14) on a synthetic history: F files of the C5 size law, C commits, each
editing E files with gen_edit(lambda).  The pairs of the whole history are one batch of chains (a file's edits in commit order).
Alternating on the same batch: tsm_diff_pairs_detail (plain kernels) and tsm_blame_pairs (DIFF_MARKS kernels + k_blame), each
timed by CUDA events inside the library (tsm_diff_last_ms, tsm_blame_last_ms); medians over the repetitions.

    python tools/bench_blame.py [--files 4000] [--commits 500] [--per-commit 40] [--lam 6] [--reps 10] [--out F]
"""
import argparse
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
import tosemscan as ts  # noqa: E402


def history(files, commits, per_commit, lam, seed=0x7053454D0014):
    base = ts.gen_corpus(seed, files, size_law=1, pinned=False)
    cur = [base.file_bytes(i) for i in range(files)]
    last = [-1] * files
    rng = random.Random(seed)
    olds, news, exts, prev, label = [], [], [], [], []
    for c in range(commits):
        for f in rng.sample(range(files), per_commit):
            new = ts.gen_edit(seed + len(olds), cur[f], lam)
            olds.append(cur[f]); news.append(new); exts.append(int(base.ext[f]))
            prev.append(last[f]); label.append(c)
            last[f] = len(olds) - 1
            cur[f] = new
    heads = {}
    for i, p in enumerate(prev):                           # the first edit of a file: its lines are boundary lines
        if p < 0:
            heads[i] = np.array([(-1, j + 1) for j in range(len(ts_lines(olds[i])))], ts.ORIGIN)
    return olds, news, exts, np.array(prev, np.int32), np.array(label, np.int32), heads


def ts_lines(b):
    if not b:
        return []
    parts = b.split(b"\n")
    return parts[:-1] if parts[-1] == b"" else parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=4000)
    ap.add_argument("--commits", type=int, default=500)
    ap.add_argument("--per-commit", type=int, default=40)
    ap.add_argument("--lam", type=float, default=6.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().split("\n")[0]
    olds, news, exts, prev, label, heads = history(a.files, a.commits, a.per_commit, a.lam)
    A, B = ts.pack(olds, exts, pinned=True), ts.pack(news, exts, pinned=True)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    plain, marks, blame, wall = [], [], [], [[], []]
    for r in range(a.reps + 2):                            # two warm-up rounds
        t0 = time.perf_counter()
        d = sc.diff_pairs(A, B, detail=True)
        t1 = time.perf_counter()
        g = sc.blame_pairs(A, B, prev, label, heads)
        t2 = time.perf_counter()
        if r < 2:
            continue
        wall[0].append(t1 - t0); wall[1].append(t2 - t1)
        blame.append(sc.blame_last_ms())
        marks.append(sc.diff_last_ms())
        sc.diff_pairs(A, B, detail=True)
        plain.append(sc.diff_last_ms())
    assert all(np.array_equal(x, y) for x, y in zip(d, g[:3]))
    med = lambda v: float(np.median(v))                    # noqa: E731
    lines = [
        "# tools/bench_blame.py: %d files (C5 size law), %d commits x %d edited files (gen_edit lambda %g) = %d pairs in %d chains; %d lines old, "
        "%d lines new; medians of %d alternating repetitions" % (a.files, a.commits, a.per_commit, a.lam, len(prev), int((prev < 0).sum()),
                                                                 sum(len(ts_lines(x)) for x in olds), len(g[4]), a.reps),
        "# card: %s" % card,
        "kernel                          tsm_diff_pairs_detail (ms)   tsm_blame_pairs (ms)",
        "k_scan (both sides)             %10.3f                  %10.3f" % (med([p[0] for p in plain]), med([m[0] for m in marks])),
        "k_diff_small (four sizes)       %10.3f                  %10.3f  (marks)" % (med([p[1] for p in plain]), med([m[1] for m in marks])),
        "k_myers + k_myers_trace         %10.3f                  %10.3f" % (med([p[2] for p in plain]), med([m[2] for m in marks])),
        "k_blame                         %10s                  %10.3f" % ("-", med(blame)),
        "whole call, host clock          %10.3f                  %10.3f" % (1e3 * med(wall[0]), 1e3 * med(wall[1])),
    ]
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)
    sc.close()


if __name__ == "__main__":
    main()
