#!/usr/bin/env python3
"""Cost of the moved code (docs/SPEC.md section 20), one GPU:

    python tools/bench_moves.py [--pairs 50000] [--steps 10] [--warmup 2] [--out F]

Five workloads, timed in alternating calls: the 50 000 pairs of BASELINE config C5 in steps of 8 pairs and in one step (as `diff`
puts a whole tree pair: blank lines and `}` of every file meet in one key); a planted-move history
(tests/test_gpu_moves.py planted: 20 000 C5-like pairs in steps of 8 with a stretch of a new side moved to another pair of its
step); the duplicate-heavy step (2 000 blank and 2 000 `}` lines per side, every line changed: the quadratic case of the reach);
and a 70 000-line whole-file move beside a 70 000-line run that matches line by line but forms no block (70 000 steps for a walk
of one step per line; none for the walk of k_move_runs, which steps from block to block).  Per workload: the median whole-call time of Scanner.diff_moves on the host clock (the call synchronises before it
returns) beside Scanner.diff_marks on the same pairs, the median device time of each phase (tsm_moves_last_ms: k_scan, the diff,
line flags + join + k_move_reach, k_move_starts + k_move_runs + k_move_mark), the counts, and one call under torch.profiler in a
separate run (device ms per kernel).  The card's name and power limit are read in the same run.  Prints one JSON line and, with --out,
writes it there too."""
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
import tosemscan as ts  # noqa: E402
from bench_cases import kernel_ms  # noqa: E402
from bench_diff_asserts import card  # noqa: E402
from test_gpu_moves import planted, stepped  # noqa: E402

PHASES = ("k_scan", "diff", "join_reach", "runs_blocks")


def workloads(n_pairs):
    a, b = ts.gen_pairs(0x7053454D0005, n_pairs)
    w = {"c5_steps_of_8": (stepped(a, [i // 8 for i in range(n_pairs)]), stepped(b, [i // 8 for i in range(n_pairs)])),
         "c5_one_step": (stepped(a, [0] * n_pairs), stepped(b, [0] * n_pairs))}
    olds, news, exts = planted(0x7053454D0020, 20_000, 8)
    st = [i // 8 for i in range(len(olds))]
    w["planted"] = (stepped(ts.pack(olds, exts, pinned=True), st), stepped(ts.pack(news, exts, pinned=True), st))

    def side(tag):
        return b"".join(b"%s_%d = compute_%d(x)\n\n}\n" % (tag, i, i) for i in range(2_000))
    w["duplicate_heavy"] = (ts.pack([side(b"a"), b""], [1, 1], pinned=True), ts.pack([b"", side(b"b")], [1, 1], pinned=True))
    whole = b"".join(b"    self.assertEqual(value_%d, other_%d)\n" % (j, j) for j in range(70_000))
    lines = [b"m%05d\n" % j for j in range(70_000)]
    olds = [whole, b"", b"".join(lines), b""]
    news = [b"", whole, b"", b"".join(lines[j ^ 1] for j in range(70_000))]
    w["move_70000"] = (ts.pack(olds, [1] * 4, pinned=True), ts.pack(news, [1] * 4, pinned=True))
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=50_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    work = workloads(args.pairs)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    cap = {}
    for k, (a, b) in work.items():
        r = sc.diff_moves(a, b)
        cap[k] = max(len(r["dels"]), len(r["ins"]), len(r["old_blocks"]), len(r["new_blocks"]))
    res = {k: {"moves": [], "marks": [], "ms": []} for k in work}
    for step in range(args.warmup + args.steps):
        for k, (a, b) in work.items():                     # alternating calls
            t0 = time.perf_counter()
            r = sc.diff_moves(a, b, cap=cap[k])
            t1 = time.perf_counter()
            ms = sc.moves_last_ms()
            sc.diff_marks(a, b, cap=cap[k])
            t2 = time.perf_counter()
            res[k]["r"] = r
            if step >= args.warmup:
                res[k]["moves"].append(1e3 * (t1 - t0))
                res[k]["marks"].append(1e3 * (t2 - t1))
                res[k]["ms"].append(ms)
    out = {"metric": "tsm_diff_pairs_moves against tsm_diff_pairs_marks on the same pairs, alternating calls", "unit": "ms",
           "steps": args.steps, "warmup": args.warmup, "gpu": card()}
    for k, (a, b) in work.items():
        r = res[k]["r"]
        out[k] = {"pairs": a.n_files, "bytes": a.source_bytes + b.source_bytes, "changed_lines": int((r["dels"] != 0).sum() + (r["ins"] != 0).sum()),
                  "old_blocks": len(r["old_blocks"]), "new_blocks": len(r["new_blocks"]),
                  "moved_lines": int((r["dels"] & 2).astype(bool).sum() + (r["ins"] & 2).astype(bool).sum()),
                  "diff_moves_ms_median": float(np.median(res[k]["moves"])), "diff_marks_ms_median": float(np.median(res[k]["marks"])),
                  "device_ms_median": dict(zip(PHASES, (float(x) for x in np.median(np.array(res[k]["ms"]), axis=0))))}
    for k, (a, b) in work.items():                         # separate run: the profiler slows the host
        out[k]["profiler_kernel_ms"] = {n: round(v, 4) for n, v in sorted(kernel_ms(lambda: sc.diff_moves(a, b, cap=cap[k])).items())
                                        if n.startswith("tsm::") or n.startswith("Memcpy")}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    sc.close()


if __name__ == "__main__":
    main()
