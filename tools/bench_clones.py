#!/usr/bin/env python3
"""Cost of the clone classes (docs/SPEC.md section 15) on a C4-scale corpus with planted copies, one GPU:

    python tools/bench_clones.py [--files 100000] [--min-lines 5] [--steps 10] [--warmup 3]

The corpus: --files files of BASELINE config C4's size law (seeded), every fourth of them replaced by tsm_gen_edit
(lambda = 6) of an earlier file (tests/orc_clones.py, c4_planted).  Reported: the median whole-call time of Scanner.clones on
the host clock (the call synchronises before it returns) and the median device time of each of its phases
(tsm_clones_last_ms: k_scan, grouping + classes, members + coverage) over --steps calls after --warmup, the counts, the serial
C reference's time on the same corpus (whose output must equal the GPU's, every array), and the card's name and power limit.
Prints one JSON line; writes nothing."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=100000)
    ap.add_argument("--min-lines", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    files, exts = ocl.c4_planted(0x7053454D0C15, args.files)
    c = ts.pack(files, exts, pinned=True)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    cap = None
    for _ in range(args.warmup):
        r = sc.clones(c, args.min_lines, cap=cap)
        cap = max(len(r["class_len"]), len(r["member"]))
    t, ms, phases = [], [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        r = sc.clones(c, args.min_lines, cap=cap)
        t.append(1e3 * (time.perf_counter() - t0))
        ms.append(sc.clones_last_ms())
    t0 = time.perf_counter()
    ref = ocl.clones(c, args.min_lines)
    cpu_s = time.perf_counter() - t0
    ocl.assert_equal(r, ref)
    lines = int(r["line_base"][-1])
    print(json.dumps({"metric": "tsm_clones over a C4-scale corpus with planted copies", "unit": "ms", "files": c.n_files,
                      "bytes": c.source_bytes, "lines": lines, "min_lines": args.min_lines, "steps": args.steps, "warmup": args.warmup,
                      "ms_median": float(np.median(t)), "ms_min": float(min(t)),
                      "device_ms_median": dict(zip(("k_scan", "grouping_classes", "members_coverage"),
                                                   (float(x) for x in np.median(np.array(ms), axis=0)))),
                      "classes": len(r["class_len"]), "fragments": len(r["member"]), "duplicated_lines": int(r["file_dup"].sum()),
                      "duplicated_assertion_lines": int(r["file_dup_assert"].sum()), "largest_class": int(np.diff(r["class_base"]).max()),
                      "cpu_reference_s": cpu_s, "equal_to_cpu_reference": True, "gpu": card()}))
    sc.close()


if __name__ == "__main__":
    main()
