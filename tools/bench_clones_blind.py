#!/usr/bin/env python3
"""Cost of the blind clones (docs/SPEC.md section 21) against the exact clones of section 15 on the same C4-scale corpus, one GPU:

    python tools/bench_clones_blind.py [--files 100000] [--min-lines 5] [--steps 10] [--warmup 3]

The corpus is bench_clones.py's: --files files of BASELINE config C4's size law (seeded), every fourth of them replaced by
tsm_gen_edit (lambda = 6) of an earlier file (tests/orc_clones.py, c4_planted).  The two calls alternate, so that both see the same
state of the card.  Reported per call: the median whole-call time on the host clock (the calls synchronise before they return)
and the median device time of each phase (tsm_clones_last_ms; tsm_clones_blind_last_ms: k_scan, lexing + compaction, grouping +
classes, members + coverage) over --steps calls after --warmup, the counts, whether the blind call equals the serial C reference
(every array), and the card's name and power limit.  Prints one JSON line; writes nothing."""
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
import blind_ref as br  # noqa: E402
import orc_blind as ob  # noqa: E402
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
    cap = cap_b = None
    for _ in range(args.warmup):
        r = sc.clones(c, args.min_lines, cap=cap)
        cap = max(len(r["class_len"]), len(r["member"]))
        rb = sc.clones(c, args.min_lines, blind=True, cap=cap_b)
        cap_b = max(len(rb["class_len"]), len(rb["member"]), len(rb["kept_line"]))
    t, tb, ms, msb = [], [], [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        r = sc.clones(c, args.min_lines, cap=cap)
        t.append(1e3 * (time.perf_counter() - t0))
        ms.append(sc.clones_last_ms())
        t0 = time.perf_counter()
        rb = sc.clones(c, args.min_lines, blind=True, cap=cap_b)
        tb.append(1e3 * (time.perf_counter() - t0))
        msb.append(sc.clones_blind_last_ms())
    br.assert_equal(rb, ob.clones_blind(c, args.min_lines))

    def counts(x):
        return {"classes": len(x["class_len"]), "fragments": len(x["member"]), "duplicated_lines": int(x["file_dup"].sum()),
                "duplicated_assertion_lines": int(x["file_dup_assert"].sum())}
    print(json.dumps({"metric": "tsm_clones_blind against tsm_clones over a C4-scale corpus with planted copies", "unit": "ms",
                      "files": c.n_files, "bytes": c.source_bytes, "lines": int(r["line_base"][-1]), "kept_lines": len(rb["kept_line"]),
                      "min_lines": args.min_lines, "steps": args.steps, "warmup": args.warmup,
                      "clones": {"ms_median": float(np.median(t)), "ms_min": float(min(t)),
                                 "device_ms_median": dict(zip(("k_scan", "grouping_classes", "members_coverage"),
                                                              (float(x) for x in np.median(np.array(ms), axis=0)))), **counts(r)},
                      "clones_blind": {"ms_median": float(np.median(tb)), "ms_min": float(min(tb)),
                                       "device_ms_median": dict(zip(("k_scan", "lexing_compaction", "grouping_classes", "members_coverage"),
                                                                    (float(x) for x in np.median(np.array(msb), axis=0)))), **counts(rb)},
                      "blind_equal_to_cpu_reference": True, "gpu": card()}))
    sc.close()


if __name__ == "__main__":
    main()
