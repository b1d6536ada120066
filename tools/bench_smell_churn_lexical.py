#!/usr/bin/env python3
"""Cost of the lexical test-smell churn (docs/SPEC.md section 26), one GPU:

    python tools/bench_smell_churn_lexical.py [--pairs 50000] [--files 20000] [--steps 10] [--warmup 2] [--out F]

Two workloads, timed in alternating calls: the 50 000 pairs of BASELINE config C5, and a planted history (tests/lexsmell_ref.py
planted_corpus files as old sides, gen_edit(lambda = 6) of each as new sides).  Per workload: the median whole-call time of
Scanner.diff_smells_lexical on the host clock (the call synchronises before it returns) beside Scanner.diff_smells on the same
pairs, the median device time of each phase of both (k_scan, the smell (and lexical) stages, the diff, case records +
k_smell_churn), the counts, and one call of each under torch.profiler in a separate run (device ms per kernel).  The card's name
and power limit are read in the same run.  Prints one JSON line and, with --out, writes it there too."""
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
import lexsmell_ref as lr  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_cases import kernel_ms  # noqa: E402
from bench_diff_asserts import card  # noqa: E402

PHASES = ("k_scan", "smell_stages", "diff", "cases_churn")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=50_000)
    ap.add_argument("--files", type=int, default=20_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    work = {"c5": ts.gen_pairs(0x7053454D0005, args.pairs)}
    olds, exts = lr.planted_corpus(0x7053454D2605, args.files)
    news = [ts.gen_edit(i, o, 6.0) for i, o in enumerate(olds)]
    work["planted"] = (ts.pack(olds, exts, pinned=True), ts.pack(news, exts, pinned=True))
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    cap = {}
    for k, (a, b) in work.items():
        r = sc.diff_smells_lexical(a, b)
        cap[k] = max(len(r[x]) for x in ("old_cases", "new_cases", "old_tests", "new_tests"))
    res = {k: {"lexical": [], "smells": [], "ms_lexical": [], "ms_smells": []} for k in work}
    for step in range(args.warmup + args.steps):
        for k, (a, b) in work.items():                     # alternating calls
            t0 = time.perf_counter()
            r = sc.diff_smells_lexical(a, b, cap=cap[k])
            t1 = time.perf_counter()
            ml = sc.diff_smells_lexical_last_ms()
            sc.diff_smells(a, b, cap=cap[k])
            t2 = time.perf_counter()
            ms = sc.diff_smells_last_ms()
            res[k]["r"] = r
            if step >= args.warmup:
                res[k]["lexical"].append(1e3 * (t1 - t0))
                res[k]["smells"].append(1e3 * (t2 - t1))
                res[k]["ms_lexical"].append(ml)
                res[k]["ms_smells"].append(ms)
    out = {"metric": "tsm_diff_pairs_smells_lexical against tsm_diff_pairs_smells, C5 pairs and a planted history, alternating calls",
           "unit": "ms", "steps": args.steps, "warmup": args.warmup, "gpu": card()}
    for k, (a, b) in work.items():
        r = res[k]["r"]
        med = {x: dict(zip(PHASES, (float(v) for v in np.median(np.array(res[k]["ms_" + x]), axis=0)))) for x in ("lexical", "smells")}
        out[k] = {"pairs": a.n_files, "bytes": a.source_bytes + b.source_bytes, "old_tests": len(r["old_tests"]),
                  "new_tests": len(r["new_tests"]), "added_lex_instances": int(r["new_lex_churn"]["churned"].sum()),
                  "removed_lex_instances": int(r["old_lex_churn"]["churned"].sum()),
                  "diff_smells_lexical_ms_median": float(np.median(res[k]["lexical"])),
                  "diff_smells_ms_median": float(np.median(res[k]["smells"])),
                  "device_ms_median_lexical": med["lexical"], "device_ms_median_smells": med["smells"]}
    for k, (a, b) in work.items():                         # separate run: the profiler slows the host
        for name, fn in (("lexical", sc.diff_smells_lexical), ("smells", sc.diff_smells)):
            out[k]["profiler_kernel_ms_" + name] = {n: round(v, 4) for n, v in sorted(kernel_ms(lambda: fn(a, b, cap=cap[k])).items())}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    sc.close()


if __name__ == "__main__":
    main()
