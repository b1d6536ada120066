#!/usr/bin/env python3
"""Cost of the test-to-code link churn (docs/SPEC.md section 28), one GPU:

    python tools/bench_link_churn.py [--files 20000] [--steps 10] [--warmup 3] [--out F]

One planted repository of --files files (tests/link_ref.py, planted_repos with one repository: a third of them test files, PY,
C++ and Java, whose tests call Zipf-distributed names) and five steps from it: 1 and 100 test files edited (a call added to
their first test), 1 and 100 definition lines edited, and the most widely defined-and-called name deleted from every production
file.  Each step is timed with tsm_link_churn against what it replaces: two tsm_test_links calls (one per revision) plus
tsm_diff_pairs_marks over the changed pairs.  Reported per step: the median whole-call time of both on the host clock (every call
synchronises before it returns), the median device time of each phase (tsm_link_churn_last_ms), the event counts by kind, and
whether the events equal the plain-Python reference (tests/link_churn_ref.py) on a 1 500-file version of the same steps; and the
card's name and power limit.  Prints one JSON line and, with --out, writes it there too."""
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
import link_churn_ref as ref  # noqa: E402
import link_ref as lk  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402

PHASES = ("k_scan", "fronts_marks_change", "link_joins", "churn_join_emit")


def steps(n_files, seed):
    """{step name: (old revision, new revision, pair_old, pair_new)}; a revision is (files, exts, role, stem)."""
    files, exts, role, stem, _, paths = lk.planted_repos(seed, n_files, n_repos=1)
    old = (files, exts, role, stem)
    tests = [i for i in range(len(files)) if role[i]]
    prods = [i for i in range(len(files)) if not role[i] and (b"def " in files[i] or b"(int a) {" in files[i])]   # functions
    production = [i for i in range(len(files)) if not role[i]]
    calls = {}
    for f in tests:
        for w in files[f].split(b"("):
            nm = w.rsplit(b" ", 1)[-1]
            calls[nm] = calls.get(nm, 0) + 1
    hot = max((nm for nm in calls if nm.startswith(b"fn_") or nm.startswith(b"a_rather")), key=lambda nm: calls[nm])

    def edit(fs, fn):
        new = list(files)
        for f in fs:
            new[f] = fn(files[f])
        changed = [f for f in range(len(files)) if new[f] != files[f]]
        return (old, (new, exts, role, stem), changed, changed)

    def add_call(d):
        return d.replace(b"x0 = ", b"y0 = helper_x(0) + ", 1)

    def edit_def(d):
        return d.replace(b"(a):", b"(a, b=0):", 1).replace(b"(int a) {", b"(int a, int b) {", 1)

    def delete_hot(d):
        for kw, end in ((b"def ", b"("), (b"int ", b"("), (b"class ", b":"), (b"class ", b" {")):   # every definition of it
            d = d.replace(kw + hot + end, kw + b"gone_" + hot + end)
        return d
    return {"tests_1": edit(tests[:1], add_call), "tests_100": edit(tests[:100], add_call), "defs_1": edit(prods[:1], edit_def),
            "defs_100": edit(prods[:100], edit_def), "delete_hot": edit(production, delete_hot)}


def pair_corpora(old, new, po, pn):
    return (ts.pack([old[0][f] for f in po], old[1][po], pinned=True), ts.pack([new[0][f] for f in pn], new[1][pn], pinned=True))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=20000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    work = steps(args.files, 0x7053454D2800)
    sc = ts.Scanner(0, 1 << 20, 16, 4)
    out = {"metric": "tsm_link_churn against two tsm_test_links + tsm_diff_pairs_marks, planted one-repository history",
           "unit": "ms", "files": args.files, "steps": args.steps, "warmup": args.warmup, "gpu": card()}
    for name, (old, new, po, pn) in work.items():
        ko, kn = ts.pack(old[0], old[1], pinned=True), ts.pack(new[0], new[1], pinned=True)
        po_a, pn_a = np.asarray(po, np.int32), np.asarray(pn, np.int32)
        po_k, pn_k = pair_corpora(old, new, po_a, pn_a)
        t_new, t_old, ms = [], [], []
        for it in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            r = sc.link_churn(ko, kn, old[2], new[2], po, pn, old[3], new[3], cap=1 << 18)
            t1 = time.perf_counter()
            sc.test_links(ko, old[2], old[3], cap=1 << 18)
            sc.test_links(kn, new[2], new[3], cap=1 << 18)
            sc.diff_marks(po_k, pn_k)
            t2 = time.perf_counter()
            if it >= args.warmup:
                t_new.append(1e3 * (t1 - t0))
                t_old.append(1e3 * (t2 - t1))
                ms.append(sc.link_churn_last_ms())
        ev = r["events"]["event"]
        out[name] = {"changed_files": len(po), "events": int(len(ev)),
                     "by_event": {ref.EVENTS[k]: int((ev == k).sum()) for k in range(len(ref.EVENTS)) if (ev == k).any()},
                     "link_churn_ms_median": float(np.median(t_new)), "two_links_plus_marks_ms_median": float(np.median(t_old)),
                     "device_ms_median": dict(zip(PHASES, (float(v) for v in np.median(np.array(ms), axis=0))))}
    small = steps(1500, 0x7053454D2801)
    eq = {}
    for name, (old, new, po, pn) in small.items():
        got = sc.link_churn(ts.pack(old[0], old[1]), ts.pack(new[0], new[1]), old[2], new[2], po, pn, old[3], new[3])
        want = ref.churn(old, new, po, pn)
        eq[name] = [tuple(int(x) for x in e) for e in got["events"]] == [tuple(e) for e in want["events"]]
    out["reference_equal_1500"] = eq
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    sc.close()


if __name__ == "__main__":
    main()
