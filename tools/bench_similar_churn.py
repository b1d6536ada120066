#!/usr/bin/env python3
"""Cost of the similar-test churn of one step (docs/SPEC.md section 24), one GPU:

    python tools/bench_similar_churn.py [--tests 500000] [--steps 5] [--warmup 1]

Workloads, one JSON line each:
* C1, the study's own test files (tests/golden/c1_testfiles.npz), with steps that touch 1, 10 and 100 tests;
* a generated corpus of --tests PY tests (tests/simtest_ref.generated, seeded), with steps that touch 0.1 % and 1 % of them.
A step touches a test by inserting one line behind its header; the files it touches are the step's pairs, all others are
unchanged.  For each, in one run and alternating: tsm_similar_churn of the step, against what it replaces - tsm_similar_tests
of both revisions plus tsm_diff_pairs_marks of the touched files.  Reported: median whole-call times on the host clock (every
call synchronises before it returns), the median device phases of tsm_similar_churn (tsm_similar_churn_last_ms), the candidates
the restricted enumeration verified per side against tsm_similar_tests' full count, the summed device phases of the two
tsm_similar_tests calls, the events, and the card's name and power limit.  The events are checked against tsm_similar_tests of
both revisions: every pair of either side with a touched test is in an event.  Writes nothing."""
import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import corpus_util as cu  # noqa: E402
import simtest_ref as sr  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402

HEADER = re.compile(rb"^[ \t]*def (test\w*)\(", re.M)


def touch(files, exts, n_touch, seed):
    """The new revision: n_touch test headers (random, over all files) each followed by one inserted line."""
    rng = np.random.default_rng(seed)
    heads = [(f, m.end()) for f, data in enumerate(files) if int(exts[f]) == 1 for m in HEADER.finditer(data)]
    pick = sorted((heads[int(i)] for i in rng.choice(len(heads), n_touch, replace=False)), reverse=True)
    new = list(files)
    for f, at in pick:
        eol = new[f].index(b"\n", at) + 1
        indent = re.match(rb"[ \t]*", new[f][eol:]).group(0) or b"    "
        new[f] = new[f][:eol] + indent + b"touched = True\n" + new[f][eol:]
    touched = sorted({f for f, _ in pick})
    return new, touched


def run(s, name, files, exts, n_touch, steps, warmup, seed=7):
    new, touched = touch(files, exts, n_touch, seed)
    old_k, new_k = ts.pack(files, exts), ts.pack(new, exts)
    po = pn = np.array(touched, np.int32)
    sub_old = ts.pack([files[f] for f in touched], exts[touched])
    sub_new = ts.pack([new[f] for f in touched], exts[touched])
    t_churn, t_base, phases, base_phases = [], [], [], []
    for it in range(warmup + steps):
        t0 = time.perf_counter()
        got = s.similar_churn(old_k, new_k, po, pn)
        t1 = time.perf_counter()
        so = s.similar_tests(old_k)
        po_ms = s.similar_tests_last_ms()
        sn = s.similar_tests(new_k)
        pn_ms = s.similar_tests_last_ms()
        s.diff_marks(sub_old, sub_new)
        t2 = time.perf_counter()
        if it >= warmup:
            t_churn.append((t1 - t0) * 1e3)
            t_base.append((t2 - t1) * 1e3)
            phases.append(s.similar_churn_last_ms())
            base_phases.append([x + y for x, y in zip(po_ms, pn_ms)])
    for side, st in (("old", so), ("new", sn)):
        dirty = got[side]["change"] != ord("=")
        want = {(int(p["a"]), int(p["b"])) for p in st["pairs"] if dirty[p["a"]] or dirty[p["b"]]}
        a, b = ("old_a", "old_b") if side == "old" else ("a", "b")
        lcs = "old_lcs" if side == "old" else "lcs"
        seen = {(int(e[a]), int(e[b])) for e in got["events"] if e[lcs] != 0xFFFFFFFF}
        assert want <= seen, (name, side)
    ph = np.median(np.array(phases), axis=0)
    ev = got["events"]
    return {"metric": "tsm_similar_churn of one step", "unit": "ms", "workload": name, "files": len(files),
            "touched_tests": n_touch, "touched_files": len(touched), "steps": steps, "warmup": warmup,
            "ms_median": float(np.median(t_churn)), "two_similar_tests_plus_marks_ms_median": float(np.median(t_base)),
            "device_ms_median": dict(zip(("k_scan", "fronts_marks_change", "tokens_lists_enumeration", "verification"),
                                         (float(x) for x in ph))),
            "two_similar_tests_device_ms_median": dict(zip(("k_scan", "spans_smells_lexer", "tokens_lists_enumeration", "verification"),
                                                           (float(x) for x in np.median(np.array(base_phases), axis=0)))),
            "tests": [len(got["old"]["tests"]), len(got["new"]["tests"])],
            "changed_tests": int(np.count_nonzero(got["new"]["change"] != ord("="))),
            "candidates_restricted": [got["old"]["n_candidates"], got["new"]["n_candidates"]],
            "candidates_full": [so["n_candidates"], sn["n_candidates"]],
            "events": len(ev), "events_by_status": {k: int(np.count_nonzero(ev["status"] == i)) for i, k in enumerate(ts.SIMILAR_STATUSES)},
            "events_checked_against_similar_tests": True, "gpu": card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tests", type=int, default=500000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    files, exts, _, _ = cu.load_fixture(os.path.join(ROOT, "tests", "golden", "c1_testfiles.npz"))
    files, exts = list(files), np.asarray(exts, np.uint8)
    s = ts.Scanner(device=0, max_arena_bytes=1 << 30, max_files=1 << 17, max_groups=4)
    for n in (1, 10, 100):
        print(json.dumps(run(s, "C1", files, exts, n, a.steps, a.warmup)), flush=True)
    k, _ = sr.generated(1, a.tests)
    gfiles = [bytes(k.arena[int(k.off[i]):int(k.off[i]) + int(k.len[i])]) for i in range(k.n_files)]
    gexts = np.ones(len(gfiles), np.uint8)
    for frac in (0.001, 0.01):
        print(json.dumps(run(s, "generated", gfiles, gexts, int(a.tests * frac), a.steps, a.warmup)), flush=True)
    s.close()


if __name__ == "__main__":
    main()
