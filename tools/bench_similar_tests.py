#!/usr/bin/env python3
"""Cost of the similar tests (docs/SPEC.md section 23), one GPU:

    python tools/bench_similar_tests.py [--tests 500000] [--steps 5] [--warmup 1]

Two workloads, each one JSON line:
* C1, the study's own test files (tests/golden/c1_testfiles.npz) at (min_lines, P) = (5, 70); the result is checked against the
  serial C brute force (tests/orc_simtest.c), every array.
* A generated corpus of --tests PY tests (seeded) at (5, 70): bodies of 4 to 20 lines drawn from 65 536 distinct blind line shapes,
  a fifth of the lines from 16 common shapes (the assertion and set-up lines every suite repeats); every tenth test is a Type-3
  copy of an earlier one with one or two lines inserted, deleted or changed.  Every reported pair's LCS is recomputed, and 8
  random tests are brute-forced against the whole corpus.
Reported: the median whole-call time on the host clock (the call synchronises before it returns), the median device time of each
phase (tsm_similar_tests_last_ms), tests, compared tests, candidates verified, pairs and classes, the card's name and power limit,
and the posting-list lengths of the prefix tokens and the virtual candidate space they span, from the filter model of
tests/simtest_ref.py (ties of equal counts broken by shape; the device breaks them by table slot, so the lists can differ
slightly).  Writes nothing."""
import argparse
import json
import os
import random
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


def shape(v):
    return "x" + "".join("[x]" if (v >> b) & 1 else "(x)" for b in range(16))


def generated(seed, n_tests):
    rng = np.random.default_rng(seed)
    shapes = [shape(v) for v in range(1 << 16)]
    klen = rng.integers(4, 21, n_tests)
    common = rng.random(int(klen.sum())) < 0.2
    ids = np.where(common, rng.integers(0, 16, common.size), rng.integers(16, 1 << 16, common.size))
    bodies, at = [], 0
    prng = random.Random(seed)
    for t in range(n_tests):
        b = ids[at:at + klen[t]].tolist()
        at += klen[t]
        if t % 10 == 9:
            b = list(bodies[prng.randrange(t)])
            for _ in range(prng.randint(1, 2)):
                r = prng.random()
                if r < 0.33 and len(b) > 1:
                    b.pop(prng.randrange(len(b)))
                elif r < 0.66:
                    b.insert(prng.randrange(len(b) + 1), prng.randrange(16, 1 << 16))
                else:
                    b[prng.randrange(len(b))] = prng.randrange(16, 1 << 16)
        bodies.append(b)
    files = []
    for f in range(0, n_tests, 100):
        files.append("".join("def test_%d():\n%s" % (t, "".join("    %s\n" % shapes[v] for v in bodies[t]))
                             for t in range(f, min(f + 100, n_tests))).encode())
    return ts.pack(files, np.ones(len(files), np.uint8), pinned=True)


def prefix_lists(seqs, min_lines, P):
    """Posting-list lengths of the prefix tokens (the filter model, vectorised) and the candidates they span."""
    k = np.array([len(s) for s in seqs], np.int64)
    cmp = k >= min_lines
    test = np.repeat(np.arange(len(seqs)), k)
    h = np.array([x for s in seqs for x in s], np.uint64)
    keep = cmp[test]
    test, h = test[keep], h[keep]
    uh, hid = np.unique(h, return_inverse=True)
    cnt = np.bincount(hid)
    order = np.lexsort((np.arange(h.size), hid, test))         # j: the occurrence of h within its test
    t_s, h_s = test[order], hid[order]
    new_run = np.r_[True, (t_s[1:] != t_s[:-1]) | (h_s[1:] != h_s[:-1])]
    run_start = np.maximum.accumulate(np.where(new_run, np.arange(h_s.size), 0))
    j = np.empty(h.size, np.int64)
    j[order] = np.arange(h_s.size) - run_start
    o2 = np.lexsort((j, hid, cnt[hid], test))                   # each test's tokens in the global order
    t2 = test[o2]
    first = np.r_[0, np.nonzero(t2[1:] != t2[:-1])[0] + 1]
    rank = np.arange(t2.size) - np.repeat(first, np.diff(np.r_[first, t2.size]))
    kk = k[t2]
    q = kk - (P * kk + 199 - P) // (200 - P) + 1
    sel = o2[rank < q]
    key = hid[sel].astype(np.int64) * (1 << 20) + j[sel]
    _, m = np.unique(key, return_counts=True)
    return {"prefix_tokens": int(sel.size), "lists": int(m.size), "list_len_p50": int(np.median(m)),
            "list_len_p99": int(np.percentile(m, 99)), "list_len_max": int(m.max()),
            "virtual_candidates": int((m * (m - 1) // 2).sum())}


def run(sc, c, min_lines, P, steps, warmup):
    cap = None
    for _ in range(warmup):
        r = sc.similar_tests(c, min_lines, P, cap=cap)
        cap = max(len(r["tests"]), len(r["pairs"]))
    t, ms = [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        r = sc.similar_tests(c, min_lines, P, cap=cap)
        t.append(1e3 * (time.perf_counter() - t0))
        ms.append(sc.similar_tests_last_ms())
    out = {"ms_median": float(np.median(t)), "ms_min": float(min(t)),
           "device_ms_median": dict(zip(("k_scan", "spans_smells_lexer", "tokens_lists_enumeration", "verification"),
                                        (float(x) for x in np.median(np.array(ms), axis=0)))),
           "tests": len(r["tests"]), "compared_tests": int((r["test_kept"] >= min_lines).sum()), "candidates": r["n_candidates"],
           "pairs": len(r["pairs"]), "classes": len(r["class_base"]) - 1}
    return r, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tests", type=int, default=500000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    gpu = card()
    files, exts, _, _ = cu.load_fixture(os.path.join(ROOT, "tests", "golden", "c1_testfiles.npz"))
    c = ts.pack(files, exts, pinned=True)
    r, out = run(sc, c, 5, 70, args.steps, args.warmup)
    sr.assert_equal(r, sr.reference(c, 5, 70))
    _, seqs = sr.c_sequences(c)
    print(json.dumps({"metric": "tsm_similar_tests over the C1 test files", "unit": "ms", "workload": "C1", "files": c.n_files,
                      "min_lines": 5, "similarity": 70, "steps": args.steps, "warmup": args.warmup, **out,
                      "prefix_model": prefix_lists(seqs, 5, 70), "equal_to_cpu_reference": True, "gpu": gpu}), flush=True)
    c = generated(0x53494D54, args.tests)
    r, out = run(sc, c, 5, 70, args.steps, args.warmup)
    _, seqs = sr.c_sequences(c)
    k = [len(s) for s in seqs]
    for a, b, l, score in r["pairs"].tolist():
        assert sr.lcs(seqs[a], seqs[b]) == l and score == 120000 * l // (k[a] + k[b]) and 200 * l >= 70 * (k[a] + k[b])
    rng = random.Random(1)
    for a in rng.sample(range(len(seqs)), 8):
        p = r["pairs"]
        got = sorted(p["b"][p["a"] == a].tolist() + p["a"][p["b"] == a].tolist())
        assert got == sr.c_partners(seqs, a, 5, 70), a
    print(json.dumps({"metric": "tsm_similar_tests over a generated corpus with planted Type-3 copies", "unit": "ms",
                      "workload": "generated", "files": c.n_files, "bytes": c.source_bytes, "min_lines": 5, "similarity": 70,
                      "steps": args.steps, "warmup": args.warmup, **out, "prefix_model": prefix_lists(seqs, 5, 70),
                      "pairs_lcs_checked": len(r["pairs"]), "tests_brute_forced": 8, "gpu": gpu}), flush=True)
    sc.close()


if __name__ == "__main__":
    main()
