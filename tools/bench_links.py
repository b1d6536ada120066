#!/usr/bin/env python3
"""Cost of the test-to-code links (docs/SPEC.md section 27), one GPU:

    python tools/bench_links.py [--files 100000] [--steps 10] [--warmup 3] [--out F]

Three corpora, each timed with tsm_test_links: --files files of three planted repositories (tests/link_ref.py, planted_repos: a
third of them test files, PY, C++ and Java, whose tests call Zipf-distributed names, some defined in several files, some in the
focal file, some nowhere); the hot name, one name defined 100 000 times and called 1 000 000 times (every call joins one name
slot and 1 000 link slots); and one test of 20 000 distinct linked names.  Reported: the median whole-call time on the host
clock (the call synchronises before it returns), the median device time of each phase (tsm_test_links_last_ms), the counts,
whether the outputs equal the plain-Python reference on a 3 000-file planted corpus and on both worst cases; and the card's name
and power limit.  Prints one JSON line and, with --out, writes it there too."""
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
import link_ref as lk  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402

PHASES = ("k_scan", "front", "k_link_lines", "join_records")


def hot_name():
    prod = b"".join(b"def hot(x%d):\n    pass\n" % i for i in range(10000))
    test = b"".join(b"def test_%d():\n" % i + b"    hot(1); hot(2); hot(3); hot(4); hot(5)\n" * 200 for i in range(100))
    return [prod] * 10 + [test] * 10, np.ones(20, np.uint8), np.array([0] * 10 + [1] * 10, np.uint8), None, np.zeros(20, np.uint16)


def many_names():
    n = 20000
    prod = b"".join(b"int f%d(int a) {\n  return a;\n}\n" % i for i in range(n))
    test = b"TEST(A, B) {\n" + b"".join(b"  f%d(%d);\n" % (i, i) for i in range(n)) + b"}\n"
    return [prod, test], np.array([2, 2], np.uint8), np.array([0, 1], np.uint8), None, np.zeros(2, np.uint16)


def equal(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("tests", "links", "defs"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    src = {"c4_planted": lk.planted_repos(0x7053454D2700, args.files)[:5], "hot_name": hot_name(), "many_names": many_names()}
    corp = {k: ts.pack(f, e, grps=g, n_groups=int(g.max()) + 1, pinned=True) for k, (f, e, _, _, g) in src.items()}
    sc = ts.Scanner(0, 1 << 20, 16, 4)
    caps = {k: max(len(v) for v in sc.test_links(c, src[k][2], src[k][3]).values()) for k, c in corp.items()}
    res = {k: {"t": [], "ms": []} for k in corp}
    for step in range(args.warmup + args.steps):
        for k, c in corp.items():
            t0 = time.perf_counter()
            r = sc.test_links(c, src[k][2], src[k][3], cap=caps[k])
            t = 1e3 * (time.perf_counter() - t0)
            res[k]["r"] = r
            if step >= args.warmup:
                res[k]["t"].append(t)
                res[k]["ms"].append(sc.test_links_last_ms())
    out = {"metric": "tsm_test_links: C4-scale planted repositories and two worst cases", "unit": "ms", "steps": args.steps,
           "warmup": args.warmup, "gpu": card()}
    for k, c in corp.items():
        r = res[k]["r"]
        out[k] = {"files": c.n_files, "bytes": c.source_bytes, "test_files": int(src[k][2].sum()), "tests": len(r["tests"]),
                  "calls": int(r["tests"]["calls"].sum()), "links": len(r["links"]), "definitions": len(r["defs"]),
                  "ambiguous_links": int((r["links"]["target"] < 0).sum()), "eager": int((r["tests"]["flags"] & 1).sum()),
                  "lazy": int((r["tests"]["flags"] >> 1 & 1).sum()),
                  "ms_median": float(np.median(res[k]["t"])), "ms_min": float(min(res[k]["t"])),
                  "device_ms_median": dict(zip(PHASES, (float(v) for v in np.median(np.array(res[k]["ms"]), axis=0))))}
    small = lk.planted_repos(0x7053454D2701, 3000)[:5]
    out["reference_equal"] = {
        "planted_3000": equal(sc.test_links(ts.pack(small[0], small[1], grps=small[4], n_groups=3), small[2], small[3]),
                              lk.py_links(small[0], small[1], small[2], small[3], small[4])),
        "hot_name": equal(res["hot_name"]["r"], lk.py_links(*src["hot_name"])),
        "many_names": equal(res["many_names"]["r"], lk.py_links(*src["many_names"]))}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    sc.close()


if __name__ == "__main__":
    main()
