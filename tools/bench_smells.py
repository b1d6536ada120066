#!/usr/bin/env python3
"""Cost of the test smells (docs/SPEC.md section 18), one GPU:

    python tools/bench_smells.py [--files 100000] [--steps 10] [--warmup 3] [--out F]

Two corpora, timed in alternating calls: --files files of BASELINE config C4's size law (seeded sizes from tsm_gen_sizes), each
filled with planted PY or C++ tests (tests/smell_ref.py, planted_file) cut to its size at a line end; and the worst case of the
duplicate search, one test of 20 000 assertion lines (10 000 distinct ones, then each again) (O(A^2 / 32) shuffles in one warp).  Reported:
the median whole-call time of Scanner.smells on the host clock (the call synchronises before it returns), the median device time
of each phase (tsm_smells_last_ms: k_scan, kinds + case spans, k_smell_lines, k_smell_tests), the counts, the serial C reference's
rate (tests/orc_smells.c, one host thread) on a sample of the corpus and on the worst case (its output must equal the GPU's, every
array), and the card's name and power limit.  Prints one
JSON line and, with --out, writes it there too."""
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
import orc_smells as ocs  # noqa: E402
import smell_ref as sr  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402

PHASES = ("k_scan", "kinds_spans", "k_smell_lines", "k_smell_tests")


def c4_smelly(seed, n_files):
    sizes = ts.gen_corpus(seed, n_files, size_law=1, pinned=False).len
    rng = random.Random(seed)
    pool = [(ext, sr.planted_file(rng, 40, ext)) for ext in [1, 3] * 256]
    files, exts = [], []
    for i, size in enumerate(sizes.tolist()):
        ext, text = pool[rng.randrange(len(pool))]
        data = text * (size // len(text) + 1)
        cut = data.rfind(b"\n", 0, size)
        files.append(data[:cut + 1])
        exts.append(ext)
    return files, np.array(exts, np.uint8)


def worst_case():
    body = b"".join(b"    assert x == %d\n" % i for i in range(10000))
    return [b"def test_worst():\n" + body + body], np.array([1], np.uint8)


def timed(sc, c):
    t0 = time.perf_counter()
    r = sc.smells(c, cap=c.cap)
    return r, 1e3 * (time.perf_counter() - t0), sc.smells_last_ms()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=5000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    files, exts = c4_smelly(0x7053454D1805, args.files)
    wf, we = worst_case()
    corp = {"c4": ts.pack(files, exts, pinned=True), "worst": ts.pack(wf, we, pinned=True)}
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    for c in corp.values():
        c.cap = None
        r = sc.smells(c)
        c.cap = max(len(r["line_smell"]), len(r["tests"]))
    res = {k: {"t": [], "ms": []} for k in corp}
    for step in range(args.warmup + args.steps):
        for k, c in corp.items():                          # alternating calls
            r, t, ms = timed(sc, c)
            res[k]["r"] = r
            if step >= args.warmup:
                res[k]["t"].append(t)
                res[k]["ms"].append(ms)
    sample = list(range(0, args.files, max(1, args.files // args.sample)))
    sc_ = ts.pack([files[i] for i in sample], exts[sample])
    t0 = time.perf_counter()
    ref = ocs.smells(sc_)
    ref_s = time.perf_counter() - t0
    ocs.assert_equal(sc.smells(sc_), ref)
    t0 = time.perf_counter()
    wref = ocs.smells(corp["worst"])
    wref_s = time.perf_counter() - t0
    ocs.assert_equal(res["worst"]["r"], wref)
    out = {"metric": "tsm_smells: C4-scale corpus of planted tests and the 20 000-assertion worst case, alternating calls", "unit": "ms",
           "steps": args.steps, "warmup": args.warmup, "gpu": card()}
    for k, c in corp.items():
        r = res[k]["r"]
        t = r["tests"]
        out[k] = {"files": c.n_files, "bytes": c.source_bytes, "lines": int(r["line_base"][-1]), "tests": len(t),
                  "tests_per_smell": {n: int((t["smells"] >> b & 1).sum()) for b, n in enumerate(ts.SMELLS)},
                  "max_assertions_in_a_test": int(t["n_assert"].max()) if len(t) else 0,
                  "ms_median": float(np.median(res[k]["t"])), "ms_min": float(min(res[k]["t"])),
                  "device_ms_median": dict(zip(PHASES, (float(x) for x in np.median(np.array(res[k]["ms"]), axis=0))))}
    out["c_reference"] = {"files": sc_.n_files, "bytes": sc_.source_bytes, "s": ref_s, "MB_per_s": sc_.source_bytes / ref_s / 1e6,
                          "worst_case_s": wref_s, "threads": 1, "equal_to_gpu": True}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    sc.close()


if __name__ == "__main__":
    main()
