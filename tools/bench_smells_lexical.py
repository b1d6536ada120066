#!/usr/bin/env python3
"""Cost of the lexical test smells (docs/SPEC.md section 25) against the test smells alone (section 18), one GPU:

    python tools/bench_smells_lexical.py [--files 100000] [--steps 10] [--warmup 3] [--out F]

Three corpora, each timed with tsm_smells and tsm_smells_lexical in alternating calls: --files files of BASELINE config C4's size
law (seeded sizes from tsm_gen_sizes), each filled with planted PY or C++ tests (tests/lexsmell_ref.py, planted_file: every
section-25 rule) cut to its size at a line end; the worst case of the statement walk, one test of 20 000 assertion lines whose
calls all stay open (each walks LEX_STMT_LINES = 64 lines); and the worst case of the distinct-name count, one test of 20 000
distinct local names (O(n^2 / 32) shuffles in one warp).  Reported: the median whole-call time of each call on the host clock (the
calls synchronise before they return), the median device time of each phase (tsm_smells_last_ms / tsm_smells_lexical_last_ms),
the counts, whether the lexical call's section-18 outputs equal those of tsm_smells, and whether its outputs equal the plain-Python
reference on a sample of the corpus and on both worst cases; and the card's name and power limit.  Prints one JSON line and, with
--out, writes it there too."""
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
import lexsmell_ref as lr  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402

PHASES = ("k_scan", "kinds_spans", "k_smell_lines", "k_smell_tests")
LEX_PHASES = ("k_scan", "front", "k_lex_body_lines", "k_lex_tests")


def c4_planted(seed, n_files):
    sizes = ts.gen_corpus(seed, n_files, size_law=1, pinned=False).len
    rng = random.Random(seed)
    pool = [(ext, lr.planted_file(rng, 40, ext)) for ext in [1, 3] * 256]
    files, exts = [], []
    for size in sizes.tolist():
        ext, text = pool[rng.randrange(len(pool))]
        data = text * (size // len(text) + 1)
        cut = data.rfind(b"\n", 0, size)
        files.append(data[:cut + 1])
        exts.append(ext)
    return files, np.array(exts, np.uint8)


def open_calls():
    return [b"def test_open(self):\n" + b"    self.assertEqual(a, (\n" * 20000], np.array([1], np.uint8)


def many_locals():
    return [b"def test_locals():\n" + b"".join(b"    v%d = %d\n" % (i, i) for i in range(20000))], np.array([1], np.uint8)


def equal(a, b, keys):
    return all(np.array_equal(a[k], b[k]) for k in keys)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=300)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    files, exts = c4_planted(0x7053454D2505, args.files)
    src = {"c4": (files, exts), "open_calls": open_calls(), "many_locals": many_locals()}
    corp = {k: ts.pack(f, e, pinned=True) for k, (f, e) in src.items()}
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    caps = {}
    for k, c in corp.items():
        r = sc.smells_lexical(c)
        caps[k] = max(len(r["line_smell"]), len(r["tests"]))
    res = {k: {m: {"t": [], "ms": []} for m in ("smells", "lexical")} for k in corp}
    for step in range(args.warmup + args.steps):
        for k, c in corp.items():                          # alternating calls
            for m in ("smells", "lexical"):
                t0 = time.perf_counter()
                r = sc.smells(c, cap=caps[k]) if m == "smells" else sc.smells_lexical(c, cap=caps[k])
                t = 1e3 * (time.perf_counter() - t0)
                ms = sc.smells_last_ms() if m == "smells" else sc.smells_lexical_last_ms()
                res[k][m]["r"] = r
                if step >= args.warmup:
                    res[k][m]["t"].append(t)
                    res[k][m]["ms"].append(ms)
    out = {"metric": "tsm_smells vs tsm_smells_lexical: C4-scale planted corpus and two worst cases, alternating calls", "unit": "ms",
           "steps": args.steps, "warmup": args.warmup, "gpu": card()}
    for k, c in corp.items():
        s, x = res[k]["smells"]["r"], res[k]["lexical"]["r"]
        lex = x["lex"]
        out[k] = {"files": c.n_files, "bytes": c.source_bytes, "lines": int(x["line_base"][-1]), "tests": len(lex),
                  "tests_per_lexical_smell": {n: int((lex["smells"] >> b & 1).sum()) for b, n in enumerate(ts.LSMELLS)},
                  "section18_outputs_equal": equal(s, x, ("line_base", "line_smell", "tests"))}
        for m, ph in (("smells", PHASES), ("lexical", LEX_PHASES)):
            out[k][m] = {"ms_median": float(np.median(res[k][m]["t"])), "ms_min": float(min(res[k][m]["t"])),
                         "device_ms_median": dict(zip(ph, (float(v) for v in np.median(np.array(res[k][m]["ms"]), axis=0))))}
    sample = list(range(0, args.files, max(1, args.files // args.sample)))
    sf, se = [files[i] for i in sample], exts[sample]
    keys = ("line_base", "line_lsmell", "lex")
    out["reference_equal"] = {"c4_sample_files": len(sample),
                              "c4_sample": equal(sc.smells_lexical(ts.pack(sf, se)), lr.py_lexsmells(sf, se), keys),
                              "open_calls": equal(res["open_calls"]["lexical"]["r"], lr.py_lexsmells(*src["open_calls"]), keys),
                              "many_locals": equal(res["many_locals"]["lexical"]["r"], lr.py_lexsmells(*src["many_locals"]), keys)}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    sc.close()


if __name__ == "__main__":
    main()
