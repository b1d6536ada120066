#!/usr/bin/env python3
"""Cost of the changed assertion lines (docs/SPEC.md section 8) on BASELINE config C5, one GPU:

    python tools/bench_diff_asserts.py [--pairs 50000] [--steps 20] [--warmup 5]

The resident diff step three ways, alternating step by step so that all three see the same clocks:
  plain    tsm_diff_resident with detail (what bench.py times for C5);
  counts   tsm_diff_resident_asserts with the [group][category] tables only (no event arrays);
  events   Scanner.diff_resident(asserts=True): tables and both event arrays, as the CLI and the Python host use it.
Each call synchronises before it returns, so a host clock around it is its whole time.  Also reported: the device time of
k_diff_small in each (tsm_diff_last_ms), and the card's name and power limit.  Prints one JSON line; writes nothing."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
import numpy as np  # noqa: E402
import tosemscan as ts  # noqa: E402


def card():
    try:
        f = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
        return {"name": f[0], "power_limit_w": float(f[1])}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=50000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    a, b = ts.gen_pairs(0x7053454D0005, args.pairs)          # the C5 pairs of bench.py
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    sc.diff_upload(a, b)
    n = a.n_files
    add, rem = np.zeros(n, np.int64), np.zeros(n, np.int64)
    det = np.zeros(n, ts.DIFF_DETAIL)
    ac, rc = np.zeros((1, ts.K), np.int64), np.zeros((1, ts.K), np.int64)

    def plain():
        return sc.diff_resident(True)

    def counts():
        r = ts._DiffAsserts(ts._p(ac), ts._p(rc), None, 0, 0, None, 0, 0)
        st = ts.lib().tsm_diff_resident_asserts(sc._ctx, ts._p(add), ts._p(rem), ts._p(det), C.byref(r), None)
        if st:
            raise ts.TsmError(st, "tsm_diff_resident_asserts")
        return r.n_aev, r.n_rev

    def events():
        return sc.diff_resident(asserts=True)

    modes = (("plain", plain), ("counts", counts), ("events", events))
    for _ in range(args.warmup):
        for _, fn in modes:
            fn()
    t = {m: [] for m, _ in modes}
    k = {m: [] for m, _ in modes}
    for _ in range(args.steps):
        for m, fn in modes:
            t0 = time.perf_counter()
            out = fn()
            t[m].append(1e3 * (time.perf_counter() - t0))
            k[m].append(sc.diff_last_ms()[1])
            if m == "events":
                last = out
    p_add, p_rem, p_det = plain()
    e_add, e_rem, e_det, e_ac, e_rc, aev, rev = last
    assert np.array_equal(p_add, e_add) and np.array_equal(p_rem, e_rem) and np.array_equal(p_det, e_det), "the diff changed"
    assert np.array_equal(e_ac, ac) and np.array_equal(e_rc, rc), "counts differ between the two calls"
    traced = e_det["added_assert"] >= 0
    assert len(aev) == int(e_ac.sum()) == int(e_det["added_assert"][traced].sum())
    assert len(rev) == int(e_rc.sum()) == int(e_det["removed_assert"][traced].sum())
    print(json.dumps({"metric": "C5 resident diff step with the changed assertion lines", "unit": "ms", "pairs": n,
                      "bytes": a.source_bytes + b.source_bytes, "steps": args.steps, "warmup": args.warmup,
                      "ms_median": {m: float(np.median(v)) for m, v in t.items()},
                      "ms_min": {m: float(min(v)) for m, v in t.items()},
                      "k_diff_small_ms_median": {m: float(np.median(v)) for m, v in k.items()},
                      "changed_assertion_lines": {"added": len(aev), "removed": len(rev)}, "gpu": card()}))
    sc.close()


if __name__ == "__main__":
    main()
