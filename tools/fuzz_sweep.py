#!/usr/bin/env python3
"""Extended differential fuzz of the scan against the oracle (GPU box): python tools/fuzz_sweep.py [first_seed] [n_seeds]."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import corpus_util as cu
import orc
import tosemscan as ts

first = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
n = int(sys.argv[2]) if len(sys.argv) > 2 else 40
sc = ts.Scanner(0, 1 << 28, 1 << 16, 16)
FLAGS = ts.SCAN_ASSERT_EVENTS | ts.SCAN_HEADER_EVENTS
bad = 0
for seed in range(first, first + n):
    small = seed % 2 == 0
    binary = seed % 4 >= 2                                 # every other pair of seeds: all 256 byte values, CR-heavy
    files, exts, grps = cu.fuzz_corpus(seed, 500 if small else 120, 3000 if small else 70000, long_lines=not small, binary=binary)
    c = ts.pack(files, exts, grps, 5)
    want = orc.scan(c.arena, c.off, c.len, c.ext, c.grp, c.n_groups)
    got = sc.scan(c, FLAGS)
    ok = all(np.array_equal(got["stats"][f], want["stats"][f]) for f in ("n_lines", "n_assert", "n_headers", "n_fixture", "digest"))
    ok &= np.array_equal(got["group_counts"], want["group_counts"]) and np.array_equal(got["global_counts"], want["global_counts"])
    ok &= len(got["assert_events"]) == len(want["assert_events"]) and all(
        np.array_equal(got["assert_events"][f], want["assert_events"][f]) for f in got["assert_events"].dtype.names)
    ok &= np.array_equal(got["header_events"], want["header_events"])
    if not ok:
        bad += 1
        print("MISMATCH seed", seed)
print("fuzz sweep: %d seeds from %d, %d mismatches" % (n, first, bad))
sys.exit(1 if bad else 0)
