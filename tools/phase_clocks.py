#!/usr/bin/env python3
"""Where the cycles of k_scan go: run C2 (law 0) or C4 (law 1) on a build with -DTSM_PHASE_CLOCKS=1 and print each
phase's share of the cycles in the chunk loop (summed over every warp of 20 resident scans).
  cd tosem-2021-replication_b200 && mkdir -p build_variants
  make VARIANT=-DTSM_PHASE_CLOCKS=1 OUT=build_variants/clocks.so build_variants/clocks.so
  TOSEMSCAN_LIB=$PWD/build_variants/clocks.so python ../tools/phase_clocks.py [files] [law]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
import tosemscan as ts

PHASES = ["wait (bulk copy)", "zero fill", "walk", "tail/entry scans", "mixed words", "line records", "finish",
          "long-line slow path", "per-file flush"]

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
law = int(sys.argv[2]) if len(sys.argv) > 2 else 0
L = ts.lib()
if not hasattr(L, "tsm_phase_clocks"):
    sys.exit("phase_clocks.py: %s was not built with -DTSM_PHASE_CLOCKS=1" % ts.LIB_PATH)
L.tsm_phase_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
buf = (C.c_ulonglong * len(PHASES))()
c = ts.gen_corpus(0x7053454D0002 if law == 0 else 0x7053454D0004, n, law, 4096, n_groups=9)
sc = ts.Scanner(0, int(c.off[-1]) + 4096, n, 16)
sc.upload(c)
for _ in range(3):
    sc.scan_resident(0)
assert L.tsm_phase_clocks(buf, len(PHASES), 1) == 0
for _ in range(20):
    sc.scan_resident(0)
assert L.tsm_phase_clocks(buf, len(PHASES), 1) == 0
tot = sum(buf)
print("k_scan phases, %s, %d files, %s: %.3g warp-cycles in the chunk loop" % (
    "C2" if law == 0 else "C4", n, os.path.basename(ts.LIB_PATH), tot))
for name, v in zip(PHASES, buf):
    print("  %-22s %6.2f %%" % (name, 100.0 * v / tot))
