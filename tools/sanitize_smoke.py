#!/usr/bin/env python3
"""Small scan (Rev A and Rev B) + line records + diff (plain, assertion lines, marks, provenance, test cases, assertion edits,
smell churn, moved code) + similarity + clones + smells + statements + reduce under compute-sanitizer (run: compute-sanitizer
--tool memcheck python tools/sanitize_smoke.py)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import corpus_util as cu
import tosemscan as ts

s = ts.Scanner(0, 1 << 24, 4096, 16)
files, exts, grps = cu.edge_corpus()
r = s.scan(ts.pack(files, exts, grps, 3), 3)
files, exts, grps = cu.fuzz_corpus(5, 120, 30000, long_lines=True)
r2 = s.scan(ts.pack(files, exts, grps, 5), 3)
c = ts.gen_corpus(3, 300, 1, n_groups=4, pinned=False)
r3 = s.scan(c, 0)
a = ts.pack([b"a\nb\nc\n", b"x\n" * 50, b""], [1, 1, 1])
b = ts.pack([b"a\nc\nd\n", b"y\n" * 40, b"q\n"], [1, 1, 1])
print(s.diff_pairs(a, b, detail=True))
far_o = [b"".join(b"o%d\n" % i for i in range(60)), b"head\n" * 10 + b"".join(b"m%d\n" % i for i in range(2500)) + b"tail\n"]
far_n = [b"".join(b"n%d\n" % i for i in range(50)), b"head\n" * 10 + b"x\n" + b"".join(b"m%d\n" % i for i in range(2500)) + b"y\ntail\n"]
print(s.diff_pairs(ts.pack(far_o, [1, 1]), ts.pack(far_n, [1, 1]), detail=True))   # the left-over path: D > 31, middle > 4 096 lines
# the pair calls with their own scratch: changed assertion lines, edit marks, provenance and rename similarity, each also
# over the far pair so that the EMIT and MARKS variants of the left-over kernels run
far_o[0] += b"assert x == 1\n"; far_n[0] += b"assertEqual(y, 2)\n"
fo, fn = ts.pack(far_o, [1, 1], [0, 1], 2), ts.pack(far_n, [1, 1], [1, 0], 2)
print([x.sum() for x in s.diff_pairs(fo, fn, asserts=True)[3:5]])
print([int(x.sum()) for x in s.diff_marks(fo, fn)[5:]])
lines0 = far_o[0].count(b"\n")
g = s.blame_pairs(ts.pack([far_o[0], far_n[0]], [1, 1]), ts.pack([far_n[0], far_o[0]], [1, 1]), [-1, 0], [1, 2],
                  {0: np.array([(-1, j + 1) for j in range(lines0)], ts.ORIGIN)})
print(len(g[4]), g[4][:3])
print(s.similarity(fo, ts.pack(far_n + [b"m1\nm2\n"], [1, 1, 1]), [0, 1, 1], [0, 1, 2]))
# the case, assertion-edit, smell and move calls over the far pair and a test file with cases, smells, an edited assertion
# and a block that moves between the files of its step
body = b"    x = compute_the_value(1, 2)\n    assert x == 3\n"
to = [far_o[0], b"import time\n\ndef test_a():\n    time.sleep(1)\n    assert f(1) == 2\n    assert f(1) == 2\n\ndef test_m():\n" + body]
tn = [far_n[0] + b"def test_m():\n" + body, b"import time\n\ndef test_a():\n    time.sleep(1)\n    assert f(1) == 3\n"]
to_, tn_ = ts.pack(to, [1, 1], [0, 0], 1), ts.pack(tn, [1, 1], [0, 0], 1)
print([len(x) for x in s.diff_cases(to_, tn_)[3:]])
print(len(s.diff_assert_edits(to_, tn_)[7]))
print(len(s.smells(to_)["tests"]))
print({k: len(v) for k, v in s.diff_smells(to_, tn_).items()})
mv = s.diff_moves(to_, tn_)
print(len(mv["old_blocks"]), len(mv["new_blocks"]))
lic = b"".join(b"# licence %d\n" % i for i in range(8))    # clone classes: warp-sorted, CTA-sorted and tiled (> 4 096 fragments)
cl = s.clones(ts.pack(far_o + far_n + [lic + (b"x\n" if i % 50 else b"") + b"f%d\n" % i for i in range(4200)], [1] * 4204), 3)
print(len(cl["class_len"]), int(cl["file_dup"].sum()), int(cl["class_len"].max()))
print([x[:4] for x in s.line_hashes(ts.pack(files[:40], exts[:40]), ngram=3)])
r4 = s.scan(ts.pack(files, exts, grps, 5), 3 | ts.SCAN_REV_B)
print(s.statements(c)[0][-1])
fl = (np.random.default_rng(1).random((500, 7)) < 0.3).astype(np.uint8)
print(s.reduce(fl, np.arange(500) % 3, np.arange(500) % 41, 3, 41)[1])
big = ts.gen_corpus(9, 9000, 0, 4096, n_groups=2)           # 37 MB through the host path: two slabs, classified slab by slab
s2 = ts.Scanner(0, int(big.off[-1]) + 4096, big.n_files, 2)
r5 = s2.scan(big, 0, reuse=True)
print("streamed", r5["totals"], int(r5["global_counts"].sum()))
print("totals", r["totals"], r2["totals"], r3["totals"])
