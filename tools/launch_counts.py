#!/usr/bin/env python3
"""tsm_last_launch_count, an output digest (sha256 of the returned arrays) and which phase times are zero after one call of
every pair and line-records entry point, plus the scan and reduce calls, on a fixed small input: 300 gen_pairs revision pairs,
two far-apart pairs that go to k_myers / k_myers_trace and two planted test files (cases, smells, a moved block).  The phase
times are every *_last_ms getter after the call, one character per entry: 0 for zero, + for non-zero.  Two builds of the
library that launch, compute and time the same phases print the same object.

    python tools/launch_counts.py [TREE]      (TREE: the repository whose build is used; default this one)"""
import hashlib
import json
import os
import sys

root = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(root, "tosem-2021-replication_b200"))
import numpy as np  # noqa: E402
import tosemscan as ts  # noqa: E402


def h(x):
    m = hashlib.sha256()
    for a in (x if isinstance(x, (tuple, list)) else [x]):
        m.update(np.ascontiguousarray(a).tobytes())
    return m.hexdigest()[:16]


def nl(b):
    return b.count(b"\n") + (1 if b and not b.endswith(b"\n") else 0)


po, pn = ts.gen_pairs(0x5EED0001, 300, lam=6.0, pinned=False)
ob = [po.file_bytes(i) for i in range(po.n_files)]
nb = [pn.file_bytes(i) for i in range(pn.n_files)]
ob.append(b"".join(b"o%d\n" % i for i in range(60)) + b"assert a == 1\n")
nb.append(b"".join(b"n%d\n" % i for i in range(50)) + b"assertEqual(b, 2)\n")
ob.append(b"head\n" * 10 + b"".join(b"m%d\n" % i for i in range(2500)) + b"tail\n")
nb.append(b"head\n" * 10 + b"x\n" + b"".join(b"m%d\n" % i for i in range(2500)) + b"y\ntail\n")
n = len(ob)
ext = [1] * n
A, B = ts.pack(ob, ext, [i % 3 for i in range(n)], 3), ts.pack(nb, ext, [(i + 1) % 3 for i in range(n)], 3)
# planted tests for the case, smell and move calls: a sleepy test with a duplicate assertion that loses it, a new print test,
# an edited assertion and a test that moves to the other file of its step
body = b"    x = compute_the_value(1, 2)\n    assert x == 3\n"
to = [b"import time\n\ndef test_sleepy():\n    time.sleep(1)\n    assert f(1) == 2\n    assert f(1) == 2\n\ndef test_moved():\n" + body,
      b"class T:\n    def test_kept(self):\n        self.assertEqual(g(), 1)\n"]
tn = [b"import time\n\ndef test_sleepy():\n    time.sleep(1)\n    assert f(1) == 2\n\ndef test_new():\n    print(1)\n",
      b"class T:\n    def test_kept(self):\n        self.assertEqual(g(), 2)\n    def test_moved():\n" + body]
AT, BT = ts.pack(ob + to, ext + [1, 1]), ts.pack(nb + tn, ext + [1, 1])
steps = [i * 16 // (n + 2) for i in range(n + 2)]            # moves: 16 steps of consecutive pairs, the same tag on both sides
AM, BM = ts.pack(ob + to, ext + [1, 1], steps, 16), ts.pack(nb + tn, ext + [1, 1], steps, 16)
s = ts.Scanner(0, 1 << 24, 4096, 16)
out = {}
TIMES = ("diff_last_ms", "similarity_last_ms", "clones_last_ms", "smells_last_ms", "diff_smells_last_ms", "assert_edits_last_ms",
         "moves_last_ms", "blame_last_ms")


def rec(name, res):
    ms = {t: "".join("+" if v else "0" for v in np.atleast_1d(getattr(s, t)())) for t in TIMES}
    out[name] = {"launches": s.last_launch_count(), "digest": h(res), "ms": ms}


c = ts.gen_corpus(0x5EED0002, 400, 1, n_groups=4, pinned=False)
r = s.scan(c, 3)
rec("scan", [r["stats"], r["group_counts"], r["assert_events"], r["header_events"]])
r = s.scan(c, 3 | ts.SCAN_REV_B)
rec("scan_rev_b", [r["stats"], r["group_counts"], r["assert_events"], r["header_events"]])
fl = (np.random.default_rng(1).random((500, 7)) < 0.3).astype(np.uint8)
rec("reduce", list(s.reduce(fl, np.arange(500) % 3, np.arange(500) % 41, 3, 41)))
rec("diff_pairs", list(s.diff_pairs(A, B)))
rec("diff_pairs_detail", list(s.diff_pairs(A, B, detail=True)))
rec("diff_pairs_asserts", list(s.diff_pairs(A, B, asserts=True)))
s.diff_upload(A, B)
rec("diff_resident", [x.copy() for x in s.diff_resident(detail=False)])
rec("diff_resident_detail", [x.copy() for x in s.diff_resident(detail=True)])
rec("diff_resident_asserts", [x.copy() for x in s.diff_resident(asserts=True)])
rec("diff_marks", list(s.diff_marks(A, B)))
prev = [-1] * n + [0]
heads = {i: np.array([(-1, j + 1) for j in range(nl(ob[i]))], ts.ORIGIN) for i in range(n)}
rec("blame_pairs", list(s.blame_pairs(ts.pack(ob + [nb[0]], ext + [1]), ts.pack(nb + [ob[0]], ext + [1]), prev,
                                      list(range(n + 1)), heads)))
co = np.array(list(range(n)) + list(range(n - 1)), np.int32)
cn = np.array(list(range(n)) + list(range(1, n)), np.int32)
rec("similarity", s.similarity(A, ts.pack(nb + [b"z\n"], ext + [1]), co, cn))
cl = s.clones(ts.pack(ob + nb, ext + ext), 3)
rec("clones", [cl[k] for k in ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len", "member")])
rec("line_hashes", list(s.line_hashes(A, ngram=3)))
rec("statements", list(s.statements(A)))
rec("diff_cases", list(s.diff_cases(AT, BT)))
rec("diff_assert_edits", list(s.diff_assert_edits(AT, BT)))
r = s.smells(AT)
rec("smells", [r["line_base"], r["line_smell"], r["tests"]])
r = s.diff_smells(AT, BT)
rec("diff_smells", [r[k] for k in sorted(r)])
r = s.diff_moves(AM, BM)
rec("diff_moves", [r[k] for k in sorted(r)])
s.close()
print(json.dumps(out, sort_keys=True))
