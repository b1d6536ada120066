#!/usr/bin/env python3
"""tsm_last_launch_count and an output digest (sha256 of the returned arrays) after one call of every pair and line-records
entry point, plus the scan and reduce calls, on a fixed small input: 300 gen_pairs revision pairs and two far-apart pairs
that go to k_myers / k_myers_trace.  Two builds of the library that launch and compute the same print the same object.

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
s = ts.Scanner(0, 1 << 24, 4096, 16)
out = {}


def rec(name, res):
    out[name] = {"launches": s.last_launch_count(), "digest": h(res)}


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
s.close()
print(json.dumps(out, sort_keys=True))
