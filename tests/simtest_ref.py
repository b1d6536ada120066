"""References of the similar tests of docs/SPEC.md section 23.  TEST INFRASTRUCTURE ONLY.

* `py_sequences(files, exts)`: the plain-Python restatement of the tests and their sequences: tests and bodies from
  `smell_ref.py_file_smells`, kept lines and blind hashes from `blind_ref.blind_lines`;
* `c_sequences(corpus)`: the same from the serial C references (`orc_smells`, `orc_blind`), for corpora at scale;
* `py_similar(seqs, min_lines, P)`: every pair by brute force with an O(nm) LCS table, no filter at all;
* `c_similar(seqs, min_lines, P)`: the serial C brute force of tests/orc_simtest.c (only the exact size filter);
* `prefix_candidates(seqs, min_lines, P)`: a model of the device's exact prefix filter (tokens, rare-first order, prefixes,
  posting lists, the first-common-token rule), which must keep every pair that passes;
* `classes(pairs, nt)`: single-linkage classes by a union-find;
* `reference(corpus, min_lines, P)`: the dict of `tosemscan.Scanner.similar_tests` from the C references.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import threading
from collections import Counter, defaultdict

import numpy as np

import blind_ref as br
import orc
import orc_blind
import orc_smells
import smell_ref

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_simtest.c")
_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(open(SRC, "rb").read()).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_simtest_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-o", tmp, SRC])
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_similar.restype = C.c_int
            L.orc_similar.argtypes = [C.c_void_p] * 3 + [C.c_int32] * 3 + [C.c_void_p] * 3 + [C.c_int64, C.c_void_p]
            L.orc_similar_row.restype = C.c_int64
            L.orc_similar_row.argtypes = [C.c_void_p] * 3 + [C.c_int32] * 4 + [C.c_void_p, C.c_int64]
            _lib = L
    return _lib


def py_sequences(files, exts):
    """(tests, seqs): tests as (file, header line, body_lines) in global line order, seqs[t] the blind hashes of t's kept lines."""
    tests, seqs = [], []
    for f, (data, ext) in enumerate(zip(files, exts)):
        forms = br.blind_lines(data, int(ext))
        for b, n, *_ in smell_ref.py_file_smells(data, int(ext))[0]:
            tests.append((f, b, n))
            seqs.append([br.blind_hash(x) for x in forms[b:b + n] if x])
    return tests, seqs


def c_sequences(corpus):
    """(SMELL_TEST records, seqs) from the C references."""
    tests = orc_smells.smells(corpus)["tests"]
    base, kept, bhash, _ = orc_blind.blind_lines(corpus)
    seqs = []
    for t in tests:
        l0 = int(base[t["file"]]) + int(t["line"])
        sl = slice(l0, l0 + int(t["body_lines"]))
        seqs.append(bhash[sl][kept[sl]].tolist())
    return tests, seqs


def lcs(a, b):
    prev = [0] * (len(b) + 1)
    for x in a:
        cur = [0]
        for j, y in enumerate(b):
            cur.append(prev[j] + 1 if x == y else max(prev[j + 1], cur[j]))
        prev = cur
    return prev[-1]


def passes(l, ka, kb, P):
    return 200 * l >= P * (ka + kb)


def score(l, ka, kb):
    return 120000 * l // (ka + kb)


def py_similar(seqs, min_lines, P):
    """[(a, b, lcs, score)] over every pair of compared tests, ascending."""
    out = []
    for a in range(len(seqs)):
        if len(seqs[a]) < min_lines:
            continue
        for b in range(a + 1, len(seqs)):
            if len(seqs[b]) < min_lines:
                continue
            l = lcs(seqs[a], seqs[b])
            if passes(l, len(seqs[a]), len(seqs[b]), P):
                out.append((a, b, l, score(l, len(seqs[a]), len(seqs[b]))))
    return out


def c_similar(seqs, min_lines, P):
    k = np.array([len(s) for s in seqs], np.uint32)
    beg = np.concatenate([[0], np.cumsum(k, dtype=np.int64)]).astype(np.int64)
    flat = np.array([h for s in seqs for h in s], np.uint64)
    if flat.size == 0:
        flat = np.zeros(1, np.uint64)
    p = orc._p
    cap = 1 << 16
    for _ in range(2):
        pa, pb, pl = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.uint32)
        n = C.c_int64()
        rc = lib().orc_similar(p(flat), p(beg), p(k), len(seqs), int(min_lines), int(P), p(pa), p(pb), p(pl), cap, C.byref(n))
        if rc == -3:
            cap = n.value
            continue
        if rc:
            raise ValueError("orc_similar failed")
        n = n.value
        return [(int(a), int(b), int(l), score(int(l), int(k[a]), int(k[b]))) for a, b, l in zip(pa[:n], pb[:n], pl[:n])]
    raise ValueError("orc_similar: capacity")


def c_partners(seqs, a, min_lines, P):
    """The tests that pair with test a, by brute force over the whole corpus (ascending)."""
    k = np.array([len(s) for s in seqs], np.uint32)
    beg = np.concatenate([[0], np.cumsum(k, dtype=np.int64)]).astype(np.int64)
    flat = np.array([h for s in seqs for h in s] or [0], np.uint64)
    other = np.zeros(len(seqs), np.int32)
    n = lib().orc_similar_row(orc._p(flat), orc._p(beg), orc._p(k), len(seqs), int(a), int(min_lines), int(P), orc._p(other), len(seqs))
    if n < 0:
        raise ValueError("orc_similar_row failed")
    return other[:n].tolist()


def tokens(seq):
    seen = Counter()
    out = []
    for h in seq:
        out.append((h, seen[h]))
        seen[h] += 1
    return out


def prefix_candidates(seqs, min_lines, P):
    """The candidate pairs of the device's filter: each compared test's tokens (h, j) in the order (count of h over the compared
    tests, h, j), its prefix of k - ceil(P k / (200 - P)) + 1 tokens, the posting lists of prefix tokens, and per list every pair
    that passes the size filter and whose first common prefix token is the list's token."""
    cmp = [t for t, s in enumerate(seqs) if len(s) >= min_lines]
    cnt = Counter(h for t in cmp for h in seqs[t])
    order = lambda tok: (cnt[tok[0]], tok[0], tok[1])
    pref, lists = {}, defaultdict(list)
    for t in cmp:
        k = len(seqs[t])
        alpha = -(-P * k // (200 - P))
        pref[t] = sorted(tokens(seqs[t]), key=order)[:k - alpha + 1]
        for tok in pref[t]:
            lists[tok].append(t)
    out = set()
    for tok, mem in lists.items():
        for i in range(len(mem)):
            for j in range(i + 1, len(mem)):
                a, b = min(mem[i], mem[j]), max(mem[i], mem[j])
                ka, kb = len(seqs[a]), len(seqs[b])
                if 200 * min(ka, kb) < P * (ka + kb):
                    continue
                pb = set(pref[b])
                first = next(x for x in pref[a] if x in pb)
                if first == tok:
                    assert (a, b) not in out
                    out.add((a, b))
    return out


def classes(pairs, nt):
    """(class_base, member): the components of at least two tests, by smallest member, members ascending."""
    root = list(range(nt))

    def find(x):
        while root[x] != x:
            root[x] = root[root[x]]
            x = root[x]
        return x
    linked = set()
    for a, b, *_ in pairs:
        ra, rb = find(a), find(b)
        root[max(ra, rb)] = min(ra, rb)
        linked.update((a, b))
    groups = defaultdict(list)
    for t in sorted(linked):
        groups[find(t)].append(t)
    base, member = [0], []
    for r in sorted(groups):
        member += groups[r]
        base.append(len(member))
    return np.array(base, np.int64), np.array(member, np.int32)


def reference(corpus, min_lines, P):
    tests, seqs = c_sequences(corpus)
    pairs = c_similar(seqs, min_lines, P)
    base, member = classes(pairs, len(seqs))
    return {"tests": tests, "test_kept": np.array([len(s) for s in seqs], np.uint32),
            "pairs": np.array(pairs, [("a", "<i4"), ("b", "<i4"), ("lcs", "<u4"), ("score", "<u4")]),
            "class_base": base, "member": member}


def assert_equal(got, want):
    for key in ("tests", "test_kept", "pairs", "class_base", "member"):
        g, w = got[key], want[key]
        assert len(g) == len(w), (key, len(g), len(w))
        assert np.array_equal(g.view(np.uint8) if g.dtype.names else g, np.asarray(w, g.dtype).view(np.uint8) if g.dtype.names else w), key
