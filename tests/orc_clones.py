"""References of the clone classes of docs/SPEC.md section 15.  TEST INFRASTRUCTURE ONLY.

* `clones(corpus, n)`: ctypes binding of tests/orc_clones.c (compiled together with the oracle's orc.c, for the line and
  n-gram hashes, into a library in the temporary directory, so that the tests never write into the tree).
* `py_clones(files, exts, n)`: the same definition in plain Python over line contents (windows are equal when their n
  contents are equal), independent of the hash.
Both return the dict of `tosemscan.Scanner.clones`.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import threading

import numpy as np

import orc
import spec_ref

HERE = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(HERE, "orc_clones.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(orc.ORC_DIR, "orc.h"), os.path.join(orc.ORC_DIR, "orc_categories.inc")]

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_clones_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_clones.restype = C.c_int
            L.orc_clones.argtypes = [C.c_void_p] * 4 + [C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int64, C.c_void_p, C.c_void_p,
                                                                                                    C.c_int64, C.c_void_p]
            _lib = L
    return _lib


def clones(corpus, n):
    """corpus: tosemscan.Corpus (or anything with arena, off, len, ext)."""
    arena = np.ascontiguousarray(corpus.arena, np.uint8)
    off = np.ascontiguousarray(corpus.off, np.int32)
    length = np.ascontiguousarray(corpus.len, np.int32)
    ext = np.ascontiguousarray(corpus.ext, np.uint8)
    nf = len(length)
    p = orc._p
    cap = 0
    for _ in range(2):
        out = {"line_base": np.zeros(nf + 1, np.int64), "file_dup": np.zeros(max(nf, 1), np.uint32),
               "file_dup_assert": np.zeros(max(nf, 1), np.uint32), "class_base": np.zeros(cap + 1, np.int64),
               "class_len": np.zeros(max(cap, 1), np.uint32), "member": np.zeros(max(cap, 1), np.int64)}
        nc, nm = C.c_int64(), C.c_int64()
        rc = lib().orc_clones(p(arena), p(off), p(length), p(ext), nf, int(n), p(out["line_base"]), p(out["file_dup"]),
                              p(out["file_dup_assert"]), p(out["class_base"]), p(out["class_len"]), cap, C.byref(nc),
                              p(out["member"]), cap, C.byref(nm))
        if rc == -3:
            cap = max(nc.value, nm.value)
            continue
        if rc != 0:
            raise ValueError("orc_clones failed")
        out["file_dup"], out["file_dup_assert"] = out["file_dup"][:nf], out["file_dup_assert"][:nf]
        out["class_base"], out["class_len"], out["member"] = out["class_base"][:nc.value + 1], out["class_len"][:nc.value], out["member"][:nm.value]
        return out
    raise ValueError("orc_clones: capacity")


def py_clones(files, exts, n):
    """Section 15 over line contents (the line minus one trailing CR)."""
    content, flag, fid, base = [], [], [], [0]
    for f, (data, e) in enumerate(zip(files, exts)):
        for line in spec_ref.py_lines(data):
            content.append(line[:-1] if line.endswith(b"\r") else line)
            flag.append(spec_ref.py_is_assert_line(line, int(e)))
            fid.append(f)
        base.append(len(content))
    T = len(content)
    groups = {}                                              # window contents -> positions, ascending
    key = [None] * T
    for p in range(T):
        if p + n > base[fid[p] + 1] or all(not c for c in content[p:p + n]):
            continue
        key[p] = tuple(content[p:p + n])
        groups.setdefault(key[p], []).append(p)

    def ext_of(g):                                          # left-extendable
        preds = set()
        for q in g:
            if q == base[fid[q]] or key[q - 1] is None:
                return False
            preds.add(key[q - 1])
        return len(preds) == 1 and len(groups[preds.pop()]) == len(g)

    extendable = {k: len(g) >= 2 and ext_of(g) for k, g in groups.items()}
    covered = [False] * T
    class_base, class_len, member = [0], [], []
    for p in range(T):
        k = key[p]
        if k is None or len(groups[k]) < 2:
            continue
        for x in range(p, p + n):
            covered[x] = True
        if extendable[k] or groups[k][0] != p:
            continue
        r = 0
        while p + r + 1 < T and fid[p + r + 1] == fid[p] and key[p + r + 1] is not None and len(groups[key[p + r + 1]]) >= 2 \
                and extendable[key[p + r + 1]]:
            r += 1
        class_len.append(n + r)
        member += groups[k]
        class_base.append(len(member))
    nf = len(files)
    dup = [sum(covered[base[f]:base[f + 1]]) for f in range(nf)]
    dup_a = [sum(1 for x in range(base[f], base[f + 1]) if covered[x] and flag[x]) for f in range(nf)]
    return {"line_base": np.array(base, np.int64), "file_dup": np.array(dup, np.uint32), "file_dup_assert": np.array(dup_a, np.uint32),
            "class_base": np.array(class_base, np.int64), "class_len": np.array(class_len, np.uint32), "member": np.array(member, np.int64)}


KEYS = ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len", "member")


def assert_equal(got, want):
    for k in KEYS:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k


def c4_planted(seed, n_files, share=4):
    """Files of BASELINE config C4's size law (seeded), every `share`-th of them replaced by tsm_gen_edit (lambda = 6) of
    another, earlier file of the corpus: planted partial copies at a realistic scale.  Returns (files, exts)."""
    import tosemscan as ts
    c = ts.gen_corpus(seed, n_files, size_law=1, pinned=False)
    files = [c.file_bytes(i) for i in range(n_files)]
    rng = np.random.default_rng(seed)
    for i in range(share, n_files, share):
        files[i] = ts.gen_edit(seed + i, files[int(rng.integers(0, i))], 6.0)
    return files, c.ext.copy()
