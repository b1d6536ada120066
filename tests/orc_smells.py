"""Serial C reference of the test smells of docs/SPEC.md section 18.  TEST INFRASTRUCTURE ONLY.

`smells(corpus)`: ctypes binding of tests/orc_smells.c (compiled together with the oracle's orc.c, for the header rule, the
assertion rule and the line hash, into a library in the temporary directory, so that the tests never write into the tree).
Returns the dict of `tosemscan.Scanner.smells`: line_base[n_files+1], line_smell[lines] and tests[n_tests] (SMELL_TEST records).
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import threading

import numpy as np

import orc

HERE = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(HERE, "orc_smells.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(orc.ORC_DIR, "orc.h"), os.path.join(orc.ORC_DIR, "orc_categories.inc")]
SMELL_TEST = np.dtype([("file", "<i4"), ("line", "<i4"), ("body_lines", "<i4"), ("n_assert", "<i4"), ("smells", "<u4"),
                       ("n_instances", "<i4")])        # the layout of tsm_smell_test

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_smells_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_smells.restype = C.c_int
            L.orc_smells.argtypes = [C.c_void_p] * 4 + [C.c_int32] + [C.c_void_p] * 2 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                                                                         C.c_void_p]
            _lib = L
    return _lib


def smells(corpus):
    """corpus: tosemscan.Corpus (or anything with arena, off, len, ext)."""
    arena = np.ascontiguousarray(corpus.arena, np.uint8)
    off = np.ascontiguousarray(corpus.off, np.int32)
    length = np.ascontiguousarray(corpus.len, np.int32)
    ext = np.ascontiguousarray(corpus.ext, np.uint8)
    nf = len(length)
    p = orc._p
    cl = ct = 0
    for _ in range(2):
        base = np.zeros(nf + 1, np.int64)
        smell = np.zeros(max(cl, 1), np.uint16)
        tests = np.zeros(max(ct, 1), SMELL_TEST)
        nl, nt = C.c_int64(), C.c_int64()
        rc = lib().orc_smells(p(arena), p(off), p(length), p(ext), nf, p(base), p(smell), cl, C.byref(nl), p(tests), ct, C.byref(nt))
        if rc == -3:
            cl, ct = nl.value, nt.value
            continue
        if rc != 0:
            raise ValueError("orc_smells failed")
        return {"line_base": base, "line_smell": smell[:nl.value], "tests": tests[:nt.value]}
    raise ValueError("orc_smells: capacity")


def assert_equal(got, want):
    """Every output array of two smell results is equal."""
    for k in ("line_base", "line_smell", "tests"):
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.shape == b.shape, "%s: %s vs %s" % (k, a.shape, b.shape)
        if k == "tests":
            a, b = a.view(np.int32).reshape(-1, 6), b.view(np.int32).reshape(-1, 6)
        bad = np.nonzero((a != b).reshape(len(a), -1).any(1))[0] if len(a) else []
        assert len(bad) == 0, "%s differs first at %s: %s vs %s" % (k, bad[:3], a[bad[:3]], b[bad[:3]])


def as_python(files, exts):
    """smell_ref.py_smells in the same dict form (with its line_base from the line counts)."""
    import smell_ref as sr
    tests, smell = sr.py_smells(files, exts)
    t = np.zeros(len(tests), SMELL_TEST)
    for i, r in enumerate(tests):
        t[i] = r
    base = np.cumsum([0] + [len(sr.py_lines(f)) for f in files]).astype(np.int64)
    return {"line_base": base, "line_smell": np.array(smell, np.uint16), "tests": t}
