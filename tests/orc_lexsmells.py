"""Serial C reference of the lexical test smells of docs/SPEC.md section 25.  TEST INFRASTRUCTURE ONLY.

`lexsmells(corpus)`: ctypes binding of tests/orc_lexsmells.c (compiled together with tests/orc_blind.c, tests/orc_smells.c and the
oracle's orc.c into a library in the temporary directory, so that the tests never write into the tree).  Returns line_base,
line_lsmell and lex, the arrays of `tosemscan.Scanner.smells_lexical` that section 25 adds.
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
SRCS = [os.path.join(HERE, "orc_lexsmells.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(HERE, "orc_blind.c"), os.path.join(HERE, "orc_smells.c"), os.path.join(orc.ORC_DIR, "orc.h"),
               os.path.join(orc.ORC_DIR, "orc_categories.inc")]
LEX_TEST = np.dtype([("n_stmts", "<i4"), ("n_unexplained", "<i4"), ("n_magic", "<i4"), ("n_locals", "<i4"), ("smells", "<u4"),
                     ("n_instances", "<i4")])          # the layout of tsm_lex_test

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_lexsmells_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-I", HERE, "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_lexsmells.restype = C.c_int
            L.orc_lexsmells.argtypes = [C.c_void_p] * 4 + [C.c_int32] + [C.c_void_p] * 2 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                                                                            C.c_void_p]
            _lib = L
    return _lib


def lexsmells(corpus):
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
        lsm = np.zeros(max(cl, 1), np.uint8)
        lex = np.zeros(max(ct, 1), LEX_TEST)
        nl, nt = C.c_int64(), C.c_int64()
        rc = lib().orc_lexsmells(p(arena), p(off), p(length), p(ext), nf, p(base), p(lsm), cl, C.byref(nl), p(lex), ct, C.byref(nt))
        if rc == -3:
            cl, ct = nl.value, nt.value
            continue
        if rc != 0:
            raise ValueError("orc_lexsmells failed")
        return {"line_base": base, "line_lsmell": lsm[:nl.value], "lex": lex[:nt.value]}
    raise ValueError("orc_lexsmells: capacity")


def assert_equal(got, want):
    """line_base, line_lsmell and lex of two results are equal (the first differing rows in the message)."""
    for k in ("line_base", "line_lsmell", "lex"):
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.shape == b.shape, "%s: %s vs %s" % (k, a.shape, b.shape)
        if k == "lex":
            a, b = a.view(np.int32).reshape(-1, 6), b.view(np.int32).reshape(-1, 6)
        bad = np.nonzero((a != b).reshape(len(a), -1).any(1))[0] if len(a) else []
        assert len(bad) == 0, "%s differs first at %s: %s vs %s" % (k, bad[:3], a[bad[:3]], b[bad[:3]])
