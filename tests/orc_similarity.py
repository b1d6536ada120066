"""References of the rename similarity of docs/SPEC.md section 13.  TEST INFRASTRUCTURE ONLY.

* `similarity(old, new, cand_old, cand_new)`: ctypes binding of tests/orc_similarity.c (compiled together with the oracle's
  orc.c, for orc_line_hash, into a library in the temporary directory, so that the tests never write into the tree).
* `py_similarity(a, b)`: the same rule in plain Python on two byte strings, with the line hash of tests/spec_ref.py.
* `git_score(common, size_a, size_b)`: git's MAX_SCORE scale, and `similarity_percent` the number git prints after `R`.
"""
import collections
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
SRCS = [os.path.join(HERE, "orc_similarity.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(orc.ORC_DIR, "orc.h"), os.path.join(orc.ORC_DIR, "orc_categories.inc")]
MAX_SCORE = 60000

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_similarity_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_similarity.restype = C.c_int
            L.orc_similarity.argtypes = [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 3 + [C.c_int32] + \
                [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
            _lib = L
    return _lib


def similarity(old, new, cand_old, cand_new):
    """old/new: tosemscan.Corpus (or anything with arena, off, len).  Returns np.int64[n_cand]."""
    co = np.ascontiguousarray(cand_old, np.int32).ravel()
    cn = np.ascontiguousarray(cand_new, np.int32).ravel()
    out = np.zeros(max(co.size, 1), np.int64)
    p = orc._p
    sides = []
    for s in (old, new):
        sides += [np.ascontiguousarray(s.arena, np.uint8), np.ascontiguousarray(s.off, np.int32), np.ascontiguousarray(s.len, np.int32)]
    rc = lib().orc_similarity(p(sides[0]), p(sides[1]), p(sides[2]), len(sides[2]), p(sides[3]), p(sides[4]), p(sides[5]),
                              len(sides[5]), p(co), p(cn), co.size, p(out))
    if rc != 0:
        raise ValueError("orc_similarity failed")
    return out[:co.size]


def line_weights(data: bytes):
    """{line hash: total weight} of one file: a line weighs its bytes, plus 1 for its LF, minus 1 for the CR of a CRLF."""
    out = collections.Counter()
    lines = data.split(b"\n")
    for k, line in enumerate(lines):
        has_lf = k + 1 < len(lines)
        if not has_lf and not line:
            break
        w = len(line) + (1 if has_lf else 0) - (1 if has_lf and line.endswith(b"\r") else 0)
        out[spec_ref.py_bytes_hash(line[:-1] if line.endswith(b"\r") else line)] += w
    return out


def py_similarity(a: bytes, b: bytes) -> int:
    wa, wb = line_weights(a), line_weights(b)
    return sum(min(w, wb[h]) for h, w in wa.items() if h in wb)


def git_score(common, size_a, size_b):
    m = max(size_a, size_b)
    return common * MAX_SCORE // m if m else MAX_SCORE


def similarity_percent(common, size_a, size_b):
    return git_score(common, size_a, size_b) // 600
