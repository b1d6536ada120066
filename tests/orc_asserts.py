"""ctypes binding of the CPU reference of the changed assertion lines (tests/orc_diff_asserts.c).  TEST INFRASTRUCTURE ONLY.

The C file is compiled together with the oracle (oracle/orc.c, whose orc_scan builds the events) into a library in the
temporary directory, so that the tests never write into the tree.
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
SRCS = [os.path.join(HERE, "orc_diff_asserts.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(orc.ORC_DIR, "orc.h"), os.path.join(orc.ORC_DIR, "orc_categories.inc")]

_lib = None
_lock = threading.Lock()                  # the first call may come from several threads at once


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_asserts_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_diff_pairs_asserts.restype = C.c_int
            L.orc_diff_pairs_asserts.argtypes = [C.c_void_p] * 10 + [C.c_int32, C.c_int32] + [C.c_void_p] * 2 + \
                [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
            _lib = L
    return _lib


def _side(s):
    arena, off, length, ext = s[:4]
    grp = s[4] if len(s) > 4 and s[4] is not None else np.zeros(len(length), np.uint16)
    return [np.ascontiguousarray(arena, np.uint8), np.ascontiguousarray(off, np.int32), np.ascontiguousarray(length, np.int32),
            np.ascontiguousarray(ext, np.uint8), np.ascontiguousarray(grp, np.uint16)]


def diff_pairs_asserts(old, new, n_groups=1):
    """old/new: (arena, off, len, ext[, grp]).  Returns (added_counts, removed_counts, added_events, removed_events):
    [n_groups][K] tables by the side's group, and the events of the inserted / deleted assertion lines."""
    a, b = _side(old), _side(new)
    n = len(a[2])
    ac, rc_ = np.zeros((n_groups, orc.K), np.int64), np.zeros((n_groups, orc.K), np.int64)
    na, nr = C.c_int64(), C.c_int64()
    p = orc._p
    args = [p(x) for x in a] + [p(x) for x in b] + [n, n_groups, p(ac), p(rc_)]
    if lib().orc_diff_pairs_asserts(*args, None, 0, C.byref(na), None, 0, C.byref(nr)) != 0:
        raise ValueError("orc_diff_pairs_asserts failed")
    aev, rev = np.zeros(max(na.value, 1), orc.ASSERT_EVENT), np.zeros(max(nr.value, 1), orc.ASSERT_EVENT)
    if lib().orc_diff_pairs_asserts(*args, p(aev), aev.size, C.byref(na), p(rev), rev.size, C.byref(nr)) != 0:
        raise ValueError("orc_diff_pairs_asserts failed")
    return ac, rc_, aev[:na.value], rev[:nr.value]
