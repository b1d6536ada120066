"""ctypes binding of the CPU reference of the edit marks (tests/orc_diff_marks.c).  TEST INFRASTRUCTURE ONLY.

The C file is compiled into a library in the temporary directory, so that the tests never write into the tree.  diff_marks
of packed sides takes the line hashes from the oracle (orc.line_records)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import threading

import numpy as np

import orc

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_diff_marks.c")
TRACE_MAX_D = 23168                          # the largest distance the device traces (include/tosemscan.h)

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(open(SRC, "rb").read()).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_marks_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-o", tmp, SRC])
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_diff_marks.restype = C.c_int64
            L.orc_diff_marks.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
            _lib = L
    return _lib


def diff_marks(a, b):
    """(D, del, ins) of the line-hash sequences a (old) and b (new): uint8 marks of the deleted / inserted lines."""
    a = np.ascontiguousarray(a, np.uint64)
    b = np.ascontiguousarray(b, np.uint64)
    dl, ins = np.zeros(max(a.size, 1), np.uint8), np.zeros(max(b.size, 1), np.uint8)
    d = lib().orc_diff_marks(orc._p(a), a.size, orc._p(b), b.size, orc._p(dl), orc._p(ins))
    if d < 0:
        raise MemoryError("orc_diff_marks")
    return int(d), dl[:a.size], ins[:b.size]


def diff_pairs_marks(old, new):
    """old/new: packed sides (arena, off, len, ext).  (line_base_old, line_base_new, del, ins) over every line of each side,
    as tsm_diff_pairs_marks gives them; both sides must be within reach of the serial search (no untraced pair)."""
    ba, ha = orc.line_records(*old)[:2]
    bb, hb = orc.line_records(*new)[:2]
    dl, ins = np.zeros(int(ba[-1]), np.uint8), np.zeros(int(bb[-1]), np.uint8)
    for i in range(len(ba) - 1):
        d, x, y = diff_marks(ha[ba[i]:ba[i + 1]], hb[bb[i]:bb[i + 1]])
        assert d <= TRACE_MAX_D
        dl[ba[i]:ba[i + 1]], ins[bb[i]:bb[i + 1]] = x, y
    return ba, bb, dl, ins
