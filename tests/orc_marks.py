"""ctypes binding of the CPU reference of the edit marks (tests/orc_diff_marks.c).  TEST INFRASTRUCTURE ONLY.

The C file is compiled into a library in the temporary directory, so that the tests never write into the tree.  The marks
of packed sides take the line hashes from the oracle (orc.scan)."""
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


def line_hashes(side):
    """(line_base, line_hash) of the packed side (arena, off, len, ext): orc.line_records without the assertion flags."""
    res = orc.scan(*side, np.zeros(len(side[2]), np.uint16), 1, events=False, line_hashes=True)
    return res["line_base"], res["line_hash"]


def middle(a, b):
    """(pre, suf) of the line-hash sequences a and b: their common prefix, then the common suffix of what the prefix leaves,
    as the diff kernels take them.  The middle is a[pre:len(a) - suf] and b[pre:len(b) - suf]."""
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    k = min(a.size, b.size)
    ne = np.flatnonzero(a[:k] != b[:k])
    pre = int(ne[0]) if ne.size else k
    k -= pre
    ne = np.flatnonzero(a[a.size - k:][::-1] != b[b.size - k:][::-1])
    return pre, int(ne[0]) if ne.size else k


def middle_marks(a, b):
    """(del, ins) with every line of the middle marked: how the device marks a pair it does not trace (D > TRACE_MAX_D)."""
    pre, suf = middle(a, b)
    dl, ins = np.zeros(len(a), np.uint8), np.zeros(len(b), np.uint8)
    dl[pre:len(a) - suf] = 1
    ins[pre:len(b) - suf] = 1
    return dl, ins


def device_marks(a, b, d=None):
    """(del, ins) of the line-hash sequences a and b as the device marks them: the serial script of a traced pair, the whole
    middle of an untraced one.  d: the pair's distance when it is known without a search (corpus_util.block_pair gives it in
    closed form); the serial search, whose memory grows as D^2, runs only when d is None or at most TRACE_MAX_D.  A pure
    hunk needs no search: its script is its whole middle, at any distance."""
    if d is not None and d > TRACE_MAX_D:
        return middle_marks(a, b)
    got, dl, ins = diff_marks(a, b)
    assert d is None or got == d, (got, d)
    assert got <= TRACE_MAX_D or not dl.any() or not ins.any(), got
    return dl, ins


def diff_pairs_marks(old, new, dist=None):
    """old/new: packed sides (arena, off, len, ext).  (line_base_old, line_base_new, del, ins) over every line of each side,
    as tsm_diff_pairs_marks gives them (device_marks per pair).  dist: {pair: D} of the pairs whose distance is known in closed
    form; every other pair must be within reach of the serial search."""
    ba, ha = line_hashes(old)
    bb, hb = line_hashes(new)
    dist = dist or {}
    dl, ins = np.zeros(int(ba[-1]), np.uint8), np.zeros(int(bb[-1]), np.uint8)
    for i in range(len(ba) - 1):
        dl[ba[i]:ba[i + 1]], ins[bb[i]:bb[i + 1]] = device_marks(ha[ba[i]:ba[i + 1]], hb[bb[i]:bb[i + 1]], dist.get(i))
    return ba, bb, dl, ins
