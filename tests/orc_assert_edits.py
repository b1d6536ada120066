"""numpy + C reference of the assertion edits of tsm_diff_pairs_assert_edits (docs/SPEC.md section 17), for inputs too large for
the plain-Python restatement (edit_ref.py_assert_edits).  TEST INFRASTRUCTURE ONLY.

The marks come from the serial tests/orc_diff_marks.c (orc_marks), the assertion lines from the oracle's events (orc_cases
.side_lines); the entries and their hunk keys are array arithmetic over them, and the scores and the greedy pairing are the
serial tests/orc_assert_edits.c, compiled into the temporary directory as orc_marks compiles its C file."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import threading

import numpy as np

import orc
import orc_cases
import orc_marks
import tosemscan as ts

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_assert_edits.c")
W = b" \t\r\x0b\x0c"

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(open(SRC, "rb").read()).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_edits_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-o", tmp, SRC])
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_assert_edits.restype = C.c_int64
            L.orc_assert_edits.argtypes = [C.c_int64] + [C.c_void_p] * 4 + [C.c_int64] + [C.c_void_p] * 7 + [C.c_int64]
            _lib = L
    return _lib


def line_ends(side, base):
    """Arena position of the end (LF or file end) of every line of a packed side, global line order."""
    arena, off, length, _ = side
    arena = np.asarray(arena, np.uint8)
    off, length = np.asarray(off, np.int64), np.asarray(length, np.int64)
    n = len(length)
    nl = np.flatnonzero(arena[:int(off[-1])] == 10) if n else np.zeros(0, np.int64)
    f = np.searchsorted(off[:n], nl, side="right") - 1
    keep = (f >= 0) & (nl < off[np.maximum(f, 0)] + length[np.maximum(f, 0)])
    nl, f = nl[keep], f[keep]
    first = np.searchsorted(f, np.arange(n))               # index of each file's first LF in nl
    ends = np.zeros(int(base[-1]), np.int64)
    ends[base[f] + np.arange(len(nl)) - first[f]] = nl
    cnt = np.bincount(f, minlength=n)
    tail = np.flatnonzero(base[1:] - base[:-1] > cnt)      # unterminated last line
    ends[base[tail + 1] - 1] = off[tail] + length[tail]
    return ends


def entries(side, base, flag, mark, traced):
    """(keys, stripped lines) of the changed assertion lines of traced pairs: key = pair << 32 | kept rank."""
    ends = line_ends(side, base)
    total = int(base[-1])
    pair = np.searchsorted(base, np.arange(total), side="right") - 1
    kept = (mark == 0).astype(np.int64)
    rank = np.cumsum(kept) - kept
    sel = np.flatnonzero((mark != 0) & (flag != 0) & traced[pair])
    arena, off = bytes(np.asarray(side[0], np.uint8)), np.asarray(side[1], np.int64)
    starts = np.where(sel == base[pair[sel]], off[pair[sel]], ends[np.maximum(sel - 1, 0)] + 1)
    lines = [arena[s:e].strip(W) for s, e in zip(starts.tolist(), ends[sel].tolist())]
    return (pair[sel].astype(np.uint64) << np.uint64(32)) | rank[sel].astype(np.uint64), lines


def assert_edits(old, new, dist=None):
    """ASSERT_EDIT array of the packed sides old / new (arena, off, len, ext) as tsm_diff_pairs_assert_edits gives it.  dist
    as orc_marks.diff_pairs_marks."""
    ba, bb, dl, ins = orc_marks.diff_pairs_marks(old, new, dist)
    _, _, fa = orc_cases.side_lines(old)
    _, _, fb = orc_cases.side_lines(new)
    cd = np.concatenate([[0], np.cumsum(dl, dtype=np.int64)])
    ci = np.concatenate([[0], np.cumsum(ins, dtype=np.int64)])
    changed = cd[ba[1:]] - cd[ba[:-1]] + ci[bb[1:]] - ci[bb[:-1]]
    traced = changed <= orc_marks.TRACE_MAX_D                # an untraced pair has its whole middle marked: more than the limit
    ko, lo_ = entries(old, ba, fa, dl, traced)
    kn, ln_ = entries(new, bb, fb, ins, traced)
    return score_pairs(ko, lo_, kn, ln_)


def score_pairs(ko, lines_old, kn, lines_new):
    """The greedy pairing of section 17 over entries sorted by key: ASSERT_EDIT array in aev order."""
    def pack(lines):
        offs = np.zeros(len(lines) + 1, np.int64)
        offs[1:] = np.cumsum([len(x) for x in lines])
        return np.frombuffer(b"".join(lines) + b"\0", np.uint8), offs[:-1].copy(), np.diff(offs)
    bo, oo, lo_ = pack(lines_old)
    bn, on, ln_ = pack(lines_new)
    ko, kn = np.ascontiguousarray(ko, np.uint64), np.ascontiguousarray(kn, np.uint64)
    cap = max(min(len(ko), len(kn)), 1)
    rev, aev, sc = np.zeros(cap, np.int64), np.zeros(cap, np.int64), np.zeros(cap, np.int64)
    m = lib().orc_assert_edits(len(ko), orc._p(ko), orc._p(oo), orc._p(lo_), orc._p(bo), len(kn), orc._p(kn), orc._p(on),
                               orc._p(ln_), orc._p(bn), orc._p(rev), orc._p(aev), orc._p(sc), cap)
    if m < 0:
        raise MemoryError("orc_assert_edits")
    out = np.zeros(m, ts.ASSERT_EDIT)
    order = np.argsort(aev[:m], kind="stable")
    out["rev"], out["aev"], out["score"] = rev[:m][order], aev[:m][order], sc[:m][order]
    return out
