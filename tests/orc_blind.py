"""ctypes binding of tests/orc_blind.c, the serial C reference of the blind clones of docs/SPEC.md section 21.  TEST
INFRASTRUCTURE ONLY.  Compiled together with the oracle's orc.c (line hashes, n-gram keys, assertion lines) into a library in
the temporary directory, so that the tests never write into the tree.

* `blind_lines(corpus)`: per line of the corpus the kept flag, the blind hash (0 when not kept) and the assertion flag;
* `clones_blind(corpus, n)`: section 15 over the kept lines, the dict of `tosemscan.Scanner.clones(..., blind=True)`.
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
SRCS = [os.path.join(HERE, "orc_blind.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(orc.ORC_DIR, "orc.h"), os.path.join(orc.ORC_DIR, "orc_categories.inc")]

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_blind_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_blind_lines.restype = C.c_int
            L.orc_blind_lines.argtypes = [C.c_void_p] * 4 + [C.c_int32] + [C.c_void_p] * 4
            L.orc_clone_walk.restype = C.c_int
            L.orc_clone_walk.argtypes = [C.c_void_p] * 3 + [C.c_int32, C.c_int32] + [C.c_void_p] * 4 + [C.c_int64, C.c_void_p,
                                                                                                         C.c_void_p, C.c_int64, C.c_void_p]
            _lib = L
    return _lib


def _arrays(corpus):
    return (np.ascontiguousarray(corpus.arena, np.uint8), np.ascontiguousarray(corpus.off, np.int32),
            np.ascontiguousarray(corpus.len, np.int32), np.ascontiguousarray(corpus.ext, np.uint8))


def blind_lines(corpus):
    """(line_base, kept, blind_hash, flag) of every line of the corpus (tosemscan.Corpus or anything with arena, off, len,
    ext)."""
    arena, off, length, ext = _arrays(corpus)
    nf = len(length)
    T = sum(int(np.count_nonzero(arena[o:o + n] == 0x0A)) + (n > 0 and arena[o + n - 1] != 0x0A) for o, n in zip(off[:nf], length))
    base = np.zeros(nf + 1, np.int64)
    kept, bhash, flag = np.zeros(max(T, 1), np.uint8), np.zeros(max(T, 1), np.uint64), np.zeros(max(T, 1), np.uint8)
    p = orc._p
    if lib().orc_blind_lines(p(arena), p(off), p(length), p(ext), nf, p(base), p(kept), p(bhash), p(flag)) != 0:
        raise ValueError("orc_blind_lines failed")
    assert base[-1] == T
    return base, kept[:T].astype(bool), bhash[:T], flag[:T]


def clone_walk(hashes, flag, base, n):
    """Section 15 over a line sequence (orc_clone_walk): file_dup, file_dup_assert, class_base, class_len and member."""
    hashes = np.ascontiguousarray(hashes, np.uint64)
    flag = np.ascontiguousarray(flag, np.uint8)
    base = np.ascontiguousarray(base, np.int64)
    nf = len(base) - 1
    p = orc._p
    cap = 0
    for _ in range(2):
        out = {"file_dup": np.zeros(max(nf, 1), np.uint32), "file_dup_assert": np.zeros(max(nf, 1), np.uint32),
               "class_base": np.zeros(cap + 1, np.int64), "class_len": np.zeros(max(cap, 1), np.uint32),
               "member": np.zeros(max(cap, 1), np.int64)}
        nc, nm = C.c_int64(), C.c_int64()
        rc = lib().orc_clone_walk(p(hashes), p(flag), p(base), nf, int(n), p(out["file_dup"]), p(out["file_dup_assert"]),
                                  p(out["class_base"]), p(out["class_len"]), cap, C.byref(nc), p(out["member"]), cap, C.byref(nm))
        if rc == -3:
            cap = max(nc.value, nm.value)
            continue
        if rc != 0:
            raise ValueError("orc_clone_walk failed")
        out["file_dup"], out["file_dup_assert"] = out["file_dup"][:nf], out["file_dup_assert"][:nf]
        out["class_base"], out["class_len"], out["member"] = out["class_base"][:nc.value + 1], out["class_len"][:nc.value], out["member"][:nm.value]
        return out
    raise ValueError("orc_clone_walk: capacity")


def clones_blind(corpus, n):
    """Section 21 from the C lexer and orc_clone_walk over the kept lines."""
    base, kept, bhash, flag = blind_lines(corpus)
    kept_line = np.nonzero(kept)[0].astype(np.int64)
    rank = np.concatenate([[0], np.cumsum(kept, dtype=np.int64)])
    kept_base = rank[base]
    kflag = flag[kept_line]
    out = clone_walk(bhash[kept_line], kflag, kept_base, n)
    fa = np.concatenate([[0], np.cumsum(kflag, dtype=np.int64)])[kept_base]
    out.update(line_base=base, kept_base=kept_base, kept_line=kept_line, blind_hash=bhash[kept_line],
               file_kept_assert=np.diff(fa).astype(np.uint32))
    return out
