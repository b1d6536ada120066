"""numpy reference of the moved code of docs/SPEC.md section 20 for C5-scale corpora (test infrastructure): the serial marks of
tests/orc_marks.py and the oracle's line hashes, then the matching (deleted, inserted) pairs of every step enumerated per key,
their diagonals by one sort, the reach by another, and the greedy block walk run by run.  No shared code with the kernels or
tests/move_ref.py."""
import numpy as np

import orc
import orc_marks as om

MIN_ALNUM = 20
_NOT_ALNUM = bytes(c for c in range(256) if not (48 <= c <= 57 or 65 <= c <= 90 or 97 <= c <= 122))
BLOCK = np.dtype([("line", "<i8"), ("partner", "<i8"), ("n_lines", "<i4"), ("n_assert", "<i4")])


class _Side:
    def __init__(self, packed, base, hashes, mark, step):
        arena, off, length, ext = packed
        self.arena, self.off, self.ext = arena, np.asarray(off, np.int64), np.asarray(ext)
        self.base, self.hash, self.mark = np.asarray(base, np.int64), np.asarray(hashes, np.uint64), mark
        T, n = len(self.hash), len(self.base) - 1
        self.file = np.repeat(np.arange(n), np.diff(self.base))
        self.step = np.asarray(step, np.int64)[self.file] if n else np.zeros(0, np.int64)
        chg = mark != 0
        first = np.zeros(T, bool)
        first[self.base[:-1][np.diff(self.base) > 0]] = True
        prev = np.zeros(T, bool)
        prev[1:] = chg[:-1]
        self.changed, self.head = chg, chg & (first | ~prev)
        self.cont = np.zeros(T, bool)                  # x + 1 lies in the run of x
        self.cont[:-1] = chg[:-1] & chg[1:] & ~self.head[1:]
        self.run = np.cumsum(self.head) - 1
        self.data = bytes(arena)
        self.ends = None

    def line_bytes(self, x):
        f = int(self.file[x])
        b = int(self.off[f])
        s = 0 if x == self.base[f] else int(self.ends[x - 1]) + 1
        return self.data[b + s:b + int(self.ends[x])]


def _reach(X, Y, ex, ey, kx, ky):
    """L(x) and partner(x) of every changed line x of X (0 / -1 without a match): kx, ky the key ids of the entries ex, ey."""
    T = len(X.hash)
    L, P = np.zeros(T, np.int64), np.full(T, -1, np.int64)
    ox, oy = np.argsort(kx, kind="stable"), np.argsort(ky, kind="stable")
    ex, kx, ey, ky = ex[ox], kx[ox], ey[oy], ky[oy]
    keys = np.intersect1d(kx, ky)
    if not len(keys):
        return L, P
    sx0, sx1 = np.searchsorted(kx, keys), np.searchsorted(kx, keys, "right")
    sy0, sy1 = np.searchsorted(ky, keys), np.searchsorted(ky, keys, "right")
    cx, cy = sx1 - sx0, sy1 - sy0
    npair = cx * cy
    tot = int(npair.sum())
    g = np.repeat(np.arange(len(keys)), npair)               # key of every pair, then its (i, j) inside the key's product
    r = np.arange(tot) - np.repeat(np.cumsum(npair) - npair, npair)
    i, j = r // cy[g], r % cy[g]
    x, c = ex[sx0[g] + i], ey[sy0[g] + j]
    succ = X.cont[x] & Y.cont[c]
    succ[succ] = X.hash[x[succ] + 1] == Y.hash[c[succ] + 1]
    o = np.lexsort((x, x - c))                                # diagonals, each in line order
    link = succ[o]                                            # sorted pair k continues to k + 1
    idx = np.arange(tot)
    end = np.where(~link, idx, tot)                           # the last pair of every diagonal, from each pair on
    end = np.minimum.accumulate(end[::-1])[::-1]
    ln = np.empty(tot, np.int64)
    ln[o] = end - idx + 1
    o2 = np.lexsort((c, -ln, x))                              # per x: the longest, then the smallest partner
    xs = x[o2]
    firsts = np.ones(tot, bool)
    firsts[1:] = xs[1:] != xs[:-1]
    L[xs[firsts]] = ln[o2][firsts]
    P[xs[firsts]] = c[o2][firsts]
    return L, P


def serial_marks(old, new, dist=None):
    """(line_base_old, line_base_new, line_hash_old, line_hash_new, dels, ins) of packed sides: the oracle's hashes and the
    serial marks of every pair (orc_marks.device_marks; dist as orc_marks.diff_pairs_marks)."""
    ba, ha = om.line_hashes(old)
    bb, hb = om.line_hashes(new)
    dist = dist or {}
    dl, ins = np.zeros(int(ba[-1]), np.uint8), np.zeros(int(bb[-1]), np.uint8)
    for i in range(len(old[2])):
        dl[ba[i]:ba[i + 1]], ins[bb[i]:bb[i + 1]] = om.device_marks(ha[ba[i]:ba[i + 1]], hb[bb[i]:bb[i + 1]], dist.get(i))
    return ba, bb, ha, hb, dl, ins


def diff_moves(old, new, steps=None, dist=None, marks=None):
    """old/new: packed sides (arena, off, len, ext); steps: the step of every pair (default 0).  Returns (line_base_old,
    line_base_new, dels, ins, old_blocks, new_blocks) as tsm_diff_pairs_moves gives them: the marks with bit 1 on moved lines,
    the blocks as BLOCK arrays in line order.  dist: as orc_marks.diff_pairs_marks; marks: serial_marks(old, new, dist) when
    the caller has it (it is not changed)."""
    n = len(old[2])
    steps = np.zeros(n, np.int64) if steps is None else np.asarray(steps, np.int64)
    ba, bb, ha, hb, dl, ins = marks if marks is not None else serial_marks(old, new, dist)
    dl, ins = dl.copy(), ins.copy()
    S = [_Side(old, ba, ha, dl, steps), _Side(new, bb, hb, ins, steps)]
    for s, packed in zip(S, (old, new)):
        s.ends = _line_ends(packed, s.base)
    ent = [np.flatnonzero(s.changed) for s in S]
    ids = {}
    key = [np.array([ids.setdefault((int(s.step[x]), int(s.hash[x])), len(ids)) for x in e], np.int64) for s, e in zip(S, ent)]
    out = []
    for a in range(2):
        X, Y = S[a], S[1 - a]
        L, P = _reach(X, Y, ent[a], ent[1 - a], key[a], key[1 - a])
        blocks = []
        for x0 in np.flatnonzero(X.head):
            x, r = int(x0), X.run[x0]
            while x < len(X.hash) and X.changed[x] and X.run[x] == r:
                k = int(L[x])
                if k and sum(len(X.line_bytes(x + q).translate(None, _NOT_ALNUM)) for q in range(k)) >= MIN_ALNUM:
                    na = 0
                    for q in range(k):
                        na += X.ext[X.file[x + q]] != 0 and orc.is_assert_line(X.line_bytes(x + q))
                    blocks.append((x, int(P[x]), k, na))
                    X.mark[x:x + k] |= 2
                    x += k
                else:
                    x += 1
        out.append(np.array(blocks, BLOCK) if blocks else np.zeros(0, BLOCK))
    return ba, bb, dl, ins, out[0], out[1]


def _line_ends(packed, base):
    """line_end of every line (file-relative position of its LF, or the file size)."""
    arena, off, length, _ = packed
    ends = np.zeros(int(base[-1]), np.int64)
    for f in range(len(length)):
        b = np.asarray(arena[int(off[f]):int(off[f]) + int(length[f])])
        nl = np.flatnonzero(b == 10)
        k = int(base[f + 1] - base[f])
        e = np.full(k, int(length[f]), np.int64)
        e[:min(k, len(nl))] = nl[:k]
        ends[int(base[f]):int(base[f + 1])] = e
    return ends
