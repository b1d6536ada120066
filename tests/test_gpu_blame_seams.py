"""GPU tests of the line provenance (docs/SPEC.md section 14) at the seams tests/test_gpu_blame.py does not reach: more chains
than the k_blame launch has warps, and the same chains in another order; untraced pairs inside chains; files emptied and
refilled; line counts and edits on the 32-line tiles of k_blame's two ballot passes; every k_diff_small limit in DIFF_MARKS
mode; a side with more lines than the first staging guess of its line records; and the raw C ABI.  Every origin and every
mark is compared with the serial references of tests/test_gpu_blame.py and tests/orc_marks.py (the marks of
tests/orc_diff_marks.c, or the whole middle of a pair whose distance is known in closed form to be above the trace limit),
and every test asserts that its shapes reach the seam it names."""
import ctypes as C
import random

import numpy as np
import pytest

import corpus_util as cu
import orc
import orc_marks
import spec_ref as sr
import tosemscan as ts
from test_gpu_blame import chain_order, provenance, reordered, same_origins, sides
from test_gpu_diff_seams import staging_lines

pytestmark = pytest.mark.gpu
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
TILE_COUNTS = (1, 31, 32, 33, 63, 64, 65, 95, 96, 97)      # line counts around the 32-line tiles of k_blame


@pytest.fixture(scope="module")
def sc():
    s = ts.Scanner(0, 1 << 20, 16, 1)
    yield s
    s.close()


def head_origins(c, f):
    o = np.zeros(len(sr.py_lines(f)), ts.ORIGIN)
    o["change"], o["line"] = -1 - c, np.arange(1, len(o) + 1)
    return o


def batch(chains, seed):
    """chains: [(files, with_origins, ext)], chain c being the pairs files[0] -> files[1] -> ...; the chains interleaved in a
    random order that keeps the pairs of each chain in order (chain_order).  A head with origins has (-1 - c, line) for its
    lines; one without (with_origins False) must have an empty old side.  Returns (olds, news, exts, prev, label, heads,
    where) with where[c][s] = the place of step s of chain c."""
    olds, news, exts, prev, heads, where = [], [], [], [], {}, []
    for c, (files, with_origins, ext) in enumerate(chains):
        assert with_origins or not files[0]
        w = []
        for s in range(len(files) - 1):
            prev.append(w[-1] if w else -1)
            w.append(len(olds))
            olds.append(files[s]); news.append(files[s + 1]); exts.append(ext)
        if with_origins:
            heads[w[0]] = head_origins(c, files[0])
        where.append(w)
    prev = np.array(prev, np.int32)
    label = (1000 + np.arange(len(prev))).astype(np.int32)
    order = chain_order(prev, seed)
    pos = np.empty(len(order), np.int64)
    pos[order] = np.arange(len(order))
    return (*reordered(order, olds, news, exts, prev, label, heads), [[int(pos[i]) for i in w] for w in where])


def run(sc, bt, dist=None):
    """blame_pairs and diff_marks of the batch against the references, origin for origin and mark for mark.  Returns
    (reference marks (line_base_old, line_base_new, del, ins), reference origins, blame_pairs result, diff_last_ms after
    blame_pairs, diff_last_ms after diff_marks)."""
    olds, news, exts, prev, label, heads, _ = bt
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    mk = orc_marks.diff_pairs_marks(*sides(a, b), dist)
    want = provenance(*mk, prev, label, heads)
    res = sc.blame_pairs(a, b, prev, label, heads)
    ms_blame = sc.diff_last_ms()
    add, rem, det, bn, org = res
    assert np.array_equal(bn, mk[1])
    same_origins(org, bn, want)
    madd, mrem, mdet, bo, bn2, dl, ins = sc.diff_marks(a, b)
    ms_marks = sc.diff_last_ms()
    assert np.array_equal(bo, mk[0]) and np.array_equal(bn2, mk[1])
    assert np.array_equal(dl, mk[2]) and np.array_equal(ins, mk[3])
    assert np.array_equal(add, madd) and np.array_equal(rem, mrem) and np.array_equal(det, mdet)
    padd, prem, pdet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(add, padd) and np.array_equal(rem, prem) and np.array_equal(det, pdet)
    return mk, want, res, ms_blame, ms_marks


def pair_marks(mk, i):
    ba, bb, dl, ins = mk
    return dl[ba[i]:ba[i + 1]], ins[bb[i]:bb[i + 1]]


# ---------------------------------------------------------------------------------------------- more chains than warps
def many_chains(seed, n_chains, cap=3000):
    """Chains of 1-4 edits of small C5-law files (capped at `cap` bytes): odd chains start from the file with origins, even
    ones from an empty file without."""
    rng = random.Random(seed)
    base = ts.gen_corpus(seed, n_chains, size_law=1, pinned=False)
    out = []
    for c in range(n_chains):
        f = base.file_bytes(c)[:cap]
        files = [f if c % 2 else b""]
        for s in range(rng.randint(1, 4)):
            g = files[-1]
            files.append(ts.gen_edit(seed * 1_000_000 + c * 8 + s, g, rng.choice((1.0, 6.0, 20.0))) if g else f)
        out.append((files, c % 2 == 1, 1 + c % 3))
    return out


@pytest.fixture(scope="module")
def wide(sc):
    """More than three chains per warp of the k_blame launch (8 warps per block, at most 8 blocks per SM)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    chains = many_chains(77, 3 * 64 * sms + 101)
    bt = batch(chains, 78)
    return sms, chains, bt, run(sc, bt)


def test_more_chains_than_warps(wide):
    sms, chains, bt, (mk, want, res, _, _) = wide
    n_chains = len(chains)
    assert n_chains > 3 * 64 * sms                          # min((n + 7) / 8, 8 sms) blocks of 8 warps: every warp takes 3+ chains
    assert sum(1 for _, o, _ in chains if o) > 1000 and sum(1 for _, o, _ in chains if not o) > 1000
    assert {len(f) - 1 for f, _, _ in chains} == {1, 2, 3, 4}
    d = mk[2].sum() + mk[3].sum()
    assert d > 100_000 and (bt[3] >= 0).sum() > n_chains


def test_chain_order_invariance(wide, sc):
    """The same chains with the pairs in another order that keeps each chain's order: per pair, the same origins.  The host
    sorts chains longest first (stable), so the chains of one length go to the warps in another order."""
    _, _, bt, (_, want, _, _, _) = wide
    olds, news, exts, prev, label, heads, _ = bt
    order = chain_order(prev, 79)
    assert (order != np.arange(len(order))).mean() > 0.9
    olds2, news2, exts2, prev2, label2, heads2 = reordered(order, olds, news, exts, prev, label, heads)
    a, b = ts.pack(olds2, exts2), ts.pack(news2, exts2)
    _, _, _, bn, org = sc.blame_pairs(a, b, prev2, label2, heads2)
    same_origins(org, bn, [want[i] for i in order])


# ---------------------------------------------------------------------------------------------- untraced steps
UNTRACED = (((11584,), (11585,)), ((6000, 5585), (6000, 5585)), ((23169,), (0,)))


def test_untraced_steps_inside_chains(sc):
    """A traced edit, then an untraced pair (D = 23 169 / 23 170: its whole middle deleted and inserted, common lines inside
    it too), then two traced edits, among small chains."""
    chains, shapes = [], []
    for i, s in enumerate(UNTRACED):
        o, n, w = cu.block_pair(b"U%d" % i, *s, n_prefix=40 + i, n_suffix=30 + i)
        e1 = ts.gen_edit(900 + i, n, 6.0)
        files = [ts.gen_edit(910 + i, o, 6.0), o, n, e1, ts.gen_edit(920 + i, e1, 6.0)]
        chains.append((files, True, 1 + i))
        shapes.append(w)
    chains += many_chains(81, 40)
    bt = batch(chains, 82)
    where, label = bt[6], bt[4]
    dist = {where[i][1]: len(w[3]) + len(w[4]) for i, w in enumerate(shapes)}
    assert sorted(dist.values()) == [23169, 23169, 23170] and min(dist.values()) > orc_marks.TRACE_MAX_D
    mk, want, (add, rem, det, _, _), _, ms = run(sc, bt, dist)
    assert ms[2] > 0
    common_inside = 0
    for i, w in enumerate(shapes):
        u, after, later = where[i][1], where[i][2], where[i][3]
        assert (add[u], rem[u]) == (len(w[4]), len(w[3]))
        if add[u] and rem[u]:                               # one hunk, assertion counts unknown (tsm_diff_pairs_detail)
            assert det[u].tolist() == (0, 0, 1, -1, -1)
        else:                                               # a pure hunk needs no trace: its detail is exact at any distance
            one = sides(ts.pack([bt[0][u]], [bt[2][u]]), ts.pack([bt[1][u]], [bt[2][u]]))
            assert det[u].tolist() == orc.diff_pairs_detail(*one)[2][0].tolist() and det[u]["removed_assert"] > 4000
        dl, ins = pair_marks(mk, u)
        assert dl.sum() >= rem[u] and ins.sum() >= add[u]
        common_inside += int(ins.sum() - add[u])            # common lines inside the middle: inserted, with the pair's label
        mid = np.flatnonzero(ins)
        assert (want[u]["change"][mid] == label[u]).all()
        if add[u]:                                          # the untraced pair's origins carried on two more pairs
            assert min((want[t]["change"] == label[u]).sum() for t in (after, later)) > 1000
    assert common_inside > 0


# ---------------------------------------------------------------------------------------------- emptied and refilled files
def unique_lines(tag, k):
    return b"".join(b"%s line %d\n" % (tag, j) for j in range(k))


def test_emptied_and_refilled_files(sc):
    f = unique_lines(b"F", 300) + b"F unterminated"
    g = unique_lines(b"G", 5000)
    chains = [([f, b"", g, ts.gen_edit(31, g, 6.0)], True, 1),     # full, emptied, refilled, edited
              ([g, b"", f, b"", g], True, 2),                      # the same past k_diff_small's middle limit
              ([b"", f, ts.gen_edit(32, f, 6.0)], False, 1),       # an empty head without origins
              ([b"", b""], False, 4),                              # one pair, empty on both sides
              ([b"a\nb\nc\n", b"a\nb\nc", b"a\nb\nc\nd\n", b"a\nb\nc\nd"], True, 1),   # unterminated = terminated twin
              ([b"x", b"x\n", b"", b"x"], True, 3)]
    chains += many_chains(83, 30)
    bt = batch(chains, 84)
    olds, news, where = bt[0], bt[1], bt[6]
    mk, want, res, _, _ = run(sc, bt)
    emptied = [p for p in range(len(olds)) if olds[p] and not news[p]]
    refilled = [p for p in range(len(olds)) if news[p] and not olds[p]]
    assert len(emptied) >= 4 and len(refilled) >= 5
    for p in emptied:
        assert pair_marks(mk, p)[0].all() and len(want[p]) == 0
    for p in refilled:
        assert pair_marks(mk, p)[1].all() and (want[p]["change"] == bt[4][p]).all()
    assert 5000 in {len(sr.py_lines(olds[p])) for p in emptied}
    twin = where[4]
    assert [int(sum(m.sum() for m in pair_marks(mk, p))) for p in twin] == [0, 1, 0]
    assert want[twin[2]]["change"].tolist() == [-5, -5, -5, bt[4][twin[1]]]
    assert len(want[where[3][0]]) == 0 and want[where[5][2]].tolist() == [(bt[4][where[5][2]], 1)]


# ---------------------------------------------------------------------------------------------- the 32-line tiles
def tile_step(rng, old, b, tag):
    """old (unique lines) edited to b lines: deletions and insertions on tile positions 0 and 31 first, kept lines unique."""
    a = len(old)
    nd = min(a, max(a - b, 0) + rng.randint(1, 4))

    def pick(size, k):
        edge = [i for i in range(size) if i % 32 in (0, 31)]
        rest = [i for i in range(size) if i % 32 not in (0, 31)]
        rng.shuffle(edge); rng.shuffle(rest)
        return set((edge + rest)[:k])
    dels, ins = pick(a, nd), pick(b, b - (a - nd))
    kept = iter([x for i, x in enumerate(old) if i not in dels])
    return [b"%s %d\n" % (tag, j) if j in ins else next(kept) for j in range(b)]


def test_tile_edges(sc):
    """Old and new line counts 1, 31, 32, 33, 63, 64, 65, 95, 96, 97, edits on lanes 0 and 31, and an insertion of more than
    65 536 lines (origin lines past 16 bits) carried on by the next pair."""
    rng = random.Random(61)
    chains = []
    for c in range(12):
        counts = list(TILE_COUNTS)
        rng.shuffle(counts)
        lines = [b"c%d head %d\n" % (c, j) for j in range(counts[0])]
        files = [b"".join(lines)]
        for s, k in enumerate(counts[1:] + counts[:1]):
            lines = tile_step(rng, lines, k, b"c%d s%d" % (c, s))
            files.append(b"".join(lines))
        chains.append((files, True, 1 + c % 3))
    small = unique_lines(b"S", 40)
    big = b"".join(small.splitlines(True)[:20]) + unique_lines(b"B", 70_000) + b"".join(small.splitlines(True)[20:])
    chains.append(([small, big, ts.gen_edit(62, big, 6.0)], True, 1))
    bt = batch(chains, 63)
    olds, news, where = bt[0], bt[1], bt[6]
    mk, want, res, _, _ = run(sc, bt)
    n_old = {len(sr.py_lines(f)) for f in olds}
    n_new = {len(sr.py_lines(f)) for f in news}
    assert set(TILE_COUNTS) <= n_old and set(TILE_COUNTS) <= n_new
    lanes_del, lanes_ins = set(), set()
    for p in range(len(olds)):
        dl, ins = pair_marks(mk, p)
        lanes_del |= set(np.flatnonzero(dl) % 32)
        lanes_ins |= set(np.flatnonzero(ins) % 32)
    assert {0, 31} <= lanes_del and {0, 31} <= lanes_ins
    b1, b2 = where[-1][0], where[-1][1]
    assert want[b1]["line"].max() == 70_020 and (want[b2]["line"] > 65_536).sum() > 4000
    assert (want[b2]["change"] == bt[4][b1]).sum() > 60_000


# ---------------------------------------------------------------------------------------------- k_diff_small limits
def limit_pairs():
    """The pairs of test_gpu_parity.test_diff_limits_of_the_one_launch_kernel, with every middle of 510-514, 1 022-1 026 and
    4 094-4 098 lines: (old, new, ext)."""
    def lines(tag, n):
        return [b"%s%05d\n" % (tag, i) for i in range(n)]
    out = []
    for total, ds in ((250, (1, 15, 30, 31, 32, 33)), (500, (62, 63, 64, 65)), (1300, (31, 64, 126, 127, 128, 129, 200))):
        for d in ds:                                        # d deletions spread over the file: D = d
            o = lines(b"assert x", total)
            keep = [x for i, x in enumerate(o) if not (i % (total // d) == 3 and i // (total // d) < d)]
            out.append((b"".join(o), b"".join(keep), 1))
    for d in (16, 31, 32, 64):                              # replacements: D = 2 d
        o = lines(b"y = ", 300)
        n = list(o)
        for j in range(d):
            n[5 + 4 * j] = b"EXPECT_EQ(%d, q);\n" % j
        out.append((b"".join(o), b"".join(n), 2))
    for total in (*range(510, 515), *range(1022, 1027), *range(4094, 4099), 6000):   # a middle of `total` lines
        half = total // 2
        o = [b"first old\n"] + lines(b"m", half - 2) + [b"last old\n"]
        n = [b"first new\n"] + lines(b"m", total - half - 2) + [b"assert last_new\n"]
        out.append((b"head\n" * 40 + b"".join(o) + b"tail\n" * 40, b"head\n" * 40 + b"".join(n) + b"tail\n" * 40, 1))
    out += [(b"", b"b\n" * 2500, 1), (b"a\n" * 3000, b"", 1), (b"".join(lines(b"p", 40)), b"".join(lines(b"q", 40)), 1),
            (b"same\n" * 5000, b"same\n" * 5000, 1)]
    return out


def test_every_kernel_limit_in_marks_mode(sc):
    """Each limit pair as a chain there and back (old -> new -> old): the limits with deletions and with insertions."""
    pairs = limit_pairs()
    bt = batch([([o, n, o], True, x) for o, n, x in pairs], 71)
    mk, want, res, ms_blame, ms_marks = run(sc, bt)
    assert ms_blame[2] > 0 and ms_marks[2] > 0              # the left-over kernels ran
    A, B = sides(ts.pack(bt[0], bt[2]), ts.pack(bt[1], bt[2]))
    (ba, ha), (bb, hb) = orc_marks.line_hashes(A), orc_marks.line_hashes(B)
    middles, dists = set(), set()
    for p in range(len(bt[0])):
        a, b = ha[ba[p]:ba[p + 1]], hb[bb[p]:bb[p + 1]]
        pre, suf = orc_marks.middle(a, b)
        middles.add(len(a) + len(b) - 2 * (pre + suf))
        dists.add(int(sum(m.sum() for m in pair_marks(mk, p))))
    assert {*range(510, 515), *range(1022, 1027), *range(4094, 4099), 6000} <= middles
    assert {31, 32, 33, 63, 64, 65, 126, 127, 128, 129, 200} <= dists


# ---------------------------------------------------------------------------------------------- a line-dense side
def dense_file(rng, k, tag):
    return [b"%s %d\n" % (tag, j) if rng.random() < 0.05 else b"\n" for j in range(k)]


def dense_edit(rng, lines, tag):
    out = []
    for j, x in enumerate(lines):
        r = rng.random()
        if r < 0.01:
            continue
        if r < 0.02:
            out.append(b"%s %d\n" % (tag, j) if rng.random() < 0.5 else b"\n")
        out.append(x)
    return out


def raw_blame(sc, a, b, prev, label, origin_in, in_base, cap):
    """tsm_blame_pairs through ctypes: (rc, added, removed, detail, line_base_old, line_base_new, origins, n_lines)."""
    n = a.n_files
    add, rem, det = np.zeros(max(n, 1), np.int64), np.zeros(max(n, 1), np.int64), np.zeros(max(n, 1), ts.DIFF_DETAIL)
    bo, bn = np.full(n + 1, -7, np.int64), np.full(n + 1, -7, np.int64)
    out = np.zeros(max(cap, 1), ts.ORIGIN)
    out["change"], out["line"] = -7, -7
    ca, cb = a.c_struct(), b.c_struct()
    nl = C.c_int64(-7)
    rc = ts.lib().tsm_blame_pairs(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), ts._p(det), ts._p(prev), ts._p(label),
                                  ts._p(origin_in), ts._p(in_base), ts._p(bo), ts._p(bn), ts._p(out), cap, C.byref(nl), None)
    return rc, add[:n], rem[:n], det[:n], bo, bn, out[:max(nl.value, 0)], nl.value


def wrapper_args(bt):
    """origin_in / in_base as the Python wrapper packs them (heads only, from 0)."""
    prev, heads = bt[3], bt[5]
    parts = [np.asarray(heads.get(i, np.zeros(0, ts.ORIGIN)), ts.ORIGIN) if prev[i] < 0 else np.zeros(0, ts.ORIGIN)
             for i in range(len(prev))]
    in_base = np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.int64)
    origin_in = np.concatenate(parts + [np.zeros(1, ts.ORIGIN)])
    return origin_in, in_base


def test_line_dense_side(sc):
    """Chains of files of mostly empty lines: each side has more lines than the staging arrays of its first k_scan pass
    hold, so the line records (and the line_base blame checks line counts with) come from the second, exact-size pass."""
    rng = random.Random(91)
    chains = []
    for c in range(4):
        lines = dense_file(rng, rng.randrange(1500, 3000), b"d%d" % c)
        files = [b"".join(lines)]
        for s in range(3):
            lines = dense_edit(rng, lines, b"d%d s%d" % (c, s))
            files.append(b"".join(lines))
        chains.append((files, True, 1 + c % 3))
    bt = batch(chains, 92)
    a, b = ts.pack(bt[0], bt[2]), ts.pack(bt[1], bt[2])
    for side, files in ((a, bt[0]), (b, bt[1])):
        assert sum(len(sr.py_lines(f)) for f in files) > staging_lines(side)
    mk, want, res, _, _ = run(sc, bt)
    origin_in, in_base = wrapper_args(bt)
    rc, add, rem, det, bo, bn, org, nl = raw_blame(sc, a, b, bt[3], bt[4], origin_in, in_base, int(mk[1][-1]))
    assert rc == 0 and nl == mk[1][-1]
    assert np.array_equal(bo, mk[0]) and np.array_equal(bn, mk[1])
    same_origins(org, bn, want)
    assert np.array_equal(add, res[0]) and np.array_equal(rem, res[1]) and np.array_equal(det, res[2])


# ---------------------------------------------------------------------------------------------- the raw C ABI
def test_raw_abi(sc):
    """What the wrapper never passes: origins behind unused entries (in_base[0] > 0), ranges of non-head pairs (not read),
    labels INT32_MIN, -1 and INT32_MAX, and an empty batch."""
    bt = batch(many_chains(101, 60) + [([b"", b"", b"a\n"], False, 1)], 102)
    olds, news, exts, prev, _, heads, _ = bt
    label = np.array([(INT32_MIN, -1, INT32_MAX)[i % 3] for i in range(len(prev))], np.int32)
    junk = np.zeros(5, ts.ORIGIN)
    junk["change"], junk["line"] = -99, -99
    parts = [junk]
    for i in range(len(prev)):
        if prev[i] < 0:
            parts.append(np.asarray(heads.get(i, np.zeros(0, ts.ORIGIN)), ts.ORIGIN))
        else:                                               # a range of a non-head pair: only the heads' ranges are read
            parts.append(junk[:3] if i % 4 == 0 else junk[:0])
    origin_in = np.concatenate(parts)
    in_base = np.cumsum([len(x) for x in parts]).astype(np.int64)
    assert in_base[0] == 5 and len(origin_in) == in_base[-1]
    assert any(in_base[i + 1] > in_base[i] for i in range(len(prev)) if prev[i] >= 0)
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    mk = orc_marks.diff_pairs_marks(*sides(a, b))
    want = provenance(*mk, prev, label, heads)
    rc, add, rem, det, bo, bn, org, nl = raw_blame(sc, a, b, prev, label, origin_in, in_base, int(mk[1][-1]))
    assert rc == 0 and nl == mk[1][-1]
    assert np.array_equal(bo, mk[0]) and np.array_equal(bn, mk[1])
    same_origins(org, bn, want)
    got = set(np.concatenate(want)["change"].tolist())
    assert {INT32_MIN, -1, INT32_MAX} <= got and -99 not in got
    padd, prem, pdet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(add, padd) and np.array_equal(rem, prem) and np.array_equal(det, pdet)
    e = ts.pack([], [])
    z32, z64 = np.zeros(1, np.int32), np.zeros(1, np.int64)
    rc, add, rem, det, bo, bn, org, nl = raw_blame(sc, e, e, z32, z32, None, z64, 0)
    assert rc == 0 and nl == 0 and bo.tolist() == [0] and bn.tolist() == [0] and len(org) == 0
