"""GPU tests of the edit marks and the line provenance (docs/SPEC.md section 14): tsm_diff_pairs_marks against the serial
reference (tests/orc_diff_marks.c) on the C5 pairs and on the shapes of every diff kernel, the trace limit and pure hunks;
tsm_blame_pairs against a serial provenance built on that reference, on chains of files edited step after step."""
import ctypes as C
import random

import numpy as np
import pytest

import corpus_util as cu
import orc_marks
import spec_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu
SIZES = ((512, 31), (1024, 63), (4096, 63), (4096, 127))   # k_diff_small: (lines of both middles, distance)


def sides(a, b):
    return (a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext)


def check_marks(sc, a, b):
    """Device marks against the reference; the marks count added / removed; the rest equals tsm_diff_pairs_detail."""
    add, rem, det, bo, bn, dl, ins = sc.diff_marks(a, b)
    wbo, wbn, wdl, wins = orc_marks.diff_pairs_marks(*sides(a, b))
    assert np.array_equal(bo, wbo) and np.array_equal(bn, wbn)
    assert np.array_equal(dl, wdl) and np.array_equal(ins, wins)
    assert _per_file(ins, bn, add) and _per_file(dl, bo, rem)
    padd, prem, pdet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(add, padd) and np.array_equal(rem, prem) and np.array_equal(det, pdet)
    return add, rem


def _per_file(mark, base, want):
    c = np.concatenate([[0], np.cumsum(mark.astype(np.int64))])
    return np.array_equal(c[base[1:]] - c[base[:-1]], want)


def test_marks_c5():
    """All 50 000 pairs of BASELINE config C5."""
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    add, rem = check_marks(sc, a, b)
    assert add.sum() > 100_000 and rem.sum() > 100_000
    sc.close()


def test_marks_every_kernel():
    """Tie-heavy pairs at every k_diff_small size and left over to k_myers_trace, pure hunks, empty files."""
    olds, news, exts = cu.tie_heavy_pairs(5, scale=2)
    for i, (ko, kn) in enumerate(((40, 0), (0, 33), (3000, 0), (0, 2500))):   # pure hunks, small and left over
        o, n, _ = cu.block_pair(b"p%d" % i, (ko,), (kn,))
        olds.append(o); news.append(n); exts.append(1)
    olds += [b"", b"x\n", b""]; news += [b"y\n", b"", b""]; exts += [1, 1, 1]
    d = []
    for o, n, x in zip(olds, news, exts):
        r = sr.py_diff_files(o, n, x, x)
        d.append(r[0] + r[1])
    assert max(d) > 127 and any(0 < x <= 31 for x in d)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    check_marks(sc, ts.pack(olds, exts), ts.pack(news, exts))
    assert sc.diff_last_ms()[2] > 0                         # the left-over kernels ran
    sc.close()


def test_marks_trace_limit():
    """Distances 23 167 .. 23 170 around the trace limit: traced pairs are marked as their script, untraced pairs over their
    whole middle (every line between the common prefix and suffix), with common lines inside that middle."""
    olds, news, wants = [], [], []
    for i, s in enumerate((((11583,), (11584,)), ((11584,), (11585,)), ((11584,), (11584,)), ((11585,), (11585,)),
                           ((6000, 5585), (6000, 5585)))):
        o, n, w = cu.block_pair(b"L%d" % i, *s, n_prefix=40 + i, n_suffix=30 + i)
        olds.append(o); news.append(n); wants.append(w)
    d = [len(w[3]) + len(w[4]) for w in wants]
    assert d == [23167, 23169, 23168, 23170, 23170]
    a, b = ts.pack(olds, [1] * 5), ts.pack(news, [1] * 5)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    add, rem, det, bo, bn, dl, ins = sc.diff_marks(a, b)
    sc.close()
    for i, (o, n, w) in enumerate(zip(olds, news, wants)):
        no, nn = len(sr.py_lines(o)), len(sr.py_lines(n))
        if d[i] <= orc_marks.TRACE_MAX_D:
            wd, wi = w[3], w[4]
        else:                                               # the middle: first changed line to the last, both sides (the
            pre, suf = 40 + i, 30 + i + 1                   # common line behind the last block belongs to the suffix)
            wd, wi = list(range(pre, no - suf)), list(range(pre, nn - suf))
        assert np.nonzero(dl[bo[i]:bo[i + 1]])[0].tolist() == wd
        assert np.nonzero(ins[bn[i]:bn[i + 1]])[0].tolist() == wi
        assert add[i] == len(w[4]) and rem[i] == len(w[3])
    assert int(dl[bo[4]:bo[5]].sum()) > rem[4]              # the untraced middle holds a common line


def provenance(ba, bb, dl, ins, prev, label, heads):
    """Serial provenance (SPEC section 14) from the marks of every pair (orc_marks.diff_pairs_marks): an ORIGIN array per pair."""
    out = []
    for i in range(len(prev)):
        src = out[prev[i]] if prev[i] >= 0 else np.asarray(heads.get(i, np.zeros(0, ts.ORIGIN)), ts.ORIGIN)
        d, s = dl[ba[i]:ba[i + 1]], ins[bb[i]:bb[i + 1]]
        assert len(src) == len(d)
        o = np.zeros(len(s), ts.ORIGIN)
        new = np.flatnonzero(s)
        o["change"][new], o["line"][new] = label[i], new + 1
        o[s == 0] = src[d == 0]
        out.append(o)
    return out


def ref_blame(a, b, prev, label, heads, dist=None):
    """provenance over the reference marks of the packed sides a, b; dist as orc_marks.diff_pairs_marks (pairs above the trace
    limit are marked over their whole middle, as the device marks them)."""
    return provenance(*orc_marks.diff_pairs_marks(a, b, dist), prev, label, heads)


def chains(seed, lengths, lam_hi=200.0):
    """Pairs of chains of edited files, the chains interleaved in the batch: (olds, news, exts, prev, label, heads).  Chain c
    starts from an empty file (c even) or from a C5-law file whose origins are given; every 7th step edits at lam_hi."""
    rng = random.Random(seed)
    base = ts.gen_corpus(seed, len(lengths), size_law=1, pinned=False)
    state = []
    for c, k in enumerate(lengths):
        f = b"" if c % 2 == 0 else base.file_bytes(c)
        state.append([f, k, -1])
    olds, news, exts, prev, label, heads = [], [], [], [], [], {}
    while any(s[1] for s in state):
        c = rng.choice([i for i, s in enumerate(state) if s[1]])
        f, left, last = state[c]
        step = len(olds)
        lam = lam_hi if step % 7 == 3 else rng.choice((1.0, 6.0, 20.0))
        g = ts.gen_edit(seed * 1000 + step, f, lam) if f else ts.gen_edit(seed * 1000 + step, base.file_bytes(c), 0.0)
        olds.append(f); news.append(g); exts.append(1 + c % 3)
        prev.append(last); label.append(1000 + step)
        if last < 0 and f:
            nl = len(sr.py_lines(f))
            heads[step] = np.array([(-1 - c, j + 1) for j in range(nl)], ts.ORIGIN)
        state[c] = [g, left - 1, step]
    return olds, news, exts, np.array(prev, np.int32), np.array(label, np.int32), heads


def chain_order(prev, seed):
    """A random order of the pairs that keeps every pair behind its prev: order[k] = the pair that goes to place k."""
    rng = np.random.default_rng(seed)
    head = np.arange(len(prev))
    for i, p in enumerate(prev):
        if p >= 0:
            head[i] = head[p]
    key = np.empty(len(prev))
    idx = np.argsort(head, kind="stable")                  # the pairs chain by chain, each chain in its order
    cut = np.flatnonzero(np.diff(head[idx])) + 1
    for members in np.split(idx, cut):
        key[members] = np.sort(rng.random(len(members)))
    return np.argsort(key, kind="stable")


def reordered(order, olds, news, exts, prev, label, heads):
    """The batch with pair order[k] at place k, prev / label / heads remapped."""
    pos = np.empty(len(order), np.int64)
    pos[order] = np.arange(len(order))
    nprev = np.array([pos[prev[i]] if prev[i] >= 0 else -1 for i in order], np.int32)
    assert (nprev < np.arange(len(order))).all()
    return ([olds[i] for i in order], [news[i] for i in order], [exts[i] for i in order], nprev, label[order].copy(),
            {int(pos[i]): h for i, h in heads.items()})


def same_origins(org, bn, want):
    """Device origins (every line of every new side) against ref_blame's, origin for origin."""
    assert len(org) == bn[-1] == sum(len(w) for w in want)
    for i, w in enumerate(want):
        assert np.array_equal(org[bn[i]:bn[i + 1]], w), i


def check_blame(sc, olds, news, exts, prev, label, heads, stream=None):
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    add, rem, det, bn, org = sc.blame_pairs(a, b, prev, label, heads, stream=stream)
    want = ref_blame(*sides(a, b), prev, label, heads)
    same_origins(org, bn, want)
    padd, prem, pdet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(add, padd) and np.array_equal(rem, prem) and np.array_equal(det, pdet)
    return add, rem


def test_blame_chains():
    """Chains of length 1, 2 and several hundred, heads with and without origins, pairs on both sides of the
    k_diff_small / k_myers_trace split inside one chain."""
    olds, news, exts, prev, label, heads = chains(21, [1, 2, 1, 2, 300, 5, 40, 3])
    assert (prev >= 0).sum() > 300 and heads
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    add, rem = check_blame(sc, olds, news, exts, prev, label, heads)
    long_chain = [i for i in range(len(prev)) if prev[i] >= 0]
    assert (add + rem > 127)[long_chain].sum() > 0 and (add + rem <= 127)[long_chain].sum() > 0
    assert sc.blame_last_ms() > 0
    sc.close()


def test_blame_capacity_then_success():
    olds, news, exts, prev, label, heads = chains(5, [3, 2])
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    L = ts.lib()
    n = a.n_files
    add, rem = np.zeros(n, np.int64), np.zeros(n, np.int64)
    bo, bn = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
    mk = ts._LineMarks(ts._p(bo), ts._p(bn), None, 0, 0, None, 0, 0)
    ca, cb = a.c_struct(), b.c_struct()
    assert L.tsm_diff_pairs_marks(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), None, C.byref(mk), None) == ts.TSM_E_CAPACITY
    assert mk.n_old == bo[-1] == sum(len(sr.py_lines(f)) for f in olds) and mk.n_new == bn[-1] > 0
    zero = np.zeros(n + 1, np.int64)
    in_base = np.cumsum([0] + [len(heads.get(i, [])) for i in range(n)]).astype(np.int64)
    origin_in = np.concatenate([heads[i] for i in sorted(heads)])
    assert len(origin_in) == in_base[-1] > 0
    nl = C.c_int64()
    bad = prev.copy()
    bad[-1] = n                                             # a prev that is not earlier in the batch
    args = (ts._p(add), ts._p(rem), None)
    assert L.tsm_blame_pairs(sc._ctx, C.byref(ca), C.byref(cb), *args, ts._p(bad), ts._p(label), ts._p(origin_in), ts._p(in_base),
                             None, None, None, 0, C.byref(nl), None) == -1
    assert L.tsm_blame_pairs(sc._ctx, C.byref(ca), C.byref(cb), *args, ts._p(prev), ts._p(label), ts._p(origin_in), ts._p(zero),
                             None, None, None, 0, C.byref(nl), None) == -1   # a head range that is not its file's line count
    assert L.tsm_blame_pairs(sc._ctx, C.byref(ca), C.byref(cb), *args, ts._p(prev), ts._p(label), ts._p(origin_in), ts._p(in_base),
                             None, ts._p(bn), None, 0, C.byref(nl), None) == ts.TSM_E_CAPACITY
    assert nl.value == bn[-1]
    check_blame(sc, olds, news, exts, prev, label, heads)
    sc.close()


def test_blame_non_blocking_stream_with_another_busy():
    import torch
    olds, news, exts, prev, label, heads = chains(9, [20, 1, 6, 2])
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    s, busy = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(busy):
        torch.cuda._sleep(50_000_000)
    check_blame(sc, olds, news, exts, prev, label, heads, stream=s.cuda_stream)
    busy.synchronize()
    sc.close()
