"""GPU tests of the assertion edits (docs/SPEC.md section 17): tsm_diff_pairs_assert_edits against tsm_diff_pairs_asserts (chg
element for element) and against the numpy + C reference (tests/orc_assert_edits.py: serial marks, oracle events, serial
scores), on the C5 pairs, on every diff kernel's shapes, at the trace limit, at the hunk-key collision between pairs, at every
pattern length class of the score kernels, on one 3 000 x 3 000 hunk, at every capacity and on a non-blocking stream."""
import ctypes as C
import random

import numpy as np
import pytest

import corpus_util as cu
import edit_ref as er
import orc_assert_edits as oae
import tosemscan as ts

pytestmark = pytest.mark.gpu

TSM_E_ARG = -1                                            # include/tosemscan.h


def sides(a, b):
    return (a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext)


def check(sc, a, b, dist=None, stream=None):
    """chg equals tsm_diff_pairs_asserts; the edits equal the reference."""
    got = sc.diff_assert_edits(a, b, stream=stream)
    want = sc.diff_pairs(a, b, asserts=True)
    for g, w in zip(got[:7], want):
        assert g.dtype == w.dtype and np.array_equal(g, w)
    ed = got[7]
    ref = oae.assert_edits(*sides(a, b), dist)
    assert ed.dtype == ts.ASSERT_EDIT and np.array_equal(ed, ref)
    assert len(ed) <= min(len(got[5]), len(got[6]))
    return got


def test_assert_edits_c5():
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    ed = check(sc, a, b)[7]
    assert len(ed) > 200 and (ed["score"] < 60000).any()
    ms = sc.assert_edits_last_ms()
    assert ms[0] > 0 and ms[1] > 0 and ms[2] > 0
    sc.close()


def test_assert_edits_every_kernel():
    """Tie-heavy pairs at every k_diff_small size and left over to k_myers_trace, and block pairs with assertion lines."""
    olds, news, exts = cu.tie_heavy_pairs(7, scale=2)
    for i, (ko, kn) in enumerate(((40, 30), (3, 5), (300, 280), (2000, 2100), (1, 1))):
        o, n, _ = cu.block_pair(b"p%d" % i, (ko, 3), (kn, 4), assert_every=2)
        olds.append(o); news.append(n); exts.append(1 + i % 2)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    ed = check(sc, ts.pack(olds, exts), ts.pack(news, exts))[7]
    assert sc.diff_last_ms()[2] > 0 and len(ed) > 500
    sc.close()


def test_assert_edits_untraced_pairs():
    """Distances 23 169 and 23 170 between traced pairs: no edits there, and their neighbours keep theirs."""
    olds, news, dist = [], [], {}
    shapes = (((30,), (20,)), ((11584,), (11585,)), ((10, 10), (12, 8)), ((11585,), (11585,)), ((6,), (6,)))
    for i, s in enumerate(shapes):
        o, n, w = cu.block_pair(b"L%d" % i, *s, n_prefix=40 + i, n_suffix=30 + i, assert_every=3)
        olds.append(o); news.append(n)
        dist[i] = len(w[3]) + len(w[4])
    assert sorted(dist.values()) == [12, 40, 50, 23169, 23170]
    a, b = ts.pack(olds, [1] * 5), ts.pack(news, [1] * 5)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    add, rem, det, _, _, aev, rev, ed = check(sc, a, b, dist)
    assert det["added_assert"][1] == -1 and det["added_assert"][3] == -1
    pairs = set(aev["file"][ed["aev"]].tolist())
    assert pairs == {0, 2, 4}
    sc.close()


def test_assert_edits_hunk_key_collision():
    """Pair p ends in a mod hunk, the next pair has no kept line and pair p + 2 starts with a mod hunk: the three hunks share
    one global kept rank, and only the pair part of the key keeps them apart."""
    olds = [b"keep 0\nassert alpha_0 == 1\n", b"assert alpha_1 == 1\nassert beta_1\n", b"assert alpha_2 == 1\nkeep 2\n"]
    news = [b"keep 0\nassert alpha_0 == 2\n", b"assert alpha_1 == 2\nassert beta_1 + 1\n", b"assert alpha_2 == 2\nkeep 2\n"]
    olds.append(b"assert alpha_0 == 2\n"); news.append(b"assert alpha_0 == 1\n")     # a fourth pair with the first's text
    a, b = ts.pack(olds, [1] * 4), ts.pack(news, [1] * 4)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    got = check(sc, a, b)
    ed, aev, rev = got[7], got[5], got[6]
    assert [(int(rev["file"][e["rev"]]), int(aev["file"][e["aev"]])) for e in ed] == [(0, 0), (1, 1), (1, 1), (2, 2), (3, 3)]
    assert [(r, a_, s) for r, a_, s in er.py_batch_edits(olds, news, [1] * 4, [1] * 4)] == \
        [(int(e["rev"]), int(e["aev"]), int(e["score"])) for e in ed]
    sc.close()


def text(rng, n):
    return b"assert " + bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz_=() 0123456789") for _ in range(n - 7))


def test_assert_edits_line_lengths():
    """Stripped lengths 6 to 16 KiB, as pattern and as text: the register paths of 1, 2 and 4 words and the global path."""
    rng = random.Random(5)
    lens = [6, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2061, 16384]
    olds, news = [], []
    for i, la in enumerate(lens):
        for lb in (la, lens[(i + 1) % len(lens)], lens[i - 1]):
            base = text(rng, max(la, lb)) if max(la, lb) > 6 else b"assert"
            x = bytearray(base[:la])
            y = bytearray(base[:lb])
            for _ in range(lb // 20):                        # a few bytes changed after "assert ": similar, not equal
                y[rng.randrange(7, lb)] = 0x41 + rng.randrange(26)
            olds.append(b"k%d\n    %s\nm\n" % (i, bytes(x)))
            news.append(b"k%d\n  %s  \nm\n" % (i, bytes(y)))
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    ed = check(sc, ts.pack(olds, [1] * len(olds)), ts.pack(news, [1] * len(news)))[7]
    assert len(ed) > len(olds) // 2
    sc.close()


def test_assert_edits_one_large_hunk():
    """3 000 deleted and 3 000 inserted assertion lines in one hunk: 9 M candidates, more than the score launch has warps,
    most of them above the threshold (the kept list grows once)."""
    k = 3000
    old = b"head\n" + b"".join(b"    assert x_%04d == %d\n" % (i, i % 7) for i in range(k)) + b"tail\n"
    new = b"head\n" + b"".join(b"    assert y_%04d == %d\n" % (i, i % 5) for i in range(k)) + b"tail\n"
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    ed = check(sc, ts.pack([old], [1]), ts.pack([new], [1]))[7]
    assert len(ed) == k
    sc.close()


def test_assert_edits_capacities():
    a, b = ts.gen_pairs(0x7053454D0005, 3000, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    full = sc.diff_assert_edits(a, b)
    n_aev, n_rev, n_ed = len(full[5]), len(full[6]), len(full[7])
    assert n_ed > 0
    L = ts.lib()
    n = a.n_files
    ca, cb = a.c_struct(), b.c_struct()

    def call(ce, ck):
        add, rem = np.zeros(n, np.int64), np.zeros(n, np.int64)
        ac, rc_ = np.zeros((1, ts.K), np.int64), np.zeros((1, ts.K), np.int64)
        aev, rev, ed = np.zeros(max(ce, 1), ts.ASSERT_EVENT), np.zeros(max(ce, 1), ts.ASSERT_EVENT), np.zeros(max(ck, 1), ts.ASSERT_EDIT)
        r = ts._DiffAsserts(ts._p(ac), ts._p(rc_), ts._p(aev), ce, 0, ts._p(rev), ce, 0)
        ne = C.c_int64(0)
        rc = L.tsm_diff_pairs_assert_edits(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), None, C.byref(r), ts._p(ed), ck,
                                           C.byref(ne), None)
        return rc, r, ne.value, ed

    big = max(n_aev, n_rev)
    rc, r, ne, _ = call(big, n_ed - 1)                      # edit_cap short
    assert rc == ts.TSM_E_CAPACITY and (r.n_aev, r.n_rev, ne) == (n_aev, n_rev, n_ed)
    rc, r, ne, _ = call(min(n_aev, n_rev) - 1, n_ed)        # an event cap short
    assert rc == ts.TSM_E_CAPACITY and (r.n_aev, r.n_rev, ne) == (n_aev, n_rev, n_ed)
    rc, r, ne, ed = call(big, n_ed)
    assert rc == 0 and np.array_equal(ed[:ne], full[7])
    r0 = ts._DiffAsserts(None, None, None, 0, 0, None, 0, 0)    # both event arrays are required
    assert L.tsm_diff_pairs_assert_edits(sc._ctx, C.byref(ca), C.byref(cb), ts._p(np.zeros(n, np.int64)), ts._p(np.zeros(n, np.int64)),
                                         None, C.byref(r0), None, 0, C.byref(C.c_int64()), None) == TSM_E_ARG
    e = ts.pack([], [])
    got = sc.diff_assert_edits(e, e)
    assert got[7].size == 0 and got[5].size == 0 and not got[3].any()
    olds = [b"k\nassert a == 1\n", b"", b"x\n"]
    news = [b"k\nassert a == 2\n", b"", b"y\n"]
    got = check(sc, ts.pack(olds, [1, 1, 0]), ts.pack(news, [1, 1, 0]))
    assert len(got[7]) == 1
    check(sc, a, b)
    sc.close()


@pytest.fixture
def busy_legacy_stream():
    """A non-blocking stream while the legacy default stream sleeps on the device (as tests/test_gpu_streams.py)."""
    import torch
    s, legacy = torch.cuda.Stream(), torch.cuda.default_stream()
    assert legacy.cuda_stream == 0
    with torch.cuda.stream(legacy):
        torch.cuda._sleep(50_000_000)
    yield s.cuda_stream
    legacy.synchronize()


def test_assert_edits_non_blocking_stream_with_another_busy(busy_legacy_stream):
    rng = random.Random(3)
    olds = [b"".join(b"def test_%d():\n    assert v == %d\n" % (i, rng.randrange(3)) for i in range(k)) for k in range(1, 200, 7)]
    news = [ts.gen_edit(i, o, 4.0) for i, o in enumerate(olds)]
    a, b = ts.pack(olds, [1] * len(olds)), ts.pack(news, [1] * len(news))
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    check(sc, a, b, stream=busy_legacy_stream)
    sc.close()
