"""GPU tests of the changed assertion lines of revision pairs (docs/SPEC.md section 8; tsm_diff_pairs_asserts and
tsm_diff_resident_asserts): the device's [group][category] tables and events against the CPU reference
(tests/orc_diff_asserts.c) field for field, and added / removed / detail against tsm_diff_pairs_detail, on pairs that land
in every kernel and branch of the diff."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import corpus_util as cu
import orc
import orc_asserts
import tosemscan as ts

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 20, max_files=16, max_groups=1)
    yield s
    s.close()


def _c5_pairs(seed, n, cap, lam):
    base = ts.gen_corpus(0x7053454D0005 + seed, n, size_law=1, pinned=False)
    olds = [base.file_bytes(i)[:cap] for i in range(n)]
    news = [ts.gen_edit(1000 + seed * 7919 + i, o, lam) for i, o in enumerate(olds)]
    return olds, news


def reference(a, b, n_groups, threads=1):
    """orc_asserts over the pairs of corpora a, b, in `threads` slices (ctypes releases the GIL)."""
    n = a.n_files
    cuts = [n * t // threads for t in range(threads + 1)]

    def one(t):
        s = slice(cuts[t], cuts[t + 1])
        side = lambda c: (c.arena, c.off[s.start:s.stop + 1], c.len[s], c.ext[s], c.grp[s])
        ac, rc, aev, rev = orc_asserts.diff_pairs_asserts(side(a), side(b), n_groups)
        aev["file"] += s.start
        rev["file"] += s.start
        return ac, rc, aev, rev
    with ThreadPoolExecutor(threads) as ex:
        parts = list(ex.map(one, range(threads)))
    return (sum(p[0] for p in parts), sum(p[1] for p in parts), np.concatenate([p[2] for p in parts]),
            np.concatenate([p[3] for p in parts]))


def check(sc, a, b, threads=1):
    add, rem, det, ac, rc, aev, rev = sc.diff_pairs(a, b, asserts=True)
    dadd, drem, ddet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(add, dadd) and np.array_equal(rem, drem) and np.array_equal(det, ddet)
    wac, wrc, waev, wrev = reference(a, b, a.n_groups, threads)
    assert np.array_equal(ac, wac) and np.array_equal(rc, wrc)
    for got, want in ((aev, waev), (rev, wrev)):
        assert len(got) == len(want), (len(got), len(want))
        for f in got.dtype.names:
            bad = np.nonzero(got[f] != want[f])[0]
            assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]])
    traced = det["added_assert"] >= 0                        # per pair, the events add up to the detail's counts
    assert np.array_equal(np.bincount(aev["file"], minlength=a.n_files)[traced], det["added_assert"][traced])
    assert np.array_equal(np.bincount(rev["file"], minlength=a.n_files)[traced], det["removed_assert"][traced])
    return add, rem, det, ac, rc, aev, rev


def pack2(olds, news, exts, grp=None, n_groups=1):
    return ts.pack(olds, exts, grp, n_groups), ts.pack(news, list(exts), grp, n_groups)


def test_replaced_assertion_and_edge_cases(scanner):
    olds = [b"", b"a\n", b"a\nb\nc\n", b"a\nb\nc", b"x\n" * 100, b"same\n" * 50, b"a\nb\n", b"q\r\nr\n", b"1\n2\n3\n4\n5\n",
            b"\n\n\n", b"only old\n", b"", b"a\nb\nc\n", b"a\nb\nc\n", b"def t():\n  assert x\n  y = 1\n", b"", b"k\n" * 9,
            b"EXPECT_EQ(a, b);\nfoo\n", b"x = 1\nself.assertEqual(a, b)\ny = 2\n"]
    news = [b"", b"a\n", b"a\nc\n", b"a\nb\nc\n", b"y\n" * 70, b"same\n" * 50, b"b\na\n", b"q\nr\r\n", b"5\n4\n3\n2\n1\n",
            b"\n", b"", b"only new\nsecond\n", b"a\nc\n", b"a\nB\nc\nd\n", b"def t():\n  assert x == 2\n  y = 1\n  assert y\n",
            b"assert q\n", b"", b"foo\nEXPECT_EQ(a, b);\n", b"x = 1\nself.assertTrue(a)\ny = 2\n"]
    exts = [1] * 17 + [2, 1]
    a, b = pack2(olds, news, exts)
    _, _, det, ac, rc, aev, rev = check(scanner, a, b)
    assert rev[-1]["cat"] == 1 and aev[-1]["cat"] == 3 and rev[-1]["file"] == aev[-1]["file"] == 18   # assertEqual -> assertTrue
    assert ac.sum() == det["added_assert"].sum() > 0 and rc.sum() == det["removed_assert"].sum() > 0


@pytest.mark.parametrize("lam", [6.0, 60.0])
def test_c5_shape(scanner, lam):
    olds, news = _c5_pairs(21, 400, 65536 if lam < 10 else 20000, lam)
    a, b = pack2(olds, news, [1 + (i % 6) for i in range(400)])
    _, _, _, ac, rc, _, _ = check(scanner, a, b, threads=8)
    assert ac.sum() > 0 and rc.sum() > 0


def test_every_kernel_and_branch(scanner):
    """Pairs on both sides of every k_diff_small size (512 / D 31, 1 024 / 63, 4 096 / 63, 4 096 / 127), pairs left to
    k_myers_trace, both pure hunks (insertion only, deletion only) and one pair too far apart to trace."""
    def lines(tag, n):
        return [b"%s%05d\n" % (tag, i) for i in range(n)]
    olds, news = [], []
    for total, ds in ((250, (1, 31, 32)), (500, (63, 64)), (1300, (64, 127, 128, 200))):
        for d in ds:
            o = lines(b"assert x", total)
            keep = [l for i, l in enumerate(o) if not (i % (total // d) == 3 and i // (total // d) < d)]
            olds.append(b"".join(o)); news.append(b"".join(keep))
    for d in (16, 31, 32, 64):
        o = lines(b"y = ", 300)
        n = list(o)
        for j in range(d):
            n[5 + 4 * j] = b"EXPECT_EQ(%d, q);\n" % j
        olds.append(b"".join(o)); news.append(b"".join(n))
    for total in (510, 514, 1022, 1026, 4094, 4098, 6000):
        half = total // 2
        o = [b"first old\n"] + lines(b"assert m", half - 2) + [b"last old\n"]
        n = [b"assertEqual(first, new)\n"] + lines(b"assert m", total - half - 2) + [b"assert last_new\n"]
        olds.append(b"head\n" * 40 + b"".join(o) + b"tail\n" * 40); news.append(b"head\n" * 40 + b"".join(n) + b"tail\n" * 40)
    olds += [b"", b"assert a\n" * 3000, b"x\n" + b"assert p\n" * 70 + b"y\n", b"x\ny\n"]
    news += [b"assert b < 1\n" * 2500, b"", b"x\ny\n", b"x\n" + b"self.assertIn(q, r)\n" * 45 + b"y\n"]
    olds.append(b"".join(b"assert a%05d\n" % i for i in range(12000)))   # D = 24 000 > 23 168: not traced
    news.append(b"".join(b"assert b%05d\n" % i for i in range(12000)))
    exts = [1] * len(olds)
    a, b = pack2(olds, news, exts)
    _, _, det, _, _, aev, rev = check(scanner, a, b, threads=8)
    last = len(olds) - 1
    assert det["added_assert"][last] == -1 and last not in aev["file"] and last not in rev["file"]
    assert (aev["file"] == last - 4).sum() == 2500 and (rev["file"] == last - 3).sum() == 3000   # the two pure hunks


@pytest.mark.parametrize("n_groups", [1, 16, 17, 300])
def test_groups_of_both_sides(n_groups):
    olds, news = _c5_pairs(23, 600, 16000, 10.0)
    rng = np.random.default_rng(n_groups)
    ga = rng.integers(0, n_groups, len(olds)).astype(np.uint16)
    gb = rng.integers(0, n_groups, len(olds)).astype(np.uint16)
    exts = [1 + (i % 3) for i in range(len(olds))]
    a, b = ts.pack(olds, exts, ga, n_groups), ts.pack(news, exts, gb, n_groups)
    sc = ts.Scanner(device=0, max_arena_bytes=1 << 20, max_files=16, max_groups=1)
    _, _, _, ac, rc, _, _ = check(sc, a, b, threads=8)
    assert ac.shape == (n_groups, ts.K) and (ac.sum(axis=1) > 0).sum() > min(n_groups, 600) // 2
    with pytest.raises(ts.TsmError) as e:                   # both sides must have the same number of groups
        sc.diff_pairs(a, ts.pack(news, exts, gb, n_groups + 1), asserts=True)
    assert e.value.status == -1
    sc.diff_upload(a, b)                                     # the resident call gives the same
    got = sc.diff_resident(asserts=True)
    want = sc.diff_pairs(a, b, asserts=True)
    for x, y in zip(got, want):
        assert np.array_equal(x, y)
    sc.close()


def test_too_small_event_arrays_report_both_counts(scanner):
    import ctypes as C
    olds, news = _c5_pairs(24, 100, 30000, 20.0)
    a, b = pack2(olds, news, [1] * 100)
    add, rem, det, ac, rc, aev, rev = scanner.diff_pairs(a, b, asserts=True)
    assert len(aev) > 2 and len(rev) > 2
    got_a, got_r = np.zeros((1, ts.K), np.int64), np.zeros((1, ts.K), np.int64)
    ev1, ev2 = np.zeros(2, ts.ASSERT_EVENT), np.zeros(len(rev), ts.ASSERT_EVENT)
    r = ts._DiffAsserts(ts._p(got_a), ts._p(got_r), ts._p(ev1), 2, 0, ts._p(ev2), len(rev), 0)
    add2, rem2, det2 = np.zeros(100, np.int64), np.zeros(100, np.int64), np.zeros(100, ts.DIFF_DETAIL)
    ca, cb = a.c_struct(), b.c_struct()
    rc2 = ts.lib().tsm_diff_pairs_asserts(scanner._ctx, C.byref(ca), C.byref(cb), ts._p(add2), ts._p(rem2), ts._p(det2), C.byref(r), None)
    assert rc2 == ts.TSM_E_CAPACITY and (r.n_aev, r.n_rev) == (len(aev), len(rev))
    assert np.array_equal(got_a, ac) and np.array_equal(got_r, rc)
    assert np.array_equal(add2, add) and np.array_equal(rem2, rem) and np.array_equal(det2, det)


def test_real_c1_test_files_edited(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    keep = [i for i, f in enumerate(files) if 0 < len(f) < 200000][:1500]
    olds = [files[i] for i in keep]
    news = [ts.gen_edit(77 + i, f, 6.0) for i, f in enumerate(olds)]
    a, b = pack2(olds, news, [int(exts[i]) for i in keep])
    _, _, _, ac, rc, _, _ = check(scanner, a, b, threads=16)
    assert ac.sum() > 0 and rc.sum() > 0


def test_full_c5_pairs():
    n = 50000
    a, b = ts.gen_pairs(0x7053454D0005, n)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    _, _, det, ac, rc, _, _ = check(sc, a, b, threads=max(1, min(64, os.cpu_count() or 1)))
    assert ac.sum() > 0 and rc.sum() > 0
    sc.close()
