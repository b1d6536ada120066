"""CPU tests of the reference of the changed assertion lines (tests/orc_diff_asserts.c, docs/SPEC.md section 8): hand
cases, and on C5-shaped fuzz the two invariants that tie it to the existing oracle - per pair the category counts add up
to the detail's added_assert / removed_assert, and every event is the scan's event of that line."""
import ctypes as C

import numpy as np

import orc
import orc_asserts
import tosemscan as ts

AEQ, ATRUE = 1, 3            # category ids of assertEqual, assertTrue (SPEC section 6)


def sides(olds, news, exts, grp_old=None, grp_new=None):
    a, b = orc.pack(olds), orc.pack(news)
    e = np.asarray(exts, np.uint8)
    return a + (e, grp_old), b + (e.copy(), grp_new)


def test_replaced_assertion_changes_category():
    old = b"class T:\n    def test_a(self):\n        x = 1\n        self.assertEqual(a, b)\n        return x\n"
    new = b"class T:\n    def test_a(self):\n        x = 1\n        self.assertTrue(a)\n        return x\n"
    a, b = sides([old], [new], [1])
    ac, rc, aev, rev = orc_asserts.diff_pairs_asserts(a, b)
    assert {int(k): int(v) for k, v in enumerate(rc[0]) if v} == {AEQ: 1}
    assert {int(k): int(v) for k, v in enumerate(ac[0]) if v} == {ATRUE: 1}
    assert len(aev) == len(rev) == 1
    assert new[aev[0]["stmt_off"]:aev[0]["stmt_off"] + aev[0]["stmt_len"]] == b"self.assertTrue"
    assert old[rev[0]["stmt_off"]:rev[0]["stmt_off"] + rev[0]["stmt_len"]] == b"self.assertEqual"
    assert rev[0]["line_off"] == old.index(b"        self.assertEqual")


def test_hand_cases():
    olds = [b"a\nassert x\nb\n", b"", b"assert p == 1\nassert q\n", b"EXPECT_EQ(a, b);\nz\n", b"assert x\n", b"k\nassert y < 2\n"]
    news = [b"a\nb\n", b"assert z != 3\nassert w\n", b"", b"z\nEXPECT_EQ(a, b);\n", b"assert x\n", b"k\nassert y < 2\nv\n"]
    a, b = sides(olds, news, [1, 1, 1, 2, 0, 1], np.arange(6, dtype=np.uint16), np.arange(6, dtype=np.uint16))
    ac, rc, aev, rev = orc_asserts.diff_pairs_asserts(a, b, n_groups=6)
    assert rc[0].sum() == 1 and rc[0][ATRUE] == 1 and ac[0].sum() == 0           # deleted bare assert
    assert ac[1][2] == 1 and ac[1][ATRUE] == 1 and rc[1].sum() == 0              # pure insertion: both lines (!= -> assertNotEqual)
    assert rc[2][AEQ] == 1 and rc[2][ATRUE] == 1 and ac[2].sum() == 0            # pure deletion
    assert rc[3][AEQ] == 1 and ac[3][AEQ] == 1                                   # moved line: deleted and inserted
    assert ac[4].sum() == rc[4].sum() == 0 and ac[5].sum() == rc[5].sum() == 0   # unchanged / ext 0 / no assertion changed
    assert sorted(aev["file"].tolist()) == aev["file"].tolist()


def _c5_pairs(seed, n, cap, lam):
    base = ts.gen_corpus(0x7053454D0005 + seed, n, size_law=1, pinned=False)
    olds = [base.file_bytes(i)[:cap] for i in range(n)]
    news = [ts.gen_edit(1000 + seed * 7919 + i, o, lam) for i, o in enumerate(olds)]
    return olds, news


def _events_by_line(res):
    return {(int(e["file"]), int(e["line_off"])): e for e in res["assert_events"]}


def check_invariants(olds, news, exts):
    n = len(olds)
    g = np.arange(n, dtype=np.uint16)                       # one group per pair: the table rows are per-pair counts
    a, b = sides(olds, news, exts, g, g)
    ac, rc, aev, rev = orc_asserts.diff_pairs_asserts(a, b, n_groups=n)
    _, _, det = orc.diff_pairs_detail(a[:4], b[:4])
    assert np.array_equal(ac.sum(axis=1), det["added_assert"]) and np.array_equal(rc.sum(axis=1), det["removed_assert"])
    for ev, side, counts in ((aev, b, ac), (rev, a, rc)):
        scan = _events_by_line(orc.scan(side[0], side[1], side[2], side[3], np.zeros(n, np.uint16), 1))
        keys = [(int(e["file"]), int(e["line_off"])) for e in ev]
        assert keys == sorted(set(keys))                        # canonical order, each line once
        for e in ev:
            assert e.tobytes() == scan[(int(e["file"]), int(e["line_off"]))].tobytes()
        assert np.array_equal(np.bincount(ev["file"], minlength=n), counts.sum(axis=1))
    return ac, rc


def test_invariants_on_c5_shaped_fuzz():
    olds, news = _c5_pairs(11, 120, 65536, 6.0)
    ac, rc = check_invariants(olds, news, [1 + (i % 3) for i in range(120)])
    assert ac.sum() > 0 and rc.sum() > 0
    olds, news = _c5_pairs(12, 40, 20000, 60.0)
    check_invariants(olds, news, [1] * 40)


def test_untraced_pair_contributes_nothing():
    old = b"".join(b"assert a%05d\n" % i for i in range(12000))
    new = b"".join(b"assert b%05d\n" % i for i in range(12000))
    a, b = sides([old, b"assert q\n"], [new, b""], [1, 1])
    ac, rc, aev, rev = orc_asserts.diff_pairs_asserts(a, b)
    assert ac.sum() == 0 and rc.sum() == 1 and len(aev) == 0 and rev["file"].tolist() == [1]


def test_struct_layouts():
    S = ts._DiffAsserts
    assert C.sizeof(S) == 64
    assert [getattr(S, f).offset for f, _ in S._fields_] == [0, 8, 16, 24, 32, 40, 48, 56]
    assert ts.ASSERT_EVENT == orc.ASSERT_EVENT and ts.ASSERT_EVENT.itemsize == 32
    hdr = open(orc.ROOT + "/include/tosemscan.h").read()
    body = hdr[hdr.index("typedef struct tsm_diff_asserts"):hdr.index("} tsm_diff_asserts;")]
    names = [w for w in ("added_counts", "removed_counts", "aev", "aev_cap", "n_aev", "rev", "rev_cap", "n_rev") if w in body]
    assert names == [f for f, _ in S._fields_]
    assert "tsm_diff_pairs_asserts" in ts.SYMBOLS and "tsm_diff_resident_asserts" in ts.SYMBOLS
