"""GPU tests of the lexical test-smell churn (docs/SPEC.md section 26): tsm_diff_pairs_smells_lexical against tsm_diff_pairs_smells,
tsm_smells_lexical on each side and the numpy reference tests/orc_lexsmell_churn.py (serial marks, serial smells and lexical
smells) on the C5 pairs, a planted history, every diff kernel's shapes, untraced pairs, bodies of 1 to 70 000 lines, one test
whose Assertion Roulette a single edit toggles on 20 000 kept lines, more tests than the launch has warps, an empty batch,
capacity retries, NULL outputs and a non-blocking stream."""
import ctypes as C
import random

import numpy as np
import pytest

import corpus_util as cu
import lexsmell_ref as lr
import orc_lexsmell_churn as olc
import spec_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu

KEYS = ("old_cases", "new_cases", "old_tests", "new_tests", "old_churn", "new_churn")
LKEYS = ("old_lex", "new_lex", "old_lex_churn", "new_lex_churn")


def sides(a, b):
    return (a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext)


def same(got, want, k):
    assert got.dtype == want.dtype and len(got) == len(want), k
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%s differs at %s: %s vs %s" % (k, bad[:3], got[bad[:3]], want[bad[:3]])


def check(sc, a, b, dist=None, stream=None, cap=None):
    """Every output equals the calls it extends and the reference; returns the result."""
    r = sc.diff_smells_lexical(a, b, stream=stream, cap=cap)
    d = sc.diff_smells(a, b)
    for k in ("added", "removed", "detail") + KEYS:
        same(r[k], d[k], k)
    for side, c in (("old", a), ("new", b)):
        same(r[side + "_lex"], sc.smells_lexical(c)["lex"], side + "_lex")
    want = olc.diff_smells_lexical(*sides(a, b), dist)
    for k in KEYS + LKEYS:
        same(r[k], want[k].astype(r[k].dtype), k)
    return r


def test_lexsmell_churn_c5():
    """All 50 000 pairs of BASELINE config C5."""
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, a, b)
    assert len(r["new_tests"]) > 10_000 and (r["new_lex_churn"]["churned"].sum(1) > 0).sum() > 100
    sc.close()


def test_lexsmell_churn_planted_history():
    """Section-25 planted test files as old sides and gen_edit(lambda = 6) of each as new sides: every event kind of every lexical
    smell, and more tests than the churn launch has warps."""
    olds, exts = lr.planted_corpus(23, 8_000)
    news = [ts.gen_edit(i, o, 6.0) for i, o in enumerate(olds)]
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, a, b)
    assert len(r["new_tests"]) > 132 * 8 * 8
    assert (r["new_lex_churn"]["churned"].sum(0)[:4] > 0).all() and (r["old_lex_churn"]["churned"].sum(0)[:4] > 0).all()
    rows = olc.churn_rows(r, olds, news, [int(x) for x in exts], [int(x) for x in exts])
    events = {(x[1], x[5]) for rs in rows.values() for x in rs if x[4] in lr.LSMELLS}
    assert {("A", "introduced"), ("D", "removed"), ("M", "introduced"), ("M", "removed"), ("M", "changed")} <= events
    sc.close()


def test_lexsmell_churn_every_kernel():
    """Tie-heavy pairs with test headers and lexically smelly lines at every k_diff_small size and left over to k_myers_trace."""
    olds, news, exts = cu.tie_heavy_pairs(11, scale=2)
    sub = {b"x\n": b"def test_x() {\n", b"x\r\n": b"TEST(S, X) {\r\n", b"{\n": b"    assert v == 7 {\n"}
    olds = [b"".join(sub.get(l, l) for l in o.splitlines(keepends=True)) for o in olds]
    news = [b"".join(sub.get(l, l) for l in n.splitlines(keepends=True)) for n in news]
    d = [sum(sr.py_diff_files(o, n, x, x)[:2]) for o, n, x in zip(olds, news, exts)]
    assert max(d) > 127 and any(0 < x <= 31 for x in d)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, exts), ts.pack(news, exts))
    assert sc.diff_last_ms()[2] > 0 and r["new_lex_churn"]["churned"].sum() > 0 and len(r["old_tests"]) > 500
    sc.close()


def test_lexsmell_churn_untraced_pairs():
    """Distances 23 169 and 23 170, just above the trace limit, between traced pairs: the whole middle is churned."""
    def body(tag, k):
        return [b"    assert %s_%d == 3\n" % (tag, j) if j % 3 else b"    assert %s_%d, 'm'\n" % (tag, j) for j in range(k)]
    olds, news, dist = [], [], {}
    for i, (ko, kn) in enumerate(((30, 20), (11584, 11585), (11585, 11585), (40, 41))):
        head = [b"def test_%d():\n" % i, b"    assert v == 7\n"]
        o = head + body(b"o%d" % i, ko) + [b"    assert v == 7\n"]
        n = head + body(b"n%d" % i, kn) + [b"    assert v == 7\n"]
        olds.append(b"".join(o)); news.append(b"".join(n))
        dist[i] = ko + kn
    a, b = ts.pack(olds, [1] * 4), ts.pack(news, [1] * 4)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, a, b, dist)
    assert (r["detail"]["added_assert"] == -1).sum() == 2
    mg = ts.LSMELLS.index("magic_number")
    c = r["new_lex_churn"][1]
    assert c["churned"][mg] == c["instances"][mg] - 2 > 7000          # all but the kept `assert v == 7` lines
    sc.close()


def test_lexsmell_churn_body_lengths():
    """Bodies of 1, 31, 32, 33 and 70 000 lines with magic numbers on the first and last line of the body and on the 32-line
    seams, edited at those places; and 20 000 one-line tests, every hundredth edited."""
    olds, news = [], []
    for k in (1, 31, 32, 33, 70_000):
        body = [b"    assert v == %d\n" % j if j in (0, 30, 31, 32, k - 2) else b"    v_%d = 1\n" % j for j in range(k - 1)]
        o = [b"import os\n", b"def test_%d():\n" % k] + body + [b"def test_after():\n", b"    pass\n"]
        n = list(o)
        for j in (2, 32, 33, k):
            if j < len(n) - 2:
                n[j] = b"    with open(f) as g: assert g\n"
        olds.append(b"".join(o)); news.append(b"".join(n))
    olds.append(b"".join(b"def test_%d(): assert x == 1\n" % i for i in range(20_000)))
    news.append(b"".join(b"def test_%d(): assert x == %s\n" % (i, b"1" if i % 100 else b"ONE") for i in range(20_000)))
    exts = [1] * len(olds)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, exts), ts.pack(news, exts))
    assert {1, 31, 32, 33, 70_000} <= set(r["new_tests"]["body_lines"].tolist()) and len(r["new_tests"]) > 20_000
    sc.close()


def test_lexsmell_churn_roulette_toggled_on_20000_kept_lines():
    """One test of 20 000 unexplained assertions; a single inserted line that opens a string makes every one of them string
    content (the old side removes 20 000 instances on kept lines), and the reverse pair introduces them."""
    body = b"".join(b"    assert f(%d)\n" % j for j in range(20_000))
    plain = b"def test_many():\n" + body
    quoted = b'def test_many():\n    s = """\n' + body
    a, b = ts.pack([plain, quoted], [1, 1]), ts.pack([quoted, plain], [1, 1])
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, a, b)
    ar = ts.LSMELLS.index("assertion_roulette")
    assert r["old_lex_churn"]["churned"][0][ar] == r["old_lex_churn"]["instances"][0][ar] == 20_000
    assert r["new_lex_churn"]["churned"][1][ar] == r["new_lex_churn"]["instances"][1][ar] == 20_000
    assert r["new_lex_churn"]["instances"][0][ar] == 0 and r["added"][0] == 1
    sc.close()


def test_lexsmell_churn_capacity_null_outputs_and_empty_batch():
    a, b = ts.gen_pairs(0x7053454D0005, 300, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    full = check(sc, a, b)
    assert len(full["old_tests"]) > 0 and len(full["new_tests"]) > 0
    assert all(np.array_equal(sc.diff_smells_lexical(a, b, cap=c)[k], full[k]) for c in (1, 10**6) for k in KEYS + LKEYS)
    for _ in range(2):                                               # repeated calls
        assert all(np.array_equal(sc.diff_smells_lexical(a, b)[k], full[k]) for k in KEYS + LKEYS)
    L = ts.lib()
    n = a.n_files
    add, rem = np.zeros(n, np.int64), np.zeros(n, np.int64)
    ca, cb = a.c_struct(), b.c_struct()

    def call(r, x):
        add[:] = 0
        return L.tsm_diff_pairs_smells_lexical(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), None, C.byref(r),
                                               None if x is None else C.byref(x), None)

    t = ts._DiffSmells(ts._DiffCases(None, 0, 0, None, 0, 0), None, None, 0, 0, None, None, 0, 0)
    assert call(t, None) == -1                                      # TSM_E_ARG: lex is required
    assert call(t, ts._DiffLexSmells(None, None, None, None)) == 0 and add.any()   # every output NULL: nothing to size
    counts = (len(full["old_cases"]), len(full["new_cases"]), len(full["old_tests"]), len(full["new_tests"]))
    assert (t.cases.n_old, t.cases.n_new, t.n_old_tests, t.n_new_tests) == counts
    bufs = {k: np.zeros(len(full[k]), full[k].dtype) for k in KEYS + LKEYS}

    def structs(p, caps):
        return (ts._DiffSmells(ts._DiffCases(p["old_cases"], caps[0], 0, p["new_cases"], caps[1], 0), p["old_tests"], p["old_churn"],
                               caps[2], 0, p["new_tests"], p["new_churn"], caps[3], 0),
                ts._DiffLexSmells(p["old_lex"], p["old_lex_churn"], p["new_lex"], p["new_lex_churn"]))

    for short in range(4):                                           # one cap one short: no diff runs
        caps = [c - (i == short) for i, c in enumerate(counts)]
        r, x = structs({k: ts._p(bufs[k]) for k in KEYS + LKEYS}, caps)
        assert call(r, x) == ts.TSM_E_CAPACITY and not add.any()
        assert (r.cases.n_old, r.cases.n_new, r.n_old_tests, r.n_new_tests) == counts
    for side, i in (("old", 2), ("new", 3)):                         # a short test cap with only the lexical outputs given
        caps = [c - (j == i) for j, c in enumerate(counts)]
        p = {k: (ts._p(bufs[k]) if k.startswith(side) and k in LKEYS else None) for k in KEYS + LKEYS}
        r, x = structs(p, caps)
        assert call(r, x) == ts.TSM_E_CAPACITY and not add.any()
    for skip in KEYS + LKEYS:                                        # each output NULL in turn
        for k in bufs:
            bufs[k][...] = 0
        r, x = structs({k: (None if k == skip else ts._p(bufs[k])) for k in KEYS + LKEYS}, counts)
        assert call(r, x) == 0
        for k in KEYS + LKEYS:
            assert np.array_equal(bufs[k], full[k]) != (k == skip), (skip, k)
    e = ts.pack([], [])
    assert all(sc.diff_smells_lexical(e, e)[k].size == 0 for k in KEYS + LKEYS)
    sc.close()


def test_lexsmell_churn_non_blocking_stream_with_another_busy():
    import torch
    rng = random.Random(5)
    olds = [b"".join(b"def test_%d():\n    assert v == %d\n    assert w\n" % (i, rng.randrange(3)) for i in range(k))
            for k in range(1, 200, 7)]
    news = [ts.gen_edit(i, o, 4.0) for i, o in enumerate(olds)]
    a, b = ts.pack(olds, [1] * len(olds)), ts.pack(news, [1] * len(news))
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    s, legacy = torch.cuda.Stream(), torch.cuda.default_stream()
    assert legacy.cuda_stream == 0
    with torch.cuda.stream(legacy):
        torch.cuda._sleep(50_000_000)
    check(sc, a, b, stream=s.cuda_stream)
    legacy.synchronize()
    sc.close()
