"""GPU tests of the test-case churn (docs/SPEC.md section 16): every record of tsm_diff_pairs_cases against the numpy reference
(tests/orc_cases.py: serial marks, oracle events) on the C5 pairs, on every diff kernel's shapes, at the trace limit, on cases
of 1 to 70 000 lines, with headers in the common prefix and suffix and on the first and last line, without headers, with more
cases than the reduce launch has warps, after a capacity error and on a non-blocking stream."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

import corpus_util as cu
import orc_cases
import spec_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu


def sides(a, b):
    return (a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext)


def check(sc, a, b, dist=None, stream=None):
    """Device records equal the reference; added / removed / detail equal tsm_diff_pairs_detail."""
    add, rem, det, oc, nc = sc.diff_cases(a, b, stream=stream)
    woc, wnc = orc_cases.diff_cases(*sides(a, b), dist)
    assert oc.dtype == ts.CASE and len(oc) == len(woc) and len(nc) == len(wnc)
    assert np.array_equal(oc, woc) and np.array_equal(nc, wnc)
    padd, prem, pdet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(add, padd) and np.array_equal(rem, prem) and np.array_equal(det, pdet)
    return oc, nc


def with_headers(data: bytes, every=40) -> bytes:
    """data with some of its lines made headers in every language (`def` for PY, `test` and `{` for CJ), chosen by content so
    that equal lines stay equal and different lines stay different."""
    out = []
    for ln in data.split(b"\n"):
        out.append(b"def test_h() { " + ln if ln and zlib.crc32(ln) % every == 0 else ln)
    return b"\n".join(out)


def test_cases_c5():
    """All 50 000 pairs of BASELINE config C5 (PY, CC and Java headers about every 48 lines): more cases than the reduce
    launch has warps."""
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    oc, nc = check(sc, a, b)
    assert len(oc) > 200_000 and (nc["match"] >= 0).sum() > 150_000 and (nc["n_changed"] > 0).sum() > 10_000
    assert len(nc) > 132 * 8 * 8 * 4
    sc.close()


def test_cases_every_kernel():
    """Tie-heavy pairs with header lines at every k_diff_small size and left over to k_myers_trace, pure hunks, empty files."""
    olds, news, exts = cu.tie_heavy_pairs(7, scale=2)
    sub = {b"x\n": b"def test_x() {\n", b"x\r\n": b"def test_x() {\r\n"}
    olds = [b"".join(sub.get(l, l) for l in o.splitlines(keepends=True)) for o in olds]
    news = [b"".join(sub.get(l, l) for l in n.splitlines(keepends=True)) for n in news]
    for i, (ko, kn) in enumerate(((40, 0), (0, 33), (3000, 0), (0, 2500))):
        o, n, _ = cu.block_pair(b"p%d" % i, (ko,), (kn,))
        olds.append(with_headers(o, 7)); news.append(with_headers(n, 7)); exts.append(1)
    olds += [b"", b"def test_a():\n", b""]; news += [b"def test_b():\n", b"", b""]; exts += [1, 1, 1]
    d = [sum(sr.py_diff_files(o, n, x, x)[:2]) for o, n, x in zip(olds, news, exts)]
    assert max(d) > 127 and any(0 < x <= 31 for x in d)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    oc, nc = check(sc, ts.pack(olds, exts), ts.pack(news, exts))
    assert sc.diff_last_ms()[2] > 0 and len(oc) > 1000 and (nc["match"] >= 0).any() and (nc["match"] < 0).any()
    sc.close()


def test_cases_untraced_pairs():
    """Distances 23 169 and 23 170, just above the trace limit, beside a traced pair: untraced pairs count every line of their
    middle as changed."""
    olds, news, dist = [], [], {}
    for i, s in enumerate((((30,), (20,)), ((11584,), (11585,)), ((11585,), (11585,)), ((6000, 5585), (6000, 5585)))):
        o, n, w = cu.block_pair(b"L%d" % i, *s, n_prefix=40 + i, n_suffix=30 + i)
        olds.append(with_headers(o)); news.append(with_headers(n))
        dist[i] = len(w[3]) + len(w[4])
    assert sorted(dist.values()) == [50, 23169, 23170, 23170]
    a, b = ts.pack(olds, [1] * 4), ts.pack(news, [2] * 4)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    oc, nc = check(sc, a, b, dist)
    assert (oc["n_changed"] > 0).sum() > 400 and (nc["n_changed"] > 0).sum() > 400
    sc.close()


def test_case_lengths_and_header_places():
    """Cases of 1, 31, 32, 33 and 70 000 lines, edited on their first and last line; headers in the common prefix and suffix
    and on a file's first and last line (also unterminated); files with no header; many one-line cases."""
    body = lambda tag, k: [b"    %s_%d = 1\n" % (tag, j) for j in range(k)]
    olds, news, exts = [], [], []
    for k in (1, 31, 32, 33, 70_000):
        case = [b"def test_%d():\n" % k] + body(b"b%d" % k, k - 1)
        for edit in ("first", "last", "none"):
            o = [b"import os\n"] + case + [b"def test_after():\n", b"    pass\n"]
            n = list(o)
            if edit == "first":
                n[1] = b"def test_%d(self):\n" % k
            elif edit == "last":
                n[k] = b"    assert changed\n"
            olds.append(b"".join(o)); news.append(b"".join(n)); exts.append(1)
    pre = b"TEST(S, Pre) {\n}\n"
    suf = b"TEST(S, Suf) {\n  EXPECT_TRUE(x);\n}"                      # header near the unterminated last line
    olds.append(pre + b"int a;\n" + suf); news.append(pre + b"int b;\nTEST(S, Mid) {\n" + suf); exts.append(2)
    olds.append(b"a\nb\nvoid test_last() {"); news.append(b"a\nc\nvoid test_last() {"); exts.append(2)
    olds.append(b"void test_first() {\nx\n"); news.append(b"void test_first() {\ny\n"); exts.append(2)
    olds.append(b"no header\nhere\n"); news.append(b"no header\nthere\n"); exts.append(4)
    olds.append(b"".join(b"def t%d(): pass\n" % i for i in range(20_000)))
    news.append(b"".join(b"def t%d(): pass\n" % i for i in range(0, 20_000, 3))); exts.append(1)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    oc, nc = check(sc, ts.pack(olds, exts), ts.pack(news, exts))
    assert nc["n_lines"].max() == 70_000 and {1, 31, 32, 33} <= set(nc["n_lines"].tolist())
    assert not ((oc["pair"] == len(olds) - 2).any() or (nc["pair"] == len(olds) - 2).any())
    sc.close()


def test_cases_capacity_then_success():
    a, b = ts.gen_pairs(0x7053454D0005, 300, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    L = ts.lib()
    n = a.n_files
    add, rem = np.zeros(n, np.int64), np.zeros(n, np.int64)
    ca, cb = a.c_struct(), b.c_struct()
    r = ts._DiffCases(None, 0, 0, None, 0, 0)
    assert L.tsm_diff_pairs_cases(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), None, C.byref(r), None) == ts.TSM_E_CAPACITY
    woc, wnc = orc_cases.diff_cases(*sides(a, b))
    assert r.n_old == len(woc) > 0 and r.n_new == len(wnc) > 0 and not add.any()       # no diff ran
    oc, nc = np.zeros(r.n_old, ts.CASE), np.zeros(r.n_new, ts.CASE)
    r2 = ts._DiffCases(ts._p(oc), r.n_old, 0, ts._p(nc), r.n_new - 1, 0)
    assert L.tsm_diff_pairs_cases(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), None, C.byref(r2), None) == ts.TSM_E_CAPACITY
    r3 = ts._DiffCases(ts._p(oc), r.n_old, 0, ts._p(nc), r.n_new, 0)
    assert L.tsm_diff_pairs_cases(sc._ctx, C.byref(ca), C.byref(cb), ts._p(add), ts._p(rem), None, C.byref(r3), None) == 0
    assert np.array_equal(oc, woc) and np.array_equal(nc, wnc) and add.any()
    e = ts.pack([], [])
    assert sc.diff_cases(e, e)[3].size == 0
    check(sc, a, b)
    sc.close()


def test_cases_non_blocking_stream_with_another_busy():
    import torch
    rng = random.Random(3)
    olds = [b"".join(b"def test_%d():\n    v = %d\n" % (i, rng.randrange(3)) for i in range(k)) for k in range(1, 200, 7)]
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
