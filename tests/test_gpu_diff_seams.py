"""GPU tests of the revision diff (docs/SPEC.md section 8) on the paths its other tests do not reach: tie-heavy scripts in
every kernel size, left-over pairs traced in more than one batch, the trace limit, sides with more lines than the first
staging guess, exclusive scans of more than 256 tiles, 65 535 groups, and the resident pair across other calls on the same
context.  The references are the oracle (oracle/orc.c), the changed-assertion reference (tests/orc_diff_asserts.c), the
plain-Python restatement of section 8 (tests/spec_ref.py) and closed forms of shapes whose script is unique.  Every test
asserts that its shapes reach the path it is about, from the formulas the host uses."""
import os
import random

import numpy as np
import pytest

import corpus_util as cu
import orc
import spec_ref as sr
import tosemscan as ts
from test_gpu_diff_asserts import check

pytestmark = pytest.mark.gpu
THREADS = max(1, min(16, os.cpu_count() or 1))
TRACE_MAX_INTS = 1 << 28                     # rows of V one batch of k_myers_trace holds (tsm_device.cuh)
TRACE_MAX_D = 23168                          # the largest distance whose rows fit: (D+1)(D+2)/2 <= 2^28
SIZES = ((512, 31), (1024, 63), (4096, 63), (4096, 127))   # k_diff_small: (lines of both middles, distance)


def trace_ints(d):
    return (d + 1) * (d + 2) // 2


def pack2(olds, news, exts, grp=None, n_groups=1):
    return ts.pack(olds, exts, grp, n_groups), ts.pack(news, list(exts), grp, n_groups)


def kernel_class(old, new, ext):
    """Which kernel finishes the pair: 1-4 = the k_diff_small size, 5 = k_myers / k_myers_trace."""
    a = [r[0] for r in sr.py_line_records(old, ext)]
    b = [r[0] for r in sr.py_line_records(new, ext)]
    pre = 0
    while pre < len(a) and pre < len(b) and a[pre] == b[pre]:
        pre += 1
    suf = 0
    while suf < len(a) - pre and suf < len(b) - pre and a[-1 - suf] == b[-1 - suf]:
        suf += 1
    n, m = len(a) - pre - suf, len(b) - pre - suf
    if n == 0 or m == 0:
        return 1
    r = sr.py_diff_script(a, b, [0] * len(a), [0] * len(b))
    d = r[0] + r[1]
    return next((i + 1 for i, (h, dc) in enumerate(SIZES) if n + m <= h and d <= dc), 5)


def changed_lines(olds, news, exts, refs):
    """(file, line_off) of the inserted and of the deleted assertion lines by the reference scripts."""
    ins, dels = [], []
    for i, (o, n, x, r) in enumerate(zip(olds, news, exts, refs)):
        fo, fn = [t[2] for t in sr.py_line_records(o, x)], [t[2] for t in sr.py_line_records(n, x)]
        so, sn = sr.py_line_starts(o), sr.py_line_starts(n)
        dels += [(i, so[j]) for j in r[7] if fo[j]]
        ins += [(i, sn[j]) for j in r[8] if fn[j]]
    return ins, dels


def keys(ev):
    return [(int(f), int(o)) for f, o in zip(ev["file"], ev["line_off"])]


def assert_detail(det, want):
    for f in det.dtype.names:
        bad = np.nonzero(det[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], det[bad[:5]], want[bad[:5]])


def check_all(sc, olds, news, exts, refs=None, grp=None, n_groups=1, threads=THREADS):
    """Device against the oracle (added, removed, detail), orc_asserts (tables, events) and, given `refs`, py_diff_script;
    detail=False too.  Returns the asserts=True result."""
    a, b = pack2(olds, news, exts, grp, n_groups)
    res = check(sc, a, b, threads)
    add, rem, det = res[:3]
    wadd, wrem, wdet = orc.diff_pairs_detail((a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext))
    assert np.array_equal(add, wadd) and np.array_equal(rem, wrem)
    assert_detail(det, wdet)
    if refs is not None:
        got = [(int(x), int(y), *(int(d[f]) for f in det.dtype.names)) for x, y, d in zip(add, rem, det)]
        assert got == [r[:7] for r in refs]
        ins, dels = changed_lines(olds, news, exts, refs)
        assert keys(res[5]) == ins and keys(res[6]) == dels
    plain = sc.diff_pairs(a, b)
    assert np.array_equal(plain[0], add) and np.array_equal(plain[1], rem)
    return res


def test_tie_heavy_scripts_at_every_size():
    olds, news, exts = cu.tie_heavy_pairs(5, scale=2)
    classes = [kernel_class(o, n, x) for o, n, x in zip(olds, news, exts)]
    assert all(classes.count(c) >= 3 for c in range(1, 6)), [classes.count(c) for c in range(1, 6)]
    refs = [sr.py_diff_files(o, n, x, x) for o, n, x in zip(olds, news, exts)]
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    res = check_all(sc, olds, news, exts, refs)
    sc.diff_pairs(*pack2(olds, news, exts), detail=True)
    assert sc.diff_last_ms()[2] > 0                         # the left-over kernels ran
    assert res[3].sum() == sum(r[5] for r in refs) > 100 and res[4].sum() == sum(r[6] for r in refs) > 100
    sc.close()


def closed_form(olds, news, exts, wants, traced):
    """added, removed, detail and changed lines of block_pair shapes; an untraced pair is one hunk with -1 / -1."""
    add, rem = np.zeros(len(olds), np.int64), np.zeros(len(olds), np.int64)
    det = np.zeros(len(olds), ts.DIFF_DETAIL)
    ins, dels = [], []
    for i, (o, n, x, w) in enumerate(zip(olds, news, exts, wants)):
        fo, fn = [t[2] for t in sr.py_line_records(o, x)], [t[2] for t in sr.py_line_records(n, x)]
        so, sn = sr.py_line_starts(o), sr.py_line_starts(n)
        add[i], rem[i] = len(w[4]), len(w[3])
        if traced[i]:
            det[i] = (w[0], w[1], w[2], sum(fn[j] for j in w[4]), sum(fo[j] for j in w[3]))
            dels += [(i, so[j]) for j in w[3] if fo[j]]
            ins += [(i, sn[j]) for j in w[4] if fn[j]]
        else:
            det[i] = (int(add[i] > 0 and rem[i] == 0), int(rem[i] > 0 and add[i] == 0), int(add[i] > 0 and rem[i] > 0), -1, -1)
    return add, rem, det, ins, dels


def scan_events(corpus, lines):
    """The events orc_scan gives the (file, line_off) in `lines` when it scans the corpus: what a changed line's event is."""
    ev = orc.scan(corpus.arena, corpus.off, corpus.len, corpus.ext, corpus.grp, corpus.n_groups)["assert_events"]
    want = set(lines)
    return ev[np.array([k in want for k in keys(ev)], bool)] if len(ev) else ev


def check_closed_form(olds, news, exts, wants, grp, n_groups):
    """The device (fresh contexts) against the closed form, the scan's events of the changed lines and orc.diff_pairs."""
    d = np.array([len(w[3]) + len(w[4]) for w in wants])
    traced = d <= TRACE_MAX_D
    add, rem, det, ins, dels = closed_form(olds, news, exts, wants, traced)
    a, b = pack2(olds, news, exts, grp, n_groups)
    lcs_add, lcs_rem = orc.diff_pairs((a.arena, a.off, a.len), (b.arena, b.off, b.len))
    assert np.array_equal(lcs_add, add) and np.array_equal(lcs_rem, rem)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    gadd, grem, gdet = sc.diff_pairs(a, b, detail=True)
    assert np.array_equal(gadd, add) and np.array_equal(grem, rem)
    assert_detail(gdet, det)
    assert sc.diff_last_ms()[2] > 0
    sc.close()
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    gadd, grem, gdet, ac, rc, aev, rev = sc.diff_pairs(a, b, asserts=True)
    sc.close()
    assert np.array_equal(gadd, add) and np.array_equal(grem, rem)
    assert_detail(gdet, det)
    assert keys(aev) == ins and keys(rev) == dels
    wa, wr = scan_events(b, ins), scan_events(a, dels)
    assert np.array_equal(aev, wa) and np.array_equal(rev, wr)
    for got, ev, side in ((ac, wa, b), (rc, wr, a)):
        want = np.zeros((n_groups, ts.K), np.int64)
        np.add.at(want, (side.grp[ev["file"]], ev["cat"]), 1)
        assert np.array_equal(got, want)
    return traced


def test_trace_batches():
    """Left-over pairs whose rows of V need more than 2^28 ints together: k_myers_trace runs in batches, each with its
    own first pair and its own slice of trace_base.  Pairs of D ~ 4 800 (one warp each), small left-over pairs and one
    untraced pair between them."""
    rng = random.Random(11)
    olds, news, wants = [], [], []
    for i in range(30):
        if i % 3 == 0:                                      # disjoint unique lines: one mod hunk
            ob, nb = (2400 + rng.randrange(-90, 90),), (2400 + rng.randrange(-90, 90),)
        else:                                               # blocks between common lines: one hunk per block pair
            total = 4800 + rng.randrange(-150, 150)
            cut = sorted(rng.sample(range(1, total), 7)) + [total]
            sizes = [y - x for x, y in zip([0] + cut, cut)]
            ob, nb = tuple(sizes[0::2]), tuple(sizes[1::2])
            if i % 3 == 2:
                ob, nb = nb, ob
        o, n, w = cu.block_pair(b"t%d" % i, ob, nb, n_prefix=rng.randrange(0, 50), n_suffix=rng.randrange(0, 50))
        olds.append(o); news.append(n); wants.append(w)
        if i % 5 == 1:                                      # small left-over pairs (D > 127) among them
            o, n, w = cu.block_pair(b"s%d" % i, (rng.randrange(60, 120), 0, 7), (0, rng.randrange(60, 120), 3))
            olds.append(o); news.append(n); wants.append(w)
        if i == 17:                                         # too far apart to trace
            o, n, w = cu.block_pair(b"u", (12000,), (11500,))
            olds.append(o); news.append(n); wants.append(w)
    d = [len(w[3]) + len(w[4]) for w in wants]
    assert all(x > 127 for x in d)                          # every pair is left to k_myers / k_myers_trace
    need = sum(trace_ints(x) if x <= TRACE_MAX_D else 1 for x in d)
    assert need > TRACE_MAX_INTS and sum(x > TRACE_MAX_D for x in d) == 1
    assert max(trace_ints(x) for x in d if x <= TRACE_MAX_D) < TRACE_MAX_INTS // 20   # D ~ 4 800: many pairs per batch
    exts = [1 + (i % 3) for i in range(len(olds))]
    grp = np.array([i % 7 for i in range(len(olds))], np.uint16)
    traced = check_closed_form(olds, news, exts, wants, grp, 7)
    assert traced.sum() == len(olds) - 1


def test_trace_limit():
    """Distances 23 167 and 23 168 are traced, 23 169 and 23 170 are not (one hunk, assertion counts -1, no events, zero
    table rows); untraced pairs with removed == 0 or added == 0 are one add or one del hunk.  Common prefixes and suffixes
    move the changed lines inside their files."""
    shapes = [((11583,), (11584,)), ((11584,), (11585,)), ((11584,), (11584,)), ((11585,), (11585,)), None, None,
              ((5, 0, 190), (0, 9, 180))]
    olds, news, wants = [], [], []
    for i, s in enumerate(shapes):
        if s is None:
            head, tail = [b"head%d\n" % k for k in range(33)], [b"assert tail%d\n" % k for k in range(21)]
            x, ys = [b"x = 1\n"], [b"assert y\n"] * 12000
            o, n = head + x + tail, head + ys + x + ys + tail
            ins = list(range(33, 33 + 12000)) + list(range(33 + 12001, 33 + 24001))
            w = (1, 0, 0, [], ins)
            if i == 5:
                o, n, w = n, o, (0, 1, 0, ins, [])
            o, n = b"".join(o), b"".join(n)
        else:
            o, n, w = cu.block_pair(b"L%d" % i, *s, n_prefix=40 + i, n_suffix=30 + i)
        olds.append(o); news.append(n); wants.append(w)
    d = [len(w[3]) + len(w[4]) for w in wants]
    assert d[:6] == [23167, 23169, 23168, 23170, 24000, 24000] and d[6] > 127
    assert [trace_ints(x) <= TRACE_MAX_INTS for x in d] == [True, False, True, False, False, False, True]
    exts = [1] * len(olds)
    grp = np.arange(len(olds), dtype=np.uint16)             # one group per pair: an untraced pair's rows stay zero
    traced = check_closed_form(olds, news, exts, wants, grp, len(olds))
    assert traced.tolist() == [True, False, True, False, False, False, True]


def staging_lines(c):
    """The line records the first k_scan pass of a side stages room for (sides_records)."""
    ab = int(c.off[c.n_files])
    return ab // 8 + 2 * (ab // 4096 + c.n_files + 1) + 64


def dense(rng, k):
    pat = rng.choice([[b"\n"], [b"a\n", b"\n"], [b"x\r\n"], [b"\n", b"\n", b"assert\n"]])
    lines = [pat[j % len(pat)] for j in range(k)]
    for _ in range(rng.randrange(3, 12)):
        lines.insert(rng.randrange(len(lines)), rng.choice([b"assert\n", b"}\n", b"\n", b"x\n"]))
    return lines


def sparse(rng, lines):
    """The same lines with long comment lines between them and a few edits: far fewer lines than bytes / 8."""
    out = []
    for j, ln in enumerate(lines):
        if j % 9 == 4:
            out.append(b"# " + bytes(rng.choice(b"abcdef ") for _ in range(150)) + b"\n")
        if rng.random() > 0.004:
            out.append(ln)
    return out


@pytest.mark.parametrize("dense_side", ["old", "new", "both"])
def test_line_dense_pairs(dense_side):
    """Sides with more lines than the staging arrays of the first k_scan pass hold are scanned again at their exact size;
    in a pair one side or both may need it, each with its own pinned control slot."""
    rng = random.Random({"old": 1, "new": 2, "both": 3}[dense_side])
    olds, news = [], []
    for i in range(5):
        base = dense(rng, rng.randrange(1500, 3000))
        d = [ln for ln in base if rng.random() > 0.01] + dense(rng, 20)
        if dense_side == "old":
            o, n = base, sparse(rng, base)
        elif dense_side == "new":
            o, n = sparse(rng, base), base
        else:
            o, n = base, d
        olds.append(b"".join(o)); news.append(b"".join(n))
    exts = [1, 2, 4, 1, 2]
    a, b = pack2(olds, news, exts)
    over = [sum(len(sr.py_lines(f)) for f in fs) > staging_lines(c) for fs, c in ((olds, a), (news, b))]
    assert over == {"old": [True, False], "new": [False, True], "both": [True, True]}[dense_side]
    refs = [sr.py_diff_files(o, n, x, x) for o, n, x in zip(olds, news, exts)]
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    check_all(sc, olds, news, exts, refs)
    sc.close()


def small_files(rng, n):
    lines = [b"\n", b"}\n", b"x = 1\n", b"    assert x == 1\n", b"def test_a():\n", b"EXPECT_EQ(a,\n", b"  b);\n",
             b"self.assertTrue(y)\n", b"// c\r\n", b"int main() {\n", b"return 0;\n", b"\t\n"]
    files = []
    for _ in range(n):
        size = 0 if rng.random() < 0.02 else rng.randrange(1, 201)
        f = b""
        while len(f) < size:
            f += rng.choice(lines)
        f = f[:size]
        if f and rng.random() < 0.3:
            f = f.rstrip(b"\n")                             # no final LF
        files.append(f)
    return files


def test_more_than_256_scan_tiles():
    """300 000 small files: more than 256 tiles of 1 024 items in the exclusive scans of files and of work units, so the
    top-level scan carries its total from one round of 256 tiles to the next."""
    n = 300_000
    rng = random.Random(17)
    files = small_files(rng, n)
    exts = [rng.choice((0, 1, 2, 4)) for _ in range(n)]
    units = sum((len(f) + 4095) // 4096 for f in files)
    assert n > 256 * 1024 and units > 256 * 1024
    c = ts.pack(files, exts)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    base, lh, le, lf, ng = sc.line_hashes(c, ngram=3)
    wbase, wlh, wle, wlf = orc.line_records(c.arena, c.off, c.len, c.ext)
    assert np.array_equal(base, wbase) and np.array_equal(lh, wlh) and np.array_equal(le, wle) and np.array_equal(lf, wlf)
    assert np.array_equal(ng, orc.ngram_hashes(wlh, wbase, 3))
    sbase, send, skind = sc.statements(c)
    wsb, wse, wsk = orc.statements(c.arena, c.off, c.len)
    assert np.array_equal(sbase, wsb) and np.array_equal(send, wse) and np.array_equal(skind, wsk)
    news = [ts.gen_edit(4000 + i, f, 2.0) for i, f in enumerate(files)]
    res = check_all(sc, files, news, exts)
    assert res[1].sum() > 0 and res[3].sum() > 0 and res[4].sum() > 0
    g = np.random.default_rng(5)                            # one batch of `tosem-scan history`: up to 65 535 groups
    ga, gb = g.integers(0, 65535, n).astype(np.uint16), g.integers(0, 65535, n).astype(np.uint16)
    ga[:2], gb[:2] = (0, 65534), (65534, 0)
    a, b = ts.pack(files, exts, ga, 65535), ts.pack(news, exts, gb, 65535)
    _, _, _, ac, rc, _, _ = check(sc, a, b, THREADS)
    assert ac.shape == (65535, ts.K) and (ac.sum(axis=1) > 0).sum() > 10000 and (rc.sum(axis=1) > 0).sum() > 10000
    sc.close()


def copies(t):
    return tuple(np.array(x, copy=True) for x in t)


def test_resident_pair_across_calls():
    """The resident pair against a fresh context, with other calls on the same context between its runs: the scratch pool
    is reused without being cleared, and diff_resident's results live in buffers the next call overwrites."""
    xo, xn, xe = cu.tie_heavy_pairs(8)
    o, n, _ = cu.block_pair(b"r", (3000, 40), (2900, 0))    # D = 5 940: traced by k_myers_trace
    xo.append(o); xn.append(n); xe.append(2)
    yo, yn, ye = cu.tie_heavy_pairs(9)
    yo, yn, ye = yo[::5], yn[::5], ye[::5]
    assert len(yo) < len(xo) and any(kernel_class(p, q, e) == 5 for p, q, e in zip(xo, xn, xe))
    X, Y = pack2(xo, xn, xe), pack2(yo, yn, ye)
    big1 = ts.gen_pairs(0x7053454D0005, 3000, pinned=False)
    big2 = ts.gen_pairs(0x7053454D0006, 6000, pinned=False)
    corpus = ts.gen_corpus(0x7053454D0002, 12, size_law=0, fixed_size=4096, pinned=False)

    fresh = ts.Scanner(0, 1 << 20, 16, 1)
    want_x = fresh.diff_pairs(*X, asserts=True)
    want_x2 = fresh.diff_pairs(*big2, detail=True)
    fresh.close()
    wx = orc.diff_pairs_detail(*((c.arena, c.off, c.len, c.ext) for c in X))
    wy = orc.diff_pairs_detail(*((c.arena, c.off, c.len, c.ext) for c in Y))
    for got, want in zip(want_x[:3], wx):
        assert np.array_equal(got, want)

    sc = ts.Scanner(0, 1 << 22, 64, 1)
    sc.diff_pairs(*big1, detail=True)                       # used slots in the pool
    sc.diff_upload(*X)
    r1 = copies(sc.diff_resident(detail=True))
    got2 = sc.diff_pairs(*big2, detail=True)
    r2 = copies(sc.diff_resident(detail=False))
    lines = sc.line_hashes(corpus)
    r3 = copies(sc.diff_resident(detail=True))
    stm = sc.statements(corpus)
    scan = sc.scan(corpus)
    r4 = copies(sc.diff_resident(asserts=True))
    sc.diff_upload(*Y)
    r5 = copies(sc.diff_resident(detail=True))
    sc.close()

    for r in (r1, r3):
        assert all(np.array_equal(g, w) for g, w in zip(r, wx))
    assert all(np.array_equal(g, w) for g, w in zip(r2, wx[:2]))
    assert len(r4) == 7 and all(np.array_equal(g, w) for g, w in zip(r4, want_x))
    assert len(r5[0]) == len(yo) and all(np.array_equal(g, w) for g, w in zip(r5, wy))
    assert all(np.array_equal(g, w) for g, w in zip(got2, want_x2))
    wl = orc.line_records(corpus.arena, corpus.off, corpus.len, corpus.ext)
    assert all(np.array_equal(g, w) for g, w in zip(lines, wl))
    assert all(np.array_equal(g, w) for g, w in zip(stm, orc.statements(corpus.arena, corpus.off, corpus.len)))
    wscan = orc.scan(corpus.arena, corpus.off, corpus.len, corpus.ext, corpus.grp, 1, events=False)
    assert np.array_equal(scan["stats"], wscan["stats"]) and np.array_equal(scan["group_counts"], wscan["group_counts"])
