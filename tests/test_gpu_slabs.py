"""The streamed scan (tsm_scan with a host arena) across its H2D slabs.

launch_scan (csrc/tsm_api.cu) cuts a host arena into slabs of about 32 MiB and runs k_plan, k_scan and k_classify once
per slab while the next slab is on the wire; only the last k_classify adds the per-file totals, and an overflow of the
event lists found by tsm_download rescans the resident arena as one slab.  Every test here restates the cut
(expected_slabs) and asserts the launch count it implies, so a scan that silently runs as one slab fails; the results
are compared field by field with the CPU oracle (stats, [group][category] tables, totals, both event arrays).

Memory of the 64-slab case, estimated from the buffer sizes (not measured): a 2 GiB pinned host arena, a 2 GiB device
arena and about 3.8 GB of default candidate / event lists; its diff and line-record calls stage about 3.5 GB of line
records for the 2 GiB side.  It runs at full size on an 80 GB H100."""
import os
import random
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import orc
import tosemscan as ts

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
EV = ts.SCAN_ASSERT_EVENTS | ts.SCAN_HEADER_EVENTS
SLAB = 32 << 20                                           # launch_scan: first slab size
MAX_SLABS = 64                                            # tsm_ctx::kMaxSlabs
TOP = (1 << 31) - 128                                     # the largest arena tsm_create accepts


def slab_starts(off):
    """The slab cut of launch_scan restated: slabs of 32 MiB, doubled while arena / slab + 1 > 64; a new slab starts at
    the first file (after the first) whose offset is at or past the start of the current slab + the slab size.  Returns
    the first file of every slab, then n."""
    off = np.asarray(off, np.int64)
    n = len(off) - 1
    if n <= 0:
        return [0]
    slab = SLAB
    while int(off[n]) // slab + 1 > MAX_SLABS:
        slab *= 2
    out, nxt, i = [0], slab, 1
    while True:
        i += int(np.searchsorted(off[i:n], nxt, "left"))
        if i >= n:
            return out + [n]
        out.append(i)
        nxt = int(off[i]) + slab
        i += 1


def expected_slabs(off):
    return len(slab_starts(off)) - 1


def streamed(sc, c, flags, at_least, **kw):
    """sc.scan(c, flags) that must have run as expected_slabs(c.off) >= at_least slabs (3 launches each)."""
    got = sc.scan(c, flags, **kw)
    n = expected_slabs(c.off)
    assert n >= at_least, ("the corpus does not reach the slabs it is meant to", n, at_least)
    assert sc.last_launch_count() == 3 * n, (sc.last_launch_count(), n)
    return got


def oracle(c, rev_b=False):
    return orc.scan(c.arena, c.off, c.len, c.ext, c.grp, c.n_groups, rev_b=rev_b)


def fold_groups(gc, n_groups):
    """The [group][category] table of groups g % n_groups from the table of groups g."""
    out = np.zeros((n_groups, gc.shape[1]), np.int64)
    np.add.at(out, np.arange(gc.shape[0]) % n_groups, gc)
    return out


def check(got, want, events=True, group_counts=None):
    for f in ts.FILE_STAT.names:
        bad = np.nonzero(got["stats"][f] != want["stats"][f])[0]
        assert bad.size == 0, (f, bad[:10], got["stats"][bad[:5]], want["stats"][bad[:5]])
    gc = want["group_counts"] if group_counts is None else group_counts
    assert np.array_equal(got["group_counts"], gc), np.argwhere(got["group_counts"] != gc)[:10]
    assert np.array_equal(got["global_counts"], want["global_counts"])
    st = want["stats"]
    tot = [int(st[f].astype(np.int64).sum()) for f in ("n_lines", "n_assert", "n_headers", "n_fixture")]
    assert got["totals"].tolist() == tot, (got["totals"].tolist(), tot)
    assert int(got["global_counts"].sum()) == tot[1]
    if events:
        for k in ("assert_events", "header_events"):
            a, b = got[k], want[k]
            assert len(a) == len(b), (k, len(a), len(b))
            for f in a.dtype.names:
                bad = np.nonzero(a[f] != b[f])[0]
                assert bad.size == 0, (k, f, a[bad[:5]], b[bad[:5]])


def same(a, b):
    """Two results of the device, equal in every array."""
    assert set(a) == set(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def place(items, n_groups=1, top=None):
    """A pinned corpus of (offset, bytes, ext, grp) items at the given 128-B aligned offsets, zero bytes between them.
    top: off[n] (default: the end of the last file rounded up to 128 B)."""
    offs = [int(o) for o, _, _, _ in items]
    lens = [len(d) for _, d, _, _ in items]
    end = top if top is not None else offs[-1] + (lens[-1] + 127) // 128 * 128
    off = np.array(offs + [end], np.int64)
    assert end < (1 << 31) and not (off % 128).any()
    assert all(offs[i] + lens[i] <= off[i + 1] for i in range(len(offs))), "files overlap"
    arena, keep = ts.host_buffer(end)
    for (o, d, _, _) in items:
        if d:
            arena[o:o + len(d)] = np.frombuffer(d, np.uint8)
    return ts.Corpus(arena, off.astype(np.int32), lens, [e for _, _, e, _ in items], [g for _, _, _, g in items],
                     n_groups, keep)


def up128(x):
    return (x + 127) // 128 * 128


# ---------------------------------------------------------------------------------------------- contents
MID_LINES = [b"    x = compute(%d)\n", b"    assert x == %d\n", b"    EXPECT_TRUE(ok_%d);\n", b"    BOOST_CHECK(v == %d);\n",
             b"    TESTEQUAL(a, %d);\n", b"    FAIL() << %d;\n", b"def test_%d(self):\n", b"TEST_F(Fix, Case%d) {\n",
             b"    self.assertEqual(a, %d)\n", b"    assert not flag_%d\n", b"class TestCase%d(unittest.TestCase):\n"]


def chunk_edge_file(size):
    """About `size` bytes in pages: the first half of 4096 B (one per 4 KiB chunk), each opening with an assertion line and
    closing with one that ends on the chunk edge; the second half of 4133 B, so that the edges fall inside lines; every
    97th page carries a 9 000-byte assertion line that spans two edges."""
    pages, total, k = [], 0, 0
    while total < size:
        plen = 4096 if total < size // 2 else 4133
        first, last = b"assert first_%07d\n" % k, b"EXPECT_EQ(k, %07d);\n" % k
        mid = b"".join(MID_LINES[(k + j) % len(MID_LINES)] % (k + j) for j in range(200))
        if k % 97 == 50:
            mid = b"    assert " + b"y" * 9000 + b"\n" + mid
            plen += 2 * 4096
        body = mid[:plen - len(first) - len(last) - 1] + b"\n"
        page = first + body + last
        assert len(page) == plen
        pages.append(page)
        total += plen
        k += 1
    return b"".join(pages)


NO_CAND = [b"value = 1\n" * 3000, b"def helper(x):\n    return x\n" * 500, b"", b"\n" * 100, b"x = 1"]   # lines, headers, no candidate


def dense_assert_files():
    return [b"assert x\n" * 30000, b"EXPECT_EQ(a, b);\n" * 10000, b"    self.assertEqual(a, b)\n" * 8000,
            b"BOOST_CHECK(x);\nTESTEQUAL(a, b);\nFAIL();\n" * 5000]


# ---------------------------------------------------------------------------------------------- 2: streamed = resident = oracle
def mixed_corpus():
    """About 200 MB: C4-shaped synthetic files, fuzzed files with long lines and with binary bytes, the edge files and
    three copies of the C1 test files, shuffled, so that every kind sits in several slabs."""
    rng = random.Random(0x51AB)
    c4 = ts.gen_corpus(0x51AB0004, 14000, 1, n_groups=1, pinned=False)
    files = [c4.file_bytes(i) for i in range(c4.n_files)]
    exts = c4.ext.tolist()
    for seed, kw in ((1, {"long_lines": True}), (2, {"binary": True})):
        f, e, _ = cu.fuzz_corpus(0x51AB00 + seed, 250, 20000, **kw)
        files += f
        exts += e.tolist()
    f, e, _ = cu.edge_corpus()
    files += f
    exts += e.tolist()
    c1, e1, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    for _ in range(3):
        files += c1
        exts += e1.tolist()
    order = list(range(len(files)))
    rng.shuffle(order)
    files = [files[i] for i in order]
    exts = np.array([exts[i] for i in order], np.uint8)
    grp = np.array([rng.randrange(300) for _ in files], np.uint16)
    return ts.pack(files, exts, grp, 300, pinned=True)


@pytest.mark.parametrize("rev_b", [False, True], ids=["revA", "revB"])
def test_streamed_equals_resident_equals_oracle(rev_b):
    c300 = mixed_corpus()
    assert 150e6 < c300.source_bytes < 250e6
    c9 = ts.Corpus(c300.arena, c300.off, c300.len, c300.ext, c300.grp % 9, 9)
    rev = ts.SCAN_REV_B if rev_b else 0
    want = oracle(c300, rev_b)
    sc = ts.Scanner(0, int(c300.off[-1]) + 4096, c300.n_files, 300)
    got300 = streamed(sc, c300, EV | rev, 5)                # > 16 groups: k_classify's global atomics
    check(got300, want)
    got9 = streamed(sc, c9, EV | rev, 5)                    # 9 groups: the shared-memory histogram
    check(got9, want, group_counts=fold_groups(want["group_counts"], 9))
    for c, got in ((c300, got300), (c9, got9)):
        sc.upload(c)                                         # the same corpus resident: one slab
        sc.scan_resident(EV | rev)
        assert sc.last_launch_count() == 3
        same(sc.download(EV | rev), got)
        plain = streamed(sc, c, rev, 5)                     # no events: the same counts and totals
        for k in ("stats", "group_counts", "global_counts", "totals"):
            assert np.array_equal(plain[k], got[k]), k
    sc.close()


# ---------------------------------------------------------------------------------------------- 3: slab-cut edges
def edges_layout():
    """Seven slabs (the cut points are in the comments; S = 32 MiB).  Returns (items, slabs, groups, candidate-free
    slabs, the dense slab)."""
    S = SLAB
    it = []
    # slab 0 at 0: an assertion line first, an unterminated assertion line last (the file 128 B below S)
    it += [(0, b"assert first_of_arena\n" + cu.PY_SAMPLE, 1), (4096, cu.CC_SAMPLE, 2), (S // 2, cu.JAVA_SAMPLE, 4),
           (S - 128, b"y = 1\n    assert last0 == 2", 1)]
    # slab 1 at exactly S: a header line first, 128 B behind it another file, a header line last (128 B below 2S)
    it += [(S, b"def test_first_of_slab1(self):\n    assert a\n", 1), (S + 128, b"EXPECT_EQ(a, b);\n", 2),
           (S + 4096, cu.JAVA_SAMPLE, 4), (2 * S - 128, b"    assert z\nclass TestLastOfSlab1(unittest.TestCase):\n", 1)]
    # slab 2 at 2S + 128 (nothing at 2S): no candidate line at all
    base = 2 * S + 128
    it += [(base + k * 262144, NO_CAND[k % len(NO_CAND)], 1 + k % 2) for k in range(40)]
    # slab 3 at 3S + 256: many candidates, a CRLF file, and an unterminated line at the slab's end
    base = 3 * S + 256
    dense = dense_assert_files()
    o = base
    for k, d in enumerate(dense + [b"assert x\r\nEXPECT_EQ(a, b);\r\n" * 100]):
        it.append((o, d, (1, 2, 1, 2, 2)[k]))
        o = up128(o + len(d) + 4096 * k)
    it.append((base + S - 256, b"\n\nTEST(Last, Unterminated) {\n  EXPECT_TRUE(x)", 2))
    # slab 4 at 4S + 256: one 40 MB file alone (longer than a slab)
    big = chunk_edge_file(40_000_000)
    o4 = 4 * S + 256
    it.append((o4, big, 1))
    # slab 5 behind it: empty files only
    o5 = up128(o4 + len(big))
    it += [(o5 + k * 128000, b"", 1 + k % 6) for k in range(100)]
    # slab 6 at o5 + S: the edge files, and the arena ends with an unterminated assertion line
    o6 = o5 + S
    o = o6
    for d, e in cu.EDGE_FILES:
        it.append((o, d, e))
        o = up128(o + len(d))
    it.append((o, b"x = 1\nassert end_of_arena", 1))
    return [(a, d, e, k % 20) for k, (a, d, e) in enumerate(it)], 7, 20, (2,), 3


def late_layout():
    """Four slabs; candidate lines only in the last one."""
    S = SLAB
    it = []
    for s in range(3):
        it += [(s * S + (k << 20), NO_CAND[(s + k) % len(NO_CAND)], 1 + k % 3) for k in range(8)]
    o = 3 * S
    for d, e in [(cu.PY_SAMPLE, 1), (cu.CC_SAMPLE, 2), (cu.JAVA_SAMPLE, 4)] + [(d, 1) for d in dense_assert_files()]:
        it.append((o, d, e))
        o = up128(o + len(d))
    it.append((o, b"def test_tail():\n    assert tail == 1", 1))
    return [(a, d, e, k % 3) for k, (a, d, e) in enumerate(it)], 4, 3, (0, 1, 2), 3


@pytest.mark.parametrize("layout", ["edges", "late"])
def test_slab_cut_edges(layout):
    items, n_slabs, n_groups, empty_slabs, many = (edges_layout if layout == "edges" else late_layout)()
    c = place(items, n_groups)
    assert expected_slabs(c.off) == n_slabs
    starts = slab_starts(c.off)
    sc = ts.Scanner(0, int(c.off[-1]) + 4096, c.n_files, n_groups)
    for rev_b in (False, True):
        want = oracle(c, rev_b)
        got = streamed(sc, c, EV | (ts.SCAN_REV_B if rev_b else 0), n_slabs)
        check(got, want)
        # the layout is what it claims: the candidate-free slabs hold no assertion line (Rev B triggers included) ...
        n_assert = want["stats"]["n_assert"].astype(np.int64)
        for s in empty_slabs:
            assert int(n_assert[starts[s]:starts[s + 1]].sum()) == 0, s
        assert int(n_assert[starts[many]:starts[many + 1]].sum()) > 1000   # ... and the slab behind them many
    sc.close()


# ---------------------------------------------------------------------------------------------- 4: overflow in a later slab
OVERFLOW = {"assert": (b"assert\n", 1, 0), "def": (b"def\n", 1, 0), "FAIL": (b"FAIL\n", 2, ts.SCAN_REV_B)}


def overflow_corpus(line, ext):
    """Three sparse slabs, then 48 MB of `line` in eight files (two slabs): more candidates or events than the default
    lists of the context (max_arena / 32 + max_files) and the default host arrays (source bytes / 8) hold."""
    it = []
    for s in range(3):
        it += [(s * SLAB, cu.PY_SAMPLE, 1), (s * SLAB + (1 << 20), cu.CC_SAMPLE, 2)]
    o = 3 * SLAB
    for _ in range(8):
        d = line * (6_000_000 // len(line))
        it.append((o, d, ext))
        o = up128(o + len(d))
    it.append((o, cu.JAVA_SAMPLE, 4))
    return place([(a, d, e, k % 4) for k, (a, d, e) in enumerate(it)], 4)


@pytest.mark.parametrize("kind", list(OVERFLOW))
def test_overflow_in_a_later_slab(kind):
    line, ext, rev = OVERFLOW[kind]
    c = overflow_corpus(line, ext)
    flags = EV | rev
    want = oracle(c, bool(rev))
    n_ev = max(len(want["assert_events"]), len(want["header_events"]))
    arena = int(c.off[-1]) + 4096
    assert n_ev > arena // 32 + c.n_files and n_ev > c.source_bytes // 8 + 16
    # the slabs the corpus reaches, on a context whose lists hold all of it
    roomy = ts.Scanner(0, arena, c.n_files, 4, max_events=n_ev + 1024)
    check(streamed(roomy, c, flags, 5), want)
    roomy.close()
    sc = ts.Scanner(0, arena, c.n_files, 4)
    got = sc.scan(c, flags)                                  # lists too short: grown, the resident arena rescanned as one slab
    assert sc.last_launch_count() == 3
    check(got, want)
    check(streamed(sc, c, flags, 5), want)                   # the grown lists hold the next streamed scan
    check(streamed(sc, c, flags, 5, event_cap=1000), want)   # host arrays too short: the events are downloaded again
    sc.close()


# ---------------------------------------------------------------------------------------------- 5: 64 slabs at the top
def ends_at(data, n, last):
    """data cut to n bytes so that it ends with `last`."""
    assert len(data) >= n
    return data[:n - len(last)] + last


def top_items():
    """One small file every 32 MiB (64 slabs, the limit), then files packed against off[n] = 2^31 - 128 whose staged
    chunk ranges end within the last 4 KiB of the arena: a three-chunk file whose last line ends on its last byte, a
    terminated and an unterminated one-line file, and a file that ends on the arena's last byte with an unterminated
    line; a multi-chunk file sits in front of them."""
    fz, fe, _ = cu.fuzz_corpus(0x70B1, 40, 9000, long_lines=True)
    small = [(cu.PY_SAMPLE, 1), (cu.CC_SAMPLE, 2), (cu.JAVA_SAMPLE, 4)] + list(zip(fz, fe.tolist())) + cu.EDGE_FILES[:21]
    it = [(k * SLAB, d, e) for k, (d, e) in enumerate(small[:MAX_SLABS])]
    assert len(it) == MAX_SLABS
    K4 = TOP - 4096                                          # the last 4 KiB
    edge = chunk_edge_file(40000)
    it += [(K4 - 6 * 4096, ends_at(edge, 3 * 4096 + 77, b"\nassert pre_top\n"), 1),
           (K4 - 2 * 4096, ends_at(edge[4096:], 2 * 4096 + 1000, b"\n    self.assertEqual(top, 1)\n"), 1),
           (K4 + 1024, b"assert tail_a\n", 1),
           (K4 + 1152, b"    assert unterminated_b == 2", 1),
           (TOP - 2816, ends_at(cu.CC_SAMPLE * 4, 2816, b"\n  EXPECT_TRUE(top_of_arena)"), 2)]
    return [(a, d, e, k % 5) for k, (a, d, e) in enumerate(it)]


def test_64_slabs_at_the_top_of_the_int32_arena():
    items = top_items()
    c = place(items, 5, top=TOP)
    assert c._keep is not None, "the 2 GiB host arena must be pinned"
    assert int(c.off[-1]) == TOP and expected_slabs(c.off) == MAX_SLABS
    files = [d for _, d, _, _ in items]
    low = ts.pack(files, c.ext, c.grp, 5, pinned=True)       # the same files at low offsets
    sc = ts.Scanner(0, TOP, c.n_files, 5)
    for rev in (0, ts.SCAN_REV_B):
        want = oracle(c, bool(rev))
        got = streamed(sc, c, EV | rev, MAX_SLABS)
        check(got, want)
        assert len(got["assert_events"]) > 100
        same(sc.scan(low, EV | rev), got)                   # event offsets are file-relative: identical
    sc.close()
    # one side of line records, statements, diffs and similarity is the 2 GiB arena
    news = ts.pack([ts.gen_edit(0x70B0 + i, f) for i, f in enumerate(files)], c.ext, c.grp, 5, pinned=True)
    dc = ts.Scanner(0, 1 << 20, 16, 5)

    def eq(x, y):
        assert len(x) == len(y)
        for a, b in zip(x, y):
            assert np.array_equal(a, b)
    eq(dc.line_hashes(c, ngram=3), dc.line_hashes(low, ngram=3))
    eq(dc.statements(c), dc.statements(low))
    for hi, lo in (((c, news), (low, news)), ((news, c), (news, low))):
        det = dc.diff_pairs(*hi, detail=True)
        assert int(det[0].sum()) > 0 and int(det[1].sum()) > 0
        eq(det, dc.diff_pairs(*lo, detail=True))
        eq(dc.diff_pairs(*hi, asserts=True), dc.diff_pairs(*lo, asserts=True))
    n = c.n_files
    co = np.concatenate([np.arange(n), np.arange(n)])
    cn = np.concatenate([np.arange(n), np.roll(np.arange(n), 1)])
    eq([dc.similarity(c, news, co, cn)], [dc.similarity(low, news, co, cn)])
    eq([dc.similarity(news, c, cn, co)], [dc.similarity(news, low, cn, co)])
    dc.close()


# ---------------------------------------------------------------------------------------------- 6: through the CLI
def test_cli_scan_one_streamed_batch_equals_single_slab_batches(tmp_path):
    c = ts.gen_corpus(0x51AB0006, 9000, 1, n_groups=1, pinned=False)
    assert 80e6 < c.source_bytes < 130e6 and int(c.len.max()) < (8 << 20) - 4096
    root = tmp_path / "proj_tests"
    os.makedirs(root)
    for i in range(c.n_files):
        (root / ("f%05d_test.%s" % (i, {1: "py", 2: "cc", 4: "java"}[int(c.ext[i])]))).write_bytes(c.file_bytes(i))
    # the default batch (1 GiB) takes every file, packed in walk (name) order: at least three slabs
    off = np.concatenate([[0], np.cumsum((c.len.astype(np.int64) + 127) // 128 * 128)])
    assert off[-1] < (1 << 30) and expected_slabs(off) >= 3
    outs = []
    for extra in ([], ["--batch-bytes", "8388608"]):           # ... and batches of at most 8 MiB: one slab each
        tag = "b" if extra else "a"
        rows_p, sum_p = str(tmp_path / ("rows_%s.csv" % tag)), str(tmp_path / ("sum_%s.csv" % tag))
        out = subprocess.run([CLI, "scan", str(root), "--rows", rows_p, "--summary", sum_p] + extra, capture_output=True)
        assert out.returncode == 0, out.stderr
        totals = out.stderr.decode().strip().split("\n")[-1].split(" on ")[0]
        outs.append((out.stdout, open(rows_p, "rb").read(), open(sum_p, "rb").read(), totals))
    assert outs[0] == outs[1]
    want = orc.scan(c.arena, c.off, c.len, c.ext, c.grp, 1, events=False)
    agg = dict(l.rsplit(",", 1) for l in outs[0][0].decode().replace("\r\n", "\n").strip().split("\n")[1:])
    assert {k: int(v) for k, v in agg.items()} == {(ts.category_name(k) if k else ""): int(v)
                                                  for k, v in enumerate(want["global_counts"]) if v}
    st = want["stats"]
    assert outs[0][3] == "tosem-scan: lines=%d assertion_lines=%d headers=%d fixture_headers=%d" % tuple(
        int(st[f].astype(np.int64).sum()) for f in ("n_lines", "n_assert", "n_headers", "n_fixture"))
