"""GPU parity tests: the sm_90a product path, through the C ABI, against the CPU oracle on the
same seeded inputs.  Integer / byte work: the bar is bit-exact equality of every output."""
import ctypes as C

import numpy as np
import pytest

import corpus_util as cu
import orc
import tosemscan as ts

pytestmark = pytest.mark.gpu

FLAGS = ts.SCAN_ASSERT_EVENTS | ts.SCAN_HEADER_EVENTS


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 18, max_groups=16)
    yield s
    s.close()


def check_against_oracle(scanner, corpus, flags=FLAGS, resident=False):
    want = orc.scan(corpus.arena, corpus.off, corpus.len, corpus.ext, corpus.grp, corpus.n_groups)
    if resident:
        scanner.upload(corpus)
        scanner.scan_resident(flags)
        got = scanner.download(flags)
    else:
        got = scanner.scan(corpus, flags)
    for f in ("n_lines", "n_assert", "n_headers", "n_fixture", "digest"):
        bad = np.nonzero(got["stats"][f] != want["stats"][f])[0]
        assert bad.size == 0, (f, bad[:10], got["stats"][bad[:5]], want["stats"][bad[:5]],
                               [corpus.len[i] for i in bad[:5]], [corpus.ext[i] for i in bad[:5]])
    assert np.array_equal(got["group_counts"], want["group_counts"])
    assert np.array_equal(got["global_counts"], want["global_counts"])
    st = want["stats"]
    assert got["totals"].tolist() == [int(st[k].astype(np.int64).sum()) for k in ("n_lines", "n_assert", "n_headers", "n_fixture")]
    if flags & ts.SCAN_ASSERT_EVENTS:
        a, b = got["assert_events"], want["assert_events"]
        assert len(a) == len(b)
        for f in a.dtype.names:
            bad = np.nonzero(a[f] != b[f])[0]
            assert bad.size == 0, (f, a[bad[:5]], b[bad[:5]])
    if flags & ts.SCAN_HEADER_EVENTS:
        a, b = got["header_events"], want["header_events"]
        assert len(a) == len(b)
        assert np.array_equal(a, b), (a[:5], b[:5])
    return got


def test_edge_cases(scanner):
    files, exts, grps = cu.edge_corpus()
    check_against_oracle(scanner, ts.pack(files, exts, grps, 3))


def test_single_files_one_by_one(scanner):
    """Each edge file alone (so that a failure names the file) and with every extension tag."""
    files, exts, _ = cu.edge_corpus()
    for i, f in enumerate(files):
        for e in {int(exts[i]), 1, 2, 4}:
            check_against_oracle(scanner, ts.pack([f], [e]))


def test_empty_corpus_and_empty_files(scanner):
    got = scanner.scan(ts.pack([], []), FLAGS)
    assert got["totals"].tolist() == [0, 0, 0, 0] and got["global_counts"].sum() == 0
    check_against_oracle(scanner, ts.pack([b""] * 70, [1] * 70))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_fuzz_small_files(scanner, seed):
    files, exts, grps = cu.fuzz_corpus(seed, 600, 3000)
    check_against_oracle(scanner, ts.pack(files, exts, grps, 5))


@pytest.mark.parametrize("seed", [11, 12])
def test_fuzz_multi_chunk_files_and_long_lines(scanner, seed):
    files, exts, grps = cu.fuzz_corpus(seed, 150, 60000, long_lines=True)
    check_against_oracle(scanner, ts.pack(files, exts, grps, 5))


def test_chunk_edge_alignment_sweep(scanner):
    """A statement sliding across the 4 KiB chunk edge and across the 240-byte look-ahead."""
    files = []
    for pad in list(range(4060, 4120)) + list(range(4096 + 200, 4096 + 260)) + [8180, 8192, 8200]:
        files.append(b"x" * pad + b"\n  self.assertEqual(a, b)\nEXPECT_NEAR(q, r, 1e-3);\n" + b"y" * 300)
        files.append(b"def test_a(self):\n" + b"z" * (pad - 18) + b" assert not q\r\n")
    check_against_oracle(scanner, ts.pack(files, [1, 2] * (len(files) // 2)))


def test_newline_storms(scanner):
    """More lines per chunk than one window of the line table holds (several windows per chunk)."""
    files = [b"\n" * 20000, b"a\n" * 9000, (b"assert x\n" + b"\n" * 700) * 9, b"\n" * 4096 + b"assert y", b"\r\n" * 5000]
    check_against_oracle(scanner, ts.pack(files, [1, 2, 1, 4, 3]))


def test_pattern_ends_next_to_newlines(scanner):
    """Every word holds a newline AND a pattern end (pass 2b: queue overflow, several line windows per chunk),
    patterns straddling stripe and word borders at every alignment, flags of lines that span stripes."""
    files, exts = [], []
    for body, ext in [(b"{\n", 3), (b"test{\n}\n", 3), (b"void test(){\n", 3), (b"TEST_F(A, b) {\n", 3),
                      (b"def\n", 1), (b"def f():\n assert x\n", 1), (b"class A:\n  class B :\n", 1),
                      (b"EXPECT_EQ(a, b);\r\n", 3), (b"\tassert(x);{\n", 6), (b"x = 1\n", 1)]:
        for pad in (0, 1, 3, 7, 129, 135, 4090):
            files.append(b"#" * pad + b"\n" + body * (20000 // len(body)))
            exts.append(ext)
    long_line = b"// " + b"y" * 700 + b" assert_that(x) test { void class " + b"z" * 300 + b"\n"   # spans 8 stripes
    files.append((long_line + b"int test_it() {\n") * 40)
    exts.append(3)
    check_against_oracle(scanner, ts.pack(files, exts))


def test_synthetic_c2_shape(scanner):
    c = ts.gen_corpus(0x7053454D0002, 3000, size_law=0, fixed_size=4096, n_groups=9, pinned=True)
    check_against_oracle(scanner, c)
    check_against_oracle(scanner, c, flags=0, resident=True)


def test_synthetic_c4_zipf_shape(scanner):
    c = ts.gen_corpus(0x7053454D0004, 2500, size_law=1, n_groups=9, pinned=True)
    assert c.len.max() > 100000
    check_against_oracle(scanner, c)


def test_resident_rescans_are_identical_and_launch_count(scanner):
    c = ts.gen_corpus(5, 1500, 0, 4096, n_groups=4)
    scanner.upload(c)
    outs = []
    for _ in range(3):
        scanner.scan_resident(0)
        outs.append(scanner.download(0))
    assert scanner.last_launch_count() == 3
    for o in outs[1:]:
        assert np.array_equal(o["stats"], outs[0]["stats"]) and np.array_equal(o["group_counts"], outs[0]["group_counts"])
    ms = scanner.last_kernel_ms()
    assert len(ms) == 4 and all(m >= 0 for m in ms)


def test_host_path_with_pinned_index_and_reused_result_buffers(scanner):
    """The path bench.py's e2e times: a pinned corpus pins its index arrays too, scan(reuse=True) returns views of
    pinned buffers the Scanner keeps - same numbers as the plain call, the buffers are overwritten by the next call."""
    a = ts.gen_corpus(11, 1200, 1, n_groups=5)                # pinned arena (a GPU is present)
    b = ts.gen_corpus(12, 1200, 1, n_groups=5)
    assert a._keep is not None and len(a._index_pins) == 4 and a.off.dtype == np.int32 and a.grp.dtype == np.uint16
    plain_a, plain_b = scanner.scan(a, 0), scanner.scan(b, 0)
    ra = scanner.scan(a, 0, reuse=True)
    keep = {k: ra[k].copy() for k in ("stats", "group_counts", "global_counts")}
    rb = scanner.scan(b, 0, reuse=True)
    assert rb["stats"] is ra["stats"]                         # the same buffer, now holding b's records
    for k in keep:
        assert np.array_equal(keep[k], plain_a[k]) and np.array_equal(rb[k], plain_b[k])
    assert np.array_equal(ra["totals"], plain_a["totals"]) and np.array_equal(rb["totals"], plain_b["totals"])
    want = orc.scan(a.arena, a.off, a.len, a.ext, a.grp, 5, events=False)
    assert np.array_equal(keep["stats"], want["stats"])


def test_shards_add_up_to_the_whole(scanner):
    """Size-independent property used at full scale: counts of round-robin shards sum to the whole."""
    n, w = 4000, 4
    whole = scanner.scan(ts.gen_corpus(9, n, 0, 4096, n_groups=9))
    acc = np.zeros_like(whole["group_counts"])
    dig = np.uint64(0)
    for r in range(w):
        part = scanner.scan(ts.gen_corpus(9, n // w, 0, 4096, first_index=r, index_stride=w, n_groups=9))
        acc += part["group_counts"]
        dig ^= np.bitwise_xor.reduce(part["stats"]["digest"])
    assert np.array_equal(acc, whole["group_counts"])
    assert dig == np.bitwise_xor.reduce(whole["stats"]["digest"])


def test_full_size_c2_properties(scanner):
    """BASELINE config C2 at full size (100k x 4 KiB): oracle-free invariants + a sampled oracle check."""
    big = ts.Scanner(device=0, max_arena_bytes=100000 * 4096 + 4096, max_files=100000, max_groups=16)
    c = ts.gen_corpus(0x7053454D0002, 100000, 0, 4096, n_groups=9)
    got = big.scan(c, 0)
    st = got["stats"]
    assert got["totals"].tolist() == [int(st[k].astype(np.int64).sum()) for k in ("n_lines", "n_assert", "n_headers", "n_fixture")]
    assert int(got["global_counts"].sum()) == got["totals"][1]
    assert np.array_equal(got["group_counts"].sum(axis=0), got["global_counts"])
    for g in range(9):
        assert int(got["group_counts"][g].sum()) == int(st["n_assert"][c.grp == g].astype(np.int64).sum())
    # sampled files against the oracle
    idx = np.arange(0, 100000, 97)
    sub = ts.pack([c.file_bytes(int(i)) for i in idx], c.ext[idx], c.grp[idx], 9)
    want = orc.scan(sub.arena, sub.off, sub.len, sub.ext, sub.grp, 9, events=False)
    assert np.array_equal(st[idx], want["stats"])
    big.close()


def test_reduce_matches_oracle_and_golden(scanner):
    import os
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g3_reduce.npz"))
    n_cases = int(d["case_id"].max()) + 1
    out, cpr = scanner.reduce(d["flags"], d["repo"], d["case_id"], len(d["repo_names"]), n_cases)
    assert np.array_equal(out, d["oracle_distinct"]) and np.array_equal(cpr, d["oracle_cases_per_repo"])
    rng = np.random.default_rng(3)
    for rows, nf, nr, nc in [(0, 3, 2, 5), (1, 1, 1, 1), (5000, 40, 7, 3000), (20000, 5, 3, 40000)]:
        flags = (rng.random((rows, nf)) < 0.2).astype(np.uint8)
        repo = rng.integers(0, nr, rows).astype(np.int32)
        case = rng.integers(0, nc, rows).astype(np.int32)
        o1, c1 = scanner.reduce(flags, repo, case, nr, nc)
        o2, c2 = orc.reduce(flags, repo, case, nr, nc)
        assert np.array_equal(o1, o2) and np.array_equal(c1, c2)


def test_errors_are_reported_not_swallowed(scanner):
    c = ts.pack([b"assert x\n"], [1])
    bad = ts.Corpus(c.arena, np.array([64, 128], np.int32), c.len, c.ext)
    with pytest.raises(ts.TsmError) as e:
        scanner.scan(bad)
    assert e.value.status == -2
    # a broken file behind the first 32 MiB slab: found while the slabs in front of it are already on the wire
    big = ts.gen_corpus(21, 12000, 0, 4096)
    sc2 = ts.Scanner(0, int(big.off[-1]) + 4096, big.n_files, 1)
    good = sc2.scan(big, 0)
    big.len[11000] = 5000                                    # runs into its neighbour
    with pytest.raises(ts.TsmError) as e:
        sc2.scan(big, 0)
    assert e.value.status == -2
    big.len[11000] = 4096
    again = sc2.scan(big, 0)                                 # the ctx is usable afterwards
    assert np.array_equal(again["stats"], good["stats"]) and np.array_equal(again["global_counts"], good["global_counts"])
    big.off[9000] = 2 ** 31 - 128                            # an offset far outside the arena, in a later slab
    with pytest.raises(ts.TsmError) as e:
        sc2.scan(big, 0)
    assert e.value.status == -2
    sc2.close()
    small = ts.Scanner(device=0, max_arena_bytes=4096, max_files=4, max_groups=1)
    with pytest.raises(ts.TsmError) as e:
        small.scan(ts.pack([b"x" * 9000], [1]))
    assert e.value.status == -3
    small.close()


OK, ARG, LAYOUT = 0, -1, -2
FAULTS = ("none", "misaligned_off", "negative_off", "negative_len", "runs_into_next", "off_far_past_arena", "misaligned_end",
          "ext_7", "ext_null", "grp_out_of_range", "no_groups", "groups_mismatch", "groups_mismatch_and_misaligned_off")
# status per fault (in FAULTS order) of every corpus-taking entry point; diff_resident(_asserts) follow a diff_upload of a
# clean pair and then one of the faulty pair, so that a rejected upload shows that the ctx keeps the clean one
STATUS = {
    "scan":                  (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, ARG, LAYOUT, ARG, OK, LAYOUT),
    "upload":                (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, ARG, LAYOUT, ARG, OK, LAYOUT),
    "diff_pairs":            (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, OK, OK, OK, OK, OK, OK, LAYOUT),
    "diff_pairs_detail":     (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, OK, LAYOUT, OK, OK, OK, OK, LAYOUT),
    "diff_pairs_asserts":    (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, OK, LAYOUT, OK, LAYOUT, ARG, ARG, ARG),
    "diff_upload":           (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, OK, LAYOUT, OK, OK, OK, OK, LAYOUT),
    "diff_resident":         (OK, OK, OK, OK, OK, OK, OK, OK, OK, OK, OK, OK, OK),
    "diff_resident_asserts": (OK, OK, OK, OK, OK, OK, OK, OK, OK, LAYOUT, LAYOUT, ARG, OK),
    "line_hashes":           (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, OK, LAYOUT, OK, OK, OK, OK, LAYOUT),
    "statements":            (OK, LAYOUT, LAYOUT, LAYOUT, LAYOUT, LAYOUT, OK, OK, OK, OK, OK, OK, LAYOUT),
}


def _fault_corpus(files, fault):
    """Three files in an arena with room past off[n], n_groups 2, and one fault of the layout or tag rules (SPEC section 1).
    Returns the tsm_corpus and the arrays it points into."""
    off = np.array([0, 128, 256, 384], np.int32)
    arena = np.zeros(1024, np.uint8)
    for o, f in zip(off, files):
        arena[o:o + len(f)] = np.frombuffer(f, np.uint8)
    a = {"arena": arena, "off": off, "len": np.array([len(f) for f in files], np.int32), "ext": np.ones(3, np.uint8),
         "grp": np.array([0, 1, 0], np.uint16)}
    n_groups = 2
    if fault in ("misaligned_off", "groups_mismatch_and_misaligned_off"):
        off[1] = 130
    elif fault == "negative_off":
        off[0] = -128
    elif fault == "negative_len":
        a["len"][1] = -1
    elif fault == "runs_into_next":
        a["len"][1] = 200
    elif fault == "off_far_past_arena":
        off[1] = 2 ** 31 - 128
    elif fault == "misaligned_end":
        off[3] = 385
    elif fault == "ext_7":
        a["ext"][1] = 7
    elif fault == "ext_null":
        a["ext"] = None
    elif fault == "grp_out_of_range":
        a["grp"][1] = 2
    elif fault == "no_groups":
        n_groups = 0
    if fault.startswith("groups_mismatch"):
        n_groups = 3
    k = ts._Corpus(*(ts._p(a[f]) for f in ("arena", "off", "len", "ext", "grp")), 3, n_groups)
    return k, a


def _call(entry, ctx, old, new, clean):
    """One call of `entry` on the corpus `new` (pair calls: on the pair (old, new)); returns its status."""
    L = ts.lib()
    add, rem, det = np.zeros(3, np.int64), np.zeros(3, np.int64), np.zeros(3, ts.DIFF_DETAIL)
    tables = np.zeros((2, 3 * ts.K), np.int64)
    out, res = ts._DiffAsserts(ts._p(tables[0]), ts._p(tables[1]), None, 0, 0, None, 0, 0), ts._Result()
    base, n_lines = np.zeros(4, np.int64), C.c_int64()
    line_end, line_kind = np.zeros(256, np.uint32), np.zeros(256, np.uint8)
    o, k = C.byref(old), C.byref(new)
    if entry == "scan":
        return L.tsm_scan(ctx, k, C.byref(res), 0, None)
    if entry == "upload":
        return L.tsm_upload(ctx, k, None)
    if entry == "diff_pairs":
        return L.tsm_diff_pairs(ctx, o, k, ts._p(add), ts._p(rem), None)
    if entry == "diff_pairs_detail":
        return L.tsm_diff_pairs_detail(ctx, o, k, ts._p(add), ts._p(rem), ts._p(det), None)
    if entry == "diff_pairs_asserts":
        return L.tsm_diff_pairs_asserts(ctx, o, k, ts._p(add), ts._p(rem), None, C.byref(out), None)
    if entry == "diff_upload":
        return L.tsm_diff_upload(ctx, o, k, None)
    if entry.startswith("diff_resident"):
        assert L.tsm_diff_upload(ctx, C.byref(clean), C.byref(clean), None) == OK
        L.tsm_diff_upload(ctx, o, k, None)
        if entry == "diff_resident":
            return L.tsm_diff_resident(ctx, ts._p(add), ts._p(rem), ts._p(det), None)
        return L.tsm_diff_resident_asserts(ctx, ts._p(add), ts._p(rem), ts._p(det), C.byref(out), None)
    if entry == "line_hashes":
        return L.tsm_line_hashes(ctx, k, ts._p(base), None, None, None, 256, C.byref(n_lines), 0, None, None)
    assert entry == "statements"
    return L.tsm_statements(ctx, k, ts._p(base), ts._p(line_end), ts._p(line_kind), 256, C.byref(n_lines), None)


@pytest.mark.parametrize("entry", sorted(STATUS))
def test_layout_and_tag_faults_give_the_same_status_everywhere(entry):
    """The exact status of every corpus-taking entry point for one fault at a time: which of the rules (ext, grp, n_groups,
    off[n]) each call checks, and in which order.  A pair call gets the fault on either side, the other side none (for
    no_groups: n_groups 0 as well)."""
    old_files = [b"assert x == 1\n", b"def test_a():\n    self.assertTrue(y)\n", b"x = 1\n"]
    new_files = [b"assert x == 2\n", b"def test_a():\n    assert y\n    z = 1\n", b"x = 1\ny = 2\n"]
    sc = ts.Scanner(device=0, max_arena_bytes=1 << 20, max_files=16, max_groups=4)
    clean, clean_arrays = _fault_corpus(new_files, "none")
    bad = {}
    for fault, want in zip(FAULTS, STATUS[entry]):
        partner = "no_groups" if fault == "no_groups" else "none"
        for faulty in ("new", "old") if entry.startswith("diff") else ("new",):
            old, old_arrays = _fault_corpus(old_files, fault if faulty == "old" else partner)
            new, new_arrays = _fault_corpus(new_files, fault if faulty == "new" else partner)
            got = _call(entry, sc._ctx, old, new, clean)
            if got != want:
                bad[fault, faulty] = (got, want)
    sc.close()
    assert not bad, bad


def _pairs(seed, n, size_cap, lam=6.0):
    """BASELINE config C5 shape: old ~ C4 law capped, new = old with Poisson(lam) line edits."""
    base = ts.gen_corpus(0x7053454D0005 + seed, n, size_law=1, pinned=False)
    olds = [base.file_bytes(i)[:size_cap] for i in range(n)]
    news = [ts.gen_edit(1000 + seed * 7919 + i, o, lam) for i, o in enumerate(olds)]
    return olds, news


def check_diff(scanner, olds, news):
    a = ts.pack(olds, [1] * len(olds))
    b = ts.pack(news, [1] * len(news))
    add, rem = scanner.diff_pairs(a, b)
    wadd, wrem = orc.diff_pairs((a.arena, a.off, a.len), (b.arena, b.off, b.len))
    bad = np.nonzero((add != wadd) | (rem != wrem))[0]
    assert bad.size == 0, (bad[:5], add[bad[:5]], wadd[bad[:5]], rem[bad[:5]], wrem[bad[:5]])
    return add, rem


def test_diff_edge_cases(scanner):
    olds = [b"", b"a\n", b"a\nb\nc\n", b"a\nb\nc", b"x\n" * 100, b"same\n" * 50, b"a\nb\n", b"q\r\nr\n", b"1\n2\n3\n4\n5\n",
            b"\n\n\n", b"only old\n", b""]
    news = [b"", b"a\n", b"a\nc\n", b"a\nb\nc\n", b"y\n" * 70, b"same\n" * 50, b"b\na\n", b"q\nr\r\n", b"5\n4\n3\n2\n1\n",
            b"\n", b"", b"only new\nsecond\n"]
    add, rem = check_diff(scanner, olds, news)
    assert (add[0], rem[0]) == (0, 0) and (add[2], rem[2]) == (0, 1) and (add[4], rem[4]) == (70, 100)
    assert (add[7], rem[7]) == (0, 0)          # a trailing CR is not part of the line content (SPEC section 3)
    assert (add[3], rem[3]) == (0, 0)          # "c" with and without a final newline is the same line


def test_diff_c5_shape(scanner):
    olds, news = _pairs(1, 400, 65536)
    add, rem = check_diff(scanner, olds, news)
    assert add.sum() > 0 and rem.sum() > 0
    # cloc = added + removed (ML-Testing-v1.xlsx!projects:R1) and the identity pair has none
    same_add, same_rem = scanner.diff_pairs(ts.pack(olds[:50], [1] * 50), ts.pack(olds[:50], [1] * 50))
    assert same_add.sum() == 0 and same_rem.sum() == 0


def test_diff_heavy_edits_and_unrelated_files(scanner):
    olds, news = _pairs(2, 60, 20000, lam=80.0)
    check_diff(scanner, olds, news)
    olds2, _ = _pairs(3, 40, 12000)
    _, news2 = _pairs(4, 40, 12000)
    check_diff(scanner, olds2, news2)          # unrelated files: D close to n + m


def check_diff_detail(scanner, olds, news, exts):
    a = ts.pack(olds, exts)
    b = ts.pack(news, exts)
    add, rem, det = scanner.diff_pairs(a, b, detail=True)
    wadd, wrem, wdet = orc.diff_pairs_detail((a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext))
    assert np.array_equal(add, wadd) and np.array_equal(rem, wrem)
    for f in det.dtype.names:
        bad = np.nonzero(det[f] != wdet[f])[0]
        assert bad.size == 0, (f, bad[:5], det[bad[:5]], wdet[bad[:5]])
    return add, rem, det


def test_diff_hunks_and_classification(scanner):
    olds = [b"a\nb\nc\n", b"a\nb\nc\n", b"def t():\n  assert x\n  y = 1\n", b"", b"k\n" * 9, b"EXPECT_EQ(a, b);\nfoo\n"]
    news = [b"a\nc\n", b"a\nB\nc\nd\n", b"def t():\n  assert x == 2\n  y = 1\n  assert y\n", b"assert q\n", b"", b"foo\nEXPECT_EQ(a, b);\n"]
    add, rem, det = check_diff_detail(scanner, olds, news, [1, 1, 1, 1, 1, 2])
    assert (det["hunks_del"][0], det["hunks_mod"][1], det["hunks_add"][1]) == (1, 1, 1)
    assert (det["added_assert"][2], det["removed_assert"][2]) == (2, 1)
    assert det["hunks_add"][3] == 1 and det["added_assert"][3] == 1 and det["hunks_del"][4] == 1
    o2, n2 = _pairs(7, 300, 40000)
    exts = [1 + (i % 2) for i in range(300)]
    add, rem, det = check_diff_detail(scanner, o2, n2, exts)
    assert int((det["hunks_add"] + det["hunks_del"] + det["hunks_mod"]).sum()) > 300
    o3, n3 = _pairs(8, 40, 15000, lam=60.0)
    check_diff_detail(scanner, o3, n3, [1] * 40)


def test_diff_limits_of_the_one_launch_kernel(scanner):
    """k_diff_small finishes a pair in the first of its four sizes that holds it (middle <= 512 lines and D <= 31,
    1 024 / 63, 4 096 / 63, 4 096 / 127); everything else goes to k_myers / k_myers_trace.  Pairs on both sides of every limit, with
    detail, against the oracle."""
    def lines(tag, n):
        return [b"%s%05d\n" % (tag, i) for i in range(n)]
    olds, news, want_rem = [], [], []
    for total, ds in ((250, (1, 15, 30, 31, 32, 33)), (500, (62, 63, 64, 65)), (1300, (31, 64, 126, 127, 128, 129, 200))):
        for d in ds:                                        # d deletions spread over the file: D = d
            o = lines(b"assert x", total)
            keep = [l for i, l in enumerate(o) if not (i % (total // d) == 3 and i // (total // d) < d)]
            assert len(o) - len(keep) == d
            olds.append(b"".join(o)); news.append(b"".join(keep)); want_rem.append(d)
    n_del = len(olds)
    for d in (16, 31, 32, 64):                              # replacements: D = 2 d, hunks of kind mod
        o = lines(b"y = ", 300)
        n = list(o)
        for j in range(d):
            n[5 + 4 * j] = b"EXPECT_EQ(%d, q);\n" % j
        olds.append(b"".join(o)); news.append(b"".join(n))
    for total in (510, 512, 514, 1022, 1024, 1026, 4094, 4096, 4098, 6000):   # middle of `total` lines on both sides together, 2 edits at its ends
        half = total // 2
        o = [b"first old\n"] + lines(b"m", half - 2) + [b"last old\n"]
        n = [b"first new\n"] + lines(b"m", total - half - 2) + [b"assert last_new\n"]
        olds.append(b"head\n" * 40 + b"".join(o) + b"tail\n" * 40); news.append(b"head\n" * 40 + b"".join(n) + b"tail\n" * 40)
    olds += [b"", b"a\n" * 3000, b"".join(lines(b"p", 40)), b"same\n" * 5000]
    news += [b"b\n" * 2500, b"", b"".join(lines(b"q", 40)), b"same\n" * 5000]
    exts = [1] * n_del + [2] * 4 + [1] * 14
    add, rem, det = check_diff_detail(scanner, olds, news, exts)
    assert [int(x) for x in rem[:n_del]] == want_rem and int(add[:n_del].sum()) == 0
    assert [int(x) for x in det["hunks_mod"][n_del:n_del + 4]] == [16, 31, 32, 64] and int(det["added_assert"][n_del + 1]) == 31
    assert (int(add[-4]), int(rem[-4])) == (2500, 0) and (int(add[-1]), int(rem[-1])) == (0, 0)
    a = ts.pack(olds, exts)
    b = ts.pack(news, exts)
    add2, rem2 = scanner.diff_pairs(a, b)                   # and without detail (no rows kept)
    assert np.array_equal(add2, add) and np.array_equal(rem2, rem)


def test_statement_kinds(scanner):
    """SPEC section 10 line kinds: GPU (SWAR parenthesis counts + clamped warp scan) against the oracle."""
    corpora = []
    files, exts, grps = cu.edge_corpus()
    corpora.append(ts.pack(files, exts))
    files, exts, grps = cu.fuzz_corpus(31, 300, 20000, long_lines=True)
    corpora.append(ts.pack(files, exts))
    corpora.append(ts.gen_corpus(0x7053454D0004, 800, 1, pinned=False))
    corpora.append(ts.pack([b"(" * 100 + b"\n" + b"x\n" * 50 + b")" * 100 + b"\ny\n", b"\n" * 3000 + b"f(\n" * 40, b""], [2, 1, 1]))
    for c in corpora:
        gb, ge, gk = scanner.statements(c)
        ob, oe, ok = orc.statements(c.arena, c.off, c.len)
        assert np.array_equal(gb, ob) and np.array_equal(ge, oe)
        bad = np.nonzero(gk != ok)[0]
        assert bad.size == 0, (bad[:10], gk[bad[:10]], ok[bad[:10]])


def check_line_records(scanner, c, ngram=3):
    gb, gh, ge, gf, gn = scanner.line_hashes(c, ngram=ngram)
    ob, oh, oe, of_ = orc.line_records(c.arena, c.off, c.len, c.ext)
    assert np.array_equal(gb, ob), (gb[:5], ob[:5])
    for name, a, b in (("hash", gh, oh), ("end", ge, oe), ("flag", gf, of_), ("ngram", gn, orc.ngram_hashes(oh, ob, ngram))):
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (name, bad[:8], a[bad[:4]], b[bad[:4]])


def test_line_records_and_ngrams(scanner):
    """S9 (SPEC section 3): line_hash / line_end / line_flag of every line in file order and the n-gram hashes over
    them, from the scan kernel's one pass, against the oracle: edge files, fuzz (long lines, many chunks), C4 shape."""
    files, exts, _ = cu.edge_corpus()
    check_line_records(scanner, ts.pack(files, exts))
    check_line_records(scanner, ts.pack(files, exts), ngram=1)
    files, exts, _ = cu.fuzz_corpus(41, 200, 30000, long_lines=True)
    check_line_records(scanner, ts.pack(files, exts), ngram=5)
    check_line_records(scanner, ts.pack([b"\n" * 9000 + b"assert x\n" * 50, b"", b"a" * 9000, b"x\n" * 5000 + b"tail"], [1, 1, 2, 3]))
    check_line_records(scanner, ts.gen_corpus(0x7053454D0004, 300, 1, pinned=False), ngram=2)
    gb, gh, ge, gf = scanner.line_hashes(ts.pack([], []))
    assert gb.tolist() == [0] and len(gh) == 0


def test_rev_b_mode_matches_the_oracle(scanner):
    """TSM_SCAN_REV_B (docs/SPEC.md section 4b): second automaton word for the extra triggers, full statements, Rev-B
    categories - every output against the oracle's Rev-B mode."""
    fl = FLAGS | ts.SCAN_REV_B
    def check(c):
        want = orc.scan(c.arena, c.off, c.len, c.ext, c.grp, c.n_groups, rev_b=True)
        got = scanner.scan(c, fl)
        for f in ("n_lines", "n_assert", "n_headers", "n_fixture", "digest"):
            bad = np.nonzero(got["stats"][f] != want["stats"][f])[0]
            assert bad.size == 0, (f, bad[:10], got["stats"][bad[:5]], want["stats"][bad[:5]])
        assert np.array_equal(got["group_counts"], want["group_counts"])
        for k in ("assert_events", "header_events"):
            a, b = got[k], want[k]
            assert len(a) == len(b), (k, len(a), len(b))
            for f in a.dtype.names:
                bad = np.nonzero(a[f] != b[f])[0]
                assert bad.size == 0, (k, f, a[bad[:5]], b[bad[:5]])
        return got
    body = (b"BOOST_AUTO_TEST_CASE(ZeroBit57) {\n  BOOST_CHECK_EQUAL(0xFF, x);\n  BOOST_CHECK(!left.full);\n  BOOST_CHECK(a == b); // c\n"
            b"  NTA_CHECK(x > 3) << \"m\";\n  TESTEQUAL(a, b);\n  FAIL();\n  SLOPPY_CHECK_CLOSE(a, b);\n  assert (n == 1); // java style\n}\n")
    files = [body, body * 300, b"x" * 4090 + b"_CHECK(\n" + body, b"FAIL", b"_CHEC\nK", b"y" * 8188 + b"TESTEQUAL(q)\n"]
    files += [b"#" * pad + b"\n" + b"a_CHECK\nFAIL\n" * 1200 for pad in (0, 3, 7, 129)]
    check(ts.pack(files, [2, 3, 2, 1, 2, 4, 2, 1, 4, 6]))
    for seed in (71, 72):
        f2, e2, g2 = cu.fuzz_corpus(seed, 300, 12000, long_lines=seed == 72)
        check(ts.pack(f2, e2, g2, 5))
    # golden G1 from the GPU's own events (the 26 bundled DeepSpeech files of the C1 fixture)
    import json, os
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    golden = json.load(open(os.path.join(gold, "g1_deepspeech.json")))
    names = cu.load_fixture_names(os.path.join(gold, "c1_testfiles.npz"))
    allf, exts, _, _ = cu.load_fixture(os.path.join(gold, "c1_testfiles.npz"))
    keep = [i for i, n in enumerate(names) if n in golden]
    sub = [allf[i] for i in keep]
    got = check(ts.pack(sub, exts[keep]))
    stm, cnt, per_file = cu.score_g1(golden, [names[i] for i in keep], sub, got["assert_events"])
    assert stm == [72, 79] and cnt == [326, 427]
    assert per_file["DeepSpeech/v0.9.3/native_client/kenlm/util/bit_packing_test.cc"] == ([1, 1], [6, 6])
