"""CPU tests: the plain-Python restatements of tests/spec_ref.py against the C oracle, on the edge corpus and on the byte
patterns tests/test_gpu_edges.py sends through the kernels (no GPU needed).  The GPU edge tests compare the device
with these references, so they are pinned here first."""
import json
import os
import random

import numpy as np

import corpus_util as cu
import orc
import spec_ref as sr

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def placed_hash_edges():
    """Every hash-edge content behind a few pads, before a CR-less last line and as an unterminated last line."""
    files = []
    for c in cu.hash_edge_contents():
        for pad in (0, 1, 7, 64):
            files.append(b"#" * pad + (b"\n" if pad else b"") + c + b"\n" + b"tail")
        files.append(b"x\n" + c)
    return files


def check_line_records(files, exts, ngrams=(1, 3, 62)):
    arena, off, ln = orc.pack(files)
    base, lh, end, flag = orc.line_records(arena, off, ln, np.array(exts, np.uint8))
    for i, f in enumerate(files):
        want = sr.py_line_records(f, exts[i])
        a, b = int(base[i]), int(base[i + 1])
        assert [(int(h), int(e), int(g)) for h, e, g in zip(lh[a:b], end[a:b], flag[a:b])] == want, (i, f[:40])
    for n in ngrams:
        got = orc.ngram_hashes(lh, base, n)
        for i in range(len(files)):
            a, b = int(base[i]), int(base[i + 1])
            assert [int(x) for x in got[a:b]] == sr.py_ngrams(lh[a:b], n), (i, n)


def test_line_records_reference_matches_the_oracle():
    files, exts, _ = cu.edge_corpus()
    check_line_records(files, [int(e) for e in exts])
    hf = placed_hash_edges()
    check_line_records(hf, [1] * len(hf), ngrams=(1, 5, 13))
    bf, bexts, _ = cu.fuzz_corpus(77, 200, 6000, binary=True)
    check_line_records(bf, [int(e) for e in bexts], ngrams=(2, 61, 200))


def test_hash_edge_contents_are_what_they_claim():
    contents = cu.hash_edge_contents()
    wraps = [c for c in contents if len(c) >= 9 and c.endswith(b"\r") and c[:-1] != b"\xff" * 8]
    assert len(wraps) == 147
    for c in wraps:
        n = len(c) - 1
        cr = 13 * pow(256, n, sr.M61) % sr.M61
        assert (int.from_bytes(c, "little")) % sr.M61 < cr           # the line's value with its CR wraps below the CR term
    zeros = [c for c in contents if c and int.from_bytes(c, "little") % sr.M61 == 0 and any(c)]
    assert len(zeros) >= 100
    for c in contents:
        assert sr.py_bytes_hash(c) == orc.bytes_hash(c)


def test_binary_fuzz_alphabet_leaves_the_ascii_seeds_alone():
    a = cu.fuzz_corpus(3, 40, 3000)
    b = cu.fuzz_corpus(3, 40, 3000, binary=False)
    assert a[0] == b[0]
    files, _, _ = cu.fuzz_corpus(3, 40, 3000, binary=True)
    blob = b"".join(files)
    assert len(set(blob)) == 256 and blob.count(b"\r") > blob.count(b"x")


def statements_for_category_checks():
    names = [n.encode() for n in sr.CATEGORY_NAMES.values()]
    ts = [b"self." + v for v in cu.table_name_variants(names)]
    ts += [r["statement"].encode("utf-8") for r in json.load(open(os.path.join(GOLD, "g4_statement_category.json")))]
    ts += [b"assert", b"assert x", b"assert not x", b"assert a not in b", b"assert a is not b", b"assert x == True",
           b"assert a == b", b"assert a != b", b"assert a <= b", b"assert a >= b", b"assert a < b", b"assert a > b",
           b"EXPECT_EQ", b"ASSERT_FLOAT_EQ", b"EXPECT_DOUBLE_EQ", b"EXPECT_STREQ", b"EXPECT_", b"x.assert_", b"assertx",
           b"assert\tx", b"GPUAssert", b"", b"assert_", b"x.assert", b"assertnot x"]
    return ts


def test_py_category_matches_the_oracle():
    rng = random.Random(9)
    ts = statements_for_category_checks()
    ts += [bytes(rng.choice(b"assertEXPCT_ notin=<>!Tue.xq") for _ in range(rng.randrange(0, 30))).strip() for _ in range(3000)]
    for t in ts:
        assert sr.py_category(t) == orc.classify(t)[0], t
        assert sr.py_category_string(t) == orc.category_string(t), t


def test_py_category_reproduces_golden_g4_with_the_ledger_misses():
    rows = json.load(open(os.path.join(GOLD, "g4_statement_category.json")))
    ledger = json.load(open(os.path.join(GOLD, "ledger.json")))["G4"]
    hit, tot, misses = 0, 0, set()
    for r in rows:
        tot += r["rows"]
        if sr.py_category_string(r["statement"].encode("utf-8")) == r["category"]:
            hit += r["rows"]
        else:
            misses.add((r["statement"], r["category"]))
    assert [hit, tot] == [11954, 11981]
    assert misses == {(m["statement"], m["sheet_says"]) for m in ledger["misses"]}


def diff_edge_pairs():
    """The hand-built pairs of the GPU diff tests: empty sides, pure hunks, CR and final-LF twins, reversed and
    repeated lines, replaced assertion lines."""
    olds = [b"", b"a\n", b"a\nb\nc\n", b"a\nb\nc", b"x\n" * 100, b"same\n" * 50, b"a\nb\n", b"q\r\nr\n", b"1\n2\n3\n4\n5\n",
            b"\n\n\n", b"only old\n", b"", b"a\nb\nc\n", b"a\nb\nc\n", b"def t():\n  assert x\n  y = 1\n", b"", b"k\n" * 9,
            b"EXPECT_EQ(a, b);\nfoo\n", b"x = 1\nself.assertEqual(a, b)\ny = 2\n", b"assert a\n" * 300, b"a\nb\n" * 40]
    news = [b"", b"a\n", b"a\nc\n", b"a\nb\nc\n", b"y\n" * 70, b"same\n" * 50, b"b\na\n", b"q\nr\r\n", b"5\n4\n3\n2\n1\n",
            b"\n", b"", b"only new\nsecond\n", b"a\nc\n", b"a\nB\nc\nd\n", b"def t():\n  assert x == 2\n  y = 1\n  assert y\n",
            b"assert q\n", b"", b"foo\nEXPECT_EQ(a, b);\n", b"x = 1\nself.assertTrue(a)\ny = 2\n", b"", b"b\na\n" * 40]
    exts = [1] * 17 + [2, 1, 4, 1]
    return olds, news, exts


def check_diff_script(olds, news, exts):
    """py_diff_script against orc.diff_pairs_detail (added, removed, hunks, assertion counts) and orc_asserts (which lines
    change: the events of the deleted / inserted assertion lines).  Returns the reference's tuples."""
    import orc_asserts
    a, b = orc.pack(olds), orc.pack(news)
    e = np.array(exts, np.uint8)
    add, rem, det = orc.diff_pairs_detail(a + (e,), b + (e,))
    _, _, aev, rev = orc_asserts.diff_pairs_asserts(a + (e,), b + (e,))
    got_a = {(int(f), int(o)) for f, o in zip(aev["file"], aev["line_off"])}
    got_r = {(int(f), int(o)) for f, o in zip(rev["file"], rev["line_off"])}
    want_a, want_r, out = set(), set(), []
    for i, (o, n, x) in enumerate(zip(olds, news, exts)):
        r = sr.py_diff_files(o, n, x, x)
        out.append(r)
        assert r[:7] == (int(add[i]), int(rem[i]), *(int(det[i][f]) for f in det.dtype.names)), (i, r[:7], add[i], rem[i], det[i])
        fo, fn = [t[2] for t in sr.py_line_records(o, x)], [t[2] for t in sr.py_line_records(n, x)]
        so, sn = sr.py_line_starts(o), sr.py_line_starts(n)
        want_r |= {(i, so[j]) for j in r[7] if fo[j]}
        want_a |= {(i, sn[j]) for j in r[8] if fn[j]}
    assert got_a == want_a and got_r == want_r
    assert len(aev) == len(got_a) and len(rev) == len(got_r)
    return out


def test_py_diff_script_on_the_diff_edge_cases():
    out = check_diff_script(*diff_edge_pairs())
    assert out[2][:5] == (0, 1, 0, 1, 0) and out[6][:5] == (1, 1, 1, 1, 0) and out[19][:7] == (0, 300, 0, 1, 0, 0, 300)
    assert out[3][:2] == (0, 0) and out[7][:2] == (0, 0)          # final-LF and CR twins are the same line


def test_py_diff_script_on_tie_heavy_pairs():
    olds, news, exts = cu.tie_heavy_pairs(31)
    out = check_diff_script(olds, news, exts)
    assert sum(r[5] + r[6] for r in out) > 100                    # assertion lines change
    assert sum(r[4] for r in out) > 50 and sum(r[2] for r in out) > 500 and sum(r[3] for r in out) > 500


def test_py_diff_script_on_closed_form_shapes():
    shapes = [((0, 5, 0), (3, 0, 7)), ((4,), (4,)), ((0,), (9,)), ((9,), (0,)), ((1, 1, 1, 1), (0, 2, 0, 2)),
              ((40, 0, 13, 2), (0, 17, 5, 0)), ((0, 0), (0, 0))]
    olds, news, wants = [], [], []
    for i, (ob, nb) in enumerate(shapes):
        o, n, want = cu.block_pair(b"s%d" % i, ob, nb, n_prefix=i % 3, n_suffix=(i + 1) % 3)
        olds.append(o)
        news.append(n)
        wants.append(want)
    out = check_diff_script(olds, news, [1] * len(olds))
    for r, want, o, n in zip(out, wants, olds, news):
        assert r[2:5] == want[:3] and r[7] == want[3] and r[8] == want[4]
        assert (r[0], r[1]) == (len(want[4]), len(want[3]))
