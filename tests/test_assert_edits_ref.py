"""CPU tests of the assertion edits of docs/SPEC.md section 17: known answers of the plain-Python restatement (edit_ref.py) on
hand-written pairs, agreement with the numpy + C reference (orc_assert_edits.py) there and on C5 pairs, and the bit-parallel LCS
recurrence the kernels run against the LCS table."""
import random

import numpy as np

import edit_ref as er
import orc_assert_edits as oae
import tosemscan as ts

PY, CC = 1, 2


def lines(*ls):
    return b"".join(l + b"\n" for l in ls)


# (name, old, new, ext_old, ext_new, edits as (old line, new line, score), 0-based lines)
CASES = [
    ("assertEqual becomes assertAlmostEqual",
     lines(b"x = 1", b"    self.assertEqual(a, b)", b"y = 2"), lines(b"x = 1", b"    self.assertAlmostEqual(a, b)", b"y = 2"), PY, PY,
     [(1, 1, 120000 * 22 // 50)]),
    ("re-indent pairs with itself at 100 %",
     lines(b"def t():", b"  assert x == 1", b"  assert y"), lines(b"def t():", b"        assert x == 1", b"\tassert y"), PY, PY,
     [(1, 1, 60000), (2, 2, 60000)]),
    ("CRLF and indentation against LF",
     b"k = 0\r\n  assert z  \r\nm = 1\r\n", b"k = 0\r\n    assert z\nm = 1\r\n", PY, PY, [(1, 1, 60000)]),
    ("exactly at the threshold: 4 lcs = |a| + |b|",
     lines(b"k", b"assertAAAAAA", b"m"), lines(b"k", b"assertBBBBBB", b"m"), PY, PY, [(1, 1, 30000)]),
    ("just below the threshold: 4 lcs = |a| + |b| - 1",
     lines(b"k", b"assertAAAAAA", b"m"), lines(b"k", b"assertBBBBBBB", b"m"), PY, PY, []),
    ("tie on the new line: the old line first wins",
     lines(b"k", b"assert foo", b"assert foo", b"m"), lines(b"k", b"assert fooo", b"m"), PY, PY, [(1, 1, 120000 * 10 // 21)]),
    ("tie on the old line: the new line first wins",
     lines(b"k", b"assert foo", b"m"), lines(b"k", b"assert fop", b"assert foq", b"m"), PY, PY, [(1, 1, 120000 * 9 // 20)]),
    ("one deleted line best for two inserted lines",
     lines(b"k", b"assert alpha == 1", b"m"), lines(b"k", b"assert alpha == 2", b"assert alpha == 1  # x", b"m"), PY, PY,
     [(1, 1, 120000 * 16 // 34)]),
    ("two deleted lines and three inserted, one left over",
     lines(b"k", b"assert len(x) == 3", b"assert y is None", b"m"),
     lines(b"k", b"assert len(x) == 4", b"assert z == 0", b"assert y is not None", b"m"), PY, PY,
     [(1, 1, 120000 * 17 // 36), (2, 3, 120000 * 16 // 36)]),
    ("two hunks around one kept line: identical text across them does not pair",
     lines(b"assert one(1)", b"K", b"assert two(2)"), lines(b"assert two(2) ", b"K", b"assert one(1) "), PY, PY,
     [(0, 0, 120000 * 10 // 26), (2, 2, 120000 * 10 // 26)]),
    ("pure insertion", lines(b"k", b"m"), lines(b"k", b"assert a", b"assert b", b"m"), PY, PY, []),
    ("pure deletion", lines(b"k", b"assert a", b"assert b", b"m"), lines(b"k", b"m"), PY, PY, []),
    ("a .py paired with a .cc",
     lines(b"def test():", b"    self.assertEqual(a, b)"), lines(b"TEST(S, T) {", b"  EXPECT_EQ(a, b);", b"}"), PY, CC,
     [(1, 1, 120000 * 7 // 38)] if 120000 * 7 // 38 >= 30000 else []),
]


def test_known_answers():
    for name, old, new, xo, xn, want in CASES:
        assert er.py_assert_edits(old, new, xo, xn) == want, name


def test_known_answer_scores_are_what_they_say():
    assert er.py_lcs(b"self.assertEqual(a, b)", b"self.assertAlmostEqual(a, b)") == 22
    assert er.py_lcs(b"assertAAAAAA", b"assertBBBBBB") == 6 and 4 * 6 == 12 + 12
    assert er.py_lcs(b"assertAAAAAA", b"assertBBBBBBB") == 6 and 4 * 6 == 12 + 13 - 1
    assert er.py_lcs(b"assert one(1)", b"assert two(2)") == 10
    assert er.py_lcs(b"assert one(1)", b"assert one(1)") == 13           # the 100 % pair lies across the kept line
    assert er.py_score(b"    self.assertEqual(a, b)", b"self.assertAlmostEqual(a, b)") // 600 == 88


def test_hunks_of_the_two_hunk_case():
    old, new = lines(b"assert one(1)", b"K", b"assert two(2)"), lines(b"assert two(2) ", b"K", b"assert one(1) ")
    assert er.py_hunks(old, new, PY, PY) == [([0], [0]), ([2], [2])]


def references_agree(olds, news, exts_old, exts_new):
    a, b = ts.pack(olds, exts_old), ts.pack(news, exts_new)
    got = oae.assert_edits((a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext))
    want = er.py_batch_edits(olds, news, exts_old, exts_new)
    assert [(int(e["rev"]), int(e["aev"]), int(e["score"])) for e in got] == want
    return want


def test_references_agree_on_the_known_answers():
    want = references_agree(*[list(x) for x in zip(*[c[1:5] for c in CASES])])
    assert len(want) == sum(len(c[5]) for c in CASES)


def test_references_agree_on_c5_pairs():
    """C5 edits rarely replace one assertion line by another: about one pair in 150 has an edit."""
    a, b = ts.gen_pairs(0x7053454D0005, 1500, pinned=False)
    olds = [a.file_bytes(i) for i in range(a.n_files)]
    news = [b.file_bytes(i) for i in range(b.n_files)]
    ext = [int(x) for x in a.ext]
    want = references_agree(olds, news, ext, ext)
    assert len(want) >= 5


def test_bit_parallel_lcs_equals_the_table():
    """Random strings of lengths 1 to 300 over small and large alphabets, including every 64-bit word edge."""
    rng = random.Random(17)
    lens = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 300] + [rng.randrange(1, 301) for _ in range(40)]
    for k, n in enumerate(lens):
        m = lens[(k * 7 + 3) % len(lens)]
        alpha = b"ab" if k % 3 == 0 else (b"abcdefgh" if k % 3 == 1 else bytes(range(256)))
        x = bytes(rng.choice(alpha) for _ in range(n))
        y = bytes(rng.choice(alpha) for _ in range(m))
        assert er.py_bitparallel_lcs(x, y) == er.py_lcs(x, y) == er.py_lcs(y, x), (n, m)


def test_scores_do_not_depend_on_pair_order():
    olds = [c[1] for c in CASES]
    news = [c[2] for c in CASES]
    xo, xn = [c[3] for c in CASES], [c[4] for c in CASES]
    fwd = er.py_batch_edits(olds, news, xo, xn)
    rev = er.py_batch_edits(olds[::-1], news[::-1], xo[::-1], xn[::-1])
    assert len(fwd) == len(rev) > 10
    assert np.array_equal(np.sort([s for *_, s in fwd]), np.sort([s for *_, s in rev]))
