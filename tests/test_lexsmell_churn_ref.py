"""CPU tests of the lexical test-smell churn references (docs/SPEC.md section 26): the plain-Python restatement
lexsmell_churn_ref.py_lexsmell_churn on hand-written pairs with known rows (the worked examples of the section among them), and
the numpy reference tests/orc_lexsmell_churn.py (serial marks, serial smells and lexical smells, oracle events) agreeing with it
there, on a planted history, on fuzz pairs with long lines and binary bytes and on C5 pairs."""
import collections

import case_ref as cr
import lexsmell_churn_ref as lcr
import lexsmell_ref as lr
import orc_lexsmell_churn as olc
import pytest
import tosemscan as ts

PY, CC = 1, 2
UT = b"class T(unittest.TestCase):\n    def test_a(self):\n"


def ut(*lines):
    return UT + b"".join(b"        " + x + b"\n" for x in lines)


def open_call(d, msg):
    """An assertEqual whose argument list closes d lines below its first line (walk line d), then one more unexplained assertion."""
    return ut(*([b"self.assertEqual(", b"    x"] + [b"    + x"] * (d - 2) + [b"    , y%s)" % msg, b"self.assertTrue(z)"]))


# (name, old, new, ext_old, ext_new, rows): rows as py_lexsmell_churn gives them
CASES = [
    ("AR introduced by an insertion: the kept line gains the bit too",
     ut(b"self.assertEqual(f(x), y)"), ut(b"self.assertEqual(f(x), y)", b"self.assertEqual(g(x), y)"), PY, PY,
     [(b"test_a", "M", 2, 2, "assertion_roulette", "introduced", 2, 0, 2, 0)]),
    ("the same insertion with a message",
     ut(b"self.assertEqual(f(x), y)"), ut(b"self.assertEqual(f(x), y)", b'self.assertEqual(g(x), y, "why")'), PY, PY, []),
    ("gtest AR removed through a kept line",
     b"TEST(S, A) {\n  EXPECT_EQ(a, b);\n  EXPECT_EQ(c, d);\n}\n", b"TEST(S, A) {\n  EXPECT_EQ(a, b) << \"why\";\n  EXPECT_EQ(c, d);\n}\n",
     CC, CC, [(b"A", "M", 1, 1, "assertion_roulette", "removed", 0, 2, 0, 2)]),
    ("a call over three lines: only its last line edited",
     ut(b"self.assertEqual(", b"    f(x),", b"    y)", b"self.assertTrue(z)"),
     ut(b"self.assertEqual(", b"    f(x),", b'    y, msg="m")', b"self.assertTrue(z)"), PY, PY,
     [(b"test_a", "M", 2, 2, "assertion_roulette", "removed", 0, 2, 0, 2)]),
    ("magic number replaced by a name",
     ut(b"self.assertEqual(n, 5)"), ut(b"self.assertEqual(n, FIVE)"), PY, PY,
     [(b"test_a", "M", 2, 2, "magic_number", "removed", 0, 1, 0, 1)]),
    ("suboptimal assert rewritten",
     ut(b'self.assertTrue(x == y, "m")'), ut(b'self.assertEqual(x, y, "m")'), PY, PY,
     [(b"test_a", "M", 2, 2, "suboptimal_assert", "removed", 0, 1, 0, 1)]),
    ("mystery guest inserted into a kept test",
     b"def test_a():\n    x = 1\n    assert x\n", b'def test_a():\n    x = 1\n    with open("data.csv") as f:\n        pass\n    assert x\n',
     PY, PY, [(b"test_a", "M", 1, 1, "mystery_guest", "introduced", 1, 0, 1, 0)]),
    ("obscure setup: the eleventh local name, the kept header gains the bit",
     b"def test_a():\n" + b"".join(b"    v%d = 0\n" % i for i in range(10)) + b"    assert v0\n",
     b"def test_a():\n" + b"".join(b"    v%d = 0\n" % i for i in range(11)) + b"    assert v0\n", PY, PY,
     [(b"test_a", "M", 1, 1, "obscure_setup", "introduced", 1, 0, 1, 0)]),
    ("obscure setup from 12 to 30 names with the header kept: no row",
     b"def test_a():\n" + b"".join(b"    v%d = 0\n" % i for i in range(12)) + b"    assert v0\n",
     b"def test_a():\n" + b"".join(b"    v%d = 0\n" % i for i in range(30)) + b"    assert v0\n", PY, PY, []),
    ("obscure setup kept with the header edited: changed",
     b"def test_a():\n" + b"".join(b"    v%d = 0\n" % i for i in range(12)) + b"    assert v0\n",
     b"def test_a(tmp):\n" + b"".join(b"    v%d = 0\n" % i for i in range(12)) + b"    assert v0\n", PY, PY,
     [(b"test_a", "M", 1, 1, "obscure_setup", "changed", 1, 1, 1, 1)]),
    ("a docstring opened above kept assertions turns them into string content",
     b"def test_a():\n    x = 1\n    assert x == 1\n    assert x == 1, 'm'\n    assert y == 2\n",
     b'def test_a():\n    s = """\n    x = 1\n    assert x == 1\n    assert x == 1, \'m\'\n    assert y == 2\n', PY, PY,
     [(b"test_a", "M", 1, 1, "assertion_free", "introduced", 1, 0, 1, 0),
      (b"test_a", "M", 1, 1, "assertion_roulette", "removed", 0, 2, 0, 2),
      (b"test_a", "M", 1, 1, "magic_number", "removed", 0, 3, 0, 3)]),
    ("CRLF lines and unterminated last lines",
     b"def test_a():\r\n    assert f(x) == y\r\n    assert g(x)",
     b"def test_a():\r\n    assert f(x) == y\r\n    assert g(x)\r\n    assert h(x) == 3", PY, PY,
     [(b"test_a", "M", 1, 1, "assertion_roulette", "changed", 3, 2, 1, 0),
      (b"test_a", "M", 1, 1, "magic_number", "introduced", 1, 0, 1, 0)]),
    (".py paired with a .cc",
     b"def test_a():\n    with open('f') as fh:\n        pass\n    assert x == 2\n",
     b"def test_a():\n    with open('f') as fh:\n        pass\n    assert x == 2\n", PY, CC,
     [(b"test_a", "D", None, 1, "magic_number", "removed", None, 1, None, 1),
      (b"test_a", "D", None, 1, "mystery_guest", "removed", None, 1, None, 1)]),
    ("smells moved between two tests",
     b"def test_a():\n    self.assertEqual(a, 5)\n    assert b\ndef test_b():\n    assert c\n",
     b"def test_a():\n    assert b\ndef test_b():\n    self.assertEqual(a, 5)\n    assert c\n", PY, PY,
     [(b"test_a", "M", 1, 1, "assertion_roulette", "removed", 0, 2, 0, 2),
      (b"test_a", "M", 1, 1, "magic_number", "removed", 0, 1, 0, 1),
      (b"test_b", "M", 3, 4, "assertion_roulette", "introduced", 2, 0, 2, 0),
      (b"test_b", "M", 3, 4, "magic_number", "introduced", 1, 0, 1, 0)]),
    ("a call left open across an edit at walk line 63: inside the cap",
     open_call(63, b""), open_call(63, b", msg='m'"), PY, PY,
     [(b"test_a", "M", 2, 2, "assertion_roulette", "removed", 0, 2, 0, 2)]),
    ("the same at walk line 64: beyond the cap", open_call(64, b""), open_call(64, b", msg='m'"), PY, PY, []),
]


def test_known_answers():
    for name, old, new, xo, xn, rows in CASES:
        assert lcr.py_lexsmell_churn(old, new, xo, xn) == rows, name


def test_obscure_setup_changed_case_is_on_the_header():
    """The changed obscure_setup row churns the header line on both sides: the statement of the old side's 12 names is unchanged."""
    _, old, new, xo, xn, _ = next(c for c in CASES if c[0].startswith("obscure setup kept"))
    deleted, inserted, _ = lcr.scr.py_script_lines(old, new, xo, xn)
    assert deleted == {0} and inserted == {0}
    assert lr.file_lexsmells(new, xn)[1][0] == lr.LBIT["obscure_setup"]


def test_untraced_pair_changes_its_whole_middle(monkeypatch):
    """Above the trace limit every line of the middle is deleted and inserted, so the kept magic number is churned on both sides
    (the limit is lowered here: a real untraced pair is too slow for the Python diff and is checked on the GPU)."""
    old = b"def test_a():\n    a = 1\n    assert n == 5\n    b = 1\n    assert a, 'm'\n"
    new = b"def test_a():\n    a = 2\n    assert n == 5\n    b = 2\n    assert a, 'm'\n"
    assert lcr.py_lexsmell_churn(old, new, PY, PY) == []
    monkeypatch.setattr(cr, "TRACE_MAX_D", 1)
    assert lcr.py_lexsmell_churn(old, new, PY, PY) == [(b"test_a", "M", 1, 1, "magic_number", "changed", 1, 1, 1, 1)]


def references_agree(olds, news, exts_old, exts_new):
    a, b = ts.pack(olds, exts_old), ts.pack(news, exts_new)
    r = olc.diff_smells_lexical((a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext))
    got = olc.churn_rows(r, olds, news, exts_old, exts_new)
    want = {}
    for i, (o, n, xo, xn) in enumerate(zip(olds, news, exts_old, exts_new)):
        rows = lcr.py_lexsmell_churn(o, n, xo, xn)
        if rows:
            want[i] = rows
    assert got == want
    return r, want


def test_references_agree_on_the_known_answers():
    references_agree(*[list(x) for x in zip(*[c[1:5] for c in CASES])])


def planted_history(seed, n):
    olds, exts = lr.planted_corpus(seed, n)
    return olds, [ts.gen_edit(i, o, 6.0) for i, o in enumerate(olds)], [int(x) for x in exts]


def test_references_agree_on_a_planted_history():
    """Section-25 planted test files as old sides, gen_edit(lambda = 6) of each as new sides."""
    olds, news, ext = planted_history(19, 80)
    r, rows = references_agree(olds, news, ext, ext)
    lex = collections.Counter((x[1], x[5]) for rs in rows.values() for x in rs if x[4] in lr.LSMELLS)
    assert lex == PLANTED_LEX_EVENTS                           # the counts docs/SPEC.md section 26 pins
    assert (len(r["old_tests"]), len(r["new_tests"])) == PLANTED_TESTS


PLANTED_LEX_EVENTS = {("A", "introduced"): 6, ("D", "removed"): 80, ("M", "introduced"): 8, ("M", "removed"): 146,
                      ("M", "changed"): 79}
PLANTED_TESTS = (564, 527)


@pytest.mark.parametrize("long_lines,binary", [(True, False), (False, True)])
def test_references_agree_on_fuzz_pairs(long_lines, binary):
    olds, exts = lr.fuzz_with_calls(0x26 + binary, long_lines=long_lines, binary=binary)
    olds, exts = olds[:60], [int(x) for x in exts[:60]]
    news = [ts.gen_edit(i, o, 6.0) for i, o in enumerate(olds)]
    references_agree(olds, news, exts, exts)


def test_references_agree_on_c5_pairs():
    a, b = ts.gen_pairs(0x7053454D0005, 120, pinned=False)
    olds = [a.file_bytes(i) for i in range(a.n_files)]
    news = [b.file_bytes(i) for i in range(b.n_files)]
    ext = [int(x) for x in a.ext]
    r, _ = references_agree(olds, news, ext, ext)
    assert len(r["old_tests"]) > 0
