"""CPU tests of the test-case churn references (docs/SPEC.md section 16): the plain-Python restatement case_ref.py_case_churn
on hand-written pairs with known answers, and the numpy reference tests/orc_cases.py (serial marks, oracle events) agreeing
with it there and on C5 pairs."""
import orc_cases
import case_ref as cr
import tosemscan as ts

PY, CC = 1, 2

# (name, old, new, ext_old, ext_new, rows): rows as py_case_churn gives them
CASES = [
    ("added, deleted and edited",
     b"import os\ndef test_a():\n    x = 1\n    assert x == 1\ndef test_b():\n    y = 2\ndef test_c():\n    z = 3\n",
     b"import os\ndef test_a():\n    x = 1\n    assert x == 2\ndef test_c():\n    z = 3\ndef test_d():\n    assert True\n",
     PY, PY,
     [(b"test_b", "D", None, 5, None, 2, None, 0, None, 2, None, 0),
      (b"test_a", "M", 2, 2, 3, 3, 1, 1, 1, 1, 1, 1),
      (b"test_d", "A", 7, None, 2, None, 1, None, 2, None, 1, None)]),
    ("header inserted in a case",
     b"def test_a():\n    a = 1\n    b = 2\n    c = 3\n",
     b"def test_a():\n    a = 1\ndef test_new():\n    b = 2\n    c = 3\n",
     PY, PY,
     [(b"test_a", "M", 1, 1, 2, 4, 0, 0, 0, 0, 0, 0),
      (b"test_new", "A", 3, None, 3, None, 0, None, 1, None, 0, None)]),
    ("header deleted",
     b"def test_a():\n    a = 1\ndef test_new():\n    b = 2\n    c = 3\n",
     b"def test_a():\n    a = 1\n    b = 2\n    c = 3\n",
     PY, PY,
     [(b"test_new", "D", None, 3, None, 3, None, 0, None, 1, None, 0),
      (b"test_a", "M", 1, 1, 4, 2, 0, 0, 0, 0, 0, 0)]),
    ("signature change matched by name",
     b"def test_x(self):\n    v = 1\n    assert v\n",
     b"def test_x(self, tmp):\n    v = 1\n    assert v\n",
     PY, PY,
     [(b"test_x", "M", 1, 1, 3, 3, 1, 1, 1, 1, 0, 0)]),
    ("duplicate names stay unmatched",
     b"def test_dup(a):\n    x = 1\ndef test_dup(b):\n    y = 2\n",
     b"def test_dup(c):\n    x = 1\ndef test_dup(d):\n    y = 2\n",
     PY, PY,
     [(b"test_dup", "D", None, 1, None, 2, None, 0, None, 1, None, 0),
      (b"test_dup", "D", None, 3, None, 2, None, 0, None, 1, None, 0),
      (b"test_dup", "A", 1, None, 2, None, 0, None, 1, None, 0, None),
      (b"test_dup", "A", 3, None, 2, None, 0, None, 1, None, 0, None)]),
    ("edits above the first header",
     b"import os\nX = 1\ndef test_a():\n    pass\n",
     b"import sys\ndef test_a():\n    pass\n",
     PY, PY, []),
    ("CRLF lines",
     b"def test_a():\r\n    x = 1\r\n",
     b"def test_a():\r\n    x = 2\r\n    assert x\r\n",
     PY, PY,
     [(b"test_a", "M", 1, 1, 3, 2, 1, 0, 2, 1, 1, 0)]),
    ("unterminated last line, same lines",
     b"def test_a():\n    x = 1", b"def test_a():\n    x = 1\n", PY, PY, []),
    ("unterminated header line added",
     b"def test_a():\n    x = 1\n", b"def test_a():\n    x = 1\ndef test_b():", PY, PY,
     [(b"test_b", "A", 3, None, 1, None, 0, None, 1, None, 0, None)]),
    ("empty old side",
     b"", b"def test_a():\n  pass\n", PY, PY,
     [(b"test_a", "A", 1, None, 2, None, 0, None, 2, None, 0, None)]),
    ("empty new side",
     b"def test_a():\n  assert 1\n", b"", PY, PY,
     [(b"test_a", "D", None, 1, None, 2, None, 1, None, 2, None, 1)]),
    ("both sides empty", b"", b"", PY, PY, []),
    ("py renamed to cc: the kept header is no header there",
     b"def test_a():\n    x = 1\nvoid test_b() {\n}\n",
     b"def test_a():\n    x = 1\nvoid test_b() {\n}\n",
     PY, CC,
     [(b"test_a", "D", None, 1, None, 4, None, 0, None, 0, None, 0),
      (b"void test_b(", "A", 3, None, 2, None, 0, None, 0, None, 0, None)]),
    ("C++ TEST macros",
     b"TEST(Suite, One) {\n  EXPECT_EQ(1, 1);\n}\nTEST(Suite, Two) {\n}\n",
     b"TEST(Suite, Two) {\n}\nTEST_F(Fix, One) {\n  EXPECT_EQ(1, 2);\n}\n",
     CC, CC,
     [(b"Two", "M", 1, 4, 2, 2, 0, 0, 1, 0, 0, 0),        # the script keeps the old `}` of Two, inserts the one behind it
      (b"One", "M", 3, 1, 3, 3, 1, 1, 2, 3, 1, 1)]),      # a rewritten header matched by its name
]


def test_known_answers():
    for name, old, new, xo, xn, rows in CASES:
        assert cr.py_case_churn(old, new, xo, xn) == rows, name


def test_header_rule_keeps_its_noise():
    """Section 5 unchanged: `default=` is a PY header, so a case starts there as it does for `body`."""
    assert cr.py_is_header(b"    parser.add_argument('--n', default=3)", PY)
    assert cr.py_case_name(b"    parser.add_argument('--n', default=3)", PY) == b"ault"
    assert cr.py_is_header(b"class SkillTest(object):", PY) and not cr.py_is_header(b"classy = 1", PY)
    assert cr.py_is_header(b"  void assign_dst_test(", CC) and not cr.py_is_header(b"def test_a():", CC)
    assert cr.py_case_name(b"BOOST_AUTO_TEST_CASE(Foo)", CC) == b"TEST_CASE(Foo)"
    assert cr.py_case_name(b"TEST_F(Fix, Bar) {", CC) == b"Bar"
    assert cr.py_case_name(b"  public void testFactory() throws Exception {", 4) == b"testFactory()throwsException{"


def references_agree(olds, news, exts_old, exts_new):
    a, b = ts.pack(olds, exts_old), ts.pack(news, exts_new)
    oc, nc = orc_cases.diff_cases((a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext))
    got = orc_cases.case_rows(oc, nc, olds, news, exts_old, exts_new)
    want = {}
    for i, (o, n, xo, xn) in enumerate(zip(olds, news, exts_old, exts_new)):
        r = cr.py_case_churn(o, n, xo, xn)
        if r:
            want[i] = r
    assert got == want
    return oc, nc, want


def test_references_agree_on_the_known_answers():
    references_agree(*[list(x) for x in zip(*[c[1:5] for c in CASES])])


def test_references_agree_on_c5_pairs():
    a, b = ts.gen_pairs(0x7053454D0005, 120, pinned=False)
    olds = [a.file_bytes(i) for i in range(a.n_files)]
    news = [b.file_bytes(i) for i in range(b.n_files)]
    ext = [int(x) for x in a.ext]
    oc, nc, rows = references_agree(olds, news, ext, ext)
    kinds = {r[1] for rs in rows.values() for r in rs}
    assert kinds == {"A", "D", "M"} and len(oc) > 500 and (nc["match"] >= 0).sum() > 400
    assert set(int(x) for x in a.ext) >= {1, 2, 4}
