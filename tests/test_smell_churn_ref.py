"""CPU tests of the test-smell churn references (docs/SPEC.md section 19): the plain-Python restatement
smell_churn_ref.py_smell_churn on hand-written pairs with known rows, and the numpy reference tests/orc_smell_churn.py (serial
marks, serial smells, oracle events) agreeing with it there, on planted histories and on C5 pairs."""
import collections

import case_ref as cr
import orc_smell_churn as osc
import smell_churn_ref as scr
import smell_ref as smr
import tosemscan as ts

PY, CC = 1, 2

# (name, old, new, ext_old, ext_new, rows): rows as py_smell_churn gives them
CASES = [
    ("test added with a sleep",
     b"import time\n",
     b"import time\ndef test_wait():\n    time.sleep(1)\n    assert done()\n", PY, PY,
     [(b"test_wait", "A", 2, None, "sleepy", "introduced", 1, None, 1, None)]),
    ("if inserted into a kept test",
     b"def test_a():\n    x = f()\n    assert x\n",
     b"def test_a():\n    x = f()\n    if x:\n        g()\n    assert x\n", PY, PY,
     [(b"test_a", "M", 1, 1, "conditional_logic", "introduced", 1, 0, 1, 0)]),
    ("the only print deleted",
     b"def test_a():\n    print(x)\n    assert x\n",
     b"def test_a():\n    assert x\n", PY, PY,
     [(b"test_a", "M", 1, 1, "print", "removed", 0, 1, 0, 1)]),
    ("a second print added",
     b"def test_a():\n    print(x)\n    assert x\n",
     b"def test_a():\n    print(x)\n    print(y)\n    assert x\n", PY, PY,
     [(b"test_a", "M", 1, 1, "print", "changed", 2, 1, 1, 0)]),
    ("skip decorator inserted above an unchanged case",
     b"import pytest\n\ndef test_a():\n    assert x\n",
     b"import pytest\n\n@pytest.mark.skip\ndef test_a():\n    assert x\n", PY, PY,
     [(b"test_a", "M", 4, 3, "ignored", "introduced", 1, 0, 1, 0)]),
    ("assertion inserted above an identical kept one",
     b"def test_a():\n    x = 1\n    assert x == 1\n",
     b"def test_a():\n    x = 2\n    assert x == 1\n    assert x == 1\n", PY, PY,
     [(b"test_a", "M", 1, 1, "duplicate_assert", "introduced", 1, 0, 1, 0)]),
    ("PY body end moved by a deleted dedented line",
     b"def test_a():\n    assert x\nfoo()\n    print(y)\n",
     b"def test_a():\n    assert x\n    print(y)\n", PY, PY,
     [(b"test_a", "M", 1, 1, "print", "introduced", 1, 0, 1, 0)]),
    ("test deleted with its smells",
     b"def test_a():\n    assert x\ndef test_b():\n    try:\n        f()\n    except E:\n        pass\n",
     b"def test_a():\n    assert x\n", PY, PY,
     [(b"test_b", "D", None, 3, "assertion_free", "removed", None, 1, None, 1),
      (b"test_b", "D", None, 3, "exception_handling", "removed", None, 2, None, 2)]),
    ("signature change matched by name",
     b"def test_x(self):\n    print(v)\n    assert v\n",
     b"def test_x(self, tmp):\n    print(v)\n    print(w)\n    assert v\n", PY, PY,
     [(b"test_x", "M", 1, 1, "print", "changed", 2, 1, 1, 0)]),
    ("noise header gives no rows",
     b"p.add_argument('-a', default=1)\nprint(1)\n",
     b"p.add_argument('-a', default=2)\nprint(2)\nprint(3)\n", PY, PY, []),
    (".py paired with a .cc",
     b"def test_a():\n    if x:\n        pass\n",
     b"def test_a():\n    if x:\n        pass\n", PY, CC,
     [(b"test_a", "D", None, 1, "assertion_free", "removed", None, 1, None, 1),
      (b"test_a", "D", None, 1, "conditional_logic", "removed", None, 1, None, 1)]),
    ("CRLF lines and unterminated last lines",
     b"def test_a():\r\n    x = 1\r\n    assert x",
     b"def test_a():\r\n    x = 1\r\n    print(x)\r\n    assert x\r\n    assert x", PY, PY,
     [(b"test_a", "M", 1, 1, "duplicate_assert", "introduced", 1, 0, 1, 0),
      (b"test_a", "M", 1, 1, "print", "introduced", 1, 0, 1, 0)]),
    ("gtest renamed to DISABLED_ with a sleep added",
     b"TEST(S, Run) {\n  EXPECT_EQ(a, b);\n}\n",
     b"TEST(S, DISABLED_Run) {\n  EXPECT_EQ(a, b);\n  sleep(1);\n}\n", CC, CC,
     [(b"DISABLED_Run", "A", 1, None, "sleepy", "introduced", 1, None, 1, None),
      (b"DISABLED_Run", "A", 1, None, "ignored", "introduced", 1, None, 1, None)]),
    ("a smell moved between two tests",
     b"def test_a():\n    print(1)\n    assert a\ndef test_b():\n    assert b\n",
     b"def test_a():\n    assert a\ndef test_b():\n    print(1)\n    assert b\n", PY, PY,
     [(b"test_a", "M", 1, 1, "print", "removed", 0, 1, 0, 1),
      (b"test_b", "M", 3, 4, "print", "introduced", 1, 0, 1, 0)]),
]


def test_known_answers():
    for name, old, new, xo, xn, rows in CASES:
        assert scr.py_smell_churn(old, new, xo, xn) == rows, name


def test_added_instance_on_a_kept_line():
    """The duplicate of the 'assertion inserted above' pair is the kept line: the script inserts the first of the two."""
    _, old, new, xo, xn, _ = CASES[5]
    _, inserted, corr = scr.py_script_lines(old, new, xo, xn)
    _, ls = smr.py_file_smells(new, xn)
    dup = [l for l, b in enumerate(ls) if b & smr.BIT["duplicate_assert"]]
    assert dup == [3] and 3 in corr and 2 in inserted


def test_untraced_pair_changes_its_whole_middle(monkeypatch):
    """Above the trace limit every line of the middle is deleted and inserted, so the kept print(1) is churned on both sides
    (the limit is lowered here: a real untraced pair is too slow for the Python diff and is checked on the GPU)."""
    old = b"def test_a():\n    a = 1\n    print(1)\n    b = 1\n    assert a\n"
    new = b"def test_a():\n    a = 2\n    print(1)\n    b = 2\n    assert a\n"
    assert scr.py_smell_churn(old, new, PY, PY) == []
    monkeypatch.setattr(cr, "TRACE_MAX_D", 1)
    assert scr.py_smell_churn(old, new, PY, PY) == [(b"test_a", "M", 1, 1, "print", "changed", 1, 1, 1, 1)]


def references_agree(olds, news, exts_old, exts_new):
    a, b = ts.pack(olds, exts_old), ts.pack(news, exts_new)
    r = osc.diff_smells((a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext))
    got = osc.churn_rows(r, olds, news, exts_old, exts_new)
    want = {}
    for i, (o, n, xo, xn) in enumerate(zip(olds, news, exts_old, exts_new)):
        rows = scr.py_smell_churn(o, n, xo, xn)
        if rows:
            want[i] = rows
    assert got == want
    return r, want


def test_references_agree_on_the_known_answers():
    references_agree(*[list(x) for x in zip(*[c[1:5] for c in CASES])])


def test_references_agree_on_a_planted_history():
    """Planted test files as old sides, gen_edit(lambda = 6) of each as new sides."""
    olds, exts = smr.planted_corpus(19, 80)
    news = [ts.gen_edit(i, o, 6.0) for i, o in enumerate(olds)]
    ext = [int(x) for x in exts]
    r, rows = references_agree(olds, news, ext, ext)
    events = collections.Counter((x[1], x[5]) for rs in rows.values() for x in rs)
    assert events == {("A", "introduced"): 15, ("D", "removed"): 108, ("M", "introduced"): 61, ("M", "removed"): 188,
                      ("M", "changed"): 15}                      # the counts docs/SPEC.md section 19 pins
    assert (len(r["old_tests"]), len(r["new_tests"])) == (511, 451)


def test_references_agree_on_c5_pairs():
    a, b = ts.gen_pairs(0x7053454D0005, 120, pinned=False)
    olds = [a.file_bytes(i) for i in range(a.n_files)]
    news = [b.file_bytes(i) for i in range(b.n_files)]
    ext = [int(x) for x in a.ext]
    r, _ = references_agree(olds, news, ext, ext)
    assert len(r["old_tests"]) > 0
