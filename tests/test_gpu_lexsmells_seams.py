"""`tsm_smells_lexical` / `Scanner.smells_lexical` (docs/SPEC.md section 25) where tests/test_gpu_lexsmells.py never reaches:
every name the kernels compare, and its one-byte variants, at every line start and name start modulo 8 (names longer than 16
bytes that differ from one only past byte 16 among them); the token that decides a statement 62 to 65 lines below it and the body
end 63 to 65 lines below it; every short token sequence in every statement form and code line; the name whose hash is the
empty-slot key, probes that wrap, 32 copies of a name in one round, 300 names on one line and more tests than the launch has
warps; header statements, docstrings and test starts on both sides of 32-line rounds.  Every output array is compared with the C
reference (tests/orc_lexsmells.c) and the plain-Python one (tests/lexsmell_ref.py), the section-18 arrays with `smells()`, and
the crafted tests with what the builders expect.  Then the lexical churn of tsm_diff_pairs_smells_lexical (section 26) against
tests/orc_lexsmell_churn.py, one call per side configuration of lex_stage: an edit below a kept open call at the walk cap, one
side without tests (with lines or without), sides whose name total is 0, and the sentinel name added and removed.  The builders are in tests/lex_seams.py, checked on the CPU by
tests/test_lexsmells_ref.py."""
import numpy as np
import pytest
import torch

import lex_seams as lx
import lexsmell_ref as lr
import orc_lexsmells as ol
import spec_ref
import tosemscan as ts
from test_gpu_lexsmell_churn import check as check_churn
from test_gpu_lexsmells import check

pytestmark = pytest.mark.gpu
AR = lr.LBIT["assertion_roulette"]


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 12, max_groups=4)
    yield s
    s.close()


def u8(exts):
    return np.asarray(exts, np.uint8)


def test_names_on_the_load_grid(scanner):
    files, exts, reach = lx.name_corpus()
    assert all(lx.fs.on_the_grid(reach["grid"]).values())
    got = check(scanner, files, u8(exts))
    misses = lx.long_name_misses()
    assert b"assert_not_callee" in misses
    # a PY call of a name that shares its first 16 bytes with assert_not_called is a numpy-style assertion: unexplained, and in
    # a test of many unexplained ones part of Assertion Roulette
    lines = [got["line_base"][f] + ln for f, ln, head, w in reach["marks"]
             if w in misses and exts[f] == 1 and (head == b"self." or w.startswith(b"assert_"))]
    assert len(lines) == 64 * (len(misses) + 1) and (got["line_lsmell"][lines] & AR).all()


def test_walk_cap_and_body_end(scanner):
    files, exts, reach = lx.cap_corpus()
    got = check(scanner, files, u8(exts))
    lex = got["lex"]
    assert len(lex) == len(reach["cases"])
    for (form, _, d, end, seen, _), r in zip(reach["cases"], lex):
        if reach["forms"][form] == "msg":
            assert (r["n_stmts"], r["n_unexplained"]) == (1, 0 if seen else 1), (form, d, end)
        else:
            assert (r["n_stmts"], r["n_magic"]) == (1, 1 if seen else 0), (form, d, end)


@pytest.mark.parametrize("lengths,both", [((1, 2, 3), True), ((4,), False)], ids=["up_to_3", "length_4"])
def test_token_automata(scanner, lengths, both):
    # up to 3 tokens: every sequence.  4 tokens: a seeded sample of 4096 sequences per form (about 3% of the 19^4 statement
    # sequences), so that the corpus stays at a few MB; it is not exhaustive
    files, exts, reach = lx.automaton_corpus(lengths, sample=None if both else 4096)
    if both:
        got = check(scanner, files, u8(exts))
    else:                                                 # the C reference only: the Python one would take minutes
        c = ts.pack(files, u8(exts))
        got = scanner.smells_lexical(c)
        ol.assert_equal(got, ol.lexsmells(c))
    assert len(got["lex"]) == sum(reach.values())


def test_name_sets(scanner):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    files, exts, reach = lx.nameset_corpus(sms=sms)
    assert reach["alternating_warps"] > 0 and reach["wraps"][4] > 0 and reach["wraps"][5] > 0
    got = check(scanner, files, u8(exts))
    lex = got["lex"]
    assert len(lex) > 2 * reach["warps"]
    assert lex["n_locals"].tolist() == [len(set(h)) for h in reach["names"]]
    assert [int(lex["n_locals"][t]) for t in reach["sentinel_tests"]] == [1, 1, 5, 300, 2]


def test_body_scans_across_rounds(scanner):
    files, exts, reach = lx.body_corpus()
    assert reach["end_lanes"] == {1: set(range(32)), 3: set(range(32))}
    got = check(scanner, files, u8(exts))
    assert (got["lex"]["n_locals"][:5] == 1).all()        # the header's keyword arguments are no local names


# ----------------------------------------------------------------------------------------------------------------- churn
def open_call(d, msg):
    """An assertEqual whose list closes d lines below it (comment lines between), then one more unexplained assertion."""
    return (b"def test_a(self):\n    self.assertEqual(a,\n" + b"        # c\n" * (d - 1) + b"        b%s)\n" % msg +
            b"    self.assertTrue(z)\n")


def churn(scanner, olds, news, exts):
    """check_churn on one call whose old side holds olds and new side news (one ext per pair)."""
    return check_churn(scanner, ts.pack(olds, list(exts)), ts.pack(news, list(exts)))


TEST_WITH_NAMES = b"def test_a():\n    v = 1\n    w = 2\n    assert v == 1\n    assert w\n"
TEST_NO_NAMES = b"def test_a():\n    assert x == 1\n    assert y\n"
GTEST = b"TEST(S, A) {\n  int v = 1;\n  EXPECT_EQ(v, 1);\n}\n"


def test_churn_walk_cap(scanner):
    """An edit 62 to 65 lines below a kept open call: the kept assertEqual line loses Assertion Roulette when the message comes
    inside its walk (offset 63), not at offset 64."""
    r = churn(scanner, [open_call(d, b"") for d in (62, 63, 64, 65)], [open_call(d, b", 'm'") for d in (62, 63, 64, 65)], [1] * 4)
    k = ts.LSMELLS.index("assertion_roulette")
    assert r["old_lex_churn"]["churned"][:, k].tolist() == [2, 2, 0, 0]


@pytest.mark.parametrize("reverse", [False, True], ids=["old", "new"])
def test_churn_one_side_without_tests(scanner, reverse):
    """lex_stage runs the lexical kernels on the side with tests and skips the other, which has lines (a PY and a C++ pair)
    or none at all (an empty file)."""
    for with_tests, without, ext in ((TEST_WITH_NAMES, b"x = 1\n", 1), (GTEST, b"int x;\n", 3), (TEST_WITH_NAMES, b"", 1),
                                     (GTEST, b"", 3)):
        old, new = (without, with_tests) if reverse else (with_tests, without)
        r = churn(scanner, [old], [new], [ext])
        side, other = ("new", "old") if reverse else ("old", "new")
        assert len(r[other + "_lex"]) == 0 and r[side + "_lex"]["n_locals"].tolist() == [2 if ext == 1 else 1]


def test_churn_sides_without_names(scanner):
    """Sides whose tests assign no local name (a name total of 0: the name buffers are allocated empty) against sides with
    names, both ways, and on both sides."""
    r = churn(scanner, [TEST_NO_NAMES], [TEST_WITH_NAMES], [1])
    assert r["old_lex"]["n_locals"].tolist() == [0] and r["new_lex"]["n_locals"].tolist() == [2]
    r = churn(scanner, [TEST_WITH_NAMES], [TEST_NO_NAMES], [1])
    assert r["old_lex"]["n_locals"].tolist() == [2] and r["new_lex"]["n_locals"].tolist() == [0]
    r = churn(scanner, [TEST_NO_NAMES, b"TEST(S, A) {\n  EXPECT_EQ(a, 1);\n}\n"],
              [b"def test_a():\n    assert x == 2\n", b"TEST(S, A) {\n  EXPECT_EQ(a, 2);\n  EXPECT_TRUE(b);\n}\n"], [1, 3])
    assert r["old_lex"]["n_locals"].tolist() == [0, 0] and r["new_lex"]["n_locals"].tolist() == [0, 0]


def test_churn_sentinel_and_empty_sides(scanner):
    """The name whose hash is the empty-slot key added and removed; then sides of empty files only."""
    S = lx.SENTINEL
    assert spec_ref.py_bytes_hash(S) == lx.M64
    r = churn(scanner, [b"def test_s():\n    a = 1\n", b"def test_s():\n    " + S + b", b = f()\n    c = 1\n"],
              [b"def test_s():\n    a = 1\n    " + S + b" = 2\n", b"def test_s():\n    c = 1\n"], [1, 1])
    assert r["old_lex"]["n_locals"].tolist() == [1, 3] and r["new_lex"]["n_locals"].tolist() == [2, 1]
    r = churn(scanner, [b"", b""], [b"", b""], [1, 3])
    assert all(r[k].size == 0 for k in ("old_lex", "new_lex", "old_lex_churn", "new_lex_churn"))
