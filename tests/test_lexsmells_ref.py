"""The references of the lexical test smells (docs/SPEC.md section 25): the plain-Python tests/lexsmell_ref.py on hand-written
files with known answers for every rule, and against the section-18 and section-21 references it builds on (its seen tokens blind
to exactly `blind_ref.lex_line`, its bodies are those of `smell_ref`), and the C1 counts of section 25; the serial C
tests/orc_lexsmells.c equal to it, every array, on the hand-written files, C1, the hazard files, planted and fuzz corpora."""
import os

import numpy as np
import pytest

import blind_ref as br
import corpus_util as cu
import front_seams as fs
import lex_seams as lx
import lexsmell_ref as lr
import orc_lexsmells as ol
import smell_ref as sr
import spec_ref
import tosemscan as ts
from spec_ref import py_lines

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
AR, MAGIC, SUB, GUEST, OBSCURE = (lr.LBIT[s] for s in lr.LSMELLS)
C1_COUNTS = {"tests": 6239, "assertion_roulette": 2854, "magic_number": 1979, "suboptimal_assert": 528, "mystery_guest": 111,
             "obscure_setup": 316}


def one_test(data, ext):
    """(record, {line: bits}) of a file with exactly one test."""
    tests, lsm = lr.file_lexsmells(data, ext)
    assert len(tests) == 1
    return tests[0], {l: b for l, b in enumerate(lsm) if b}


UNITTEST, PYTEST, NUMPY, GTEST, JUNIT = (d for _, _, d in lr.HAND[:5])


def test_unittest():
    r, bits = one_test(UNITTEST, 1)
    assert r[2:6] == (7, 3, 2, 1)                          # statements, unexplained, magic, locals
    assert bits == {5: AR, 7: AR, 9: AR | MAGIC, 10: MAGIC}


def test_pytest_asserts():
    r, bits = one_test(PYTEST, 1)
    # 1, 3, 4, 7, 8, 9 have no message; the multi-line assert on 4-6 ends at its closing line, its -3 is not at depth 0
    assert r[2:6] == (8, 6, 4, 0)
    assert bits == {1: AR | MAGIC, 2: MAGIC, 3: AR, 4: AR, 7: AR | MAGIC, 8: AR, 9: AR | MAGIC}


def test_numpy_mock_suboptimal():
    r, bits = one_test(NUMPY, 1)
    assert r[2:6] == (11, 7, 2, 0)
    assert bits == {1: AR, 3: AR | MAGIC, 4: MAGIC, 6: AR | SUB, 7: AR | SUB, 8: AR | SUB, 9: AR | SUB, 10: AR}


def test_gtest_c_static():
    r, bits = one_test(GTEST, 3)
    assert r[2:6] == (10, 7, 3, 2)
    assert bits == {1: MAGIC, 2: AR, 3: AR | SUB, 4: AR, 5: SUB, 7: AR, 8: AR, 9: MAGIC, 10: AR | MAGIC, 11: GUEST, 12: GUEST,
                    15: AR}


def test_junit():
    r, bits = one_test(JUNIT, 4)
    assert r[2:6] == (9, 5, 3, 1)
    assert bits == {2: AR | MAGIC, 5: AR, 6: AR | SUB, 8: MAGIC, 9: AR | MAGIC, 10: GUEST, 11: GUEST, 12: AR}


@pytest.mark.parametrize("k,explained", [(1, True), (2, True), (63, True), (64, True), (65, False)])
def test_statement_line_cap(k, explained):
    """A call over k lines whose message is on its last line: seen up to LEX_STMT_LINES = 64 lines."""
    call = [b"        self.assertEqual(a, b, 'm')"] if k == 1 else \
        [b"        self.assertEqual("] + [b"            # c"] * (k - 2) + [b"            a, b, 'm')"]
    data = b"def test_cap(self):\n" + b"\n".join(call) + b"\n        self.assertTrue(y)\n"
    r, _ = one_test(data, 1)
    assert r[2] == 2 and r[3] == (1 if explained else 2)


def test_unterminated_at_body_end():
    data = b"def test_open(self):\n    self.assertEqual(a,\n        b, 'm'\ndef later():\n    pass)\n"
    r, bits = one_test(data, 1)
    assert r[1] == 3 and r[2:4] == (1, 0)                  # a, b, 'm': three positional arguments before the body ends
    data = b"def test_open(self):\n    self.assertEqual(a,\ndef later():\n    b, 'm')\n    self.assertTrue(x)\n"
    r, bits = one_test(data, 1)
    assert r[1] == 2 and r[2:4] == (1, 1)


@pytest.mark.parametrize("n,obscure", [(10, False), (11, True)])
def test_locals_threshold(n, obscure):
    body = b"".join(b"    v%d = %d\n" % (i, i) for i in range(n)) + b"    v0 = 2\n    a, b = 1, 2\n    self.x = 1\n    f(k=1)\n"
    data = b"def test_locals():\n" + body.replace(b"    a, b = 1, 2\n", b"") + b"    assert v0\n"
    r, bits = one_test(data, 1)
    assert r[5] == n and ((r[6] & OBSCURE) != 0) == obscure and bits.get(0, 0) == (OBSCURE if obscure else 0)
    data = b"def test_locals():\n" + b"".join(b"    v%d = 0\n" % i for i in range(n - 2)) + b"    a, b = 1, 2\n"
    assert one_test(data, 1)[0][5] == n


def test_cj_locals():
    data = b"TEST(S, Locals) {\n  int x = 5;\n  auto y = f();\n  std::vector<int> v = {1};\n  x = 5;\n  a.b = 1;\n" \
           b"  if (x) z = 1;\n  int c == d;\n  x += 1;\n  const char* s = \"a\";\n}\n"
    r, _ = one_test(data, 3)
    assert r[5] == 4                                       # x, y, v, s


def test_docstring_and_comment_not_counted():
    data = b'def test_doc():\n    """assert x == 5"""\n    # assert 7\n    assert y\n'
    r, bits = one_test(data, 1)
    assert r[2:5] == (1, 1, 0) and bits == {}


def test_mystery_guest_py():
    data = b"def test_io(tmp):\n    with open('f') as fh:\n        pass\n    os.listdir(d)\n    x = reopen(1)\n    pd.read_csv\n"
    _, bits = one_test(data, 1)
    assert bits == {1: GUEST, 3: GUEST}


def test_call_only_when_followed_by_paren():
    assert lr.find_call(lr.lex_tokens(b"x = self.assertEqual", 1, 0)[0], 1) is None
    assert lr.find_call(lr.lex_tokens(b"check_assert (x)", 1, 0)[0], 1) == (0, "call")
    assert lr.find_call(lr.lex_tokens(b"assert(x)", 3, 0)[0], 3) == (0, "call")
    assert lr.find_call(lr.lex_tokens(b"assert x", 2, 0)[0], 3) is None


def test_seen_tokens_blind_to_lex_line():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_hazard_files.npz"))
    files2, exts2, _ = cu.fuzz_corpus(0x1E55, 200, 6000, binary=True)
    for data, e in list(zip(files, exts)) + list(zip(files2, exts2)):
        fam = br.family(int(e))
        if fam == br.NONE:
            continue
        st = br.CODE
        for line in py_lines(data):
            a, s1 = br.lex_line(line, fam, st)
            b, s2 = lr.lex_tokens(line, fam, st)
            assert a == [lr.blind(t) for t in b] and s1 == s2
            st = s1


def test_bodies_match_smell_ref():
    files, exts = sr.planted_corpus(0x1E57, 300)
    for data, e in zip(files, exts):
        got = [(b, bend - b) for b, bend, _, _ in lr.bodies(py_lines(data), int(e))]
        want = [(t[0], t[1]) for t in sr.py_file_smells(data, int(e))[0]]
        assert got == want


def test_c1_counts():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    r = lr.py_lexsmells(files, exts)
    lex = r["lex"]
    counts = {"tests": len(lex)}
    counts.update({n: int(((lex["smells"] >> k) & 1).sum()) for k, n in enumerate(lr.LSMELLS)})
    assert counts == C1_COUNTS
    assert int(lex["n_stmts"].sum()) == 20197 and int(lex["n_unexplained"].sum()) == 19517 and int(lex["n_magic"].sum()) == 8603
    assert int(lex["n_locals"].max()) == 41 and int(lex["n_instances"].sum()) == 28477
    assert int(np.unpackbits(r["line_lsmell"]).sum()) == 28477


def corpora():
    c1, e1, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    hz, eh, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_hazard_files.npz"))
    yield "hand", [d for _, _, d in lr.HAND], np.array([e for _, e, _ in lr.HAND], np.uint8)
    yield "c1", c1, e1
    yield "hazard", hz, eh
    yield ("planted",) + lr.planted_corpus(0x1E58, 500)
    for lo, bi in ((False, False), (True, False), (False, True)):
        yield ("fuzz",) + lr.fuzz_with_calls(0x1E25 + 7 * lo + 3 * bi, lo, bi)


@pytest.mark.parametrize("name", ["hand", "c1", "hazard", "planted", "fuzz"])
def test_c_reference_equals_python(name):
    for n, files, exts in corpora():
        if n == name:
            ol.assert_equal(ol.lexsmells(ts.pack(files, exts)), lr.py_lexsmells(files, exts))


# ------------------------------------------------------------------------------------------------------ the seams corpora
def test_kernel_names_equal_reference_tables():
    """Every name the kernels compare an identifier with is one of the reference's, and the other way round."""
    assert lx.kernel_names() == lx.reference_names()
    assert b"assert_not_called" in lx.kernel_names() and b"assert_not_callee" in lx.long_name_misses()


def test_sentinel_name_hashes_to_the_empty_slot():
    assert spec_ref.py_bytes_hash(lx.SENTINEL) == (1 << 64) - 1
    assert lr.lex_tokens(b"    " + lx.SENTINEL + b" = 1", br.PY, br.CODE)[0][0] == (lr.IDENT, lx.SENTINEL)


SEAMS = {"names": lx.name_corpus, "cap": lx.cap_corpus, "automata": lambda: lx.automaton_corpus((1, 2, 3)),
         "name_sets": lx.nameset_corpus, "body": lx.body_corpus}


def test_seams_corpora_reach_their_seams():
    c = {k: b() for k, b in SEAMS.items()}
    _, _, reach = c["names"]
    assert all(fs.on_the_grid(reach["grid"]).values()) and len(reach["grid"]) > 800
    assert {w for _, _, _, w in reach["marks"]} >= lx.kernel_names() | lx.long_name_misses()
    _, _, reach = c["cap"]
    assert {(d, end, seen) for _, _, d, end, seen, _ in reach["cases"]} == \
        {(62, None, True), (63, None, True), (64, None, False), (65, None, False), (62, 63, True), (63, 64, True),
         (64, 65, False), (63, 63, False), (64, 64, False), (65, 65, False)}
    _, _, reach = c["automata"]
    assert reach[("stmt", 1, b"assert ")] == 19 + 19 ** 2 + 19 ** 3 and reach[("code", 3)] == 15 + 15 ** 2 + 15 ** 3
    _, _, reach = c["name_sets"]
    assert reach["wraps"][4] > 0 and reach["wraps"][5] > 0 and reach["alternating_warps"] > 0
    assert len(reach["names"]) > 2 * reach["warps"] and reach["sentinel_tests"] == [0, 1, 2, 3, 13]
    assert [len(set(h)) for h in reach["names"][:14]] == [1, 1, 5, 300, 5, 300, 2, 1, 300, 10, 11, 0, 0, 2]
    assert len(reach["names"][6]) == 33 and len(reach["names"][3]) > 256
    assert {len(set(h)) for h in reach["names"][14:]} >= set(range(21)) | {257, 300}
    _, _, reach = c["body"]
    assert [x[1] for x in reach["head_end"]] == [(30, 0), (31, 0), (0, 1), (1, 1), (2, 1)]
    assert sorted({(o, c) for o, c in reach["doc"]}) == [((31, 0), (16, r)) for r in (1, 2, 3)]
    assert reach["end_lanes"] == {1: set(range(32)), 3: set(range(32))}


@pytest.mark.parametrize("name", ["names", "cap", "automata", "name_sets", "body"])
def test_seams_references_agree(name):
    files, exts, reach = SEAMS[name]()
    want = lr.py_lexsmells(files, exts)
    ol.assert_equal(ol.lexsmells(ts.pack(files, np.asarray(exts, np.uint8))), want)
    if name == "cap":
        for (form, _, d, end, seen, _), r in zip(reach["cases"], want["lex"]):
            if reach["forms"][form] == "msg":
                assert r["n_unexplained"] == (0 if seen else 1), (form, d, end)
            else:
                assert r["n_magic"] == int(seen), (form, d, end)
    if name == "names":
        lsm = want["line_lsmell"]
        hits = [want["line_base"][f] + ln for f, ln, _, w in reach["marks"] if w == b"assert_not_callee" and exts[f] == 1]
        assert len(hits) == 128 and (lsm[hits] & AR).all()
    if name == "name_sets":
        assert want["lex"]["n_locals"].tolist() == [len(set(h)) for h in reach["names"]]
