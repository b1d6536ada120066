"""The plain-Python smell reference (smell_ref.py, docs/SPEC.md section 18) on hand-written files with known answers: every smell
in unittest and pytest files, gtest TEST / TEST_F, Boost and JUnit 3 / 4, and the edges of section 18 - `if __name__` after the
last test, a black-style signature, a column-0 comment inside a body, docstrings holding "if" and two triple quotes, a commented
sleep, sprintf( and fingerprint(, stacked decorators, DISABLED_, duplicates differing in indentation or CR, assertEqual(a, a) and
assertEqual(f(a, b), f(a, b)), a C-family one-liner, brace counts that never open or go negative, CRLF, an unterminated last
line, headerless and empty files; the C1 counts that SPEC section 18 pins; and the planted corpus generator.  The serial C reference
(orc_smells.c, on the oracle's header and assertion rules and line hash) agrees with it, every output array, on the hand-written
files, C1, planted corpora and fuzz corpora with long lines and binary bytes, and on the crafted seam corpora of
tests/front_seams.py, which give their crafted lines the smell bits the builders expect and reach the seams they name."""
import os

import numpy as np

import pytest

import corpus_util as cu
import front_seams as fs
import orc_smells as ocs
import smell_ref as sr
import tosemscan as ts

HERE = os.path.dirname(os.path.abspath(__file__))

# per file: (1-based header line, body lines, assertion lines, [(instance line, smell), ...])
KNOWN = {
    'unittest.py': [
        (8, 4, 0, [(8, 'assertion_free'), (10, 'print')]),
        (12, 6, 4, [(14, 'duplicate_assert'), (15, 'redundant_assert'), (16, 'redundant_assert')]),
        (18, 13, 1, [(19, 'conditional_logic'), (21, 'conditional_logic'), (23, 'exception_handling'), (24, 'sleepy'), (25, 'exception_handling'), (26, 'exception_handling'), (29, 'print')]),
        (31, 4, 1, [(32, 'ignored')]),
        (35, 3, 0, [(35, 'empty'), (35, 'assertion_free')]),
        (38, 9, 1, []),
    ],
    'pytest_style.py': [
        (6, 4, 1, [(6, 'ignored')]),
        (10, 4, 1, []),
        (14, 10, 2, [(21, 'duplicate_assert')]),
        (28, 6, 3, [(29, 'redundant_assert'), (31, 'redundant_assert')]),
    ],
    'crlf.py': [
        (1, 6, 3, [(3, 'duplicate_assert'), (5, 'conditional_logic')]),
        (7, 2, 0, [(7, 'empty'), (7, 'assertion_free')]),
    ],
    'gtest.cc': [
        (3, 7, 2, [(5, 'duplicate_assert'), (6, 'conditional_logic'), (7, 'print')]),
        (11, 5, 1, [(11, 'ignored'), (12, 'redundant_assert'), (13, 'sleepy'), (14, 'print')]),
        (17, 1, 0, [(17, 'empty'), (17, 'assertion_free')]),
        (20, 2, 0, [(20, 'empty'), (20, 'assertion_free')]),
        (23, 3, 1, [(24, 'redundant_assert')]),
        (26, 1, 0, [(26, 'empty'), (26, 'assertion_free')]),
    ],
    'boost.cpp': [
        (1, 6, 0, [(1, 'assertion_free'), (5, 'conditional_logic'), (5, 'sleepy')]),
        (7, 4, 0, [(7, 'assertion_free'), (8, 'print')]),
    ],
    'Junit4Test.java': [
        (3, 3, 1, [(3, 'ignored'), (4, 'redundant_assert')]),
        (6, 5, 1, [(7, 'print'), (8, 'conditional_logic')]),
        (11, 1, 0, [(11, 'empty'), (11, 'assertion_free'), (11, 'ignored')]),
    ],
    'Junit3Test.java': [
        (2, 7, 2, [(3, 'sleepy'), (7, 'duplicate_assert')]),
    ],
    'headerless.py': [
    ],
    'empty.py': [
    ],
    'other.txt': [
    ],
}


def test_known_answers():
    for name, ext, data in sr.HAND:
        tests, line_smell = sr.py_file_smells(data, ext)
        got = [(b + 1, n, a, [(l + 1, sr.SMELLS[bit.bit_length() - 1]) for l, bit in inst]) for b, n, a, _, _, inst in tests]
        assert got == KNOWN[name], name
        for b, n, a, smells, k, inst in tests:
            assert k == len(inst) == sum(bin(line_smell[l]).count("1") for l in range(b, b + n))
            assert smells == np.bitwise_or.reduce([bit for _, bit in inst] or [0])


def test_edges():
    t = {name: sr.py_file_smells(d, e)[0] for name, e, d in sr.HAND}
    assert t["pytest_style.py"][-1][1] == 6                 # `if __name__` ends the last test: not conditional logic
    assert sr.is_redundant(b"self.assertEqual(a, a)") and sr.is_redundant(b"self.assertEqual(f(a, b), f(a, b))")
    assert not sr.is_redundant(b"self.assertEqual(f(a, b), f(a, c))") and sr.is_redundant(b"assert  True")
    assert not sr.has_print(b"sprintf(x) + fingerprint(y)") and sr.has_print(b"pprint(y)") and sr.has_print(b"std::cout << x;")
    assert sr.is_test_header(b"async  def test_x():", 1) and not sr.is_test_header(b"asyncdef test_x():", 1)
    assert not sr.is_test_header(b"    parser.add_argument(default=1)", 1)


def test_c1_counts():
    files, exts, _, _ = cu.load_fixture(os.path.join(HERE, "golden", "c1_testfiles.npz"))
    tests, line_smell = sr.py_smells(files, exts)
    assert len(line_smell) == 294387 and len(tests) == 6239
    counts = [sum(1 for t in tests if t[4] >> k & 1) for k in range(len(sr.SMELLS))]
    assert counts == [363, 1812, 866, 8, 1190, 98, 70, 114, 98]
    assert max(t[3] for t in tests) == 107 and sum(t[5] for t in tests) == 8492


def test_planted_corpus():
    files, exts = sr.planted_corpus(7, 200)
    tests, _ = sr.py_smells(files, exts)
    assert len(tests) > 400 and all(any(t[4] >> k & 1 for t in tests) for k in range(len(sr.SMELLS)))
    assert sr.planted_corpus(7, 200)[0] == files


def both_agree(files, exts):
    exts = np.asarray(exts, np.uint8)
    got = ocs.smells(ts.pack(files, exts))
    ocs.assert_equal(got, ocs.as_python(files, exts))
    return got


def test_c_reference_hand_and_c1():
    got = both_agree([d for _, _, d in sr.HAND], [e for _, e, _ in sr.HAND])
    assert len(got["tests"]) == 24
    files, exts, _, _ = cu.load_fixture(os.path.join(HERE, "golden", "c1_testfiles.npz"))
    got = both_agree(files, exts)
    assert len(got["tests"]) == 6239 and len(got["line_smell"]) == 294387


def test_c_reference_planted():
    files, exts = sr.planted_corpus(0x5E13, 1500)
    got = both_agree(files, exts)
    assert all((got["tests"]["smells"] >> k & 1).any() for k in range(len(sr.SMELLS)))


@pytest.mark.parametrize("long_lines,binary", [(False, False), (True, False), (False, True)])
def test_c_reference_fuzz(long_lines, binary):
    files, exts, _ = cu.fuzz_corpus(0x5E14 + 7 * long_lines + 3 * binary, 300, 20000, long_lines=long_lines, binary=binary)
    rng = np.random.default_rng(6)
    heads = [b"def test_a():", b"    def test_b(self):", b"TEST(A, B) {", b"  public void testX() {", b"@pytest.mark.skip", b"@Ignore"]
    for i in range(0, len(files), 3):                       # plant headers of every family between the fuzz lines
        lines = files[i].split(b"\n")
        for _ in range(max(1, len(lines) // 20)):
            lines.insert(int(rng.integers(0, len(lines) + 1)), heads[int(rng.integers(0, len(heads)))])
        files[i] = b"\n".join(lines)
    got = both_agree(files, exts)
    assert len(got["tests"]) > 50


# The crafted corpora of tests/front_seams.py, on which tests/test_gpu_smells_seams.py runs the kernels: the two references agree
# on each, give the crafted lines the smell bits their builders expect, and each corpus reaches the seams it names.
def bits_as_built(got, want):
    """The crafted lines whose smell bits (under their mask) differ from what the builder expects."""
    base, smell = got["line_base"], got["line_smell"]
    return [(f, ln, w, int(smell[base[f] + ln])) for f, ln, m, w in want if int(smell[base[f] + ln]) & m != w]


@pytest.mark.parametrize("build", [fs.pattern_corpus, fs.token_corpus, fs.redundant_corpus])
def test_grid_corpora(build):
    files, exts, reach, want = build()
    assert reach and all(fs.on_the_grid(reach).values())
    got = both_agree(files, exts)
    assert bits_as_built(got, want) == []
    assert got["tests"]["body_lines"].tolist() == [len(sr.py_lines(f)) for f in files]      # every line is in the test


def test_pattern_prefix_checks_meet_equality():
    files, exts, reach, want = fs.pattern_corpus()
    # gtest body from column 0: `sleep_for(` / `_until(` / `System.` start at the line's first byte
    assert (0, 0) in reach[(3, "sleep_for")] and (0, 0) in reach[(3, "sleep_until")] and (0, 0) in reach[(3, "system_out")]
    lines = sr.py_lines(files[0])
    assert lines[[ln for f, ln, _, w in want if f == 0][0]].startswith(b"print(")


def test_facts_corpus():
    files, exts = fs.facts_corpus()
    got = both_agree(files, exts)
    t = got["tests"]
    n = len(fs.EMPTY_BODIES)
    want = [int(e) for _, e in fs.EMPTY_BODIES]
    assert (t["smells"][:n] & 1).tolist() == want and (t["smells"][n:2 * n] & 1).tolist() == want
    quotes = got["line_smell"][got["line_base"][2]:got["line_base"][3]]
    assert 0 < int((quotes & fs.COND).astype(bool).sum()) < 2 * len(fs.QUOTE_LINES)   # some `if` lines are in a docstring


def test_scan_smell_corpus_lanes():
    files, exts = fs.scan_smell_corpus()
    both_agree(files, exts)
    py, java, cc = (fs.scan_facts(d, e) for d, e in zip(files, exts))
    assert [fs.lane_round(hs, b + 1) for b, hs, _, _ in py[:4]] == [(31, 0), (0, 1), (1, 1), (8, 1)]
    assert [fs.lane_round(bend, hs) for _, hs, bend, _ in py[4:12]] == [(31, 0)] * 2 + [(0, 1)] * 2 + [(31, 1)] * 2 + [(0, 2)] * 2
    b, _, bend, _ = py[12]
    lines = sr.py_lines(files[0])
    doc = [ln for ln in range(b, bend) if lines[ln].strip() == b'"""']
    assert [fs.lane_round(ln, b) for ln in doc] == [(31, 0), (31, 2)]
    assert [fs.lane_round(br, b) for b, _, _, br in java[::2]] == [(31, 0), (0, 1)]              # Allman `{`
    jl = sr.py_lines(files[1])
    assert [fs.lane_round(next(ln for ln in range(b, bend) if b"}" in jl[ln]), b) for b, _, bend, _ in java[1::2]] == \
        [(31, 0), (0, 1)]                                                                            # `}` ahead of the `{`
    assert [bend - b for b, _, bend, _ in cc] == [1, 1]


def test_header_corpus():
    files, exts = fs.header_corpus()
    got = both_agree(files, exts)
    t = got["tests"]
    ignored = [(int(f), int(ln)) for f, ln, s in zip(t["file"], t["line"], t["smells"]) if s >> 8 & 1]
    assert ignored == [(1, 2), (4, 2), (4, 4), (4, 8), (4, 19), (5, 97)]
    names = [sr.py_lines(files[int(f)])[int(ln)] for f, ln in zip(t["file"], t["line"])]
    assert b"asyncdef test_c():" not in names and {b"async  def\ttest_b():", b"def  test_d():", b"async\tdef test_e():"} <= set(names)
    assert sum(1 for n in names if n.startswith((b"TEST", b"TYPED", b"BOOST"))) == 8 + 3 + 2
    assert [int(f) for f in t["file"][-4:]] == [6, 7, 8, 9]             # a header on the last line, with and without the LF
