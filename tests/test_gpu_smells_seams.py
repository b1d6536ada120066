"""`tsm_smells` / `Scanner.smells` (docs/SPEC.md section 18) where tests/test_gpu_smells.py never reaches: the print and sleep
patterns of k_smell_lines' Shift-And automaton at every line start and statement start modulo 8, with the prefix checks that
count from the line start brought to equality and a rejected match ahead of an accepted one; first tokens of 8 bytes and
longer ones that begin with a keyword, behind '}' and W bytes; `pass` and bracket-only bodies; quote runs of 2 to 7; the
redundant forms; k_smell_tests' header-statement, body-end, brace and docstring scans on both sides of a 32-line round;
decorator walks to the file's first line and cut short, the ignore markers of every family, the async forms, the gtest and
Boost macros and their one-byte changes, and headers on a file's last line.  Every output array is compared with the C
reference (tests/orc_smells.c) and the plain-Python one (tests/smell_ref.py), and the crafted lines' smell bits with what the
builders expect.  The builders are in tests/front_seams.py, checked on the CPU by tests/test_smells_ref.py; each test asserts
that its corpus reaches its seams."""
import numpy as np
import pytest

import front_seams as fs
import orc_smells as ocs
import smell_ref as sr
import tosemscan as ts
from test_smells_ref import bits_as_built

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 12, max_groups=4)
    yield s
    s.close()


def check(s, files, exts):
    exts = np.asarray(exts, np.uint8)
    c = ts.pack(files, exts)
    got = s.smells(c)
    ocs.assert_equal(got, ocs.smells(c))
    ocs.assert_equal(got, ocs.as_python(files, exts))
    return got


@pytest.mark.parametrize("build", [fs.pattern_corpus, fs.token_corpus, fs.redundant_corpus], ids=["patterns", "tokens", "redundant"])
def test_lines_on_the_load_grid(scanner, build):
    files, exts, reach, want = build()
    assert reach and all(fs.on_the_grid(reach).values())
    got = check(scanner, files, exts)
    assert bits_as_built(got, want) == []
    assert got["tests"]["body_lines"].tolist() == [len(sr.py_lines(f)) for f in files]


def test_empty_bodies_and_quote_runs(scanner):
    files, exts = fs.facts_corpus()
    got = check(scanner, files, exts)
    n, want = len(fs.EMPTY_BODIES), [int(e) for _, e in fs.EMPTY_BODIES]
    assert (got["tests"]["smells"][:2 * n] & 1).tolist() == want * 2
    quotes = got["line_smell"][got["line_base"][2]:got["line_base"][3]]
    assert 0 < int((quotes & fs.COND).astype(bool).sum()) < 2 * len(fs.QUOTE_LINES)


def test_scans_across_rounds(scanner):
    files, exts = fs.scan_smell_corpus()
    py, java, cc = (fs.scan_facts(d, e) for d, e in zip(files, exts))
    assert [fs.lane_round(hs, b + 1) for b, hs, _, _ in py[:4]] == [(31, 0), (0, 1), (1, 1), (8, 1)]
    assert [fs.lane_round(bend, hs) for _, hs, bend, _ in py[4:12]] == [(31, 0)] * 2 + [(0, 1)] * 2 + [(31, 1)] * 2 + [(0, 2)] * 2
    assert [fs.lane_round(br, b) for b, _, _, br in java[::2]] == [(31, 0), (0, 1)]
    got = check(scanner, files, exts)
    t = got["tests"]
    assert [(int(f), int(ln), int(n)) for f, ln, n in zip(t["file"], t["line"], t["body_lines"])] == \
        [(f, b, bend - b) for f, facts in enumerate((py, java, cc)) for b, _, bend, _ in facts]


def test_decorators_and_headers(scanner):
    files, exts = fs.header_corpus()
    got = check(scanner, files, exts)
    t = got["tests"]
    assert [(int(f), int(ln)) for f, ln, s in zip(t["file"], t["line"], t["smells"]) if s >> 8 & 1] == \
        [(1, 2), (4, 2), (4, 4), (4, 8), (4, 19), (5, 97)]
    assert [int(f) for f in t["file"][-4:]] == [6, 7, 8, 9]
