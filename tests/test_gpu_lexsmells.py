"""`tsm_smells_lexical` / `Scanner.smells_lexical` (docs/SPEC.md section 25) against the serial C reference orc_lexsmells and the
plain-Python reference lexsmell_ref.py_lexsmells, every output array, and its section-18 outputs against `tsm_smells`: the
hand-written files, the C1 test files with their counts, the hazard files, planted smells at scale, fuzz corpora with long lines
and binary bytes, tests of many assertion lines, the line cap's worst case, tests of 256, 257 and 20 000 local names (the shared and
the global name sets), more tests than the launch has warps, no tests and an empty corpus; the raw ABI's caps and NULL outputs,
repeated calls and a non-blocking stream while the legacy stream is busy."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import corpus_util as cu
import lexsmell_ref as lr
import orc_lexsmells as ol
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
C1_COUNTS = {"tests": 6239, "assertion_roulette": 2854, "magic_number": 1979, "suboptimal_assert": 528, "mystery_guest": 111,
             "obscure_setup": 316}


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


def check(s, files, exts, **kw):
    """Every output array equals both references; line_base, line_smell and tests equal those of smells()."""
    c = ts.pack(files, exts)
    got = s.smells_lexical(c, **kw)
    ol.assert_equal(got, ol.lexsmells(c))
    want = lr.py_lexsmells(files, exts)
    assert np.array_equal(got["line_base"], want["line_base"])
    assert got["line_lsmell"].dtype == np.uint8 and np.array_equal(got["line_lsmell"], want["line_lsmell"])
    assert got["lex"].dtype == ts.LEX_TEST and np.array_equal(got["lex"], want["lex"].astype(ts.LEX_TEST))
    plain = s.smells(c)
    for k in ("line_base", "line_smell", "tests"):
        assert np.array_equal(got[k], plain[k]), k
    return got


def test_hand(scanner):
    files = [d for _, _, d in lr.HAND]
    exts = np.array([e for _, e, _ in lr.HAND], np.uint8)
    got = check(scanner, files, exts)
    assert all((got["lex"]["smells"] >> k & 1).any() for k in range(4))


def test_c1_counts(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    got = check(scanner, files, exts)
    lex = got["lex"]
    counts = {"tests": len(lex)}
    counts.update({n: int(((lex["smells"] >> k) & 1).sum()) for k, n in enumerate(ts.LSMELLS)})
    assert counts == C1_COUNTS
    ms = scanner.smells_lexical_last_ms()
    assert len(ms) == 4 and all(m > 0 for m in ms)


def test_hazard_files(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_hazard_files.npz"))
    check(scanner, files, exts)


def test_c4_scale_planted():
    files, exts = lr.planted_corpus(0x7053454D2500, 20000)
    s = ts.Scanner(device=0, max_arena_bytes=1 << 26, max_files=1 << 16, max_groups=4)
    try:
        got = check(s, files, exts)
        assert len(got["lex"]) > 50000 and all((got["lex"]["smells"] >> k & 1).any() for k in range(5))
    finally:
        s.close()


@pytest.mark.parametrize("long_lines,binary", [(False, False), (True, False), (False, True)])
def test_fuzz(scanner, long_lines, binary):
    # fuzz tokens seldom form a test or an assertion call: every third file gets both planted between its lines
    files, exts = lr.fuzz_with_calls(0x1E25 + 7 * long_lines + 3 * binary, long_lines, binary)
    check(scanner, files, exts)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 20000])
def test_assertion_counts(scanner, n):
    py = b"def test_many(self):\n" + b"".join(b"    self.assertEqual(v%d, %d)\n    x%d = 1\n" % (i % 7, i, i % 13) for i in range(n))
    cc = b"TEST(A, B) {\n" + b"".join(b"  EXPECT_EQ(%d, x)%s\n" % (i % 40, b" << \"m\";" if i % 3 else b";") for i in range(n)) + b"}\n"
    got = check(scanner, [py, cc], np.array([1, 3], np.uint8))
    assert list(got["lex"]["n_stmts"]) == [n, n]
    assert got["lex"]["n_locals"][0] == min(n, 13)


def test_statement_cap_worst_case(scanner):
    # every line of a 20 000-line body is an assertion line whose call stays open: each walks the full LEX_STMT_LINES lines
    py = b"def test_open(self):\n" + b"    self.assertEqual(a, (\n" * 20000
    cc = b"TEST(A, B) {\n" + b"  EXPECT_EQ(a, (\n" * 20000 + b"}\n"
    got = check(scanner, [py, cc], np.array([1, 3], np.uint8))
    assert list(got["lex"]["n_unexplained"]) == [20000, 20000]


@pytest.mark.parametrize("n", [256, 257, 20000])
def test_many_locals(scanner, n):
    # a test of up to 256 names (repeats included) is counted in its warp's shared set, a larger one in its own slots of the
    # global table
    py = b"def test_locals():\n" + b"".join(b"    v%d = %d\n" % (i, i) for i in range(n)) + b"    v0 = 1\n    v%d = 2\n" % (n - 1)
    cc = b"TEST(A, B) {\n" + b"".join(b"  int v%d = %d;\n" % (i % (n - 1), i) for i in range(n)) + b"}\n"
    got = check(scanner, [py, cc, py], np.array([1, 3, 1], np.uint8))
    assert list(got["lex"]["n_locals"]) == [n, n - 1, n]


def test_more_tests_than_warps(scanner):
    files = [b"".join(b"def test_%d():\n    assert x == %d\n    assert y\n" % (i, i) for i in range(3000)) for _ in range(4)]
    got = check(scanner, files, np.array([1] * 4, np.uint8))
    assert len(got["lex"]) == 12000 > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 8
    assert (got["lex"]["smells"] == 3).all()


def test_no_tests_and_empty(scanner):
    got = check(scanner, [b"def helper():\n    assert 1\n", b"x\n"], np.array([1, 3], np.uint8))
    assert len(got["lex"]) == 0 and not got["line_lsmell"].any()
    got = scanner.smells_lexical(ts.pack([], np.zeros(0, np.uint8)))
    assert len(got["lex"]) == 0 and len(got["line_lsmell"]) == 0 and list(got["line_base"]) == [0]


def test_raw_caps_and_null_outputs(scanner):
    files = [d for _, _, d in lr.HAND]
    c = ts.pack(files, np.array([e for _, e, _ in lr.HAND], np.uint8))
    cs = c.c_struct()
    want = scanner.smells_lexical(c)
    L, T = len(want["line_smell"]), len(want["tests"])
    lib = ts.lib()
    nl, nt = C.c_int64(), C.c_int64()

    def call(base, smell, lsmell, lcap, tests, lex, tcap):
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731
        return lib.tsm_smells_lexical(scanner._ctx, C.byref(cs), p(base), p(smell), p(lsmell), lcap, C.byref(nl), p(tests), p(lex),
                                      tcap, C.byref(nt), None)

    def arrays():
        return (np.zeros(len(files) + 1, np.int64), np.zeros(L, np.uint16), np.zeros(L, np.uint8), np.zeros(T, ts.SMELL_TEST),
                np.zeros(T, ts.LEX_TEST))

    base, smell, lsmell, tests, lex = arrays()
    assert call(base, smell, lsmell, L, tests, lex, T) == 0 and (nl.value, nt.value) == (L, T)
    for k, a in zip(("line_base", "line_smell", "line_lsmell", "tests", "lex"), (base, smell, lsmell, tests, lex)):
        assert np.array_equal(a, want[k]), k
    assert call(base, smell, lsmell, L - 1, tests, lex, T) == ts.TSM_E_CAPACITY and (nl.value, nt.value) == (L, T)
    assert call(None, None, lsmell, L - 1, None, None, 0) == ts.TSM_E_CAPACITY
    assert call(base, smell, lsmell, L, tests, lex, T - 1) == ts.TSM_E_CAPACITY and (nl.value, nt.value) == (L, T)
    assert call(None, None, None, 0, None, lex, T - 1) == ts.TSM_E_CAPACITY
    assert call(None, None, None, 0, None, None, 0) == 0 and (nl.value, nt.value) == (L, T)
    for k, i in (("line_base", 0), ("line_smell", 1), ("line_lsmell", 2), ("tests", 3), ("lex", 4)):
        outs = [None] * 5
        outs[i] = arrays()[i]
        assert call(outs[0], outs[1], outs[2], L, outs[3], outs[4], T) == 0 and np.array_equal(outs[i], want[k]), k


def test_repeated_calls_and_stream(scanner):
    files, exts = lr.planted_corpus(0x1E26, 400)
    c = ts.pack(files, exts)
    first = scanner.smells_lexical(c)
    for _ in range(3):
        again = scanner.smells_lexical(c)
        assert all(np.array_equal(first[k], again[k]) for k in first)
    busy = torch.empty(1 << 26, device="cuda:0")
    st = torch.cuda.Stream(device=0)                      # (created non-blocking by torch)
    for _ in range(20):
        busy.mul_(1.0001)                                  # the legacy stream is busy while the call runs on st
    got = scanner.smells_lexical(c, stream=st.cuda_stream)
    torch.cuda.synchronize()
    assert all(np.array_equal(first[k], got[k]) for k in first)
