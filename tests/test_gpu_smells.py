"""`tsm_smells` / `Scanner.smells` (docs/SPEC.md section 18) against the serial C reference orc_smells and the plain-Python
reference smell_ref.py_smells, every output array: the hand-written files, the C1 test files with their counts, planted smells at scale, fuzz corpora, tests of many assertion
lines with duplicates at every lane and tile seam, bodies ending at the seams of a 32-line round, a 70 000-line test, more tests
than the launch has warps, no tests and an empty corpus; the raw ABI's caps and NULL outputs, repeated calls and a non-blocking
stream while the legacy stream is busy."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import corpus_util as cu
import orc_smells as ocs
import smell_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
C1_COUNTS = {"tests": 6239, "empty": 363, "assertion_free": 1812, "duplicate_assert": 866, "redundant_assert": 8,
             "conditional_logic": 1190, "exception_handling": 98, "sleepy": 70, "print": 114, "ignored": 98}


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


def check(s, files, exts, **kw):
    """Every output array equals the C reference, and the plain-Python reference (which the CPU tests pin to the C one)."""
    c = ts.pack(files, exts)
    got = s.smells(c, **kw)
    ocs.assert_equal(got, ocs.smells(c))
    ocs.assert_equal(got, ocs.as_python(files, exts))
    return got


def test_hand(scanner):
    files = [d for _, _, d in sr.HAND]
    exts = np.array([e for _, e, _ in sr.HAND], np.uint8)
    got = check(scanner, files, exts)
    assert len(got["tests"]) == 24


def test_c1_counts(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    got = check(scanner, files, exts)
    t = got["tests"]
    counts = {"tests": len(t)}
    counts.update({n: int(((t["smells"] >> k) & 1).sum()) for k, n in enumerate(ts.SMELLS) if n in C1_COUNTS})
    assert counts == C1_COUNTS
    assert int(t["n_assert"].max()) == 107
    ms = scanner.smells_last_ms()
    assert len(ms) == 4 and all(m > 0 for m in ms)


def test_c4_scale_planted():
    files, exts = sr.planted_corpus(0x7053454D1800, 20000)
    s = ts.Scanner(device=0, max_arena_bytes=1 << 26, max_files=1 << 16, max_groups=4)
    try:
        got = check(s, files, exts)
        assert len(got["tests"]) > 50000 and all((got["tests"]["smells"] >> k & 1).any() for k in range(9))
    finally:
        s.close()


@pytest.mark.parametrize("long_lines,binary", [(False, False), (True, False), (False, True)])
def test_fuzz(scanner, long_lines, binary):
    files, exts, _ = cu.fuzz_corpus(0x5E11 + 7 * long_lines + 3 * binary, 300, 20000, long_lines=long_lines, binary=binary)
    # fuzz tokens seldom form a test header: every third file gets headers of each family planted between its lines
    rng = np.random.default_rng(5)
    heads = [b"def test_a():", b"    def test_b(self):", b"TEST(A, B) {", b"  public void testX() {", b"@pytest.mark.skip"]
    for i in range(0, len(files), 3):
        lines = files[i].split(b"\n")
        for _ in range(max(1, len(lines) // 20)):
            lines.insert(int(rng.integers(0, len(lines) + 1)), heads[int(rng.integers(0, len(heads)))])
        files[i] = b"\n".join(lines)
    check(scanner, files, exts)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 64, 65, 20000])
def test_assertion_counts(scanner, n):
    # n distinct assertion lines; then the repeats go where the duplicate search has its seams: at lane 0 and lane 31 of the tile
    # after the distinct ones (each a repeat of one from an earlier tile, or of tile 0 when n < 32) and one of line 0 at lane 31
    # of the first tile when that lane holds a distinct line (a repeat within the tile)
    rows = [b"    assert x == %d" % i for i in range(n)]
    if n > 31:
        rows[31] = b"    assert x == 0"
    t = (n + 31) // 32 * 32                                 # first lane of the next tile
    rows += [b"    assert x == %d" % (n - 1)] + [b"    assert y == %d" % i for i in range(t - n - 1)] if t > n else []
    rows += [b"    assert x == 1" if n > 1 else b"    assert x == 0"] + [b"    assert z == %d" % i for i in range(30)]
    rows += [b"    assert x == %d" % (n // 2)]
    files = [b"def test_many():\n" + b"\n".join(rows) + b"\n",
             b"TEST(A, B) {\n" + b"".join(b"  EXPECT_EQ(%d, 1);\n" % (i % 40) for i in range(n)) + b"}\n"]
    got = check(scanner, files, np.array([1, 3], np.uint8))
    assert got["tests"]["n_assert"][0] == len(rows)
    dup = np.nonzero(got["line_smell"][1:1 + len(rows)] & 4)[0]    # assertion k is line k + 1 of the file
    want = ([31] if n > 31 else []) + ([n] if t > n else []) + [max(t, n), max(t, n) + 31]
    assert list(dup) == sorted(want)


@pytest.mark.parametrize("end", [31, 32, 33])
def test_body_end_seams(scanner, end):
    py = b"def test_a():\n" + b"    x = 1\n" * (end - 1) + b"y = 2\n" + b"    z = 3\n" * 40
    cc = b"TEST(A, B) {\n" + b"  x();\n" * (end - 2) + b"}\n" + b"int y;\n" * 40
    doc = b"def test_d():\n" + b'    """\n' + b"    if x:\n" * (end - 3) + b'    """\n' + b"    if y:\n"
    got = check(scanner, [py, cc, doc], np.array([1, 2, 1], np.uint8))
    assert list(got["tests"]["body_lines"][:2]) == [end, end]


def test_70000_line_test(scanner):
    body = b"".join(b"    if x:\n        assert y == %d\n" % (i % 500) for i in range(35000))
    check(scanner, [b"def test_long():\n" + body, b"TEST(A, B) {\n" + body.replace(b":", b"") + b"}\n"], np.array([1, 3], np.uint8))


def test_more_tests_than_warps(scanner):
    files = [b"".join(b"def test_%d():\n    assert x\n    assert x\n" % i for i in range(3000)) for _ in range(4)]
    got = check(scanner, files, np.array([1] * 4, np.uint8))
    assert len(got["tests"]) == 12000 > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 8


def test_no_tests_and_empty(scanner):
    got = check(scanner, [b"def helper():\n    assert 1\n", b"x\n"], np.array([1, 3], np.uint8))
    assert len(got["tests"]) == 0
    got = scanner.smells(ts.pack([], np.zeros(0, np.uint8)))
    assert len(got["tests"]) == 0 and len(got["line_smell"]) == 0 and list(got["line_base"]) == [0]


def test_raw_caps_and_null_outputs(scanner):
    files = [d for _, _, d in sr.HAND]
    c = ts.pack(files, np.array([e for _, e, _ in sr.HAND], np.uint8))
    cs = c.c_struct()
    want = scanner.smells(c)
    L, T = len(want["line_smell"]), len(want["tests"])
    lib = ts.lib()
    nl, nt = C.c_int64(), C.c_int64()

    def call(base, smell, lcap, tests, tcap):
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        return lib.tsm_smells(scanner._ctx, C.byref(cs), p(base), p(smell), lcap, C.byref(nl), p(tests), tcap, C.byref(nt), None)

    base, smell, tests = np.zeros(len(files) + 1, np.int64), np.zeros(L, np.uint16), np.zeros(T, ts.SMELL_TEST)
    assert call(base, smell, L, tests, T) == 0 and (nl.value, nt.value) == (L, T)
    assert np.array_equal(smell, want["line_smell"]) and np.array_equal(tests, want["tests"])
    assert call(base, smell, L - 1, tests, T) == ts.TSM_E_CAPACITY and (nl.value, nt.value) == (L, T)
    assert call(base, smell, L, tests, T - 1) == ts.TSM_E_CAPACITY and (nl.value, nt.value) == (L, T)
    assert call(None, None, 0, None, 0) == 0 and (nl.value, nt.value) == (L, T)
    tests2 = np.zeros(T, ts.SMELL_TEST)
    assert call(None, None, 0, tests2, T) == 0 and np.array_equal(tests2, want["tests"])
    smell2 = np.zeros(L, np.uint16)
    assert call(None, smell2, L, None, 0) == 0 and np.array_equal(smell2, want["line_smell"])
    base2 = np.zeros(len(files) + 1, np.int64)
    assert call(base2, None, 0, None, 0) == 0 and np.array_equal(base2, want["line_base"])


def test_repeated_calls_and_stream(scanner):
    files, exts = sr.planted_corpus(0x5E12, 400)
    c = ts.pack(files, exts)
    first = scanner.smells(c)
    for _ in range(3):
        again = scanner.smells(c)
        assert all(np.array_equal(first[k], again[k]) for k in first)
    busy = torch.empty(1 << 26, device="cuda:0")
    st = torch.cuda.Stream(device=0)                      # (created non-blocking by torch)
    for _ in range(20):
        busy.mul_(1.0001)                                  # the legacy stream is busy while the call runs on st
    got = scanner.smells(c, stream=st.cuda_stream)
    torch.cuda.synchronize()
    assert all(np.array_equal(first[k], got[k]) for k in first)
