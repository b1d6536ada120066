"""`tsm_similar_tests` (docs/SPEC.md section 23) where tests/test_gpu_similar_tests.py never reaches: the prefix filter at its
boundary for every P (the least partner size, which shares one token of the other test's prefix, and the size filter's
equality), pairs whose shared lines are one line repeated, warps that verify more than one candidate on the register and the
scratch paths of the LCS, carries across its blocks of 32 words, a corpus of many chunks with real filtering, output that does not depend on the filter's order, a
context pool left dirty by larger calls, and the section's boundaries (min_lines, the corpus' last line, CRLF, two tests in a
file, gtest and JUnit next to PY).  Each test asserts that it reached its seam; the builders are in tests/simtest_ref.py and
are checked on the CPU by tests/test_similar_tests_ref.py."""
import random

import numpy as np
import pytest
import torch

import simtest_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu

ARRAYS = ("tests", "test_kept", "pairs", "class_base", "member")


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 17, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def warps():
    """The warps of k_st_verify: sms x 4 blocks of 8 warps (csrc/tsm_api.cu)."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 32


def one_file(seqs):
    return ts.pack([sr.py_file(seqs)], np.array([1], np.uint8))


def check(s, corpus, min_lines, P):
    got = s.similar_tests(corpus, min_lines, P)
    sr.assert_equal(got, sr.reference(corpus, min_lines, P))
    return got


def pair_set(got):
    return set(zip(got["pairs"]["a"].tolist(), got["pairs"]["b"].tolist()))


def same_arrays(x, y):
    for key in ARRAYS:
        assert np.array_equal(x[key], y[key]), key


def test_tight_prefixes_at_every_P(scanner):
    eq = 0
    for P in range(1, 101):
        seqs, cases = sr.tight_cases(P)
        got = check(scanner, one_file(seqs), 1, P)
        assert got["test_kept"].tolist() == [len(s) + 1 for s in seqs]
        found = pair_set(got)
        for a, b, b2, e in cases:
            assert (min(a, b), max(a, b)) in found, (P, a, b)
            assert b2 is None or (min(a, b2), max(a, b2)) not in found, (P, a, b2)
            eq += e
    assert eq >= 30                                       # cases on 200 k_b == P (k_a + k_b)


@pytest.mark.parametrize("P", [40, 60, 80])
def test_pairs_of_repeated_lines(scanner, P):
    seqs, cases = sr.repeat_cases(P)
    got = check(scanner, one_file(seqs), 1, P)
    found = pair_set(got)
    p = {(a, b): l for a, b, l, _ in got["pairs"].tolist()}
    assert any(c2 < c for *_, c, c2 in cases)             # prefixes that end inside the run of R's tokens
    for a, b, c, c2 in cases:
        assert (a, b) in found and p[(a, b)] == c2 + 1, (a, b, c, c2)


@pytest.mark.parametrize("n", [999, 2099], ids=["register", "scratch"])
def test_warps_verify_more_than_one_candidate(scanner, warps, n):
    # 120 copies of n base lines (k = n + 1: V in registers for 1 000, in the warp's scratch slot for 2 100), every pair a
    # candidate: 7 140 > the warps, so a warp verifies a second pair after one of another lcs.
    P = 90
    seqs, sets = sr.copies(n, 120, P, n)
    want = sr.copies_pairs(n, sets, P)
    T = (n + 1) * (100 - P) // 100
    union = [len(sets[a] | sets[b]) for a in range(len(sets)) for b in range(a + 1, len(sets))]
    assert union.count(T) > 50 and union.count(T + 1) > 50   # pairs exactly on the threshold, and one line below it
    got = scanner.similar_tests(one_file(seqs), 1, P)
    assert got["n_candidates"] > warps
    assert np.all(got["test_kept"] == n + 1)
    assert got["pairs"].tolist() == want
    check(scanner, one_file(seqs[:10]), 1, P)             # every array against the C reference on 10 copies


@pytest.mark.parametrize("split", [2047, 2048, 2049])
def test_carry_across_the_32_word_blocks(scanner, split):
    # a = the header, A, B (split + 60 kept lines: V in scratch, two blocks of 32 words); b = the header, B, A.  B's lines are
    # matched first and leave zeros in V at and above bit split; each line of A then carries up through the ones below them,
    # across bit 2047 into the second block when split >= 2048.  lcs = 1 + |A| = split.
    A, B = list(range(split - 1)), list(range(split - 1, split + 59))
    got = check(scanner, one_file([A + B, B + A]), 1, 1)
    assert got["test_kept"].tolist() == [split + 60] * 2 and got["pairs"]["lcs"].tolist() == [split]


@pytest.fixture(scope="module")
def big():
    c, planted = sr.generated(0x53494D54, 200000)
    return c, planted, sr.c_sequences(c)


def test_many_chunks_with_real_filtering(scanner, big):
    c, planted, (tests, seqs) = big
    assert c.source_bytes < 1 << 28
    got = scanner.similar_tests(c, 5, 70)
    assert got["n_candidates"] > 2 * (1 << 22)            # three chunks or more of survivors
    assert np.array_equal(got["tests"], tests)
    k = np.array([len(s) for s in seqs], np.int64)
    assert np.array_equal(got["test_kept"], k.astype(np.uint32))
    flat = sr.flatten(seqs)
    p = got["pairs"]
    a, b = p["a"].astype(np.int64), p["b"].astype(np.int64)
    assert np.all((a[1:] > a[:-1]) | ((a[1:] == a[:-1]) & (b[1:] > b[:-1])))
    assert np.array_equal(p["lcs"], sr.c_lcs_pairs(flat, a, b))
    assert np.array_equal(p["score"], 120000 * p["lcs"].astype(np.int64) // (k[a] + k[b]))
    assert np.all(200 * p["lcs"].astype(np.int64) >= 70 * (k[a] + k[b])) and np.all(np.minimum(k[a], k[b]) >= 5)
    assert got["n_candidates"] > 4 * len(p)               # most survivors fail the LCS
    pc, po = np.array(planted).T
    lo, hi = np.minimum(pc, po), np.maximum(pc, po)
    pl = sr.c_lcs_pairs(flat, lo, hi).astype(np.int64)
    should = (k[lo] >= 5) & (k[hi] >= 5) & (200 * pl >= 70 * (k[lo] + k[hi]))
    assert should.sum() > 10000
    found = pair_set(got)
    missed = [(x, y) for x, y, s in zip(lo.tolist(), hi.tolist(), should) if s and (x, y) not in found]
    assert not missed, missed[:10]
    for t in random.Random(16).sample(range(len(seqs)), 16):
        mine = sorted(b[a == t].tolist() + a[b == t].tolist())
        assert mine == sr.c_partners(flat, t, 5, 70), t
    base, member = sr.classes(p.tolist(), len(seqs))
    assert np.array_equal(got["class_base"], base) and np.array_equal(got["member"], member)


@pytest.fixture(scope="module")
def mid():
    c, _ = sr.generated(0x4F524452, 50000)
    return c


def test_order_invariance(scanner, mid):
    files = [mid.file_bytes(i) for i in range(mid.n_files)]
    got = scanner.similar_tests(mid, 5, 70)
    assert len(got["pairs"]) > 2000
    key = {(int(t["file"]), int(t["line"])): i for i, t in enumerate(got["tests"])}
    # the files permuted: the pairs map through the permutation
    perm = np.random.default_rng(7).permutation(len(files))
    inv = np.argsort(perm)
    pc = ts.pack([files[i] for i in perm], np.ones(len(files), np.uint8))
    pg = scanner.similar_tests(pc, 5, 70)
    to_new = {i: (int(inv[f]), ln) for (f, ln), i in key.items()}
    new_key = {(int(t["file"]), int(t["line"])): i for i, t in enumerate(pg["tests"])}
    mapped = sorted((min(x, y), max(x, y), l, s) for x, y, l, s in
                    ((new_key[to_new[a]], new_key[to_new[b]], l, s) for a, b, l, s in got["pairs"].tolist()))
    assert pg["pairs"].tolist() == mapped
    # 50 000 filler tests appended: they pair with nothing, and the pairs of the others stay
    fill = sr.filler(50000, 0)
    fc = ts.pack(files + fill, np.ones(len(files) + len(fill), np.uint8))
    fg = scanner.similar_tests(fc, 5, 70)
    nt = len(got["tests"])
    assert len(fg["tests"]) == nt + 50000 and np.array_equal(fg["tests"][:nt], got["tests"])
    assert fg["pairs"].tolist() == got["pairs"].tolist()
    # a fresh context, and one whose pool a larger similar_tests and a blind clones call just used
    fresh = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 17, max_groups=4)
    try:
        same_arrays(fresh.similar_tests(mid, 5, 70), got)
    finally:
        fresh.close()
    scanner.similar_tests(fc, 3, 50)
    scanner.clones(fc, 5, blind=True)
    same_arrays(scanner.similar_tests(mid, 5, 70), got)


def body(name, lines):
    return "def %s():\n" % name + "".join("    %s\n" % x for x in lines)


def test_section_boundaries(scanner):
    five = ["a = f(1)", "b = g(a)", "c = h(b)", "assert c"]                   # 5 kept lines with the header
    # min_lines and min_lines - 1 kept lines, otherwise alike
    c = ts.pack([(body("test_a", five) + body("test_b", five) + body("test_c", five[:3]) + body("test_d", five[:3])).encode()],
                np.array([1], np.uint8))
    got = check(scanner, c, 5, 50)
    assert got["test_kept"].tolist() == [5, 5, 4, 4] and pair_set(got) == {(0, 1)}
    assert pair_set(check(scanner, c, 4, 50)) == {(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)}
    # a test on the corpus' last line, without a newline; CRLF; two tests in one file
    last = body("test_e", five).rstrip("\n").encode()
    crlf = body("test_f", five).replace("\n", "\r\n").encode()
    two = (body("test_g", five) + "\n" + body("test_h", five[:3] + ["assert b"])).encode()
    c = ts.pack([two, crlf, last], np.array([1, 1, 1], np.uint8))
    got = check(scanner, c, 5, 70)
    assert got["test_kept"].tolist() == [5, 5, 5, 5] and len(got["member"]) == 4
    assert pair_set(got) == {(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)}
    # gtest and JUnit next to PY: each family's tests pair within it
    cpp = b"TEST(S, A) {\n  int a = f(1);\n  int b = g(a);\n  EXPECT_EQ(b, 2);\n}\nTEST(S, B) {\n  int a = f(1);\n  int b = g(a);\n  EXPECT_EQ(b, 3);\n}\n"
    java = (b"class T {\n  @Test\n  public void testA() {\n    int a = f(1);\n    assertEquals(1, a);\n  }\n"
            b"  @Test\n  public void testB() {\n    int a = f(2);\n    assertEquals(2, a);\n  }\n}\n")
    c = ts.pack([cpp, two, java], np.array([3, 1, 4], np.uint8))
    got = check(scanner, c, 3, 70)
    fam = got["tests"]["file"]
    assert sorted(set(fam.tolist())) == [0, 1, 2]
    assert {(int(fam[a]), int(fam[b])) for a, b in pair_set(got)} >= {(0, 0), (1, 1), (2, 2)}
