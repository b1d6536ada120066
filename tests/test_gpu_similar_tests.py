"""`tsm_similar_tests` / `Scanner.similar_tests` (docs/SPEC.md section 23) against the serial C reference, every output array:
the worked example, the C1 test files, planted Type-3 copies, pattern lengths around the word and block seams of the LCS, a
long test against a copy with known deletions, a hot prefix token whose candidate space passes 2^32, more survivors than one
chunk holds, corpora without tests; the raw ABI (argument checks, each output NULL, each cap exact and one short), repeated calls
and a non-blocking stream while the legacy stream is busy."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

import corpus_util as cu
import simtest_ref as sr
import tosemscan as ts
from test_similar_tests_ref import EXAMPLE

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 17, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def c1():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    return ts.pack(files, exts)


def check(s, corpus, min_lines, P, **kw):
    got = s.similar_tests(corpus, min_lines, P, **kw)
    sr.assert_equal(got, sr.reference(corpus, min_lines, P))
    assert np.array_equal(got["tests"], s.smells(corpus)["tests"])
    return got


def test_worked_example(scanner):
    c = ts.pack([EXAMPLE], np.array([1], np.uint8))
    got = check(scanner, c, 5, 70)
    assert got["pairs"].tolist() == [(0, 1, 5, 54545), (0, 2, 4, 48000), (1, 2, 4, 43636)]
    got = check(scanner, c, 5, 75)
    assert len(got["pairs"]) == 2 and got["member"].tolist() == [0, 1, 2]
    assert len(check(scanner, c, 5, 95)["pairs"]) == 0


@pytest.mark.parametrize("min_lines,P", [(5, 70), (10, 90), (5, 100), (1, 50)])
def test_c1(scanner, c1, min_lines, P):
    got = check(scanner, c1, min_lines, P)
    assert len(got["tests"]) == 6239
    assert got["n_candidates"] >= len(got["pairs"])
    ms = scanner.similar_tests_last_ms()
    assert len(ms) == 4 and all(m >= 0 for m in ms) and ms[0] > 0


def planted(seed, n_files):
    """Files of PY tests: distinct random bodies, and Type-3 copies of earlier tests with lines inserted, deleted and changed."""
    rng = random.Random(seed)
    words = ["alpha", "beta", "f", "g", "h", "x", "y", "z", "self.a", "self.b"]
    ops = [" = %s(%s)", " += %s[%s]", ".append(%s, %s)", " = [%s for _ in %s]", "(%s).%s()"]
    pool, files = [], []
    for _ in range(n_files):
        tests = []
        for t in range(rng.randrange(1, 5)):
            if pool and rng.random() < 0.4:
                body = list(rng.choice(pool))
                for _ in range(rng.randrange(0, 3)):
                    r = rng.random()
                    if r < 0.33 and len(body) > 1:
                        body.pop(rng.randrange(len(body)))
                    elif r < 0.66:
                        body.insert(rng.randrange(len(body) + 1), "print(x)")
                    else:
                        body[rng.randrange(len(body))] = "assert %s" % rng.choice(words)
            else:
                body = [rng.choice(words) + rng.choice(ops) % (rng.choice(words), rng.choice(words)) for _ in range(rng.randrange(1, 20))]
                pool.append(body)
            tests.append("def test_%d():\n" % t + "".join("    %s\n" % x for x in body))
        files.append("\n".join(tests).encode())
    return files, np.ones(n_files, np.uint8)


def test_planted_type3_copies(scanner):
    c = ts.pack(*planted(5, 4000))          # 10 000 tests: the brute-force reference stays within seconds
    for min_lines, P in ((5, 70), (3, 90)):
        got = check(scanner, c, min_lines, P)
        assert len(got["pairs"]) > 4000


def seq_file(seqs):
    """One PY file with a test per sequence; element e of a sequence is the line `v<e> = 0` (a distinct blind form per e)."""
    out = []
    for i, s in enumerate(seqs):
        out.append("def test_%d():\n" % i + "".join("    " + "(" * (e % 5) + "x" + ")" * (e % 5) + "." * (e // 5 + 1) + "y\n" for e in s))
    return "".join(out).encode()


@pytest.mark.parametrize("m", [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 2047, 2048, 2049, 3000])
def test_pattern_lengths(scanner, m):
    rng = random.Random(m)
    a = [rng.randrange(12) for _ in range(m - 1)]
    b = list(a)
    for _ in range(max(1, m // 20)):
        b.insert(rng.randrange(len(b) + 1), rng.randrange(12))
    short = a[: max(1, m // 2 - 1)]
    c = ts.pack([seq_file([a, b, short, list(reversed(a))])], np.array([1], np.uint8))
    for P in (1, 60, 95):
        check(scanner, c, 1, P)


@pytest.mark.parametrize("k", [100, 3000])
def test_exact_threshold_on_both_verify_paths(scanner, k):
    # k kept lines each (header included), k / 10 body lines replaced by lines the other test lacks: lcs = 0.9 k exactly, so
    # 200 lcs == 90 (k + k): the pair passes at P = 90 and fails at 91 (k = 100: V in a register; 3000: V in scratch).
    a = list(range(k - 1))
    b = list(a)
    for i in range(k // 10):
        b[1 + 9 * i] = k + i
    c = ts.pack([seq_file([a, b])], np.array([1], np.uint8))
    lcs = k - k // 10
    assert 200 * lcs == 90 * 2 * k
    got = check(scanner, c, 1, 90)
    assert got["pairs"].tolist() == [(0, 1, lcs, 54000)]
    assert len(check(scanner, c, 1, 91)["pairs"]) == 0


def test_long_test_with_known_deletions(scanner):
    n = 70000
    a = list(range(n))
    drop = set(range(0, n, 7))
    b = [e for e in a if e not in drop]
    c = ts.pack([seq_file([a, b])], np.array([1], np.uint8))
    got = scanner.similar_tests(c, 1, 90)
    lcs = n - len(drop) + 1                                  # the header lines are equal too
    assert got["pairs"].tolist() == [(0, 1, lcs, 120000 * lcs // (2 * n + 2 - len(drop)))]


def test_hot_token_passes_2_32(scanner):
    # 93 000 tests: the header, `t = 1` and k - 2 lines `q`, with k = 2 + (i mod 500).  The header and `t = 1` are the rarest
    # lines of every test, so at P = 100 every prefix is the same token and its list holds every test: 4.3e9 candidates.  The
    # size filter keeps the pairs of equal k, which are all 100 % alike.
    nt, M = 93000, 500
    k = 2 + np.arange(nt) % M
    tests = ["def test_%d():\n    t = 1\n%s" % (i, "    q\n" * (int(k[i]) - 2)) for i in range(nt)]
    files = ["".join(tests[i:i + 1000]).encode() for i in range(0, nt, 1000)]
    c = ts.pack(files, np.ones(len(files), np.uint8))
    got = scanner.similar_tests(c, 1, 100)
    assert nt * (nt - 1) // 2 > 1 << 32
    groups = [np.nonzero(k == v)[0] for v in range(2, 2 + M)]
    want = sum(len(g) * (len(g) - 1) // 2 for g in groups)
    assert got["n_candidates"] == len(got["pairs"]) == want > 1 << 22
    assert np.array_equal(got["test_kept"], k.astype(np.uint32))
    p = got["pairs"]
    assert np.all(k[p["a"]] == k[p["b"]]) and np.all(p["score"] == 60000)
    assert len(got["class_base"]) - 1 == M and np.array_equal(got["member"][:len(groups[0])], groups[0])


def test_more_survivors_than_one_chunk(scanner):
    nt = 3000                                              # 4.5 M survivors > the chunk of 2^22
    files = ["".join("def test_%d():\n    q = %d\n    assert q\n" % (i * 100 + j, j) for j in range(100)).encode() for i in range(nt // 100)]
    c = ts.pack(files, np.ones(len(files), np.uint8))
    got = scanner.similar_tests(c, 3, 100)
    assert len(got["pairs"]) == nt * (nt - 1) // 2 > 1 << 22
    p = got["pairs"]
    assert np.all((p["a"][1:] > p["a"][:-1]) | ((p["a"][1:] == p["a"][:-1]) & (p["b"][1:] > p["b"][:-1])))


def test_no_tests(scanner):
    for files, exts in (([], []), ([b"x = 1\n"], [1]), ([b"def test_a():\n    pass\n"], [0]), ([b""], [1])):
        got = scanner.similar_tests(ts.pack(files, np.array(exts, np.uint8)))
        assert len(got["tests"]) == len(got["pairs"]) == len(got["member"]) == 0 and got["class_base"].tolist() == [0]


def raw(s, corpus, min_lines, P, caps, null=()):
    cs = corpus.c_struct()
    ct, cp, cc, cm = caps
    arrs = {"tests": np.zeros(max(ct, 1), ts.SMELL_TEST), "test_kept": np.zeros(max(ct, 1), np.uint32),
            "pairs": np.zeros(max(cp, 1), ts.SIMILAR_PAIR), "class_base": np.zeros(cc + 1, np.int64), "member": np.zeros(max(cm, 1), np.int32)}
    ptr = {k: (None if k in null else ts._p(v)) for k, v in arrs.items()}
    r = ts._SimilarResult(ptr["tests"], ptr["test_kept"], ct, 0, ptr["pairs"], cp, 0, ptr["class_base"], cc, 0, ptr["member"], cm, 0, 0)
    rc = ts.lib().tsm_similar_tests(s._ctx, C.byref(cs), min_lines, P, C.byref(r), None)
    return rc, r, arrs


def test_abi(scanner):
    c = ts.pack([EXAMPLE, EXAMPLE], np.array([1, 1], np.uint8))
    want = sr.reference(c, 5, 70)
    exact = (len(want["tests"]), len(want["pairs"]), len(want["class_base"]) - 1, len(want["member"]))
    rc, r, a = raw(scanner, c, 5, 70, exact)
    assert rc == 0 and (r.n_tests, r.n_pairs, r.n_classes, r.n_members) == exact
    assert a["pairs"].tolist() == want["pairs"].tolist() and a["member"].tolist() == want["member"].tolist()
    for i in range(4):
        short = list(exact)
        short[i] -= 1
        rc, r, _ = raw(scanner, c, 5, 70, short)
        assert rc == ts.TSM_E_CAPACITY and (r.n_tests, r.n_pairs, r.n_classes, r.n_members) == exact
    for key in ("tests", "test_kept", "pairs", "class_base", "member"):
        rc, r, _ = raw(scanner, c, 5, 70, (0, 0, 0, 0), null=("tests", "test_kept", "pairs", "class_base", "member"))
        assert rc == 0 and (r.n_tests, r.n_pairs, r.n_classes, r.n_members) == exact
        rc, r, a = raw(scanner, c, 5, 70, exact, null=(key,))
        assert rc == 0 and (r.n_tests, r.n_pairs, r.n_classes, r.n_members) == exact
        for other in ("tests", "test_kept", "pairs", "class_base", "member"):   # the outputs that are given are still filled
            if other != key:
                n = len(want[other])
                assert a[other][:n].tobytes() == np.asarray(want[other], a[other].dtype).tobytes(), (key, other)
    for ml, P in ((0, 70), (5, 0), (5, 101)):
        assert raw(scanner, c, ml, P, exact)[0] == -1           # TSM_E_ARG


def test_repeated_calls_and_busy_stream(scanner, c1):
    first = scanner.similar_tests(c1, 5, 70)
    with torch.cuda.device(0):
        side = torch.cuda.Stream(device=0)                 # non-blocking against the legacy stream
        a = torch.randn(4096, 4096, device="cuda:0")
        for _ in range(8):
            a = a @ a
            a /= a.norm()
        got = scanner.similar_tests(c1, 5, 70, stream=C.c_void_p(side.cuda_stream))
        torch.cuda.synchronize()
    for key in ("tests", "test_kept", "pairs", "class_base", "member"):
        assert np.array_equal(got[key], first[key])
    # n_candidates depends on how the count table's slots break ties between lines of equal counts, which may differ per call
    assert got["n_candidates"] >= len(got["pairs"]) and first["n_candidates"] >= len(first["pairs"])
