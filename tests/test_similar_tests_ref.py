"""The similar tests of docs/SPEC.md section 23 on the CPU: the worked example, thresholds and edge cases with known answers, the
plain-Python and serial C references against each other, and the model of the device's prefix filter against brute force."""
import random

import numpy as np
import pytest

import simtest_ref as sr

EXAMPLE = b'''import unittest


class TestAdd(unittest.TestCase):
    def test_add(self):
        x = f(1)
        y = g(x, 2)
        self.assertEqual(y, 3)
        self.assertTrue(ok)

    def test_add_print(self):
        x = f(1)
        y = g(x, 2)
        print(y)
        self.assertEqual(y, 3)
        self.assertTrue(ok)

    def test_add_one_arg(self):
        # one argument
        x = f(1)
        y = g(x)
        self.assertEqual(y, 3)
        self.assertTrue(ok)
'''


def test_worked_example():
    tests, seqs = sr.py_sequences([EXAMPLE], [1])
    assert [(b + 1, len(s)) for (_, b, _), s in zip(tests, seqs)] == [(5, 5), (11, 6), (18, 5)]
    assert sr.py_similar(seqs, 5, 70) == [(0, 1, 5, 54545), (0, 2, 4, 48000), (1, 2, 4, 43636)]
    assert [p[3] // 600 for p in sr.py_similar(seqs, 5, 70)] == [90, 80, 72]
    at75 = sr.py_similar(seqs, 5, 75)
    assert [(a, b) for a, b, *_ in at75] == [(0, 1), (0, 2)]
    base, member = sr.classes(at75, 3)                     # single linkage: B and C are one class at 72 %
    assert base.tolist() == [0, 3] and member.tolist() == [0, 1, 2]
    assert sr.py_similar(seqs, 5, 95) == []
    renamed = EXAMPLE.replace(b"test_add(self)", b"test_other(self)").replace(b"x = f(1)", b"zz = h(7)")
    _, s2 = sr.py_sequences([renamed], [1])
    assert sr.lcs(seqs[0], s2[0]) == 5                     # a Type-2 copy is 100 %


def body(name, lines, indent=b"    "):
    return b"def " + name + b"():\n" + b"".join(indent + x + b"\n" for x in lines)


def test_exact_threshold_and_below():
    # k = 5 and 5, lcs 4: 200 * 4 = 800 = 80 * 10 passes at P = 80 and fails at 81
    a = body(b"test_a", [b"a = 1", b"b = f(a)", b"c = g(b)", b"assert c"])
    b = body(b"test_b", [b"a = 1", b"b = f(a)", b"c = g[b]", b"assert c"])
    _, seqs = sr.py_sequences([a + b"\n" + b], [1])
    assert sr.lcs(*seqs) == 4
    assert len(sr.py_similar(seqs, 5, 80)) == 1 and sr.py_similar(seqs, 5, 81) == []
    assert len(sr.py_similar(seqs, 5, 1)) == 1


def test_min_lines_edges_and_kept_lines():
    lines = [b"x = 1", b"", b"# comment", b'"""', b"inner docstring line", b'"""', b"assert x"]
    a = body(b"test_a", lines)
    _, seqs = sr.py_sequences([a + b"\n" + a.replace(b"test_a", b"test_b")], [1])
    # header, x = 1, the docstring's opening line (a string token) and assert x; blank, comment and inner lines are not kept
    assert [len(s) for s in seqs] == [4, 4]
    assert len(sr.py_similar(seqs, 4, 100)) == 1 and sr.py_similar(seqs, 5, 1) == []


def test_crlf_tag0_header_only_and_families():
    a = body(b"test_a", [b"x = 1", b"assert x"]).replace(b"\n", b"\r\n")
    b = body(b"test_b", [b"x = 1", b"assert x"])
    tests, seqs = sr.py_sequences([a, b, b], [1, 1, 0])
    assert len(tests) == 2 and sr.py_similar(seqs, 1, 100) == [(0, 1, 3, 60000)]
    cpp = b"TEST(S, A) {\n  EXPECT_EQ(f(1), 2);\n}\nBOOST_AUTO_TEST_CASE(b) {\n  EXPECT_EQ(f(3), 4);\n}\n"
    java = b"class T {\n  @Test\n  public void testA() {\n    assertEquals(1, f());\n  }\n}\n"
    tests, seqs = sr.py_sequences([cpp, java, b"def test_h(): pass\n"], [3, 4, 1])
    assert len(tests) == 4
    pairs = sr.py_similar(seqs, 1, 50)
    assert (0, 1) in [(a, b) for a, b, *_ in pairs]
    assert sr.py_similar(seqs, 1, 50) == sr.c_similar(seqs, 1, 50)


def random_corpus(rng, n_tests, alphabet):
    out = []
    base = [rng.randrange(alphabet) for _ in range(rng.randint(1, 14))]
    for _ in range(n_tests):
        s = list(base) if rng.random() < 0.5 else [rng.randrange(alphabet) for _ in range(rng.randint(1, 14))]
        for _ in range(rng.randint(0, 3)):
            if s and rng.random() < 0.5:
                s.pop(rng.randrange(len(s)))
            else:
                s.insert(rng.randrange(len(s) + 1), rng.randrange(alphabet))
        out.append(s)
    return out


@pytest.mark.parametrize("seed", range(6))
def test_prefix_filter_model_equals_brute_force(seed):
    rng = random.Random(seed)
    for P in list(range(1, 101, 9)) + [100]:
        seqs = random_corpus(rng, 30, rng.randint(2, 8))
        for min_lines in (1, 3):
            want = sr.py_similar(seqs, min_lines, P)
            cand = sr.prefix_candidates(seqs, min_lines, P)
            assert {(a, b) for a, b, *_ in want} <= cand
            assert sr.c_similar(seqs, min_lines, P) == want


def test_references_agree_on_planted_files():
    import smell_ref
    files, exts = smell_ref.planted_corpus(23, 40)
    tests, seqs = sr.py_sequences(files, exts)
    import tosemscan as ts
    ctests, cseqs = sr.c_sequences(ts.pack(files, exts))
    assert [(int(t["file"]), int(t["line"]), int(t["body_lines"])) for t in ctests] == tests and cseqs == seqs
    for P in (50, 90):
        assert sr.c_similar(seqs, 3, P) == sr.py_similar(seqs, 3, P)


# SPEC section 23's C1 counts: (min_lines, P) -> (compared tests, pairs, classes, tests in a class)
C1_PINNED = {(5, 70): (4640, 8561, 598, 2331), (10, 90): (3183, 1604, 255, 744), (5, 100): (4640, 2593, 289, 880),
             (1, 50): (6141, 282306, 418, 4981)}


@pytest.fixture(scope="module")
def c1_seqs():
    import os
    import corpus_util as cu
    import tosemscan as ts
    files, exts, _, _ = cu.load_fixture(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "c1_testfiles.npz"))
    return files, exts, sr.c_sequences(ts.pack(files, exts))


def test_c1_sequences_agree(c1_seqs):
    files, exts, (ctests, cseqs) = c1_seqs
    tests, seqs = sr.py_sequences(files, exts)
    assert len(tests) == 6239
    assert [(int(t["file"]), int(t["line"]), int(t["body_lines"])) for t in ctests] == tests and cseqs == seqs


@pytest.mark.parametrize("setting", [(5, 70), (10, 90), (5, 100)])
def test_c1_counts(c1_seqs, setting):
    _, _, (_, seqs) = c1_seqs
    pairs = sr.c_similar(seqs, *setting)
    base, member = sr.classes(pairs, len(seqs))
    assert (sum(len(s) >= setting[0] for s in seqs), len(pairs), len(base) - 1, len(member)) == C1_PINNED[setting]
    if setting == (5, 70):                                 # the filter model keeps every C1 pair
        assert {(a, b) for a, b, *_ in pairs} <= sr.prefix_candidates(seqs, *setting)


def test_prefix_filter_model_on_planted_corpora():
    import smell_ref
    for seed in (3, 4):
        files, exts = smell_ref.planted_corpus(seed, 60)
        _, seqs = sr.py_sequences(files, exts)
        for P in (1, 30, 70, 99, 100):
            want = sr.c_similar(seqs, 2, P)
            assert {(a, b) for a, b, *_ in want} <= sr.prefix_candidates(seqs, 2, P)
