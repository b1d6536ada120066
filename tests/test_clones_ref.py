"""The references of the clone classes (docs/SPEC.md section 15), without a GPU: the serial C reference `orc_clones` (line and
n-gram hashes) equals the plain-Python `py_clones` (line contents) on hand-made cases, on generated corpora with planted
copies and on the study's C1 test files, where the counts are the ones content equality gives."""
import os
import random

import numpy as np
import pytest

import corpus_util as cu
import orc_clones as ocl
import tosemscan as ts

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def both(files, n, exts=None):
    exts = [1] * len(files) if exts is None else exts
    got = ocl.clones(ts.pack(files, exts), n)
    want = ocl.py_clones(files, exts, n)
    ocl.assert_equal(got, want)
    return got


def fragments(r):
    """[(length, [starts])] per class."""
    b = r["class_base"]
    return [(int(r["class_len"][c]), r["member"][b[c]:b[c + 1]].tolist()) for c in range(len(r["class_len"]))]


def test_abcd_cdefg_example():
    f = [b"A\nB\nC\nD\nE\nF\nG\n", b"x\nA\nB\nC\nD\nE\nF\nG\n", b"A\nB\nC\nD\n"]
    r = both(f, 3)
    assert fragments(r) == [(4, [0, 8, 15]), (5, [2, 10])]     # ABCD x3, CDEFG x2
    assert r["file_dup"].tolist() == [7, 7, 4]


def test_runs_of_repeated_lines():
    r = both([b"a\n" * 10], 3)
    assert fragments(r) == [(3, list(range(8)))]
    r = both([b"a\nb\n" * 6 + b"c\n", b"a\nb\na\n"], 2)
    assert r["file_dup"].tolist() == [12, 3]
    both([b"a\n" * 5, b"a\n" * 7, b"b\na\na\na\nb\n"], 1)
    both([b"a\n" * 5, b"a\n" * 7, b"b\na\na\na\nb\n"], 3)


def test_empty_windows_and_crlf():
    r = both([b"\n\n\n\n", b"\r\n\n\r\n\n"], 2)                  # windows of empty content only are not windows
    assert len(r["class_len"]) == 0 and r["file_dup"].tolist() == [0, 0]
    r = both([b"\n\nx\n", b"\r\n\r\nx\n"], 2)                    # ... but one empty line inside a window is content
    assert fragments(r) == [(2, [1, 4])]                        # (the window at 0 is all empty)
    lf = b"def test():\n    assert a == b\n\n    assert c\n"
    r = both([lf, lf.replace(b"\n", b"\r\n")], 3)               # a CRLF copy of an LF file is a clone
    assert fragments(r) == [(4, [0, 4])] and r["file_dup_assert"].tolist() == [2, 2]


def test_unterminated_short_files_and_limits():
    both([b"a\nb\nc", b"a\nb\nc\n", b"a\nb\nc\r"], 3)
    both([b"", b"a", b"a\nb", b"a\n", b"a\nb\n"], 3)             # files shorter than n have no windows
    both([b"", b"", b"x\n"], 1)
    r = both([b"q\n" + b"".join(b"l%d\n" % i for i in range(1100))] * 2 + [b"x\n"], 1024)
    assert fragments(r) == [(1101, [0, 1101])]
    r = both([b"a\nb\n", b"b\na\n", b"a\n"], 1)
    assert fragments(r) == [(1, [0, 3, 4]), (1, [1, 2])]
    r = both([b"l%d\n" % i for i in range(100)], 5)             # every file one line: no window of 5
    assert len(r["member"]) == 0


def planted(seed, n_files):
    rng = random.Random(seed)
    vocab = [b"x = %d" % i for i in range(30)] + [b"", b"\r", b"    assert a == %d" % 1, b"EXPECT_EQ(a, b);", b"}"]
    files = []
    for i in range(n_files):
        if files and rng.random() < 0.3:                         # a copy of a block of an earlier file, maybe CRLF
            src = files[rng.randrange(len(files))].split(b"\n")
            a = rng.randrange(len(src))
            block = b"\n".join(src[a:a + rng.randrange(1, 40)])
            pre = b"".join(rng.choice(vocab) + b"\n" for _ in range(rng.randrange(0, 5)))
            data = pre + block + (b"\n" if rng.random() < 0.8 else b"")
            files.append(data.replace(b"\n", b"\r\n") if rng.random() < 0.2 else data)
        else:
            files.append(b"".join(rng.choice(vocab[:rng.randrange(3, len(vocab))]) + b"\n" for _ in range(rng.randrange(0, 60))))
    return files


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_planted_copies(n):
    files = planted(0xC10E + n, 300)
    exts = [(i % 7) for i in range(len(files))]
    r = both(files, n, exts)
    assert len(r["class_len"]) > 10 and r["file_dup_assert"].sum() > 0


# The counts of the C1 test files under section 15, counted once with content equality instead of the hash:
# window -> (classes, fragments, duplicated lines, fragments of the largest class)
C1 = {3: (11678, 56315, 154383, 716), 5: (5771, 28227, 121252, 689), 10: (1844, 9467, 81449, 632)}


@pytest.fixture(scope="module")
def c1():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    return files, exts


@pytest.mark.parametrize("n", [3, 5, 10])
def test_c1_counts(c1, n):
    files, exts = c1
    r = both(files, n, exts)
    sizes = np.diff(r["class_base"])
    assert (len(r["class_len"]), len(r["member"]), int(r["file_dup"].sum()), int(sizes.max())) == C1[n]
    assert r["line_base"][-1] == 294387
    if n == 5:
        assert int(r["file_dup_assert"].sum()) == 6319
        assert int(r["class_len"][np.argmax(sizes)]) == 6
