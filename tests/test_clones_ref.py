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


LF = b"def test():\n    assert a == b\n\n    assert c\n"
# The hand-made cases: name -> (files, n), every file with ext 1.  tests/test_gpu_clones_seams.py runs them on the GPU.
HAND_MADE = {
    "abcd_cdefg": ([b"A\nB\nC\nD\nE\nF\nG\n", b"x\nA\nB\nC\nD\nE\nF\nG\n", b"A\nB\nC\nD\n"], 3),
    "run_of_one_line": ([b"a\n" * 10], 3),
    "run_of_two_lines": ([b"a\nb\n" * 6 + b"c\n", b"a\nb\na\n"], 2),
    "runs_n1": ([b"a\n" * 5, b"a\n" * 7, b"b\na\na\na\nb\n"], 1),
    "runs_n3": ([b"a\n" * 5, b"a\n" * 7, b"b\na\na\na\nb\n"], 3),
    "empty_windows": ([b"\n\n\n\n", b"\r\n\n\r\n\n"], 2),
    "empty_line_inside": ([b"\n\nx\n", b"\r\n\r\nx\n"], 2),
    "crlf_copy": ([LF, LF.replace(b"\n", b"\r\n")], 3),
    "unterminated": ([b"a\nb\nc", b"a\nb\nc\n", b"a\nb\nc\r"], 3),
    "shorter_than_n": ([b"", b"a", b"a\nb", b"a\n", b"a\nb\n"], 3),
    "empty_files_n1": ([b"", b"", b"x\n"], 1),
    "n1024": ([b"q\n" + b"".join(b"l%d\n" % i for i in range(1100))] * 2 + [b"x\n"], 1024),
    "n1": ([b"a\nb\n", b"b\na\n", b"a\n"], 1),
    "one_line_files": ([b"l%d\n" % i for i in range(100)], 5),
}


def test_abcd_cdefg_example():
    r = both(*HAND_MADE["abcd_cdefg"])
    assert fragments(r) == [(4, [0, 8, 15]), (5, [2, 10])]     # ABCD x3, CDEFG x2
    assert r["file_dup"].tolist() == [7, 7, 4]


def test_runs_of_repeated_lines():
    r = both(*HAND_MADE["run_of_one_line"])
    assert fragments(r) == [(3, list(range(8)))]
    r = both(*HAND_MADE["run_of_two_lines"])
    assert r["file_dup"].tolist() == [12, 3]
    both(*HAND_MADE["runs_n1"])
    both(*HAND_MADE["runs_n3"])


def test_empty_windows_and_crlf():
    r = both(*HAND_MADE["empty_windows"])                       # windows of empty content only are not windows
    assert len(r["class_len"]) == 0 and r["file_dup"].tolist() == [0, 0]
    r = both(*HAND_MADE["empty_line_inside"])                   # ... but one empty line inside a window is content
    assert fragments(r) == [(2, [1, 4])]                        # (the window at 0 is all empty)
    r = both(*HAND_MADE["crlf_copy"])                           # a CRLF copy of an LF file is a clone
    assert fragments(r) == [(4, [0, 4])] and r["file_dup_assert"].tolist() == [2, 2]


def test_unterminated_short_files_and_limits():
    both(*HAND_MADE["unterminated"])
    both(*HAND_MADE["shorter_than_n"])                          # files shorter than n have no windows
    both(*HAND_MADE["empty_files_n1"])
    r = both(*HAND_MADE["n1024"])
    assert fragments(r) == [(1101, [0, 1101])]
    r = both(*HAND_MADE["n1"])
    assert fragments(r) == [(1, [0, 3, 4]), (1, [1, 2])]
    r = both(*HAND_MADE["one_line_files"])                      # every file one line: no window of 5
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


# ---------------------------------------------------------------------------------------------- windows with chosen keys
def oracle_keys(files, n):
    c = ts.pack([ocl.text(f) for f in files], [1] * len(files))
    return ocl.window_groups(c, n)["key"]


def test_crafted_keys():
    """orc.ngram_hashes gives the crafted windows exactly the keys asked for: 0, a chosen home slot, one key for two contents."""
    rng = random.Random(0xC0DE)
    for n in (5, 13):
        assert ocl.key_reachable(0, n)
        w = ocl.window_with_key(0, n, [b"t%d" % k for k in range(1, n)], rng)
        assert int(oracle_keys([[b"before"] + w], n)[1]) == 0
    for n in (3, 4, 6):                                         # n x 0x9E3779B97F4A7C15 mod 2^64 >= 2^61 - 1: no key 0
        with pytest.raises(ValueError):
            ocl.window_with_key(0, n, [b"t"] * (n - 1), rng)
    mask = ocl.table_mask(3000)
    assert mask == 8191 and ocl.table_mask(4096) == 8191 and ocl.table_mask(4097) == 16383
    for slot in (0, 1, mask):
        key = ocl.key_at_slot(slot, mask, 5, rng)
        got = int(oracle_keys([ocl.window_with_key(key, 5, [b"a", b"b", b"c", b"d"], rng)], 5)[0])
        assert got == key and got & mask == slot and got >> 13
    key = ocl.key_at_slot(17, mask, 3, rng)
    a = ocl.window_with_key(key, 3, [b"x", b"y"], rng)
    b = ocl.window_with_key(key, 3, [b"u", b"v"], rng)
    assert a != b and oracle_keys([a, b], 3)[[0, 3]].tolist() == [key, key]


@pytest.mark.parametrize("n", [5, 13])
@pytest.mark.parametrize("case", ["head", "middle", "once", "wide"])
def test_key0_corpora(case, n):
    files, _ = ocl.key0_corpus(case, n, 0xC10E0 + n)
    g = ocl.window_groups(ts.pack([ocl.text(f) for f in files], [1] * len(files)), n)
    assert ((g["key"] == 0) & g["valid"]).sum() == {"head": 3, "middle": 2, "once": 1, "wide": 40}[case]
    both([ocl.text(f) for f in files], n)


@pytest.mark.parametrize("extra", [0, 1])
def test_probe_corpus_without_collision(extra):
    files, mask = ocl.probe_corpus(extra, 0x9B0BE + extra, collide=False)
    r = both([ocl.text(f) for f in files], 3)
    assert len(r["class_len"]) == 560 and r["line_base"][-1] == 4096 + extra


def test_collision_pair_the_key_decides():
    """Section 15.1: windows are equal when their keys are.  The reference over keys puts two contents with one key in one
    group (a class of two fragments); content equality keeps them apart (no class)."""
    files, mask = ocl.probe_corpus(0, 0x9B0BE, collide=True)
    data = [ocl.text(f) for f in files]
    got = ocl.clones(ts.pack(data, [1] * len(data)), 3)
    want = ocl.py_clones(data, [1] * len(data), 3)
    pair = [i for i, f in enumerate(files) if f and f[1].startswith(b"p")]
    assert len(pair) == 2 and files[pair[0]] != files[pair[1]]
    starts = [int(got["line_base"][i]) for i in pair]
    extra = [c for c in range(len(got["class_len"])) if got["member"][got["class_base"][c]:got["class_base"][c + 1]].tolist() == starts]
    assert len(extra) == 1 and got["class_len"][extra[0]] == 3
    keep = np.ones(len(got["class_len"]), bool)
    keep[extra[0]] = False
    assert fragments(want) == [fr for fr, k in zip(fragments(got), keep) if k]
    assert np.array_equal(want["file_dup"] + np.isin(np.arange(len(files)), pair) * 3, got["file_dup"])
