"""CPU tests: the plain-Python restatements of tests/spec_ref.py against the C oracle, on the edge corpus and on the byte
patterns tests/test_gpu_edges.py sends through the kernels (no GPU needed).  The GPU edge tests compare the device
with these references, so they are pinned here first."""
import json
import os
import random

import numpy as np

import corpus_util as cu
import orc
import spec_ref as sr

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def placed_hash_edges():
    """Every hash-edge content behind a few pads, before a CR-less last line and as an unterminated last line."""
    files = []
    for c in cu.hash_edge_contents():
        for pad in (0, 1, 7, 64):
            files.append(b"#" * pad + (b"\n" if pad else b"") + c + b"\n" + b"tail")
        files.append(b"x\n" + c)
    return files


def check_line_records(files, exts, ngrams=(1, 3, 62)):
    arena, off, ln = orc.pack(files)
    base, lh, end, flag = orc.line_records(arena, off, ln, np.array(exts, np.uint8))
    for i, f in enumerate(files):
        want = sr.py_line_records(f, exts[i])
        a, b = int(base[i]), int(base[i + 1])
        assert [(int(h), int(e), int(g)) for h, e, g in zip(lh[a:b], end[a:b], flag[a:b])] == want, (i, f[:40])
    for n in ngrams:
        got = orc.ngram_hashes(lh, base, n)
        for i in range(len(files)):
            a, b = int(base[i]), int(base[i + 1])
            assert [int(x) for x in got[a:b]] == sr.py_ngrams(lh[a:b], n), (i, n)


def test_line_records_reference_matches_the_oracle():
    files, exts, _ = cu.edge_corpus()
    check_line_records(files, [int(e) for e in exts])
    hf = placed_hash_edges()
    check_line_records(hf, [1] * len(hf), ngrams=(1, 5, 13))
    bf, bexts, _ = cu.fuzz_corpus(77, 200, 6000, binary=True)
    check_line_records(bf, [int(e) for e in bexts], ngrams=(2, 61, 200))


def test_hash_edge_contents_are_what_they_claim():
    contents = cu.hash_edge_contents()
    wraps = [c for c in contents if len(c) >= 9 and c.endswith(b"\r") and c[:-1] != b"\xff" * 8]
    assert len(wraps) == 147
    for c in wraps:
        n = len(c) - 1
        cr = 13 * pow(256, n, sr.M61) % sr.M61
        assert (int.from_bytes(c, "little")) % sr.M61 < cr           # the line's value with its CR wraps below the CR term
    zeros = [c for c in contents if c and int.from_bytes(c, "little") % sr.M61 == 0 and any(c)]
    assert len(zeros) >= 100
    for c in contents:
        assert sr.py_bytes_hash(c) == orc.bytes_hash(c)


def test_binary_fuzz_alphabet_leaves_the_ascii_seeds_alone():
    a = cu.fuzz_corpus(3, 40, 3000)
    b = cu.fuzz_corpus(3, 40, 3000, binary=False)
    assert a[0] == b[0]
    files, _, _ = cu.fuzz_corpus(3, 40, 3000, binary=True)
    blob = b"".join(files)
    assert len(set(blob)) == 256 and blob.count(b"\r") > blob.count(b"x")


def statements_for_category_checks():
    names = [n.encode() for n in sr.CATEGORY_NAMES.values()]
    ts = [b"self." + v for v in cu.table_name_variants(names)]
    ts += [r["statement"].encode("utf-8") for r in json.load(open(os.path.join(GOLD, "g4_statement_category.json")))]
    ts += [b"assert", b"assert x", b"assert not x", b"assert a not in b", b"assert a is not b", b"assert x == True",
           b"assert a == b", b"assert a != b", b"assert a <= b", b"assert a >= b", b"assert a < b", b"assert a > b",
           b"EXPECT_EQ", b"ASSERT_FLOAT_EQ", b"EXPECT_DOUBLE_EQ", b"EXPECT_STREQ", b"EXPECT_", b"x.assert_", b"assertx",
           b"assert\tx", b"GPUAssert", b"", b"assert_", b"x.assert", b"assertnot x"]
    return ts


def test_py_category_matches_the_oracle():
    rng = random.Random(9)
    ts = statements_for_category_checks()
    ts += [bytes(rng.choice(b"assertEXPCT_ notin=<>!Tue.xq") for _ in range(rng.randrange(0, 30))).strip() for _ in range(3000)]
    for t in ts:
        assert sr.py_category(t) == orc.classify(t)[0], t
        assert sr.py_category_string(t) == orc.category_string(t), t


def test_py_category_reproduces_golden_g4_with_the_ledger_misses():
    rows = json.load(open(os.path.join(GOLD, "g4_statement_category.json")))
    ledger = json.load(open(os.path.join(GOLD, "ledger.json")))["G4"]
    hit, tot, misses = 0, 0, set()
    for r in rows:
        tot += r["rows"]
        if sr.py_category_string(r["statement"].encode("utf-8")) == r["category"]:
            hit += r["rows"]
        else:
            misses.add((r["statement"], r["category"]))
    assert [hit, tot] == [11954, 11981]
    assert misses == {(m["statement"], m["sheet_says"]) for m in ledger["misses"]}
