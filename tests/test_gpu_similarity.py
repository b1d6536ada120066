"""`tsm_similarity` / `Scanner.similarity` (docs/SPEC.md section 13) bit for bit against the C reference orc_similarity,
which splits, hashes and weighs the raw bytes itself.  Covers C5-shaped corpora at several edit rates, a full matrix, one
old file against thousands of new ones, repeated candidates, files above the shared-memory sort limit, empty files,
n_cand = 0 and every error status."""
import ctypes as C
import random

import numpy as np
import pytest

import orc_similarity as osim
import tosemscan as ts

pytestmark = pytest.mark.gpu

SMEM_LINES = 4096                                          # SIM_SMEM_LINES of csrc/tsm_similar_kernels.cuh


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


def check(s, olds, news, co, cn):
    got = s.similarity(olds, news, co, cn)
    want = osim.similarity(olds, news, co, cn)
    assert got.dtype == np.int64 and got.shape == want.shape
    assert np.array_equal(got, want)
    return got


@pytest.mark.parametrize("lam", [0, 1, 6, 40, 200])
def test_c5_pairs(scanner, lam):
    olds, news = ts.gen_pairs(0x51A0 + lam, 3000, cap=65536, lam=float(lam), pinned=False)
    n = olds.n_files
    rng = np.random.default_rng(lam)
    co = np.concatenate([np.arange(n), rng.integers(0, n, 20000)]).astype(np.int32)
    cn = np.concatenate([np.arange(n), rng.integers(0, n, 20000)]).astype(np.int32)
    got = check(scanner, olds, news, co, cn)
    if lam == 0:                                            # unedited pairs: everything in common but the CRs of CRLFs
        sizes = olds.len.astype(np.int64)
        crlf = np.array([olds.file_bytes(i).count(b"\r\n") for i in range(n)], np.int64)
        assert np.array_equal(got[:n], sizes - crlf)
    ms = scanner.similarity_last_ms()
    assert len(ms) == 3 and all(m > 0 for m in ms)


def test_full_matrix(scanner):
    olds, news = ts.gen_pairs(0x51A1, 2000, cap=8192, lam=6.0, pinned=False)
    co, cn = np.meshgrid(np.arange(2000, dtype=np.int32), np.arange(2000, dtype=np.int32), indexing="ij")
    got = check(scanner, olds, news, co.ravel(), cn.ravel())
    assert got.size == 4_000_000 and (got > 0).sum() > 2000


def test_one_old_file_against_thousands(scanner):
    olds, news = ts.gen_pairs(0x51A2, 5000, cap=16384, lam=6.0, pinned=False)
    one = ts.pack([olds.file_bytes(17)], [1])
    cn = np.arange(5000, dtype=np.int32)
    got = check(scanner, one, news, np.zeros(5000, np.int32), cn)
    assert got[17] > 0
    check(scanner, news, one, cn, np.zeros(5000, np.int32))    # and the other way round: different file counts per side


def test_repeated_candidates(scanner):
    olds, news = ts.gen_pairs(0x51A3, 64, cap=8192, lam=6.0, pinned=False)
    co = np.array([3] * 500 + [5, 3, 5, 3] * 100, np.int32)
    cn = np.array([3] * 500 + [5, 5, 3, 3] * 100, np.int32)
    got = check(scanner, olds, news, co, cn)
    assert len(set(got[:500].tolist())) == 1


def big_file(rng, n_lines, distinct):
    vocab = [b"line %d of many\n" % i for i in range(distinct)] + [b"\n", b"x\r\n", b"    assert q\n"]
    return b"".join(rng.choice(vocab) for _ in range(n_lines))


def test_files_above_the_shared_memory_sort_limit(scanner):
    rng = random.Random(0x51A4)
    files = [big_file(rng, SMEM_LINES + 1, 3000), big_file(rng, 9000, 8000), big_file(rng, 70000, 50000),
             big_file(rng, 61000, 50), big_file(rng, SMEM_LINES, 4000), big_file(rng, 300, 100)]
    edits = [ts.gen_edit(k, f, 40.0) for k, f in enumerate(files)]
    assert max(f.count(b"\n") for f in files) > 16 * SMEM_LINES
    olds, news = ts.pack(files, [1] * len(files)), ts.pack(edits + files, [1] * (2 * len(files)))
    co, cn = np.meshgrid(np.arange(len(files), dtype=np.int32), np.arange(2 * len(files), dtype=np.int32), indexing="ij")
    got = check(scanner, olds, news, co.ravel(), cn.ravel())
    assert got.reshape(len(files), -1)[2, 8] == len(files[2]) - files[2].count(b"\r\n")


def test_empty_files(scanner):
    files = [b"", b"a\n", b"", b"\n", b"a", b""]
    k = ts.pack(files, [0] * len(files))
    co, cn = np.meshgrid(np.arange(6, dtype=np.int32), np.arange(6, dtype=np.int32), indexing="ij")
    got = check(scanner, k, k, co.ravel(), cn.ravel())
    assert got.reshape(6, 6)[0].tolist() == [0] * 6
    allempty = ts.pack([b"", b""], [1, 1])
    assert check(scanner, allempty, allempty, [0, 1], [1, 0]).tolist() == [0, 0]


def test_no_candidates(scanner):
    olds, news = ts.gen_pairs(0x51A5, 8, cap=4096, lam=6.0, pinned=False)
    assert scanner.similarity(olds, news, [], []).shape == (0,)
    assert scanner.similarity_last_ms() == [0.0, 0.0, 0.0]
    empty = ts.Corpus(np.zeros(128, np.uint8), np.zeros(1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.uint8))
    assert scanner.similarity(empty, empty, [], []).shape == (0,)


def test_error_statuses(scanner):
    L = ts.lib()
    olds, news = ts.gen_pairs(0x51A6, 4, cap=4096, lam=6.0, pinned=False)
    a, b = olds.c_struct(), news.c_struct()
    out = np.zeros(4, np.int64)
    p = ts._p

    def call(co, cn, n=None, ka=a, kb=b, common=out, ctx=scanner._ctx):
        co = np.asarray(co, np.int32)
        cn = np.asarray(cn, np.int32)
        return L.tsm_similarity(ctx, C.byref(ka) if ka is not None else None, C.byref(kb) if kb is not None else None, p(co), p(cn),
                                co.size if n is None else n, p(common) if common is not None else None, None)

    assert call([0, 1], [1, 3]) == 0
    for co, cn in (([4], [0]), ([0], [4]), ([-1], [0]), ([0], [-1])):
        assert call(co, cn) == -1
    assert call([0], [0], n=-1) == -1
    assert call([0], [0], common=None) == -1
    assert call([0], [0], ka=None) == -1
    assert L.tsm_similarity(None, C.byref(a), C.byref(b), None, None, 0, None, None) == -1
    assert L.tsm_similarity(scanner._ctx, C.byref(a), C.byref(b), None, None, 0, None, None) == 0   # n_cand = 0: nothing is read
    assert call([0], [0], n=1 << 40) == -5                                     # 16 TiB of candidates: TSM_E_NOMEM, nothing read
    bad = olds.off.copy()
    bad[1] += 1                                                                 # a misaligned file start
    ka = ts._Corpus(p(olds.arena), p(bad), p(olds.len), p(olds.ext), None, olds.n_files, 1)
    assert call([0], [0], ka=ka) == -2
    kb = ts._Corpus(p(news.arena), p(news.off), p(news.len), p(news.ext), None, news.n_files, 1)
    assert call([0], [0], kb=kb) == 0
    ms = (C.c_float * 3)()
    assert L.tsm_similarity_last_ms(None, C.byref(ms)) == -1
    assert L.tsm_similarity_last_ms(scanner._ctx, None) == -1
    # the context still works after every refusal
    check(scanner, olds, news, np.arange(4, dtype=np.int32), np.arange(4, dtype=np.int32))
