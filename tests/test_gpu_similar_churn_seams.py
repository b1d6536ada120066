"""`tsm_similar_churn` (docs/SPEC.md section 24) where the suite never reaches: posting lists with d = 0, 1, m - 1 and m dirty
tests of m; one list of 2^17 tests with one dirty member (2^17 - 1 restricted candidates, where the full space exceeds 2^32);
more restricted candidates than one 2^22 chunk; cross scores on the register and on the scratch path (tests over 2 048 kept
lines); a cross pair on a side with no compared test; a one-sided edit that changes a test's sequence but marks none of its
body lines; and 200 000 generated tests with a step that touches 0.1 % of them, every event rechecked by the serial C LCS.
Builders: tests/simtest_ref.py (py_file: one line of its own blind form per id)."""
import numpy as np
import pytest

import similar_churn_ref as ref
import simtest_ref as sr
import test_similar_churn_ref as ex
import tosemscan as ts

pytestmark = pytest.mark.gpu
NONE = ref.NONE
CHANGED, DIVERGED, CONVERGED = 0, 3, 6


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


def churn(s, old_files, new_files, po, pn, ml=5, P=70):
    return s.similar_churn(ts.pack(old_files, np.ones(len(old_files), np.uint8)), ts.pack(new_files, np.ones(len(new_files), np.uint8)),
                           po, pn, ml, P)


BASE = list(range(5))                                      # five lines of their own: k = 6 with the header


@pytest.mark.parametrize("d", [0, 1, 39, 40])
def test_list_with_d_dirty_of_m(scanner, d):
    m = 40
    old = [sr.py_file([BASE] * m)]
    new = [sr.py_file([BASE + [100 + i] if i < d else BASE for i in range(m)])]
    got = churn(scanner, old, new, [0], [0])
    ref.assert_equal(got, ref.churn((old, [1]), (new, [1]), [0], [0]))
    want = d * m - d * (d + 1) // 2                          # every pair with a dirty test, each verified once
    assert got["old"]["n_candidates"] == want and got["new"]["n_candidates"] == want
    assert len(got["events"]) == want


def test_one_dirty_test_in_a_list_of_2_17(scanner):
    m, per = 1 << 17, 1000
    assert m * (m - 1) // 2 > 1 << 32
    files = [sr.py_file([BASE] * min(per, m - f)) for f in range(0, m, per)]
    new = list(files)
    new[0] = sr.py_file([BASE + [100]] + [BASE] * (per - 1))
    got = churn(scanner, files, new, [0], [0])
    assert got["old"]["n_candidates"] == m - 1 and got["new"]["n_candidates"] == m - 1
    ev = got["events"]
    assert len(ev) == m - 1 and bool(np.all(ev["status"] == CHANGED))
    assert bool(np.all(ev["a"] == 0)) and np.array_equal(np.sort(ev["b"]), np.arange(1, m))
    assert bool(np.all(ev["old_a"] == 0)) and np.array_equal(ev["old_b"], ev["b"])
    assert bool(np.all(ev["old_lcs"] == 6)) and bool(np.all(ev["old_score"] == 120000 * 6 // 12))
    assert bool(np.all(ev["lcs"] == 6)) and bool(np.all(ev["score"] == 120000 * 6 // 13))
    assert bytes(got["new"]["change"][:2]) == b"M="


def test_restricted_candidates_beyond_one_chunk(scanner):
    m, d = 3200, 2000
    want = d * m - d * (d + 1) // 2
    assert want > 1 << 22
    per = 400
    old = [sr.py_file([BASE] * per) for _ in range(m // per)]
    new = [sr.py_file([BASE + [100] if f * per + i < d else BASE for i in range(per)]) for f in range(m // per)]
    pairs = [f for f in range(m // per) if f * per < d]
    got = churn(scanner, old, new, pairs, pairs)
    assert got["old"]["n_candidates"] == want and got["new"]["n_candidates"] == want
    ev = got["events"]
    assert len(ev) == want and bool(np.all(ev["status"] == CHANGED))
    a, b = ev["a"].astype(np.int64), ev["b"].astype(np.int64)
    assert bool(np.all(a < b)) and bool(np.all(a < d))
    assert len(np.unique(a * m + b)) == want                  # every pair with a dirty test, once
    both = b < d
    assert bool(np.all(ev["score"][both] == 120000 * 7 // 14)) and bool(np.all(ev["score"][~both] == 120000 * 6 // 13))


@pytest.mark.parametrize("n", [100, 2100])
def test_cross_scores_register_and_scratch(scanner, n):
    base = list(range(n))
    cut = base[: n * 3 // 8]                                  # lcs with the base: the kept lines, below P = 70 against it
    old = [sr.py_file([base, base])]
    new = [sr.py_file([base, cut])]
    got = churn(scanner, old, new, [0], [0])
    ev = got["events"]
    assert len(ev) == 1 and ev[0]["status"] == DIVERGED
    k, kc = n + 1, len(cut) + 1
    assert ev[0]["lcs"] == kc and ev[0]["score"] == 120000 * kc // (k + kc)
    assert ev[0]["old_lcs"] == k and ev[0]["old_score"] == 60000
    # and back: the same pair converges, scored on the old side
    got = churn(scanner, new, old, [0], [0])
    ev = got["events"]
    assert len(ev) == 1 and ev[0]["status"] == CONVERGED and ev[0]["old_lcs"] == kc and ev[0]["lcs"] == k


def test_cross_pair_on_a_side_with_no_compared_test(scanner):
    old = [sr.py_file([[1, 2], [1, 2]])]                     # k = 3: no test of the old side is compared at min_lines 5
    new = [sr.py_file([[1, 2, 3, 4, 5], [1, 2, 3, 4, 5]])]
    got = churn(scanner, old, new, [0], [0])
    ref.assert_equal(got, ref.churn((old, [1]), (new, [1]), [0], [0]))
    ev = got["events"]
    assert len(ev) == 1 and ev[0]["status"] == CONVERGED and ev[0]["old_lcs"] == 3 and ev[0]["old_score"] == 60000
    assert got["old"]["n_candidates"] == 0


def test_sequence_changed_without_a_marked_body_line(scanner):
    new = ex.HEAD + b'    """\n' + ex.A + b'    """\n' + b"\n" + ex.B
    old = ex.HEAD + b"\n" + ex.A + b"\n" + b"\n" + ex.B
    got = churn(scanner, [old], [new], [0], [0])
    want = ref.churn(([old], [1]), ([new], [1]), [0], [0])
    assert want["new"]["change"][:1] == b"M"
    ref.assert_equal(got, want)


def test_generated_200k_with_a_small_step(scanner):
    k, _ = sr.generated(3, 200000)
    files = [bytes(k.arena[int(k.off[i]):int(k.off[i]) + int(k.len[i])]) for i in range(k.n_files)]
    exts = np.ones(len(files), np.uint8)
    rng = np.random.default_rng(11)
    new = list(files)
    for t in sorted(rng.choice(200000, 200, replace=False).tolist(), reverse=True):   # one line inserted behind 0.1 % of the headers
        f, h = t // 100, b"def test_%d():\n" % t
        at = new[f].index(h) + len(h)
        new[f] = new[f][:at] + b"    touched = True\n" + new[f][at:]
    touched = [f for f in range(len(files)) if new[f] != files[f]]
    okp, nkp = ts.pack(files, exts), ts.pack(new, exts)
    got = scanner.similar_churn(okp, nkp, touched, touched)
    ev = got["events"]
    assert len(ev) > 0
    for side, kp, a, b, lcs, score in (("old", okp, "old_a", "old_b", "old_lcs", "old_score"), ("new", nkp, "a", "b", "lcs", "score")):
        _, seqs = sr.c_sequences(kp)
        flat = sr.flatten(seqs)
        has = ev[lcs] != NONE
        x, y = ev[a][has], ev[b][has]
        lo, hi = np.minimum(x, y), np.maximum(x, y)
        want_lcs = sr.c_lcs_pairs(flat, lo, hi)
        assert np.array_equal(ev[lcs][has], want_lcs), side
        kk = flat[2]
        assert np.array_equal(ev[score][has], (120000 * want_lcs.astype(np.int64) // (kk[lo].astype(np.int64) + kk[hi])).astype(np.uint32))
        st = scanner.similar_tests(kp)
        dirty = got[side]["change"] != ord("=")
        want = {(int(p["a"]), int(p["b"])) for p in st["pairs"] if dirty[p["a"]] or dirty[p["b"]]}
        passing = {(int(min(p, q)), int(max(p, q))) for p, q, l in zip(x, y, want_lcs)
                   if kk[p] >= 5 and kk[q] >= 5 and 200 * int(l) >= 70 * (int(kk[p]) + int(kk[q]))}
        assert want == passing, side
