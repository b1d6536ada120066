"""`tsm_similar_churn` / `Scanner.similar_churn` (docs/SPEC.md section 24) against the reference of tests/similar_churn_ref.py,
every array of both sides and every event: the worked examples, C1 test files with a scripted step (pastes with edits, one-copy
fixes, deletions, renames, name-matched headers) at (5, 70), (10, 90) and (1, 50), no pairs, every file in a pair and empty
revisions.  Each side's tests equal tsm_smells of its revision alone, its pairs with a dirty test equal tsm_similar_tests of
that revision filtered by change, and with every test dirty n_candidates equals tsm_similar_tests'.  The raw ABI: argument
errors, NULL outputs, exact and one-short caps."""
import ctypes as C
import os

import numpy as np
import pytest

import corpus_util as cu
import similar_churn_ref as ref
import test_similar_churn_ref as ex
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TSM_OK, TSM_E_ARG, TSM_E_CAPACITY = 0, -1, -3             # include/tosemscan.h


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 26, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def c1():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    keep = [i for i, (f, e) in enumerate(zip(files, exts)) if int(e) == 1 and 200 < len(f) < 6000][:60]
    return [files[i] for i in keep], np.asarray([exts[i] for i in keep], np.uint8)


def packed(files, exts):
    return ts.pack(list(files), np.asarray(exts, np.uint8)) if len(files) else ts.pack([], np.zeros(0, np.uint8))


def check(s, old, new, po, pn, ml=5, P=70):
    got = s.similar_churn(packed(*old), packed(*new), po, pn, ml, P)
    ref.assert_equal(got, ref.churn(old, new, po, pn, ml, P))
    for side, rev in (("old", old), ("new", new)):
        if not len(rev[0]):
            assert len(got[side]["tests"]) == 0
            continue
        alone = s.smells(packed(*rev))["tests"]
        assert np.array_equal(alone.view(np.uint8), got[side]["tests"].view(np.uint8)), side
        st = s.similar_tests(packed(*rev), ml, P)
        dirty = got[side]["change"] != ord("=")
        want = {(int(p["a"]), int(p["b"])) for p in st["pairs"] if dirty[p["a"]] or dirty[p["b"]]}
        kk = got[side]["test_kept"].astype(np.int64)
        a, b, lcs = ("old_a", "old_b", "old_lcs") if side == "old" else ("a", "b", "lcs")
        passing = {(int(min(e[a], e[b])), int(max(e[a], e[b]))) for e in got["events"] if e[lcs] != ref.NONE and
                   kk[e[a]] >= ml and kk[e[b]] >= ml and 200 * int(e[lcs]) >= P * (kk[e[a]] + kk[e[b]])}
        assert want == passing, side                       # the side's pairs with a dirty test: the events that pass there
        if dirty.all():
            assert got[side]["n_candidates"] == st["n_candidates"]
    return got


def test_worked_examples(scanner):
    for i in range(len(ex.R) - 1):
        check(scanner, ([ex.R[i]], [1]), ([ex.R[i + 1]], [1]), [0], [0])
    other = ex.py(ex.A.replace(b"test_add", b"test_sub"))
    check(scanner, ([ex.R[1]], [1]), ([ex.R[1], other], [1, 1]), [-1], [1])
    check(scanner, ([ex.R[1], other], [1, 1]), ([ex.R[1]], [1]), [1], [-1])
    check(scanner, ([ex.R[1]], [1]), ([ex.R[1]], [2]), [0], [0])
    new = ex.py(ex.A.replace(b"def test_add(self):", b"def test_add(self, tmp_path):"), ex.B)
    check(scanner, ([ex.R[1]], [1]), ([new], [1]), [0], [0])
    old = ex.HEAD + b"\n" + ex.A + b"\n" + b"\n" + ex.B        # a docstring opened above A: its sequence changes, no body line marked
    new = ex.HEAD + b'    """\n' + ex.A + b'    """\n' + b"\n" + ex.B
    assert check(scanner, ([old], [1]), ([new], [1]), [0], [0])["new"]["change"][0] == ord("M")


def scripted(files, exts, seed):
    """A step over C1 files: test bodies pasted into a new file with one line changed, one-copy fixes (a literal), line
    deletions, a rename of a file with a header change, a deleted file; the rest unchanged.  Returns old, new, po, pn."""
    rng = np.random.default_rng(seed)
    nf = len(files)
    idx = [int(i) for i in rng.permutation(nf)]
    fix, cut, ren, dele, src = idx[:6], idx[6:10], idx[10:14], idx[14:16], idx[16:22]
    new_files, new_exts, po, pn = [], [], [], []
    for f in range(nf):
        if f in dele:
            po.append(f); pn.append(-1)
            continue
        data = files[f]
        if f in fix:
            data = data.replace(b"1", b"2", 1)
        elif f in cut:
            lines = data.split(b"\n")
            del lines[len(lines) // 2]
            data = b"\n".join(lines)
        elif f in ren:
            data = data.replace(b"(self):", b"(self, tmp_path):", 1)
        new_files.append(data)
        new_exts.append(exts[f])
        if f in fix or f in cut or f in ren:
            po.append(f); pn.append(len(new_files) - 1)
    for f in src:                                             # pasted copies: the file again with one line changed
        lines = files[f].split(b"\n")
        k = int(rng.integers(0, len(lines)))
        lines[k] = lines[k] + b"  # pasted"
        lines.insert(k, b"    x = 1")
        new_files.append(b"\n".join(lines))
        new_exts.append(1)
        po.append(-1); pn.append(len(new_files) - 1)
    return (files, exts), (new_files, np.asarray(new_exts, np.uint8)), po, pn


@pytest.mark.parametrize("ml,P", [(5, 70), (10, 90), (1, 50)])
def test_c1_scripted_step(scanner, c1, ml, P):
    old, new, po, pn = scripted(*c1, seed=ml * 100 + P)
    got = check(scanner, old, new, po, pn, ml, P)
    assert len(got["events"]) > 0


def test_no_pairs_every_pair_and_empty(scanner, c1):
    files, exts = c1[0][:30], c1[1][:30]
    got = check(scanner, (files, exts), (files, exts), [], [])
    assert len(got["events"]) == 0 and got["old"]["n_candidates"] == 0 and got["new"]["n_candidates"] == 0
    n = len(files)
    check(scanner, (files, exts), (files, exts), list(range(n)), list(range(n)))
    check(scanner, ([], []), (files, exts), [-1] * n, list(range(n)))
    check(scanner, (files, exts), ([], []), list(range(n)), [-1] * n)
    check(scanner, ([], []), ([], []), [], [])


def test_all_dirty_candidates_equal_similar_tests(scanner, c1):
    files, exts = c1
    got = scanner.similar_churn(packed([], []), packed(files, exts), [-1] * len(files), list(range(len(files))))
    st = scanner.similar_tests(packed(files, exts))
    assert got["new"]["n_candidates"] == st["n_candidates"]
    assert sorted((int(e["a"]), int(e["b"])) for e in got["events"]) == [(int(p["a"]), int(p["b"])) for p in st["pairs"]]


def test_abi(scanner):
    L = ts.lib()
    old, new = packed([ex.R[0]], [1]), packed([ex.R[1], ex.R[0]], [1, 1])
    cs = [old.c_struct(), new.c_struct()]
    po, pn = np.array([0], np.int32), np.array([0], np.int32)
    n = C.c_int64(-7)

    def call(po=po, pn=pn, cap=64, ev_cap=64, ml=5, P=70, k=None):
        outs = [{"tests": np.zeros(cap + 1, ts.SMELL_TEST), "kept": np.zeros(cap + 1, np.uint32), "match": np.zeros(cap + 1, np.int32),
                 "change": np.zeros(cap + 1, np.uint8)} for _ in range(2)]
        sides = [ts._SimilarChurnSide(*[ts._p(o[x]) for x in ("tests", "kept", "match", "change")], cap, -1, -1) for o in outs]
        ev = np.zeros(ev_cap + 1, ts.SIMILAR_EVENT)
        rc = L.tsm_similar_churn(scanner._ctx, C.byref(cs[0]), C.byref(k or cs[1]), ts._p(po), ts._p(pn), po.size, ml, P,
                                 C.byref(sides[0]), C.byref(sides[1]), ts._p(ev), ev_cap, C.byref(n), None)
        return rc, sides
    rc, _ = call()                                             # unpaired: none in old, R[0] in new: counts differ
    assert rc == TSM_E_ARG
    po2, pn2 = np.array([0], np.int32), np.array([1], np.int32)   # unpaired: none in old, R[1] in new
    assert call(po2, pn2)[0] == TSM_E_ARG
    kp = packed([ex.R[2]], [1])                               # no pairs: R[0] and R[2] unpaired, of different lengths
    k1 = kp.c_struct()
    assert call(np.zeros(0, np.int32), np.zeros(0, np.int32), k=k1)[0] == TSM_E_ARG
    assert call(ml=0)[0] == TSM_E_ARG and call(P=0)[0] == TSM_E_ARG and call(P=101)[0] == TSM_E_ARG
    assert call(np.array([-1], np.int32), np.array([-1], np.int32))[0] == TSM_E_ARG
    good_po, good_pn = np.array([0, -1], np.int32), np.array([0, 1], np.int32)
    rc, sides = call(good_po, good_pn)
    assert rc == TSM_OK
    ne, nt = n.value, sides[1].n_tests
    assert ne > 0 and nt == 3
    assert call(good_po, good_pn, ev_cap=ne)[0] == TSM_OK
    assert call(good_po, good_pn, ev_cap=ne - 1)[0] == TSM_E_CAPACITY and n.value == ne
    rc, sides = call(good_po, good_pn, cap=nt - 1)
    assert rc == TSM_E_CAPACITY and sides[1].n_tests == nt and n.value == ne
    sides = [ts._SimilarChurnSide(None, None, None, None, 0, 0, 0) for _ in range(2)]
    rc = L.tsm_similar_churn(scanner._ctx, C.byref(cs[0]), C.byref(cs[1]), ts._p(good_po), ts._p(good_pn), 2, 5, 70,
                             C.byref(sides[0]), C.byref(sides[1]), None, 0, C.byref(n), None)
    assert rc == TSM_OK and n.value == ne and sides[1].n_tests == nt


def test_busy_legacy_stream_and_repeats(scanner):
    torch = pytest.importorskip("torch")
    old, new = ([ex.R[2]], [1]), ([ex.R[4]], [1])
    want = ref.churn(old, new, [0], [0])
    a = torch.ones(1 << 24, device="cuda")
    s = torch.cuda.Stream()
    for _ in range(3):
        b = a * 2                                                 # keeps the legacy stream busy
        ref.assert_equal(scanner.similar_churn(packed(*old), packed(*new), [0], [0], stream=C.c_void_p(s.cuda_stream)), want)
    torch.cuda.synchronize()
    assert float(b[0]) == 2.0
