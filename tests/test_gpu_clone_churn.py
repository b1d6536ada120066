"""`tsm_clone_churn` / `Scanner.clone_churn` (docs/SPEC.md section 22) against the reference of tests/clone_churn_ref.py, every
output array of both sides, exact and blind: C1 as the old revision with a step of edits, pastes, one-copy fixes, deletions and
renames at n = 1, 5 and 10; pairs with -1 on either side, no pairs and every file in a pair; classes of 2, 32, 33, 4 097 and
100 000 fragments and a 60 000-line file copied; the raw ABI (argument checks, NULL outputs, exact and one-short caps) and a non-blocking
stream while the legacy stream is busy.  Each side's classes also equal tsm_clones / tsm_clones_blind of that revision alone."""
import ctypes as C
import os

import numpy as np
import pytest

import clone_churn_ref as cr
import corpus_util as cu
import orc_clones as oc
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BLIND_KEYS = ("kept_base", "kept_line", "blind_hash", "file_kept_assert")
TSM_OK, TSM_E_ARG, TSM_E_CAPACITY = 0, -1, -3             # include/tosemscan.h


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 17, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def c1():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    return list(files), np.asarray(exts, np.uint8)


def check(s, old, new, po, pn, n, blind=False, **kw):
    """The device against the reference, and each side's classes against clones() of its revision alone."""
    got = s.clone_churn(ts.pack(*old) if len(old[0]) else ts.pack([], np.zeros(0, np.uint8)),
                        ts.pack(*new) if len(new[0]) else ts.pack([], np.zeros(0, np.uint8)), po, pn, n, blind, **kw)
    cr.assert_equal(got, cr.churn(old, new, po, pn, n, blind), blind)
    for side, rev in (("old", old), ("new", new)):
        if len(rev[0]):
            alone = s.clones(ts.pack(*rev), n, blind=blind)
            for k in oc.KEYS + (BLIND_KEYS if blind else ()):
                assert np.array_equal(alone[k], got[side][k]), (side, k)
    return got


def step(files, exts, seed, n_edit=40, n_fix=10, n_paste=10, n_del=5, n_rename=20):
    """A step over (files, exts): gen_edit (lambda = 6) of n_edit files, one line changed inside a duplicated window of n_fix files
    (a one-copy fix), n_paste files pasted into new files, n_del files deleted, n_rename unchanged files paired under a new index;
    the new revision's files in a shuffled order.  Returns (old, new, pair_old, pair_new)."""
    rng = np.random.default_rng(seed)
    nf = len(files)
    idx = rng.permutation(nf)
    edit, fix = idx[:n_edit], idx[n_edit:n_edit + n_fix]
    dele = set(int(i) for i in idx[n_edit + n_fix:n_edit + n_fix + n_del])
    ren = idx[n_edit + n_fix + n_del:n_edit + n_fix + n_del + n_rename]
    paste = idx[-n_paste:] if n_paste else []
    new = list(files)
    for i in edit:
        new[i] = ts.gen_edit(seed + int(i), files[i], 6.0)
    for i in fix:
        lines = files[i].split(b"\n")
        k = int(rng.integers(0, max(len(lines) - 1, 1)))
        lines[k] = lines[k] + b"  # fixed"
        new[i] = b"\n".join(lines)
    keep = [i for i in range(nf) if i not in dele]
    order = [keep[j] for j in rng.permutation(len(keep))]
    new_files = [new[i] for i in order] + [files[i] for i in paste]
    new_exts = np.concatenate([exts[order], exts[list(paste)]]).astype(np.uint8) if len(order) + len(paste) else np.zeros(0, np.uint8)
    at = {old_i: j for j, old_i in enumerate(order)}
    po, pn = [], []
    for i in list(edit) + list(fix) + list(ren):
        po.append(int(i)); pn.append(at[int(i)])
    for i in dele:
        po.append(i); pn.append(-1)
    for j in range(len(paste)):
        po.append(-1); pn.append(len(order) + j)
    perm = rng.permutation(len(po))
    return (files, exts), (new_files, new_exts), [po[k] for k in perm], [pn[k] for k in perm]


@pytest.mark.parametrize("blind", [False, True])
@pytest.mark.parametrize("n", [1, 5, 10])
def test_c1_step(scanner, c1, n, blind):
    old, new, po, pn = step(*c1, seed=22 + n)
    got = check(scanner, old, new, po, pn, n, blind)
    touched = [int((got[s]["status"] > 0).sum()) for s in ("old", "new")]
    assert touched[0] > 0 and touched[1] > 0
    ms = scanner.clone_churn_last_ms()
    assert len(ms) == 4 and all(m > 0 for m in ms)


def test_no_pairs_touches_nothing(scanner, c1):
    files, exts = c1
    got = check(scanner, (files[:500], exts[:500]), (files[500:900], exts[500:900]), [], [], 5)
    for s in ("old", "new"):
        assert len(got[s]["status"]) > 0 and not got[s]["status"].any() and not got[s]["changed"].any()


def test_every_file_in_a_pair_and_empty_sides(scanner, c1):
    files, exts = c1
    old, new = (files[:300], exts[:300]), (files[300:500], exts[300:500])
    rng = np.random.default_rng(5)
    po = list(rng.permutation(300)) + []
    pn = list(rng.permutation(200)) + [-1] * 100
    check(scanner, old, new, [int(x) for x in po], [int(x) for x in pn], 5)
    check(scanner, old, new, [int(x) for x in po], [int(x) for x in pn], 5, blind=True)
    empty = ([], np.zeros(0, np.uint8))
    got = check(scanner, empty, new, [-1] * 200, list(range(200)), 5)
    assert set(got["new"]["status"]) <= {0, 5}
    got = check(scanner, old, empty, list(range(300)), [-1] * 300, 5, blind=True)
    assert set(got["old"]["status"]) <= {0, 2}


def wide(k, tag):
    """k files that each hold one 6-line block X between unique lines: one class of k fragments at n = 5."""
    X = [b"    self.assertEqual(f(%d), %d)" % (j, j * j) for j in range(6)]
    return [b"".join(x + b"\n" for x in [b"def test_%s_%d():" % (tag, i)] + X + [b"    u_%s_%d = 0" % (tag, i)]) for i in range(k)]


@pytest.mark.parametrize("k", [2, 32, 33, 4097])
def test_class_sizes(scanner, k):
    files = wide(k, b"w")
    exts = np.ones(k, np.uint8)
    rng = np.random.default_rng(k)
    new = list(files)
    fixed = sorted(int(i) for i in rng.choice(k, size=max(1, k // 3), replace=False))
    for i in fixed:
        new[i] = new[i].replace(b"f(2), 4", b"f(2), 5")
    dele = [i for i in range(k) if i not in fixed][: max(1, k // 5)] if k > 2 else []
    keep = [i for i in range(k) if i not in dele]
    new_files = [new[i] for i in keep] + wide(3, b"p")
    po = fixed + dele + [-1] * 3
    pn = [keep.index(i) for i in fixed] + [-1] * len(dele) + [len(keep), len(keep) + 1, len(keep) + 2]
    for blind in (False, True):
        got = check(scanner, (files, exts), (new_files, np.ones(len(new_files), np.uint8)), po, pn, 5, blind)
        if not blind:                                         # (blind, the block's six lines are one form: windows overlap)
            big = int(np.argmax(np.diff(got["old"]["class_base"])))
            assert got["old"]["class_counts"][big].sum() == k


def test_class_of_100000_fragments(scanner):
    k = 100000
    files = wide(k, b"h")
    new = list(files)
    for i in (0, 77, 50000, k - 1):                           # one-copy fixes
        new[i] = new[i].replace(b"f(2), 4", b"f(2), 5")
    po = pn = [0, 77, 50000, k - 1]
    got = check(scanner, (files, np.ones(k, np.uint8)), (new, np.ones(k, np.uint8)), po, pn, 5)
    big = int(np.argmax(np.diff(got["old"]["class_base"])))
    assert list(got["old"]["class_counts"][big]) == [k - 4, 4, 0] and got["old"]["status"][big] == 3


def test_60000_line_file_copied(scanner):
    F = b"".join(b"x%d = g(%d)\n" % (i, i * 7) for i in range(60000))
    old = ([F, b"y = 1\n"], np.array([1, 1], np.uint8))
    new = ([F, b"y = 1\n", F], np.array([1, 1, 1], np.uint8))
    got = check(scanner, old, new, [-1], [2], 5)
    assert list(got["new"]["status"]) == [6] and list(got["new"]["class_len"]) == [60000]
    assert list(got["new"]["state"]) == [0, 2]


# ------------------------------------------------------------------------------------------------------------- the raw ABI
def side(n_files, cc, cm, ck, blind, arrays):
    a = {"line_base": np.zeros(n_files + 1, np.int64), "file_dup": np.zeros(max(n_files, 1), np.uint32),
         "file_dup_assert": np.zeros(max(n_files, 1), np.uint32), "class_base": np.zeros(cc + 1, np.int64),
         "class_len": np.zeros(max(cc, 1), np.uint32), "member": np.zeros(max(cm, 1), np.int64), "changed": np.zeros(max(cm, 1), np.uint32),
         "changed_assert": np.zeros(max(cm, 1), np.uint32), "state": np.zeros(max(cm, 1), np.uint8),
         "class_counts": np.zeros((max(cc, 1), 3), np.uint32), "status": np.zeros(max(cc, 1), np.uint8),
         "kept_base": np.zeros(n_files + 1, np.int64), "kept_line": np.zeros(max(ck, 1), np.int64),
         "blind_hash": np.zeros(max(ck, 1), np.uint64), "file_kept_assert": np.zeros(max(n_files, 1), np.uint32)}
    p = (lambda k: ts._p(a[k]) if arrays else None)
    cr_ = ts._CloneResult(p("line_base"), p("file_dup"), p("file_dup_assert"), p("class_base"), p("class_len"), cc, 0, p("member"), cm, 0)
    br = ts._BlindResult(p("kept_base"), p("kept_line"), p("blind_hash"), p("file_kept_assert"), ck, 0)
    return ts._CloneChurnSide(cr_, br, p("changed"), p("changed_assert"), p("state"), p("class_counts"), p("status")), a


def raw(s, old, new, po, pn, n, blind, caps, arrays=True):
    ko, kn = ts.pack(*old), ts.pack(*new)                  # (kept alive: the structs point into their arenas)
    a, b = ko.c_struct(), kn.c_struct()
    po = np.ascontiguousarray(po, np.int32)
    pn = np.ascontiguousarray(pn, np.int32)
    so, ao = side(len(old[0]), *caps[0], blind, arrays)
    sn, an = side(len(new[0]), *caps[1], blind, arrays)
    rc = ts.lib().tsm_clone_churn(s._ctx, C.byref(a), C.byref(b), ts._p(po) if po.size else None, ts._p(pn) if pn.size else None, po.size,
                                  n, int(blind), C.byref(so), C.byref(sn), None)
    return rc, (so, ao), (sn, an)


def counts(sd, blind):
    return (sd.clones.n_classes, sd.clones.n_members) + ((sd.blind.n_kept,) if blind else ())


@pytest.mark.parametrize("blind", [False, True])
def test_abi_caps_and_null_outputs(scanner, blind):
    files = wide(40, b"a")
    ex = np.ones(40, np.uint8)
    new = [f.replace(b"f(3), 9", b"f(3), 8") if i % 4 == 0 else f for i, f in enumerate(files)]
    old_r, new_r = (files, ex), (new, ex)
    po = pn = list(range(0, 40, 4))
    want = scanner.clone_churn(ts.pack(*old_r), ts.pack(*new_r), po, pn, 5, blind)
    need = [(len(want[s]["class_len"]), len(want[s]["member"]), len(want[s]["kept_line"]) if blind else 0) for s in ("old", "new")]
    rc, (so, _), (sn, _) = raw(scanner, old_r, new_r, po, pn, 5, blind, [(0, 0, 0), (0, 0, 0)], arrays=False)
    assert rc == TSM_OK and counts(so, blind) == need[0][:2 + blind] and counts(sn, blind) == need[1][:2 + blind]
    rc, (so, ao), (sn, an) = raw(scanner, old_r, new_r, po, pn, 5, blind, need)
    assert rc == TSM_OK
    for sd, a, w in ((so, ao, want["old"]), (sn, an, want["new"])):
        nc, nm = sd.clones.n_classes, sd.clones.n_members
        for k, m in (("changed", nm), ("changed_assert", nm), ("state", nm), ("class_counts", nc), ("status", nc), ("member", nm)):
            assert np.array_equal(a[k][:m], w[k]), k
    for which in range(3):
        for s_i in range(2):
            caps = [list(c) for c in need]
            if caps[s_i][which] == 0:
                continue
            caps[s_i][which] -= 1
            if which == 2 and not blind:
                continue
            rc, (so, _), (sn, _) = raw(scanner, old_r, new_r, po, pn, 5, blind, caps)
            assert rc == TSM_E_CAPACITY, (which, s_i)
            assert counts(so, blind) == need[0][:2 + blind] and counts(sn, blind) == need[1][:2 + blind]


def test_abi_arguments(scanner):
    files = wide(4, b"a")
    ex = np.ones(4, np.uint8)
    r = (files, ex)
    caps = [(0, 0, 0), (0, 0, 0)]
    for n in (0, 1025):
        assert raw(scanner, r, r, [0], [0], n, False, caps)[0] == TSM_E_ARG
    for po, pn in (([4], [0]), ([0], [4]), ([-2], [0]), ([0, 0], [0, 1]), ([0, 1], [2, 2]), ([-1], [-1])):
        assert raw(scanner, r, r, po, pn, 5, False, caps)[0] == TSM_E_ARG, (po, pn)
    k = ts.pack(*r)
    a = k.c_struct()
    so, _ = side(4, 0, 0, 0, False, False)
    assert ts.lib().tsm_clone_churn(scanner._ctx, C.byref(a), C.byref(a), None, None, 0, 5, 0, C.byref(so), None, None) == TSM_E_ARG
    assert ts.lib().tsm_clone_churn(scanner._ctx, C.byref(a), C.byref(a), None, None, 1, 5, 0, C.byref(so), C.byref(so), None) == TSM_E_ARG
    assert raw(scanner, r, r, [], [], 1024, False, caps)[0] == TSM_OK


def test_nonblocking_stream_with_the_legacy_stream_busy(scanner, c1):
    torch = pytest.importorskip("torch")
    old, new, po, pn = step(c1[0][:2000], c1[1][:2000], seed=9)
    first = check(scanner, old, new, po, pn, 5, True)
    s = torch.cuda.Stream()
    legacy = torch.cuda.default_stream()
    with torch.cuda.stream(legacy):
        torch.cuda._sleep(50_000_000)                                  # a bounded spin (well under a second)
    got = scanner.clone_churn(ts.pack(*old), ts.pack(*new), po, pn, 5, True, stream=C.c_void_p(s.cuda_stream))
    legacy.synchronize()
    s.synchronize()
    cr.assert_equal(got, first, True)
