"""`tsm_link_churn` / `Scanner.link_churn` (docs/SPEC.md section 28) against the restatement of tests/link_churn_ref.py: every
array of both sides and every event on the worked examples, the CJ example and the known limits; each side's links equal
tsm_test_links of that revision alone; an 8 000-file planted history with production-only, test-only and mixed steps; C1 with a
scripted step (no production files: no links, so no rows); fuzz pairs with long lines and binary bytes; production pairs at
every k_diff_small size and left over to k_myers_trace; untraced pairs at distances 23 169 and 23 170 (and a traced 23 168)
with definitions in their middle; one definition called by
100 000 tests and then deleted (more tests than the launch has warps); no pairs and empty revisions; the raw ABI (argument
errors, NULL outputs, exact and one-short caps) and a busy legacy stream."""
import ctypes as C
import os

import numpy as np
import pytest

import corpus_util as cu
import link_churn_ref as ref
import smell_churn_ref as scr
import link_ref as lr
import test_link_churn_ref as ex
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TSM_OK, TSM_E_ARG, TSM_E_CAPACITY = 0, -1, -3             # include/tosemscan.h


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 26, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


def packed(rev):
    files, exts = rev[0], rev[1]
    return ts.pack(list(files), np.asarray(exts, np.uint8)) if len(files) else ts.pack([], np.zeros(0, np.uint8))


def check(s, old, new, po, pn, alone=True):
    got = s.link_churn(packed(old), packed(new), old[2], new[2], po, pn, old[3], new[3])
    ref.assert_equal(got, ref.churn(old, new, po, pn))
    for side, rev in (("old", old), ("new", new)):
        if alone and len(rev[0]):
            want = s.test_links(packed(rev), rev[2], rev[3])
            for k in ("tests", "links", "defs"):
                assert np.array_equal(want[k].view(np.uint8), got[side][k].view(np.uint8)), (side, k)
    return got


def check_step(s, old, new, renames=None):
    (a, _), (b, _) = ex.rev(old), ex.rev(new)
    po, pn = ex.pairs(old, new, renames)
    return check(s, a, b, po, pn)


def test_worked_examples_and_limits(scanner):
    for k in range(1, len(ex.REVS)):
        check_step(scanner, ex.REVS[k - 1], ex.REVS[k])
    check_step(scanner, ex.REVS[4], ex.REVS[5], {"tests/test_calc.py": "tests/test_math.py"})
    got = check_step(scanner, ex.CJ_OLD, ex.CJ_NEW)
    assert [(ref.EVENTS[int(e["event"])], chr(got["new"]["change"][e["test"]])) for e in got["events"]] == [("redefined", "=")]
    q = b'"' * 3
    for new in ({"calc.py": ex.CALC.replace(b"return a + b", b"return b + a")},
                {"calc.py": b"def sub(a, b):\n    return a - b\n\n\ndef add(a, b):\n    return a + b\n"},
                {"tests/test_calc.py": ex.TEST.replace(b"    def test_sub", b"    x = " + q + b"a\n    def test_sub")},
                {"ops.py": ex.OPS}, {"calc.py": ex.CALC.replace(b"\n", b"\r\n")},
                {"tests/test_calc.py": ex.TEST1.rstrip(b"\n"), "calc.py": ex.CALC.rstrip(b"\n")}):
        check_step(scanner, ex.REVS[0], dict(ex.REVS[0], **new))
    check_step(scanner, ex.REVS[0], {"calc.py": ex.CALC, "calc_helpers.py": ex.TEST}, {"tests/test_calc.py": "calc_helpers.py"})


def test_planted_history(scanner):
    hist = ex.planted_history(11, 8000, 3, n_edit=60)
    kinds = set()
    for k in range(1, len(hist)):
        (a, pa), (b, pb) = ex.rev(hist[k - 1]), ex.rev(hist[k])
        po, pn = ex.pairs(hist[k - 1], hist[k])
        kinds.add(tuple(sorted({bool(lr.is_test_path(pa[f] if f >= 0 else pb[g])) for f, g in zip(po, pn)})))
        got = check(scanner, a, b, po, pn, alone=k == 1)
        assert len(got["events"]) > 0
    assert kinds == {(False,), (True,), (False, True)}       # production-only, test-only and mixed steps


def test_c1_scripted_step(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    keep = [i for i, (f, e) in enumerate(zip(files, exts)) if int(e) == 1 and 200 < len(f) < 6000][:80]
    files, exts = [files[i] for i in keep], np.asarray([exts[i] for i in keep], np.uint8)
    role = np.ones(len(files), np.uint8)
    stem = np.full(len(files), -1, np.int32)
    new = list(files)
    po, pn = [], []
    for f in range(0, len(files), 5):
        new[f] = files[f].replace(b"(self):", b"(self, tmp_path):", 1)
        po.append(f); pn.append(f)
    new.append(files[1] + b"\ndef test_extra():\n    assert helper(1)\n")
    po.append(-1); pn.append(len(new) - 1)
    got = check(scanner, (files, exts, role, stem), (new, np.append(exts, 1), np.append(role, 1), np.append(stem, -1)), po, pn)
    assert len(got["events"]) == 0 and len(got["new"]["links"]) == 0 and b"A" in bytes(got["new"]["change"])


def test_fuzz_pairs_long_lines_and_binary(scanner):
    rng = np.random.default_rng(5)
    old = {"calc.py": ex.CALC + b"x = '" + b"y" * 70000 + b"'\n", "tests/test_calc.py": ex.TEST,
           "blob.py": rng.integers(0, 256, 5000, np.uint8).tobytes()}
    new = {"calc.py": b"def add(a, b):  # " + b"z" * 90000 + b"\n" + ex.CALC[15:],
           "tests/test_calc.py": ex.TEST1 + b"\x00\xff(add(\n", "blob.py": rng.integers(0, 256, 5000, np.uint8).tobytes()}
    check_step(scanner, old, new)
    for seed in range(4):
        edited = {p: ts.gen_edit(seed * 10 + i, d, 4.0) for i, (p, d) in enumerate(sorted(old.items()))}
        check_step(scanner, old, edited)


def test_every_diff_kernel(scanner):
    """Tie-heavy production pairs with definitions, at every k_diff_small size and left over to k_myers_trace, whose focal tests
    call those names: the targets move with the kept ranks of each script."""
    olds, news, _ = cu.tie_heavy_pairs(13)
    names = sorted({ln for o in olds for ln in o.splitlines(keepends=True)})
    sub = {ln: b"def f%d(a):\n" % i for i, ln in enumerate(names)}
    calls = b"".join(b"        f%d(1)\n" % i for i in range(len(names)))
    old, new = {}, {}
    for i, (o, n) in enumerate(zip(olds, news)):
        old["m%d.py" % i] = b"".join(sub[ln] for ln in o.splitlines(keepends=True))
        new["m%d.py" % i] = b"".join(sub.get(ln, b"x = 0\n") for ln in n.splitlines(keepends=True))
        old["tests/test_m%d.py" % i] = new["tests/test_m%d.py" % i] = b"class T(unittest.TestCase):\n    def test_a(self):\n" + calls
    d = [sum(scr.sr.py_diff_files(old["m%d.py" % i], new["m%d.py" % i], 1, 1)[:2]) for i in range(len(olds))]
    assert max(d) > 127 and any(0 < x <= 31 for x in d)
    got = check_step(scanner, old, new)
    assert sum(int(e["event"]) == ref.REDEFINED for e in got["events"]) > 0


def untraced_step(d):
    """A production file whose script has d edits split around `def mid(a):`; `def first` and `def last` are its common prefix and
    suffix.  Returns (old, new, the script of the pair as smell_churn_ref.py_script_lines gives it)."""
    ko = d // 2
    ka, kb = ko // 2, ko - ko // 2
    old = [b"def first(a):"] + [b"o%d = 0" % j for j in range(ka)] + [b"def mid(a):"] + [b"p%d = 0" % j for j in range(kb)] + [b"def last(a):"]
    new = ([b"def first(a):"] + [b"n%d = 0" % j for j in range(ka)] + [b"def mid(a):"] + [b"q%d = 0" % j for j in range(kb)] +
           ([b"extra = 1"] if d % 2 else []) + [b"def last(a):"])
    n_old, n_new = len(old), len(new)
    if d > 23168:                                              # untraced: the whole middle
        deleted, inserted = set(range(1, n_old - 1)), set(range(1, n_new - 1))
    else:
        deleted = set(range(1, n_old - 1)) - {1 + ka}
        inserted = set(range(1, n_new - 1)) - {1 + ka}
    corr = dict(zip([j for j in range(n_new) if j not in inserted], [i for i in range(n_old) if i not in deleted]))
    assert len(deleted) + len(inserted) >= d - (2 if d <= 23168 else 0)
    test = b"def test_calc():\n    first(1)\n    mid(2)\n    last(3)\n"
    return ({"calc.py": b"\n".join(old) + b"\n", "tests/test_calc.py": test},
            {"calc.py": b"\n".join(new) + b"\n", "tests/test_calc.py": test}, (deleted, inserted, corr))


@pytest.mark.parametrize("d", [23168, 23169, 23170])
def test_untraced_distances(scanner, monkeypatch, d):
    old, new, script = untraced_step(d)
    monkeypatch.setattr(scr, "py_script_lines", lambda *a: script)   # (the script is known by construction)
    got = check_step(scanner, old, new)
    want = [] if d <= 23168 else [("redefined", "mid")]
    (_, _), (b, _) = ex.rev(old), ex.rev(new)
    names = []
    for e in got["events"]:
        df = got["new"]["defs"][int(got["new"]["links"][int(e["link"])]["name_def"])]
        names.append((ref.EVENTS[int(e["event"])], b[0][int(df["file"])][int(df["name_off"]):int(df["name_off"]) + int(df["name_len"])].decode()))
    assert names == want


def test_definition_called_by_100k_tests(scanner):
    n = 100000
    test = b"".join(b"def test_%d():\n    f(%d)\n" % (i, i) for i in range(n))
    old = ([b"def f(a):\n    return a\n", test], np.array([1, 1], np.uint8), np.array([0, 1], np.uint8), np.array([0, 0], np.int32))
    new = ([b"def g(a):\n    return a\n", test], old[1], old[2], old[3])
    got = scanner.link_churn(packed(old), packed(new), old[2], new[2], [0], [0], old[3], new[3])
    ev = got["events"]
    assert len(ev) == 2 * n
    assert bytes(got["new"]["change"]) == b"=" * n
    lazy, rem = ev[0::2], ev[1::2]
    assert (lazy["event"] == 7).all() and (rem["event"] == 1).all() and (rem["cause"] == 2).all()
    assert (rem["test"] == np.arange(n)).all() and (rem["old_calls"] == 1).all() and (rem["calls"] == 1).all()
    assert (rem["defs"] == 0).all() and (rem["old_defs"] == 1).all()


def test_no_pairs_and_empty_revisions(scanner):
    (a, _), = [ex.rev(ex.REVS[1])]
    got = check(scanner, a, a, [], [])
    assert len(got["events"]) == 0 and bytes(got["new"]["change"]) == b"=="
    n = len(a[0])
    empty = ([], np.zeros(0, np.uint8), np.zeros(0, np.uint8), np.zeros(0, np.int32))
    assert len(check(scanner, empty, a, [-1] * n, list(range(n)))["events"]) > 0
    assert len(check(scanner, a, empty, list(range(n)), [-1] * n)["events"]) > 0
    check(scanner, empty, empty, [], [])
    blank = ([b"", b""], np.ones(2, np.uint8), np.array([0, 1], np.uint8), np.array([0, 0], np.int32))
    check(scanner, blank, a, [0, 1], [0, 1])


def test_abi(scanner):
    L = ts.lib()
    (a, _), (b, _) = ex.rev(ex.REVS[0]), ex.rev(ex.REVS[1])
    ka, kb = packed(a), packed(b)
    cs = [ka.c_struct(), kb.c_struct()]
    n = C.c_int64(-7)
    role = [np.ascontiguousarray(a[2]), np.ascontiguousarray(b[2])]
    stem = [np.ascontiguousarray(a[3]), np.ascontiguousarray(b[3])]

    def call(po=(1,), pn=(1,), cap=64, ev_cap=64, roles=None, stems=None, kn=None, null=()):
        po, pn = np.asarray(po, np.int32), np.asarray(pn, np.int32)
        roles = roles or role
        stems = stems or stem
        sides, keep = [], []
        for _ in range(2):
            o = {"tests": np.zeros(cap + 1, ts.LINK_TEST), "links": np.zeros(cap + 1, ts.LINK), "defs": np.zeros(cap + 1, ts.LINK_DEF),
                 "match": np.zeros(cap + 1, np.int32), "change": np.zeros(cap + 1, np.uint8)}
            keep.append(o)
            p = {k: None if k in null else ts._p(v) for k, v in o.items()}
            r = ts._LinksResult(tests=p["tests"], test_cap=cap, links=p["links"], link_cap=cap, defs=p["defs"], def_cap=cap)
            sides.append(ts._LinkChurnSide(r, p["match"], p["change"]))
        ev = np.zeros(ev_cap + 1, ts.LINK_EVENT)
        rc = L.tsm_link_churn(scanner._ctx, C.byref(cs[0]), C.byref(kn or cs[1]), ts._p(roles[0]), ts._p(stems[0]), ts._p(roles[1]),
                              ts._p(stems[1]), ts._p(po), ts._p(pn), po.size, C.byref(sides[0]), C.byref(sides[1]),
                              None if "events" in null else ts._p(ev), ev_cap, C.byref(n), None)
        return rc, sides, ev
    rc, sides, ev = call()
    assert rc == TSM_OK
    ne, nt, nk, nd = n.value, sides[1].links.n_tests, sides[1].links.n_links, sides[1].links.n_defs
    assert ne == 4 and nt == 2 and nk == 3 and nd == 2
    assert call(ev_cap=ne)[0] == TSM_OK
    assert call(ev_cap=ne - 1)[0] == TSM_E_CAPACITY and n.value == ne
    assert call(cap=nk)[0] == TSM_OK
    rc, sides, _ = call(cap=nk - 1)
    assert rc == TSM_E_CAPACITY and sides[1].links.n_links == nk and n.value == ne
    for out in ("tests", "links", "defs", "match", "change", "events"):
        null = {"tests", "links", "defs", "match", "change", "events"} - {out}
        assert call(cap=0, ev_cap=0, null=null)[0] == TSM_E_CAPACITY
        assert call(null=null | {out}, cap=0, ev_cap=0)[0] == TSM_OK and n.value == ne
    assert call(po=(1, 1), pn=(0, 1))[0] == TSM_E_ARG          # a file in two pairs
    assert call(po=(2,), pn=(1,))[0] == TSM_E_ARG              # out of range
    assert call(po=(-1,), pn=(-1,))[0] == TSM_E_ARG            # (-1, -1)
    assert call(po=(1,), pn=(-1,))[0] == TSM_E_ARG             # unpaired counts differ
    assert call(po=(), pn=())[0] == TSM_E_ARG                  # test files of other lengths unpaired
    assert call(roles=[role[0], np.array([1, 1], np.uint8)])[0] == TSM_E_ARG   # an unpaired file of another role
    assert call(stems=[stem[0], np.array([0, -2], np.int32)])[0] == TSM_E_ARG
    rc = L.tsm_link_churn(scanner._ctx, C.byref(cs[0]), C.byref(cs[1]), None, None, ts._p(role[1]), None, None, None, 0,
                          C.byref(ts._LinkChurnSide()), C.byref(ts._LinkChurnSide()), None, 0, C.byref(n), None)
    assert rc == TSM_E_ARG                                     # a NULL role
    lines = [(["a = 1\nb = 2\n", "def test_x():\n    a(1)\n"], ["a = 1 b = 2\n", "def test_x():\n    a(1)\n"])]
    for o, w in lines:                                         # an unpaired file of equal bytes but other line count
        ro = ([x.encode() for x in o], np.ones(2, np.uint8), np.array([0, 1], np.uint8), np.array([0, 0], np.int32))
        rw = ([x.encode() for x in w], ro[1], ro[2], ro[3])
        assert len(ro[0][0]) == len(rw[0][0])
        with pytest.raises(ts.TsmError) as err:
            scanner.link_churn(packed(ro), packed(rw), ro[2], rw[2], [], [], ro[3], rw[3])
        assert err.value.status == TSM_E_ARG


def test_busy_legacy_stream_and_repeats(scanner):
    torch = pytest.importorskip("torch")
    (a, _), (b, _) = ex.rev(ex.REVS[0]), ex.rev(ex.REVS[1])
    po, pn = ex.pairs(ex.REVS[0], ex.REVS[1])
    want = ref.churn(a, b, po, pn)
    x = torch.ones(1 << 24, device="cuda")
    s = torch.cuda.Stream()
    for _ in range(3):
        y = x * 2                                             # keeps the legacy stream busy
        ref.assert_equal(scanner.link_churn(packed(a), packed(b), a[2], b[2], po, pn, a[3], b[3], stream=C.c_void_p(s.cuda_stream)), want)
    torch.cuda.synchronize()
    assert float(y[0]) == 2.0
