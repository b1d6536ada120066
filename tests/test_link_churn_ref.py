"""The plain-Python restatement of docs/SPEC.md section 28 (link_churn_ref) on the worked examples of the section, its CJ
example, every known limit, a role change through a rename, CRLF and unterminated last lines, the untraced rule with the trace
limit lowered, and a planted history of production and test edits (tsm_gen_edit: a host function, no GPU)."""
import numpy as np
import pytest

import case_ref as cr
import link_churn_ref as ref
import link_ref as lr
import tosemscan as ts

CALC = b"def add(a, b):\n    return a + b\n\n\ndef sub(a, b):\n    return a - b\n"
TEST = b"""import unittest
from calc import add, sub


class TestCalc(unittest.TestCase):
    def test_add(self):
        self.assertEqual(add(1, 2), 3)

    def test_sub(self):
        self.assertEqual(sub(3, 2), 1)
"""
TEST1 = TEST.replace(b"self.assertEqual(sub(3, 2), 1)", b"self.assertEqual(sub(3, 2), 1)\n        self.assertEqual(add(0, 1), 1)")
CALC2 = CALC.replace(b"def add(a, b):\n    return a + b", b"def add(a, b, c=0):\n    return a + b + c")
CALC3 = b"def add(a, b, c=0):\n    return a + b + c\n"
OPS = b"def add(x, y):\n    return x + y\n"
# the revisions of the worked examples: commit k turns REVS[k - 1] into REVS[k]
REVS = [
    {"calc.py": CALC, "tests/test_calc.py": TEST},
    {"calc.py": CALC, "tests/test_calc.py": TEST1},
    {"calc.py": CALC2, "tests/test_calc.py": TEST1},
    {"calc.py": CALC3, "tests/test_calc.py": TEST1},
    {"calc.py": CALC3, "ops.py": OPS, "tests/test_calc.py": TEST1},
    {"calc.py": CALC3, "ops.py": OPS, "tests/test_math.py": TEST1},
]
EXT = {".py": 1, ".cc": 2, ".java": 4, ".h": 6}


def ext_of(path):
    return next((e for s, e in EXT.items() if path.endswith(s)), 0)


def rev(files):
    """A revision {path: bytes} as (files, exts, role, stem) in path order, and its paths."""
    paths = sorted(files)
    role = np.array([lr.is_test_path(p) for p in paths], np.uint8)
    return ([files[p] for p in paths], np.array([ext_of(p) for p in paths], np.uint8), role, lr.focal_stems(paths, role)), paths


def pairs(old, new, renames=None):
    """The changed files of a step as git names them: same path and other bytes, deleted, added; renames {old path: new path}
    pair a file with its new path whatever its bytes."""
    renames = renames or {}
    po, pn = [], []
    po_paths, pn_paths = sorted(old), sorted(new)
    moved = {renames.get(p, p) for p in old}
    for i, p in enumerate(po_paths):
        q = renames.get(p, p)
        if q in new:
            if old[p] != new[q] or q != p:
                po.append(i); pn.append(pn_paths.index(q))
        else:
            po.append(i); pn.append(-1)
    for j, q in enumerate(pn_paths):
        if q not in moved:
            po.append(-1); pn.append(j)
    return po, pn


def step(old, new, renames=None):
    """(old revision, new revision, pair_old, pair_new, reference result) of one step."""
    (a, _), (b, _) = rev(old), rev(new)
    po, pn = pairs(old, new, renames)
    return a, b, po, pn, ref.churn(a, b, po, pn)


def short(rows):
    return [(r[0].decode(), r[1].decode(), r[2]) + tuple(x.decode() if isinstance(x, bytes) else x for x in r[3:5]) for r in rows]


def test_worked_examples():
    def rows(k, renames=None):
        a, b, po, pn, res = step(REVS[k - 1], REVS[k], renames)
        return ref.rows(a, b, res)
    r = rows(1)
    assert short(r) == [("test_add", "=", "lazy_introduced", None, None), ("test_sub", "M", "eager_introduced", None, None),
                        ("test_sub", "M", "lazy_introduced", None, None), ("test_sub", "M", "added", "add", "call")]
    assert r[3][5:] == (1, 0, 1, 1, 1, None)
    r = rows(2)
    assert short(r) == [("test_add", "=", "redefined", "add", None), ("test_sub", "=", "redefined", "add", None)]
    assert all(x[9:] == (1, 1) for x in r)
    r = rows(3)
    assert short(r) == [("test_sub", "=", "eager_removed", None, None), ("test_sub", "=", "removed", "sub", "definition")]
    assert r[1][5:9] == (1, 1, 0, 1)
    assert rows(4) == []
    r = rows(5, {"tests/test_calc.py": "tests/test_math.py"})
    assert short(r) == [("test_add", "=", "retargeted", "add", None), ("test_sub", "=", "retargeted", "add", None)]
    assert all(x[9] is None and x[10] == 1 for x in r)
    r = rows(5)
    assert short(r) == [("test_add", "D", "lazy_removed", None, None), ("test_add", "D", "removed", "add", "test"),
                        ("test_sub", "D", "lazy_removed", None, None), ("test_sub", "D", "removed", "add", "test"),
                        ("test_add", "A", "lazy_introduced", None, None), ("test_add", "A", "added", "add", "test"),
                        ("test_sub", "A", "lazy_introduced", None, None), ("test_sub", "A", "added", "add", "test")]
    assert r[5][7] == 2


CJ_OLD = {"w/widget.h": lr.GTEST_H, "w/widget.cc": lr.GTEST_CC, "w/widget_unittest.cc": lr.GTEST_TEST}
CJ_NEW = dict(CJ_OLD, **{"w/widget.cc": lr.GTEST_CC.replace(b"int Widget::size() const {", b"int Widget::size() const noexcept {")})


def test_cj_signature_edit_in_the_cc_only():
    a, b, po, pn, res = step(CJ_OLD, CJ_NEW)
    r = ref.rows(a, b, res)
    assert short(r) == [("Size", "=", "redefined", "size", None)]
    assert r[0][9:] == (4, 4)                                # `int size() const;` of the header is no definition


def test_known_limits():
    body = dict(REVS[0], **{"calc.py": CALC.replace(b"return a + b", b"return b + a")})
    assert step(REVS[0], body)[4]["events"] == []            # only the definition line is compared
    moved = dict(REVS[0], **{"calc.py": b"def sub(a, b):\n    return a - b\n\n\ndef add(a, b):\n    return a + b\n"})
    a, b, po, pn, res = step(REVS[0], moved)                  # a moved definition is redefined (the script keeps the other)
    assert {(x[0], x[2]) for x in short(ref.rows(a, b, res))} in ({("test_add", "redefined")}, {("test_sub", "redefined")})
    q = b'"' * 3                                              # a string opened above test_sub, outside every body: its lines
    old = dict(REVS[0], **{"tests/test_calc.py": TEST.replace(b"    def test_sub", b"    x = " + q + b"a" + q + b"\n    def test_sub")})
    new = dict(REVS[0], **{"tests/test_calc.py": TEST.replace(b"    def test_sub", b"    x = " + q + b"a\n    def test_sub")})
    a, b, po, pn, res = step(old, new)                        # are kept, but its call is now inside the string
    assert res["new"]["change"] == b"==" and short(ref.rows(a, b, res)) == [("test_sub", "=", "removed", "sub", "call")]
    twice = dict(REVS[0], **{"ops.py": OPS})                 # add defined twice: the focal file keeps the target
    assert step(REVS[0], twice)[4]["events"] == []


def test_untraced_pair_has_its_middle_redefined(monkeypatch):
    old = dict(REVS[0], **{"calc.py": b"x = 0\n" + CALC + b"y = 0\n"})
    new = dict(REVS[0], **{"calc.py": b"x = 1\n" + CALC + b"y = 1\n"})   # the whole file is the middle
    assert step(old, new)[4]["events"] == []
    monkeypatch.setattr(cr, "TRACE_MAX_D", 1)
    a, b, po, pn, res = step(old, new)
    assert sorted(x[2] for x in ref.rows(a, b, res)) == ["redefined", "redefined"]


def test_role_change_through_a_rename():
    new = {"calc.py": CALC, "calc_helpers.py": TEST}
    a, b, po, pn, res = step(REVS[0], new, {"tests/test_calc.py": "calc_helpers.py"})
    assert res["old"]["change"] == b"DD" and res["new"]["change"] == b""
    assert [x[2] for x in ref.rows(a, b, res)] == ["removed", "removed"]


def test_crlf_and_unterminated_last_lines():
    crlf = {p: d.replace(b"\n", b"\r\n") for p, d in REVS[0].items()}
    edited = dict(crlf, **{"calc.py": crlf["calc.py"].replace(b"def add(a, b):", b"def add(a, b, c=0):")})
    a, b, po, pn, res = step(crlf, edited)
    assert short(ref.rows(a, b, res)) == [("test_add", "=", "redefined", "add", None)]
    cut = {p: d.rstrip(b"\n") for p, d in REVS[1].items()}
    a, b, po, pn, res = step(REVS[0], cut)
    assert ("test_sub", "M", "added", "add", "call") in short(ref.rows(a, b, res))


def planted_history(seed, n_files, n_steps, n_edit=20):
    """Revisions of link_ref.planted_repos (one repository: every file under r0/), each edited from the last by tsm_gen_edit on
    a few test and production files, with one step that edits production files only and one that edits tests only."""
    files, exts, role, stem, grp, paths = lr.planted_repos(seed, n_files, n_repos=1)
    cur = {p.decode(): f for p, f in zip(paths, files)}
    out = [cur]
    rng = np.random.default_rng(seed)
    names = sorted(cur)
    for s in range(n_steps):
        nxt = dict(cur)
        pool = [p for p in names if (s % 3 != 1 or not lr.is_test_path(p)) and (s % 3 != 2 or lr.is_test_path(p))]
        for p in rng.choice(pool, size=min(n_edit, len(pool)), replace=False):
            nxt[str(p)] = ts.gen_edit(int(rng.integers(1 << 30)), nxt[str(p)], 2.0)
        out.append(nxt)
        cur = nxt
    return out


def test_planted_history():
    hist = planted_history(7, 240, 4)
    counts = []
    for k in range(1, len(hist)):
        a, b, po, pn, res = step(hist[k - 1], hist[k])
        assert len(po) > 0
        counts.append(len(res["events"]))
        if k == 2:                                             # production files only: the row counts docs/SPEC.md section 28 states
            kinds = sorted((ref.EVENTS[e[0]], e[1]) for e in res["events"])
            assert kinds == [("eager_removed", -1)] + [("removed", 2)] * 7 + [("retargeted", -1)] * 3
            assert set(res["new"]["change"]) == {ord("=")}
        for e in res["events"]:
            ev, cause, ot, nt, jo, jn = e[:6]
            assert ot >= 0 or nt >= 0
            if jo >= 0:
                assert int(res["old"]["links"][jo]["test"]) == ot
            if jn >= 0:
                assert int(res["new"]["links"][jn]["test"]) == nt
            if ev in (ref.ADDED, ref.REMOVED):
                assert (cause == 0) == (ot < 0 or nt < 0)
        same = ref.churn(b, b, [], [])
        assert same["events"] == [] and set(same["new"]["change"]) <= {ord("=")}
    assert counts == [27, 11, 55, 20]
