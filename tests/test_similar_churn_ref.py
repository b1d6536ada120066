"""The similar-test churn of docs/SPEC.md section 24 on the CPU: the worked examples with their hand-derived numbers, the edge
cases the section names, and the reference (tests/similar_churn_ref.py) against a second restatement built on the serial C
tests and pairs (tests/orc_simtest.c), on the examples and on planted steps."""
import random

import pytest

import similar_churn_ref as ref
import simtest_ref as sr

HEAD = b"import unittest\n\n\nclass TestAdd(unittest.TestCase):\n"
A = b"""    def test_add(self):
        x = f(1)
        y = g(x, 2)
        self.assertEqual(y, 3)
        self.assertTrue(ok)
"""
B = b"""    def test_add_print(self):
        x = f(1)
        y = g(x, 2)
        print(y)
        self.assertEqual(y, 3)
        self.assertTrue(ok)
"""
C = b"""    def test_add_one_arg(self):
        # one argument
        x = f(1)
        y = g(x)
        self.assertEqual(y, 3)
        self.assertTrue(ok)
"""
B_FIX = B.replace(b"assertEqual(y, 3)", b"assertEqual(y, 4)")
B_CUT = B.replace(b"        x = f(1)\n        y = g(x, 2)\n", b"")


def py(*tests):
    return HEAD + b"\n".join(tests) + b"\n"


def step(old_files, new_files, pairs=None, exts_old=None, exts_new=None, min_lines=5, P=70):
    """The reference rows of one step; by default file i of both revisions is pair i."""
    old = (list(old_files), exts_old or [1] * len(old_files))
    new = (list(new_files), exts_new or [1] * len(new_files))
    if pairs is None:
        pairs = [(i, i) for i in range(max(len(old_files), len(new_files)))]
        pairs = [(o if o < len(old_files) else -1, n if n < len(new_files) else -1) for o, n in pairs]
    po, pn = zip(*pairs) if pairs else ((), ())
    return ref.churn(old, new, list(po), list(pn), min_lines, P)


def rows(r):
    return ref.rows(r)


# The revisions of the worked examples, one file each: R1 = A, R2 = A B, ..., R7 = A B (restored)
R = [py(A), py(A, B), py(A, B, C), py(A, B_FIX, C), py(A, B_CUT, C), py(A, B_CUT), py(A, B)]


def test_example_1_paste():
    r = step([R[0]], [R[1]])
    assert r["new"]["change"] == b"=A"
    assert rows(r) == [("copied", 0, -1, 0, 1, None, 90)]


def test_example_2_second_paste():
    r = step([R[1]], [R[2]])
    assert r["new"]["change"] == b"==A"
    assert rows(r) == [("copied", 0, -1, 0, 2, None, 80), ("copied", 1, -1, 1, 2, None, 72)]


def test_example_3_one_sided_fix():
    r = step([R[2]], [R[3]])
    assert r["new"]["change"] == b"=M="
    _, s2 = sr.py_sequences([R[3]], [1])
    _, s1 = sr.py_sequences([R[2]], [1])
    assert s1 == s2                                          # the fix leaves every blind sequence as it was
    assert rows(r) == [("changed", 0, 1, 0, 1, 90, 90), ("changed", 1, 2, 1, 2, 72, 72)]


def test_example_4_diverged():
    r = step([R[3]], [R[4]])
    assert r["new"]["test_kept"] == [5, 4, 5]                # B is no longer compared at min_lines 5
    assert rows(r) == [("diverged", 0, 1, 0, 1, 90, 66), ("diverged", 1, 2, 1, 2, 72, 66)]
    assert [e[7] for e in r["events"]] == [3, 3]             # lcs 3 of 5 + 4


def test_example_5_dropped():
    r = step([R[4]], [R[5]])
    assert r["old"]["change"] == b"==D"
    assert rows(r) == [("dropped", 0, 2, 0, -1, 80, None)]


def test_example_6_converged():
    r = step([R[5]], [R[6]])
    assert r["new"]["change"] == b"=M"
    assert rows(r) == [("converged", 0, 1, 0, 1, 66, 90)]


def test_created_and_removed_file():
    # two tests unlike A: a statement of another shape on each line
    body = b"        for k in range(3):\n            s += k\n        assert s == 3\n        return\n"
    other = py(b"    def test_sum(self):\n" + body, b"    def test_sum_twice(self):\n" + body + b"        del s\n")
    r = step([R[0]], [R[0], other], pairs=[(-1, 1)])
    assert rows(r) == [("created", -1, -1, 1, 2, None, 90)]
    r = step([R[0], other], [R[0]], pairs=[(1, -1)])
    assert rows(r) == [("removed", 1, 2, -1, -1, 90, None)]


def test_header_matched_by_name():
    new = py(A.replace(b"def test_add(self):", b"def test_add(self, tmp_path):"), B)
    r = step([R[1]], [new])
    assert r["old"]["match"] == [0, 1] and r["new"]["change"] == b"M="
    assert rows(r) == [("changed", 0, 1, 0, 1, 90, 72)]


def test_score_exactly_at_p_and_one_below():
    # A-B is 200 * 5 / 11 = 90.9 %: a pair at P = 90, none at P = 91
    new = py(A, B_FIX)
    assert rows(step([R[1]], [new], P=90)) == [("changed", 0, 1, 0, 1, 90, 90)]
    assert rows(step([R[1]], [new], P=91)) == []
    # A step that lowers A-B from 90.9 % to exactly 80 % (lcs 4 of 5 + 5): diverged at P = 81, changed at P = 80
    new = py(A, B.replace(b"        print(y)\n", b"").replace(b"y = g(x, 2)", b"y = g(x)"))
    assert rows(step([R[1]], [new], P=80)) == [("changed", 0, 1, 0, 1, 90, 80)]
    assert rows(step([R[1]], [new], P=81)) == [("diverged", 0, 1, 0, 1, 90, 80)]


def test_falls_under_min_lines():
    r = step([R[1]], [py(A, B_CUT)], min_lines=5)
    assert rows(r) == [("diverged", 0, 1, 0, 1, 90, 66)]
    r = step([R[1]], [py(A, B_CUT)], min_lines=4, P=60)
    assert rows(r) == [("changed", 0, 1, 0, 1, 90, 66)]


def test_comment_and_literal_edits_are_m():
    for new_b in (B.replace(b"print(y)", b"print(y)  # show"), B.replace(b"f(1)", b"f(2)")):
        r = step([R[1]], [py(A, new_b)])
        assert r["new"]["change"] == b"=M"
        assert rows(r) == [("changed", 0, 1, 0, 1, 90, 90)]


def test_rename_to_cc_is_no_test():
    # a .py file renamed to .cc: its tests are no tests there, so both old tests are D
    r = step([R[1]], [R[1]], exts_new=[2])
    assert r["new"]["tests"] == [] and r["old"]["change"] == b"DD"
    assert rows(r) == [("removed", 0, 1, -1, -1, 90, None)]


def test_docstring_above_changes_sequence_without_marked_body_line():
    # a line above test A opens a docstring that runs into A: A's body lines are unmarked but its sequence changes
    new = HEAD + b'    """\n' + A + b'    """\n' + b"\n" + B
    old = HEAD + b"\n" + A + b"\n" + b"\n" + B
    r = step([old], [new])
    assert r["new"]["match"][:1] == [0]
    assert r["new"]["change"][:1] == b"M"


# ---------------------------------------------------------------------------------------------- second restatement
def restate(old, new, pair_old, pair_new, min_lines, P):
    """Section 24's statuses from the serial C tests and pairs (orc_smells, orc_blind, orc_simtest.c) of both revisions, with
    the pairs of two unchanged tests dropped first, as the device does: {(status, a, b)}, old (a, b) for the old-side
    statuses and new (a, b) for the others."""
    to, so = sr.c_sequences(_corpus(*old))
    tn, sn = sr.c_sequences(_corpus(*new))
    key = lambda tests: [(int(t["file"]), int(t["line"]), int(t["body_lines"])) for t in tests]
    ko, kn = key(to), key(tn)
    mo, mn, marked = ref.identity(old, new, pair_old, pair_new, ko, kn)
    unmarked = lambda side, f, h, n: not any((f, l) in marked[side] for l in range(h, h + n))
    same = lambda a, b: ko[a][2] == kn[b][2] and so[a] == sn[b] and unmarked(0, *ko[a]) and unmarked(1, *kn[b])
    dirty_o = [b < 0 or not same(a, b) for a, b in enumerate(mo)]
    dirty_n = [a < 0 or not same(a, b) for b, a in enumerate(mn)]
    po = {(a, b) for a, b, _, _ in sr.c_similar(so, min_lines, P) if dirty_o[a] or dirty_o[b]}
    pn = {(a, b) for a, b, _, _ in sr.c_similar(sn, min_lines, P) if dirty_n[a] or dirty_n[b]}
    img = lambda m, a, b: (min(m[a], m[b]), max(m[a], m[b])) if m[a] >= 0 and m[b] >= 0 else None
    out = set()
    for a, b in po:
        i = img(mo, a, b)
        if i not in pn:
            out.add(("diverged" if i else "removed" if mo[a] < 0 and mo[b] < 0 else "dropped", a, b))
    images = {img(mo, a, b) for a, b in po} - {None}
    for a, b in pn:
        i = img(mn, a, b)
        out.add(("changed" if (a, b) in images else "converged" if i else "created" if mn[a] < 0 and mn[b] < 0 else "copied", a, b))
    return out


def _corpus(files, exts):
    from clone_churn_ref import _Packed
    p = _Packed(files, exts)
    p.n_files = len(files)
    return p


def summary(res):
    out = set()
    for st, oa, ob, a, b, *_ in res["events"]:
        name = ref.STATUSES[st]
        out.add((name, oa, ob) if name in ("removed", "dropped", "diverged") else (name, a, b))
    return out


def planted_step(seed):
    rng = random.Random(seed)
    bodies = [[b"        v%d = f(%d)\n" % (i, i) for i in range(rng.randint(4, 9))] for _ in range(4)]
    tests = []
    for k in range(12):
        base = list(rng.choice(bodies))
        for _ in range(rng.randint(0, 2)):
            base.insert(rng.randrange(len(base) + 1), b"        w = h(%d)\n" % rng.randint(0, 5))
        tests.append(b"    def test_%d(self):\n" % k + b"".join(base) + b"        self.assertTrue(v0)\n")
    old = [HEAD + b"\n".join(tests[:8]), HEAD + b"\n".join(tests[8:])]
    new_tests = list(tests)
    for _ in range(rng.randint(1, 4)):
        k = rng.randrange(len(new_tests))
        lines = new_tests[k].split(b"\n")
        op = rng.randrange(3)
        i = rng.randrange(1, len(lines) - 1)
        if op == 0:
            lines.insert(i, b"        z = q(1)")
        elif op == 1 and len(lines) > 4:
            del lines[i]
        else:
            lines[i] = lines[i].replace(b"f(", b"f(9 + ")
        new_tests[k] = b"\n".join(lines)
    if rng.random() < 0.5:
        new_tests.append(tests[rng.randrange(8)].replace(b"def test_", b"def test_copy_"))
    new = [HEAD + b"\n".join(new_tests[:8]), HEAD + b"\n".join(new_tests[8:])]
    return (old, [1, 1]), (new, [1, 1])


@pytest.mark.parametrize("seed", range(12))
def test_restatement_agrees_on_planted_steps(seed):
    old, new = planted_step(seed)
    # both files in a pair, and only the first (the second unchanged when the step left it alone)
    layouts = [([0, 1], [0, 1])] + ([([0], [0])] if old[0][1] == new[0][1] else [([1], [1])] if old[0][0] == new[0][0] else [])
    for po, pn in layouts:
        for ml, P in ((5, 70), (3, 50), (1, 90)):
            want = ref.churn(old, new, po, pn, ml, P)
            assert summary(want) == restate(old, new, po, pn, ml, P), (seed, ml, P)


def test_examples_restated():
    for i in range(len(R) - 1):
        old, new = ([R[i]], [1]), ([R[i + 1]], [1])
        assert summary(ref.churn(old, new, [0], [0])) == restate(old, new, [0], [0], 5, 70)
