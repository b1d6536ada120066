"""The clone churn of docs/SPEC.md section 22 on the CPU: the worked examples of the section with their statuses derived by hand,
exact and blind, and the reference (tests/clone_churn_ref.py: classes from orc_clones / orc_blind, marks from orc_marks) against
a second restatement over line contents (py_clones, py_diff_files) on planted and fuzzed steps."""
import random

import numpy as np
import pytest

import clone_churn_ref as cr

T = [b"def test_total(self):", b"    cart = Cart()", b"    cart.add(3)", b"    cart.add(4)", b"    self.assertEqual(cart.total(), 7)",
     b"    self.assertTrue(cart.items)"]


def text(lines):
    return b"".join(ln + b"\n" for ln in lines)


def rows(res, side):
    """[(status, [(fragment's first line, state, changed, changed_assert)])] of the touched classes of one side."""
    s = res[side]
    out = []
    for c in range(len(s["class_len"])):
        if s["status"][c] == 0:
            continue
        b, e = s["class_base"][c], s["class_base"][c + 1]
        out.append((cr.STATUSES[s["status"][c]], [(int(s["member"][j]), cr.STATES[s["state"][j]], int(s["changed"][j]),
                                                   int(s["changed_assert"][j])) for j in range(b, e)]))
    return out


def both(old, new, po, pn, n=5, blind=False):
    got = cr.churn(old, new, po, pn, n, blind)
    if not blind:
        cr.assert_equal(cr.py_churn(old, new, po, pn, n), got)
    return got


A = [b"import unittest", b"class TestA(unittest.TestCase):"] + [b"  " + x for x in T]
B = [b"class TestB(unittest.TestCase):"] + [b"  " + x for x in T]


def test_paste_into_new_file():
    old = ([text(A)], [1])
    new = ([text(A), text(B)], [1, 1])
    got = both(old, new, [-1], [1])
    assert rows(got, "old") == []
    assert rows(got, "new") == [("copied", [(2, "kept", 0, 0), (len(A) + 1, "whole", 6, 2)])]


def test_one_copy_edited():
    old = ([text(A), text(B)], [1, 1])
    A2 = list(A)
    A2[4] = b"    cart.add(5)"
    new = ([text(A2), text(B)], [1, 1])
    got = both(old, new, [0], [0])
    assert rows(got, "old") == [("diverged", [(2, "edited", 1, 0), (len(A) + 1, "kept", 0, 0)])]
    assert rows(got, "new") == [] and len(got["new"]["class_len"]) == 0       # no 5-line window survives the edit


def test_both_copies_edited_alike():
    old = ([text(A), text(B)], [1, 1])
    A2, B2 = list(A), list(B)
    A2[4] = B2[3] = b"    cart.add(5)"
    new = ([text(A2), text(B2)], [1, 1])
    got = both(old, new, [0, 1], [0, 1])
    assert rows(got, "old") == [("changed", [(2, "edited", 1, 0), (len(A) + 1, "edited", 1, 0)])]
    assert rows(got, "new") == [("changed", [(2, "edited", 1, 0), (len(A) + 1, "edited", 1, 0)])]


def test_copy_deleted():
    old = ([text(A), text(B)], [1, 1])
    new = ([text(A)], [1])
    got = both(old, new, [1], [-1])
    assert rows(got, "old") == [("dropped", [(2, "kept", 0, 0), (len(A) + 1, "whole", 6, 2)])]
    assert rows(got, "new") == []


def test_blind_renamed_copy_then_one_expected_value_fixed():
    Bt = [x.replace(b"cart", b"basket").replace(b"test_total", b"test_sum").replace(b"3", b"1") for x in T]
    Bf = [b"class TestB(unittest.TestCase):"] + [b"  " + x for x in Bt]
    fixed = list(Bf)
    fixed[5] = b"      self.assertEqual(basket.total(), 5)"   # the copy's expected value fixed (blind form unchanged)
    old = ([text(A), text(Bf)], [1, 1])
    new = ([text(A), text(fixed)], [1, 1])
    exact = both(old, new, [1], [1])
    assert rows(exact, "old") == [] and rows(exact, "new") == []             # no exact copy: nothing to report
    got = both(old, new, [1], [1], blind=True)
    assert rows(got, "old") == [("diverged", [(1, "kept", 0, 0), (len(A), "edited", 1, 1)])]   # the class lines match blind
    assert rows(got, "new") == [("joined", [(1, "kept", 0, 0), (len(A), "edited", 1, 1)])]


def test_status_rules():
    for new_side, want in ((False, {(0, 0, 2): 2, (1, 1, 0): 3, (1, 1, 1): 3, (1, 0, 1): 4, (0, 2, 0): 1, (0, 1, 1): 1, (2, 0, 0): 0}),
                           (True, {(0, 0, 2): 5, (1, 0, 1): 6, (1, 1, 1): 6, (1, 1, 0): 7, (0, 2, 0): 1, (0, 1, 1): 1, (2, 0, 0): 0})):
        for counts, st in want.items():
            assert cr.status_of(*counts, new_side) == st, (new_side, counts)


def planted_step(seed, n_files=12):
    """A step over small PY files with pasted tests, one-copy edits, deletions, additions and renames."""
    rng = random.Random(seed)
    pool = [[b"    v%d_%d = f(%d)" % (t, k, rng.randrange(3)) for k in range(rng.randrange(3, 9))] + [b"    assert v%d_0 == 1" % t]
            for t in range(6)]
    files = []
    for i in range(n_files):
        body = [b"import x%d" % i]
        for _ in range(rng.randrange(1, 4)):
            body += [b"def test_%d_%d():" % (i, rng.randrange(99))] + rng.choice(pool)
            if rng.random() < 0.3:
                body.append(b"")
        files.append(body)
    new_files, po, pn = [], [], []
    for i, f in enumerate(files):
        r = rng.random()
        if r < 0.1:
            po.append(i); pn.append(-1)                       # deleted
            continue
        g = list(f)
        if r < 0.5:
            for _ in range(rng.randrange(1, 3)):              # edited lines, inserted and deleted lines
                k = rng.randrange(len(g))
                op = rng.randrange(3)
                if op == 0:
                    g[k] = g[k] + b"  # fix"
                elif op == 1:
                    g.insert(k, rng.choice(rng.choice(pool)))
                elif len(g) > 1:
                    del g[k]
            po.append(i); pn.append(len(new_files))
        elif r < 0.6:
            po.append(i); pn.append(len(new_files))          # unchanged but paired (a rename)
        new_files.append(g)
    for _ in range(rng.randrange(1, 4)):                      # pasted tests in new files
        po.append(-1); pn.append(len(new_files))
        new_files.append([b"def test_paste():"] + rng.choice(pool) + rng.choice(pool))
    order = list(range(len(po)))
    rng.shuffle(order)
    old = ([text(f) for f in files], [1] * len(files))
    new = ([text(f) for f in new_files], [1] * len(new_files))
    return old, new, [po[k] for k in order], [pn[k] for k in order]


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("n", [1, 3, 5])
def test_reference_agrees_with_restatement(seed, n):
    old, new, po, pn = planted_step(seed)
    got = both(old, new, po, pn, n)
    assert any(len(got[s]["class_len"]) for s in ("old", "new")) or n == 5


@pytest.mark.parametrize("seed", range(6))
def test_fuzz(seed):
    rng = random.Random(100 + seed)
    alphabet = [b"a", b"b", b"assert x", b"", b"c = 1", b"d\r"]
    old_files = [text([rng.choice(alphabet) for _ in range(rng.randrange(0, 40))]) for _ in range(6)]
    new_files = [text([rng.choice(alphabet) for _ in range(rng.randrange(0, 40))]) for _ in range(5)]
    po, pn = [0, 1, 2, -1, 3], [0, -1, 1, 2, 4]
    for n in (1, 2, 4):
        both((old_files, [1] * 6), (new_files, [1] * 5), po, pn, n)


def test_empty_revisions_and_no_pairs():
    got = both(([], []), ([text(A), text(B)], [1, 1]), [-1, -1], [0, 1])
    assert rows(got, "new") == [("created", [(2, "whole", 6, 2), (len(A) + 1, "whole", 6, 2)])]
    got = both(([text(A), text(B)], [1, 1]), ([text(A), text(B)], [1, 1]), [], [])
    assert rows(got, "old") == [] and rows(got, "new") == [] and list(got["new"]["status"]) == [0]
