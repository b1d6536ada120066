"""`tosem-scan history --asserts / --assert-churn` (docs/SPEC.md section 8, changed assertion lines) on a git repository
built so that every edit is unambiguous - assertion lines replaced, inserted or deleted among unique lines - so that the
canonical script's changed lines are exactly the `+` / `-` lines of `git diff --minimal -U0`.  Those lines are classified
by the plain-Python restatement of SPEC sections 4 and 6 (tests/spec_ref.py), independent of the device and the oracle."""
import collections
import csv
import os
import re
import shutil
import subprocess

import pytest

import spec_ref
import tosemscan as ts
from test_history import CLI, EMPTY_TREE, git

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

ASSERTS = [b"self.assertEqual(a%d, b)", b"assert x%d == 4", b"self.assertAlmostEqual(q%d, 2)", b"self.assertFooBar(z%d)",
           b"assert not y%d", b"self.assertIn(k%d, d)", b"EXPECT_EQ(r%d, 1);", b"self.assertTrue(t%d)", b"assert_(w%d)"]


def body(tag, n, asserts):
    """n unique plain lines with the given assertion lines (kind index, number) spliced in at fixed places."""
    out = [b"v_%s_%d = %d\n" % (tag, i, i) for i in range(n)]
    for pos, (kind, num) in sorted(asserts, reverse=True):
        out.insert(pos, b"    " + ASSERTS[kind] % num + b"\n")
    return out


def build(root):
    repo = root / "repo"
    os.makedirs(repo / "tests")
    git(repo, "init", "-q", ".")
    A = body(b"a", 40, [(3, (0, 1)), (10, (1, 2)), (20, (3, 3)), (30, (4, 4))])
    B = body(b"b", 30, [(5, (5, 5)), (15, (7, 6))])
    files = {"tests/test_a.py": A, "tests/test_b.py": B}

    def commit(msg):
        for nm in list(os.listdir(repo / "tests")):
            if "tests/" + nm not in files:
                os.remove(repo / "tests" / nm)
        for nm, lines in files.items():
            (repo / nm).write_bytes(b"".join(lines))
        git(repo, "add", "-A")
        git(repo, "commit", "-q", "-m", msg)
    commit("initial")
    A[A.index(b"    self.assertEqual(a1, b)\n")] = b"    self.assertAlmostEqual(a1, b)\n"     # replaced: category changes
    A.insert(25, b"    self.assertFooBar(z9)\n")                                             # inserted
    del B[B.index(b"    self.assertIn(k5, d)\n")]                                            # deleted
    commit("edit assertions")
    files["tests/test_c.py"] = body(b"c", 12, [(2, (8, 7)), (6, (0, 8)), (9, (1, 9))])       # new file: every line added
    del files["tests/test_b.py"]                                                             # removed file: every line deleted
    commit("add c, remove b")
    A[7] = b"v_a_changed = 1\n"                                                              # no assertion line changes
    commit("plain edit")
    A[A.index(b"    assert not y4\n")] = b"    assert y4 != 5\n"
    A.insert(1, b"    self.assertTrue(t11)\n")
    commit("more")
    return repo


def category_cell(stmt):
    cat = spec_ref.py_category(stmt)
    if cat == 127:
        o, n = spec_ref.py_ident(stmt)
        return cat, stmt[o:o + n].decode()
    return cat, ts.category_name(cat)


def expected(repo):
    rows, churn = [], collections.defaultdict(lambda: [0, 0])
    log = git(repo, "log", "--first-parent", "--reverse", "--format=%H %P %ct").split("\n")
    for entry in filter(None, log):
        parts = entry.split()
        commit, parent, t = parts[0], (parts[1] if len(parts) > 2 else ""), parts[-1]
        diff = git(repo, "diff", "--minimal", "-U0", "--no-color", "--no-renames", parent or EMPTY_TREE, commit, text=False)
        path, lo, ln = None, 0, 0
        for line in diff.split(b"\n"):
            if line.startswith(b"+++ ") or line.startswith(b"--- "):
                if line[4:] != b"/dev/null":
                    path = line[6:].decode()
                continue
            m = re.match(rb"@@ -(\d+)(?:,\d+)? \+(\d+)(?:,\d+)? @@", line)
            if m:                                            # first deleted / inserted line (unused when that side is empty)
                lo, ln = int(m.group(1)), int(m.group(2))
                continue
            if line[:1] in (b"+", b"-") and path:
                text = line[1:]
                num = lo if line[:1] == b"-" else ln
                if line[:1] == b"-":
                    lo += 1
                else:
                    ln += 1
                if not spec_ref.py_is_assert_line(text, 1):
                    continue
                stmt = spec_ref.py_statement(text)
                cat, cell = category_cell(stmt)
                rows.append((commit, parent, t, path, line[:1].decode(), str(num), stmt.decode(), cell))
                churn[(commit, cat)][0 if line[:1] == b"+" else 1] += 1
    return rows, churn


def test_history_assert_rows_equal_git_diff(tmp_path):
    repo = build(tmp_path)
    out, ar, cr = tmp_path / "h.csv", tmp_path / "a.csv", tmp_path / "c.csv"
    r = subprocess.run([CLI, "history", str(repo), "--out", str(out), "--asserts", str(ar), "--assert-churn", str(cr)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [tuple(x) for x in list(csv.reader(open(ar, newline="")))[1:]]
    want, churn = expected(repo)
    assert sorted(got) == sorted(want) and len(want) == 17
    cells = {row[6]: row[7] for row in want}
    assert cells["self.assertAlmostEqual"] == "assertAlmostEqual" and cells["self.assertFooBar"] == "assertFooBar"
    got_churn = {(c[0], c[1]): (int(c[2]), int(c[3])) for c in list(csv.reader(open(cr, newline="")))[1:]}
    want_churn = {(commit, ts.category_name(cat)): tuple(v) for (commit, cat), v in churn.items()}
    assert got_churn == want_churn
    # the plain rows and stdout do not change with the new options
    out2 = tmp_path / "h2.csv"
    r2 = subprocess.run([CLI, "history", str(repo), "--out", str(out2)], capture_output=True, text=True)
    assert r2.returncode == 0 and r2.stdout == r.stdout and open(out2, "rb").read() == open(out, "rb").read()
