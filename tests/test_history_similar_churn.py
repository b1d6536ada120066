"""`tosem-scan history --similar-tests` and `diff --similar-tests` (docs/SPEC.md section 24) on a repository built in the test.  Its
commits play the worked examples of section 24 (a paste, a second paste, a one-copy fix, a cut that makes a pair diverge, a
deletion, a restore), then rename a file that holds two similar tests, add a binary test file that holds a copy, modify it, and
change a header so that its test is matched by name.  Checks: the rows equal a restatement over `git ls-tree` / `git cat-file` of
every revision (tests/similar_churn_ref.py), with and without `--find-renames`, and over a `--max-commits` window; `diff
--similar-tests` of two checkouts gives the commit's rows without the lead columns; `--clones` rows and every other output are
byte-identical with and without `--similar-tests`, and `--dry-run` is refused with it."""
import os
import shutil
import subprocess

import pytest

import case_ref
import similar_churn_ref as ref
import spec_ref
import test_similar_churn_ref as ex
from test_history import CLI, git
from test_history_clones import EXT, binary, changes, checkout, commit, commits, read, revision, run, write

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

HEAD = ["status", "fileName", "test", "oldLine", "line", "change", "otherFileName", "otherTest", "otherOldLine", "otherLine",
        "otherChange", "oldLcs", "oldSimilarity", "lcs", "similarity"]
OTHER = b"""class TestOther(unittest.TestCase):
    def test_sum(self):
        for k in range(3):
            s += k
        assert s == 3
        return

    def test_sum_twice(self):
        for k in range(3):
            s += k
        assert s == 3
        return
        del s
"""


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    r = str(tmp_path_factory.mktemp("similar") / "repo")
    os.makedirs(r)
    git(r, "init", "-q", ".")
    write(r, "tests/test_add.py", ex.R[0])
    write(r, "tests/unit/test_other.py", ex.HEAD + OTHER)
    commit(r, "root")
    for i, msg in enumerate(["paste", "second paste", "one-copy fix", "cut", "delete a copy", "restore"], start=1):
        write(r, "tests/test_add.py", ex.R[i])
        commit(r, msg)
    git(r, "mv", "tests/unit/test_other.py", "tests/unit/test_more.py")
    commit(r, "rename a file with two similar tests")
    write(r, "tests/test_bin.py", ex.py(ex.A.replace(b"test_add", b"test_bin")) + b"\x00\x01\n")
    commit(r, "add a binary test file")
    write(r, "tests/test_bin.py", ex.py(ex.A.replace(b"test_add", b"test_bin")) + b"\x00\x01\nmore = 1\n")
    commit(r, "modify the binary test file")
    write(r, "tests/test_add.py", ex.py(ex.A.replace(b"def test_add(self):", b"def test_add(self, tmp_path):"), ex.B))
    commit(r, "header matched by name")
    return r


def step_rows(repo, parent, child, ml, P, renames):
    po_, po = revision(repo, parent)
    pn_, pn = revision(repo, child)
    pairs = []
    for o, nw in changes(repo, parent, child, renames):
        a, b = (po_.index(o) if o else -1), (pn_.index(nw) if nw else -1)
        if a >= 0 and b >= 0 and (binary(po[o]) or binary(pn[nw])):
            pairs += [(a, -1), (-1, b)]
        else:
            pairs.append((a, b))
    old = ([po[p] for p in po_], [EXT[p.rsplit(".", 1)[1]] for p in po_])
    new = ([pn[p] for p in pn_], [EXT[p.rsplit(".", 1)[1]] for p in pn_])
    res = ref.churn(old, new, [a for a, _ in pairs], [b for _, b in pairs], ml, P)
    sides = [(res["old"], old, po_), (res["new"], new, pn_)]

    def cells(o, n):
        s = 1 if n >= 0 else 0
        side, (files, exts), paths = sides[s]
        f, h, _ = side["tests"][n if s else o]
        name = case_ref.py_case_name(spec_ref.py_lines(files[f])[h], exts[f]).decode("latin-1")
        line = lambda k, t: str(sides[k][0]["tests"][t][1] + 1) if t >= 0 else ""
        change = chr(side["change"][n if s else o])
        old_path = po_[res["old"]["tests"][o][0]] if o >= 0 else ""
        return [paths[f], name, line(0, o), line(1, n), change], old_path
    rows = []
    for st, oa, ob, a, b, ol, os_, l, s in res["events"]:
        ca, pa = cells(oa, a)
        cb, pb = cells(ob, b)
        num = lambda v, d: "" if v == ref.NONE else str(v // d)
        row = [ref.STATUSES[st]] + ca + cb + [num(ol, 1), num(os_, 600), num(l, 1), num(s, 600)]
        rows.append(row + ([pa, pb] if renames else []))
    return rows


def want(repo, chain, ml, P, renames):
    return [[c, p, t] + r for c, p, t in chain for r in step_rows(repo, p, c, ml, P, renames)]


@pytest.mark.parametrize("renames", [False, True])
def test_history_rows_equal_the_restatement(repo, tmp_path, renames):
    out = tmp_path / "s.csv"
    run("history", repo, "--similar-tests", out, *(["--find-renames", 50] if renames else []))
    table = read(out)
    assert table[0] == ["commit", "parent", "time"] + HEAD + (["oldFileName", "otherOldFileName"] if renames else [])
    assert table[1:] == want(repo, commits(repo), 5, 70, renames)
    statuses = {r[3] for r in table[1:]}
    assert {"copied", "changed", "diverged", "dropped", "converged"} <= statuses, statuses
    by_msg = {c: git(repo, "log", "-1", "--format=%s", c).strip() for c, _, _ in commits(repo)}
    rename_rows = [r for r in table[1:] if by_msg[r[0]].startswith("rename")]
    assert (rename_rows == []) == renames                   # an exact rename under -M touches no test
    fix = [r for r in table[1:] if by_msg[r[0]] == "one-copy fix"]
    assert [(r[3], r[5], r[8], r[15], r[17]) for r in fix] == [("changed", "test_add", "=", "90", "90"),
                                                               ("changed", "test_add_print", "M", "72", "72")]


def test_max_commits_window_and_settings(repo, tmp_path):
    out = tmp_path / "w.csv"
    run("history", repo, "--max-commits", 5, "--min-lines", 4, "--similarity", 60, "--similar-tests", out)
    assert read(out)[1:] == want(repo, commits(repo)[-5:], 4, 60, False)


def test_diff_equals_the_commit_rows(repo, tmp_path):
    hist = tmp_path / "h.csv"
    run("history", repo, "--similar-tests", hist, "--find-renames", 50)
    table = read(hist)[1:]
    for c, p, _ in commits(repo)[1:]:
        checkout(repo, p, tmp_path / ("o_" + c))
        checkout(repo, c, tmp_path / ("n_" + c))
        out = tmp_path / ("d_%s.csv" % c)
        run("diff", tmp_path / ("o_" + c), tmp_path / ("n_" + c), "--similar-tests", out, "--find-renames", 50)
        got = read(out)
        assert got[0] == HEAD + ["oldFileName", "otherOldFileName"]
        assert got[1:] == [r[3:] for r in table if r[0] == c], c


def test_clones_and_other_outputs_are_unchanged(repo, tmp_path):
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(); b.mkdir()
    r1 = run("history", repo, "--out", a / "o.csv", "--cases", a / "k.csv", "--clones", a / "c.csv", "--find-renames", 50)
    r2 = run("history", repo, "--out", b / "o.csv", "--cases", b / "k.csv", "--clones", b / "c.csv", "--find-renames", 50,
             "--similar-tests", b / "s.csv")
    assert r1.stdout == r2.stdout
    for f in ("o.csv", "k.csv", "c.csv"):
        assert open(a / f, "rb").read() == open(b / f, "rb").read(), f
    both = read(b / "s.csv")
    alone = tmp_path / "s.csv"
    run("history", repo, "--similar-tests", alone, "--find-renames", 50)
    assert read(alone) == both


def test_dry_run_is_refused(repo, tmp_path):
    r = subprocess.run([CLI, "history", repo, "--dry-run", "--similar-tests", str(tmp_path / "s.csv")], capture_output=True)
    assert r.returncode != 0 and b"--similar-tests" in r.stderr
