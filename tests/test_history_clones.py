"""`tosem-scan history --clones` and `diff --clones` (docs/SPEC.md section 22) on a repository built in the test.  Its commits
paste a test into a new file, edit both copies of a duplicated test alike, edit one copy, rename a file that holds a copy, add and
then modify a binary test file that holds a copy, and delete a copy.  Three checks: the rows equal a plain-Python restatement over
`git ls-tree` / `git cat-file` of every revision (tests/clone_churn_ref.py), exact and blind, with and without `--find-renames`,
and over a `--max-commits` window whose boundary revision is read whole; every row's class, fileName and lines are a row of
`clones --git --rev <parent|commit> --out`; `diff --clones` of two checkouts gives the commit's rows without the lead columns."""
import csv
import io
import os
import shutil
import subprocess
import tarfile

import pytest

import clone_churn_ref as cr
from test_history import CLI, git

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

HEAD = ["side", "class", "status", "fragments", "fileName", "first_line", "last_line", "state", "changed_lines", "changed_assert_lines"]
EXT = {"py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}

T = [b"def test_total(self):", b"    cart = Cart()", b"    cart.add(3)", b"    cart.add(4)", b"    self.assertEqual(cart.total(), 7)",
     b"    self.assertTrue(cart.items)"]
X = [b"def test_parse():", b"    p = Parser()", b"    r = p.parse('a b')", b"    assert r.words == ['a', 'b']", b"    assert r.ok",
     b"    assert not r.errors"]


def text(lines):
    return b"".join(ln + b"\n" for ln in lines)


def write(repo, path, data):
    os.makedirs(os.path.dirname(os.path.join(repo, path)), exist_ok=True)
    with open(os.path.join(repo, path), "wb") as f:
        f.write(data)


def commit(repo, msg):
    git(repo, "add", "-A")
    git(repo, "commit", "-q", "-m", msg)


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    r = str(tmp_path_factory.mktemp("clones") / "repo")
    os.makedirs(r)
    git(r, "init", "-q", ".")
    a = [b"import unittest", b"class TestA(unittest.TestCase):"] + [b"  " + x for x in T]
    b = [b"class TestB(unittest.TestCase):"] + [b"  " + x for x in T]
    write(r, "tests/test_a.py", text(a))
    write(r, "tests/test_x.py", text([b"import parser"] + X))
    write(r, "tests/unit/test_c.py", text([b"import parser as q"] + X + [b"# end"]))
    write(r, "src/lib.py", text(T))                                        # not a test file: never selected
    commit(r, "root")
    write(r, "tests/test_b.py", text(b))
    commit(r, "paste a test into a new file")
    a[4], b[3] = b"    cart.add(5)", b"    cart.add(5)"
    write(r, "tests/test_a.py", text(a)); write(r, "tests/test_b.py", text(b))
    commit(r, "edit both copies alike")
    a[6] = b"    self.assertEqual(cart.total(), 9)"
    write(r, "tests/test_a.py", text(a))
    commit(r, "edit one copy")
    git(r, "mv", "tests/unit/test_c.py", "tests/unit/test_d.py")
    commit(r, "rename a file that holds a copy")
    write(r, "tests/test_bin.py", text([b"# data"] + X) + b"\x00\x01\n")
    commit(r, "add a binary test file")
    write(r, "tests/test_bin.py", text([b"# data"] + X) + b"\x00\x01\nmore = 1\n")
    commit(r, "modify the binary test file")
    git(r, "rm", "-q", "tests/unit/test_d.py")
    commit(r, "delete a copy")
    return r


def commits(repo):
    out = []
    for entry in filter(None, git(repo, "log", "--first-parent", "--reverse", "--format=%H %P %ct").split("\n")):
        p = entry.split()
        out.append((p[0], p[1] if len(p) > 2 else "", p[-1]))
    return out


def selected(path):
    ext = path.rsplit(".", 1)[-1] if "." in path.rsplit("/", 1)[-1] else ""
    return "test" in path.lower() and ext in EXT


def revision(repo, rev):
    """(paths, {path: bytes}) of the selected files at rev, in the order of `clones --git` (path components compared in turn)."""
    if not rev:
        return [], {}
    paths = [p for p in git(repo, "ls-tree", "-r", "--name-only", rev).split("\n") if p and selected(p)]
    paths.sort(key=lambda p: p.split("/"))
    return paths, {p: git(repo, "cat-file", "blob", "%s:%s" % (rev, p), text=False) for p in paths}


def changes(repo, parent, child, renames):
    """[(old path or None, new path or None)] of the selected files, from `git diff-tree` (with -M50% under renames)."""
    args = ["diff-tree", "-r", "--no-commit-id", "--name-status"] + (["-M50%"] if renames else []) + [parent or "--root", child]
    out = []
    for line in filter(None, git(repo, *args).split("\n")):
        f = line.split("\t")
        k = f[0][0]
        if k == "R":
            out.append((f[1], f[2]))
        elif k == "D":
            out.append((f[1], None))
        elif k == "A":
            out.append((None, f[1]))
        else:
            out.append((f[1], f[1]))
    return [(o, n) for o, n in out if (o is None or selected(o)) and (n is None or selected(n))]


def binary(b):
    return b"\x00" in b[:8000]


def step_rows(repo, parent, child, n, blind, renames):
    """The rows of one commit without the lead columns, from the reference."""
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
    res = cr.churn(old, new, [a for a, _ in pairs], [b for _, b in pairs], n, blind)
    rows = []
    for side, sign, paths in (("old", "-", po_), ("new", "+", pn_)):
        s = res[side]
        base = s["line_base"]
        fbase = s["kept_base"] if blind else base
        for c in range(len(s["class_len"])):
            if s["status"][c] == 0:
                continue
            b0, b1 = s["class_base"][c], s["class_base"][c + 1]
            L = int(s["class_len"][c])
            for j in range(b0, b1):
                m = int(s["member"][j])
                f = max(k for k in range(len(paths)) if fbase[k] <= m)
                first, last = (s["kept_line"][m], s["kept_line"][m + L - 1]) if blind else (m, m + L - 1)
                rows.append([sign, str(c + 1), cr.STATUSES[s["status"][c]], str(b1 - b0), paths[f], str(first - base[f] + 1),
                             str(last - base[f] + 1), cr.STATES[s["state"][j]], str(s["changed"][j]), str(s["changed_assert"][j])])
    return rows


def run(*args):
    r = subprocess.run([CLI] + [str(a) for a in args], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return r


def read(path):
    return list(csv.reader(open(path, newline="", encoding="latin-1")))


def want(repo, chain, n, blind, renames):
    out = []
    for c, p, t in chain:
        for r in step_rows(repo, p, c, n, blind, renames):
            out.append([c, p, t] + r)
    return out


@pytest.mark.parametrize("blind", [False, True])
@pytest.mark.parametrize("renames", [False, True])
def test_history_rows_equal_the_restatement(repo, tmp_path, blind, renames):
    out = tmp_path / "c.csv"
    args = ["history", repo, "--clones", out] + (["--blind"] if blind else []) + (["--find-renames", 50] if renames else [])
    run(*args)
    table = read(out)
    assert table[0] == ["commit", "parent", "time"] + HEAD
    assert table[1:] == want(repo, commits(repo), 5, blind, renames)
    statuses = {r[5] for r in table[1:]}
    assert {"copied", "diverged", "changed", "dropped"} <= statuses, statuses
    by_msg = {c: git(repo, "log", "-1", "--format=%s", c).strip() for c, _, _ in commits(repo)}
    rename_rows = [r for r in table[1:] if by_msg[r[0]].startswith("rename")]
    assert (rename_rows == []) == renames                  # an exact rename under -M touches nothing
    binary_rows = [r for r in table[1:] if by_msg[r[0]].startswith("modify the binary")]
    assert any(r[7] == "tests/test_bin.py" and r[10] == "whole" for r in binary_rows)


def test_max_commits_window_and_min_lines(repo, tmp_path):
    out = tmp_path / "w.csv"
    run("history", repo, "--max-commits", 4, "--min-lines", 3, "--clones", out)
    assert read(out)[1:] == want(repo, commits(repo)[-4:], 3, False, False)


def test_rows_match_clones_out(repo, tmp_path):
    out = tmp_path / "c.csv"
    run("history", repo, "--clones", out)
    table = read(out)[1:]
    frags = {}
    for rev in {r[1] if r[3] == "-" else r[0] for r in table}:
        f = tmp_path / ("f_%s.csv" % rev)
        run("clones", "--git", repo, "--rev", rev, "--out", f)
        frags[rev] = {(r[0], r[2], r[3], r[4]) for r in read(f)[1:]}
    for r in table:
        rev = r[1] if r[3] == "-" else r[0]
        assert (r[4], r[7], r[8], r[9]) in frags[rev], r


def checkout(repo, rev, dest):
    os.makedirs(dest)
    data = git(repo, "archive", "--format=tar", rev, text=False)
    with tarfile.open(fileobj=io.BytesIO(data)) as t:
        t.extractall(dest, filter="data")


def test_diff_equals_the_commit_rows(repo, tmp_path):
    hist = tmp_path / "h.csv"
    run("history", repo, "--clones", hist, "--find-renames", 50)
    table = read(hist)[1:]
    for c, p, _ in commits(repo)[1:]:
        checkout(repo, p, tmp_path / ("o_" + c))
        checkout(repo, c, tmp_path / ("n_" + c))
        out = tmp_path / ("d_%s.csv" % c)
        run("diff", tmp_path / ("o_" + c), tmp_path / ("n_" + c), "--clones", out, "--find-renames", 50)
        got = read(out)
        assert got[0] == HEAD
        assert got[1:] == [r[3:] for r in table if r[0] == c], c


def test_other_outputs_are_unchanged(repo, tmp_path):
    a, b = tmp_path / "a.csv", tmp_path / "b.csv"
    r1 = run("history", repo, "--out", a)
    r2 = run("history", repo, "--out", b, "--clones", tmp_path / "c.csv")
    assert open(a, "rb").read() == open(b, "rb").read() and r1.stdout == r2.stdout
