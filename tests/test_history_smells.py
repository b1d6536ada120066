"""`tosem-scan history --smells` and `diff --smells` (docs/SPEC.md section 19) on a repository built here from the scenarios of
tests/test_smell_churn_ref.py: every row equals smell_churn_ref.py_smell_churn over the `git cat-file` blobs of each commit, also
after `git gc --aggressive` and in batches of 4 KiB, `diff` of two `git archive` checkouts gives the commit's rows,
`--find-renames 50` turns an edited move into M rows, and every other output is byte-identical with and without `--smells`."""
import csv
import os
import shutil
import subprocess
import tarfile

import pytest

import smell_churn_ref as scr
from test_history import CLI, EMPTY_TREE, git
from test_smell_churn_ref import CASES

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

EXT = {"py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}
SUFFIX = {1: "py", 2: "cc"}
HEAD = ["commit", "parent", "time", "fileName", "test", "change", "line", "oldLine", "smell", "event", "instances", "oldInstances",
        "addedInstances", "removedInstances"]


def ext_of(path):
    name = path.rsplit("/", 1)[-1]
    return EXT.get(name.rsplit(".", 1)[-1], 0) if "." in name else 0


def selected(path):
    return "test" in path.lower() and ext_of(path) != 0


def build(root):
    """Commit 1: the old side of every scenario whose two sides share a tag; commit 2: the new sides; commit 3: an edited move
    that adds a print; commit 4: one file deleted."""
    repo = root / "repo"
    os.makedirs(repo)
    git(repo, "init", "-q", ".")
    files = {}

    def commit(msg):
        for dp, _, fns in os.walk(repo):
            if ".git" in dp:
                continue
            for fn in fns:
                rel = os.path.relpath(os.path.join(dp, fn), repo)
                if rel not in files:
                    os.remove(os.path.join(dp, fn))
        for nm, data in files.items():
            os.makedirs(os.path.dirname(repo / nm), exist_ok=True)
            (repo / nm).write_bytes(data)
        git(repo, "add", "-A")
        git(repo, "commit", "-q", "--allow-empty", "-m", msg)

    same = [c for c in CASES if c[3] == c[4]]
    for k, (_, old, _, x, _, _) in enumerate(same):
        files["tests/test_s%02d.%s" % (k, SUFFIX[x])] = old
    files["tests/test_move.py"] = b"".join(b"def test_m%d(self):\n    v = %d\n    assert v\n" % (i, i) for i in range(12))
    commit("old sides")
    for k, (_, _, new, x, _, _) in enumerate(same):
        files["tests/test_s%02d.%s" % (k, SUFFIX[x])] = new
    commit("new sides")
    m = files.pop("tests/test_move.py")
    files["tests/moved/test_move.py"] = m.replace(b"    v = 3\n", b"    v = 3\n    print(v)\n")
    commit("move with an edit")
    files.pop("tests/test_s00.py")
    commit("delete")
    return repo


def commits(repo):
    out = []
    for entry in filter(None, git(repo, "log", "--first-parent", "--reverse", "--format=%H %P %ct").split("\n")):
        p = entry.split()
        out.append((p[0], p[1] if len(p) > 2 else "", p[-1]))
    return out


def blob(repo, rev, path):
    if not rev:
        return b""
    try:
        return git(repo, "cat-file", "blob", "%s:%s" % (rev, path), text=False)
    except subprocess.CalledProcessError:
        return b""


def cells(row):
    return [("" if x is None else x.decode("latin-1") if isinstance(x, bytes) else str(x)) for x in row]


def want_rows(repo):
    """Rows of smell_churn_ref.py_smell_churn over the blobs of every changed selected file (no renames), per commit in path order."""
    out = []
    for commit, parent, time in commits(repo):
        names = git(repo, "diff", "--name-only", "--no-renames", "-z", parent or EMPTY_TREE, commit).split("\0")
        for path in sorted(n for n in names if n and selected(n)):
            for r in scr.py_smell_churn(blob(repo, parent, path), blob(repo, commit, path), ext_of(path), ext_of(path)):
                out.append([commit, parent, time, path] + cells(r))
    return out


def run(*args):
    r = subprocess.run([CLI] + [str(a) for a in args], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return r


def read(path):
    return list(csv.reader(open(path, newline="", encoding="latin-1")))


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    return build(tmp_path_factory.mktemp("smells"))


def test_history_smells_equal_the_reference(repo, tmp_path):
    out = tmp_path / "s.csv"
    run("history", repo, "--smells", out)
    table = read(out)
    assert table[0] == HEAD
    want = want_rows(repo)
    assert table[1:] == want
    events = {(r[5], r[9]) for r in table[1:]}
    assert {("A", "introduced"), ("D", "removed"), ("M", "introduced"), ("M", "removed"), ("M", "changed")} <= events
    small = tmp_path / "s4k.csv"
    run("history", repo, "--smells", small, "--batch-bytes", 4096)
    assert open(small, "rb").read() == open(out, "rb").read()
    git(repo, "gc", "-q", "--aggressive")
    out2 = tmp_path / "s2.csv"
    run("history", repo, "--smells", out2)
    assert open(out2, "rb").read() == open(out, "rb").read()


def test_find_renames_gives_m_rows_for_an_edited_move(repo, tmp_path):
    out = tmp_path / "r.csv"
    run("history", repo, "--smells", out, "--find-renames", "50")
    table = read(out)
    assert table[0] == HEAD + ["oldFileName"]
    c = commits(repo)
    mine = [r for r in table[1:] if r[0] == c[2][0]]
    assert mine == [[c[2][0], c[1][0], c[2][2], "tests/moved/test_move.py", "test_m3", "M", "10", "10", "print", "introduced",
                     "1", "0", "1", "0", "tests/test_move.py"]]
    plain = {tuple(r[:14]) for r in table[1:] if "move" not in r[3]}
    assert plain == {tuple(r) for r in want_rows(repo) if "move" not in r[3]}


def test_outputs_are_byte_identical_with_and_without_smells(repo, tmp_path):
    for extra in ([], ["--find-renames", "50"]):
        keys = ("out", "asserts", "churn", "cases")
        flags = {"out": "--out", "asserts": "--asserts", "churn": "--assert-churn", "cases": "--cases"}
        a = {k: tmp_path / ("a_%s%d.csv" % (k, len(extra))) for k in keys}
        b = {k: tmp_path / ("b_%s%d.csv" % (k, len(extra))) for k in keys}
        sm = tmp_path / ("sm%d.csv" % len(extra))
        ra = run("history", repo, *[x for k in keys for x in (flags[k], a[k])], "--smells", sm, *extra)
        rb = run("history", repo, *[x for k in keys for x in (flags[k], b[k])], *extra)
        assert ra.stdout == rb.stdout
        for k in keys:
            assert open(a[k], "rb").read() == open(b[k], "rb").read(), k
        alone = tmp_path / ("alone%d.csv" % len(extra))
        rc = run("history", repo, "--smells", alone, *extra)
        assert rc.stdout == rb.stdout and open(alone, "rb").read() == open(sm, "rb").read()
        cases = tmp_path / ("c%d.csv" % len(extra))
        run("history", repo, "--smells", alone, "--cases", cases, *extra)
        assert open(cases, "rb").read() == open(a["cases"], "rb").read()


def test_diff_of_archives_gives_the_commit_rows(repo, tmp_path):
    c = commits(repo)
    hist = tmp_path / "h.csv"
    run("history", repo, "--smells", hist)
    table = read(hist)
    roots = {}
    for rev in (c[0][0], c[1][0]):
        d = tmp_path / ("tree_%s" % rev[:8])
        os.makedirs(d)
        tar = tmp_path / ("t_%s.tar" % rev[:8])
        tar.write_bytes(git(repo, "archive", "--format=tar", rev, text=False))
        with tarfile.open(tar) as t:
            t.extractall(d, filter="data")
        roots[rev] = str(d)
    out = tmp_path / "d.csv"
    a = run("diff", roots[c[0][0]], roots[c[1][0]], "--smells", out)
    got = read(out)
    assert got[0] == HEAD[3:]
    want = [r[3:] for r in table[1:] if r[0] == c[1][0]]
    assert got[1:] == want and len(want) >= 10
    b = run("diff", roots[c[0][0]], roots[c[1][0]])
    assert a.stdout == b.stdout
