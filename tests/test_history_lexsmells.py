"""`tosem-scan history --smells F --lexical` and `diff --smells F --lexical` (docs/SPEC.md section 26) on a repository built here
from the scenarios of tests/test_lexsmell_churn_ref.py: every row equals lexsmell_churn_ref.py_lexsmell_churn over the
`git cat-file` blobs of each commit, also in batches of 4 KiB; `diff` of two `git archive` checkouts gives the commit's rows;
`--find-renames 50` turns an edited move into M rows; every other output, and `--smells` without `--lexical`, is byte-identical
with and without `--lexical`."""
import os
import shutil
import tarfile

import pytest

import lexsmell_churn_ref as lcr
from test_history import EMPTY_TREE, git
from test_history_smells import HEAD, blob, cells, commits, ext_of, read, run, selected
from test_lexsmell_churn_ref import CASES

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

SUFFIX = {1: "py", 2: "cc"}


def build(root):
    """Commit 1: the old side of every scenario whose two sides share a tag; commit 2: the new sides; commit 3: an edited move
    that adds a magic number; commit 4: one file deleted."""
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
    files["tests/test_move.py"] = b"".join(b"def test_m%d(self):\n    v = %d\n    assert v, 'm'\n" % (i, i) for i in range(12))
    commit("old sides")
    for k, (_, _, new, x, _, _) in enumerate(same):
        files["tests/test_s%02d.%s" % (k, SUFFIX[x])] = new
    commit("new sides")
    m = files.pop("tests/test_move.py")
    files["tests/moved/test_move.py"] = m.replace(b"    v = 3\n", b"    v = 3\n    assert v == 42, 'm'\n")
    commit("move with an edit")
    files.pop("tests/test_s00.py")
    commit("delete")
    return repo


def want_rows(repo):
    """Rows of py_lexsmell_churn over the blobs of every changed selected file (no renames), per commit in path order."""
    out = []
    for commit, parent, time in commits(repo):
        names = git(repo, "diff", "--name-only", "--no-renames", "-z", parent or EMPTY_TREE, commit).split("\0")
        for path in sorted(n for n in names if n and selected(n)):
            for r in lcr.py_lexsmell_churn(blob(repo, parent, path), blob(repo, commit, path), ext_of(path), ext_of(path)):
                out.append([commit, parent, time, path] + cells(r))
    return out


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    return build(tmp_path_factory.mktemp("lexsmells"))


def test_history_lexical_smells_equal_the_reference(repo, tmp_path):
    out = tmp_path / "s.csv"
    run("history", repo, "--smells", out, "--lexical")
    table = read(out)
    assert table[0] == HEAD
    assert table[1:] == want_rows(repo)
    events = {(r[5], r[9]) for r in table[1:] if r[8] in lcr.lr.LSMELLS}
    assert {("A", "introduced"), ("D", "removed"), ("M", "introduced"), ("M", "removed"), ("M", "changed")} <= events
    assert {r[8] for r in table[1:]} >= set(lcr.lr.LSMELLS)
    small = tmp_path / "s4k.csv"
    run("history", repo, "--smells", small, "--lexical", "--batch-bytes", 4096)
    assert open(small, "rb").read() == open(out, "rb").read()


def test_find_renames_gives_m_rows_for_an_edited_move(repo, tmp_path):
    out = tmp_path / "r.csv"
    run("history", repo, "--smells", out, "--lexical", "--find-renames", "50")
    table = read(out)
    assert table[0] == HEAD + ["oldFileName"]
    c = commits(repo)
    mine = [r for r in table[1:] if r[0] == c[2][0]]
    assert mine == [[c[2][0], c[1][0], c[2][2], "tests/moved/test_move.py", "test_m3", "M", "10", "10", "magic_number",
                     "introduced", "1", "0", "1", "0", "tests/test_move.py"]]


def test_outputs_are_byte_identical_with_and_without_lexical(repo, tmp_path):
    flags = {"out": "--out", "asserts": "--asserts", "churn": "--assert-churn", "cases": "--cases", "edits": "--assert-edits",
             "moves": "--moves", "clones": "--clones", "similar": "--similar-tests"}
    for extra in ([], ["--find-renames", "50"]):
        a = {k: tmp_path / ("a_%s%d.csv" % (k, len(extra))) for k in flags}
        b = {k: tmp_path / ("b_%s%d.csv" % (k, len(extra))) for k in flags}
        ra = run("history", repo, *[x for k in flags for x in (flags[k], a[k])], "--lexical", *extra)
        rb = run("history", repo, *[x for k in flags for x in (flags[k], b[k])], *extra)
        assert ra.stdout == rb.stdout
        for k in flags:
            assert open(a[k], "rb").read() == open(b[k], "rb").read(), k
        lex, plain, base = (tmp_path / ("%s%d.csv" % (n, len(extra))) for n in ("lex", "plain", "base"))
        rl = run("history", repo, "--smells", lex, "--cases", tmp_path / "lc.csv", "--lexical", *extra)
        run("history", repo, "--smells", plain, *extra)
        rp = run("history", repo, "--smells", base, "--cases", tmp_path / "pc.csv", *extra)
        assert rl.stdout == rp.stdout and open(tmp_path / "lc.csv", "rb").read() == open(tmp_path / "pc.csv", "rb").read()
        assert open(plain, "rb").read() == open(base, "rb").read()
        nine = [r for r in read(lex) if r[8] not in lcr.lr.LSMELLS]   # the lexical rows come on top of the nine
        assert nine == read(plain)


def test_diff_of_archives_gives_the_commit_rows(repo, tmp_path):
    c = commits(repo)
    hist = tmp_path / "h.csv"
    run("history", repo, "--smells", hist, "--lexical")
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
    a = run("diff", roots[c[0][0]], roots[c[1][0]], "--smells", out, "--lexical")
    got = read(out)
    assert got[0] == HEAD[3:]
    want = [r[3:] for r in table[1:] if r[0] == c[1][0]]
    assert got[1:] == want and len(want) >= 10
    b = run("diff", roots[c[0][0]], roots[c[1][0]])
    assert a.stdout == b.stdout
