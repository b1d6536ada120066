"""`tosem-scan history --moves` and `diff --moves` (docs/SPEC.md section 20) on the planted history of tests/move_repo.py: every
row equals move_ref.py_moves over the `git cat-file` blobs of each commit and agrees with git's `--color-moved=blocks`, also in
batches of 4 KiB and after `git gc --aggressive`; `diff` of two `git archive` checkouts gives the commit's rows; under
`--find-renames 50` an edited rename moves only the lines the pair does not keep; every other output is byte-identical with and
without `--moves`."""
import csv
import os
import shutil
import subprocess
import tarfile

import pytest

import move_ref as mr
import move_repo as rp
from test_history import CLI, git

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

HEAD = ["commit", "parent", "time", "fileName", "change", "line", "lines", "asserts", "otherFileName", "otherLine"]


def commits(repo):
    out = []
    for entry in filter(None, git(repo, "log", "--first-parent", "--reverse", "--format=%H %P %ct").split("\n")):
        p = entry.split()
        out.append((p[0], p[1] if len(p) > 2 else "", p[-1]))
    return out


def want_rows(repo):
    """The rows of move_ref.py_moves over the blobs of every commit's changed files (no renames), pair by pair."""
    out = []
    for commit, parent, time in commits(repo):
        if not parent:
            continue                                             # the root commit only adds: nothing moves
        paths = rp.changed_paths(repo, parent, commit)
        res = mr.py_moves([(rp.blob(repo, parent, p), rp.blob(repo, commit, p), 1, 1) for p in paths])
        for i, p in enumerate(paths):
            for s, sign in (("old", "-"), ("new", "+")):
                o = "new" if s == "old" else "old"
                here, there = res[s]["base"], res[o]["base"]
                for line, partner, n, a in res[s]["blocks"]:
                    if here[i] <= line < here[i + 1]:
                        j = max(k for k in range(len(paths)) if there[k] <= partner)
                        out.append([commit, parent, time, p, sign, str(line - here[i] + 1), str(n), str(a), paths[j],
                                    str(partner - there[j] + 1)])
    return out


def run(*args):
    r = subprocess.run([CLI] + [str(a) for a in args], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return r


def read(path):
    return list(csv.reader(open(path, newline="", encoding="latin-1")))


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    r = tmp_path_factory.mktemp("moves") / "repo"
    rp.build(str(r))
    return r


def test_history_moves_equal_the_reference_and_git(repo, tmp_path):
    out = tmp_path / "m.csv"
    run("history", repo, "--moves", out)
    table = read(out)
    assert table[0] == HEAD
    assert table[1:] == want_rows(repo) and len(table) > 20
    for commit, parent, _ in commits(repo)[1:]:                     # the moved lines are git's
        paths = rp.changed_paths(repo, parent, commit)
        g = rp.git_moved(repo, parent, commit, paths)
        mine = {p: (set(), set()) for p in paths}
        for r in table[1:]:
            if r[0] == commit:
                mine[r[3]][r[4] == "+"].update(range(int(r[5]) - 1, int(r[5]) - 1 + int(r[6])))
        assert mine == {p: (g.get(p, (set(), set()))[0], g.get(p, (set(), set()))[1]) for p in paths}, commit
    for bb in (4096, 64):                                           # 64 bytes: every commit larger than a batch, one per batch
        small = tmp_path / ("m%d.csv" % bb)
        run("history", repo, "--moves", small, "--batch-bytes", bb)
        assert open(small, "rb").read() == open(out, "rb").read()
    git(repo, "gc", "-q", "--aggressive")
    out2 = tmp_path / "m2.csv"
    run("history", repo, "--moves", out2)
    assert open(out2, "rb").read() == open(out, "rb").read()


def test_find_renames_moves_only_what_the_pair_does_not_keep(repo, tmp_path):
    out, plain = tmp_path / "r.csv", tmp_path / "p.csv"
    run("history", repo, "--moves", out, "--find-renames", "50")
    run("history", repo, "--moves", plain)
    c = commits(repo)[-1][0]
    mine = [r[3:] for r in read(out)[1:] if r[0] == c]
    assert mine == [["test_ren_dst.py", "+", "2", "1", "1", "test_ren_old.py", "11"],     # the pairs in new path order
                    ["test_ren_old.py", "-", "11", "1", "1", "test_ren_dst.py", "2"]]
    before = [r[3:] for r in read(plain)[1:] if r[0] == c]           # without the pairing the whole file moves
    assert ["test_ren_old.py", "-", "1", "10", "0", "test_ren_new.py", "1"] in before


def test_outputs_are_byte_identical_with_and_without_moves(repo, tmp_path):
    flags = {"out": "--out", "asserts": "--asserts", "churn": "--assert-churn", "cases": "--cases", "edits": "--assert-edits",
             "smells": "--smells"}
    for extra in ([], ["--find-renames", "50"], ["--batch-bytes", "4096"]):
        tag = "".join(extra).replace("-", "")
        a = {k: tmp_path / ("a_%s_%s.csv" % (k, tag)) for k in flags}
        b = {k: tmp_path / ("b_%s_%s.csv" % (k, tag)) for k in flags}
        ra = run("history", repo, *[x for k in flags for x in (flags[k], a[k])], "--moves", tmp_path / ("mv_%s.csv" % tag), *extra)
        rb = run("history", repo, *[x for k in flags for x in (flags[k], b[k])], *extra)
        assert ra.stdout == rb.stdout
        for k in flags:
            assert open(a[k], "rb").read() == open(b[k], "rb").read(), (k, extra)


def test_diff_of_archives_gives_the_commit_rows(repo, tmp_path):
    c = commits(repo)
    hist = tmp_path / "h.csv"
    run("history", repo, "--moves", hist)
    table = read(hist)
    roots = {}
    for rev in (c[1][1], c[1][0]):                                  # the "two files" commit and its parent
        d = tmp_path / ("tree_%s" % rev[:8])
        os.makedirs(d)
        tar = tmp_path / ("t_%s.tar" % rev[:8])
        tar.write_bytes(git(repo, "archive", "--format=tar", rev, text=False))
        with tarfile.open(tar) as t:
            t.extractall(d, filter="data")
        roots[rev] = str(d)
    out = tmp_path / "d.csv"
    a = run("diff", roots[c[1][1]], roots[c[1][0]], "--moves", out, "--batch-bytes", 64)
    got = read(out)
    assert got[0] == HEAD[3:]
    want = [r[3:] for r in table[1:] if r[0] == c[1][0]]
    assert got[1:] == want and len(want) == 4
    b = run("diff", roots[c[1][1]], roots[c[1][0]])
    assert a.stdout == b.stdout
