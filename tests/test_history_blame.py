"""`tosem-scan blame` (docs/SPEC.md section 14) on a repository built here: every --out row equals `git blame --line-porcelain
--first-parent --minimal` (commit, original file name, original line, boundary) for every selected file, at HEAD and at an older
revision, over windows cut by --max-commits (boundary rows), with --find-renames 50 across a move, after `git gc --aggressive`
and with batches of one change (chains of origins carried between batches on the host).  --asserts equals the --out rows of the
spec_ref assertion lines with their statement and category; stdout equals the rows aggregated per commit."""
import collections
import csv
import os
import shutil
import subprocess

import pytest

import spec_ref
import tosemscan as ts
from test_blame_ref import build_history, git, git_blame

HERE = os.path.dirname(os.path.abspath(__file__))
CLI = os.path.join(HERE, "..", "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs git")]


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    """build_history's repository plus one commit that inserts assertion lines into every file."""
    r = str(tmp_path_factory.mktemp("blame") / "r")
    os.makedirs(r)
    build_history(r)
    env = dict(os.environ, GIT_AUTHOR_NAME="t", GIT_AUTHOR_EMAIL="t@e", GIT_COMMITTER_NAME="t", GIT_COMMITTER_EMAIL="t@e",
               GIT_AUTHOR_DATE="1600000100 +0000", GIT_COMMITTER_DATE="1600000100 +0000")
    for k, p in enumerate(sorted(git(r, "ls-files").decode().split())):
        lines = open(os.path.join(r, p), "rb").read().split(b"\n")
        for j in range(2, len(lines), 7):
            lines.insert(j, b"    self.assertEqual(v%d_%d, %d)" % (k, j, j) if j % 2 else b"    assert w%d_%d > 0" % (k, j))
        open(os.path.join(r, p), "wb").write(b"\n".join(lines))
    git(r, "commit", "-q", "-a", "-m", "asserts", env=env)
    return r


def run_blame(repo, tmp, *args):
    out, asserts = os.path.join(tmp, "o.csv"), os.path.join(tmp, "a.csv")
    r = subprocess.run([CLI, "blame", repo, "--out", out, "--asserts", asserts] + list(args), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(out, newline="") as f:
        rows = list(csv.reader(f))
    with open(asserts, newline="") as f:
        arows = list(csv.reader(f))
    return rows, arows, r.stdout


def check(repo, tmp, rev, *args, window=None, min_asserts=10):
    rows, arows, stdout = run_blame(repo, tmp, "--rev", rev, *args)
    assert rows[0] == ["fileName", "line", "commit", "time", "origFileName", "origLine", "boundary"]
    by_path = collections.defaultdict(list)
    for r in rows[1:]:
        by_path[r[0]].append(r)
    paths = [p for p in git(repo, "ls-tree", "-r", "--name-only", rev).decode().split() if "test" in p and p.endswith(".py")]
    assert sorted(by_path) == sorted(paths)
    rng = "%s~%d..%s" % (rev, window, rev) if window else rev
    times = {}
    for p in paths:
        want = git_blame(repo, rng, p, window is None)
        got = by_path[p]
        assert [int(r[1]) for r in got] == list(range(1, len(want) + 1))
        assert [(r[2], r[4], int(r[5]), int(r[6])) for r in got] == want, p
        for r in got:
            times[r[2]] = r[3]
    for sha, t in times.items():
        assert t == git(repo, "show", "-s", "--format=%ct", sha).decode().strip()
    # --asserts: the rows of the assertion lines (spec_ref) with their statement and category
    assert arows[0] == rows[0] + ["statement", "category"]
    want_a = []
    for p in sorted(by_path, key=lambda q: [r[0] for r in rows[1:]].index(q)):
        text = git(repo, "show", "%s:%s" % (rev, p))
        for j, line in enumerate(spec_ref.py_lines(text)):
            if spec_ref.py_is_assert_line(line, ts.EXT["py"]):
                stmt = spec_ref.py_statement(line)
                cat = spec_ref.py_category(stmt)
                want_a.append(by_path[p][j] + [stmt.decode(), spec_ref.py_category_string(stmt) if cat == 127 else ts.category_name(cat)])
    assert arows[1:] == want_a and len(want_a) >= min_asserts
    # stdout: lines and assertion lines per commit, window order, the boundary commit first
    order = git(repo, "rev-list", "--first-parent", "--reverse", rng if window else rev).decode().split()
    if window:
        order = [git(repo, "rev-parse", "%s~%d" % (rev, window)).decode().strip()] + order
    lines, asserts = collections.Counter(r[2] for r in rows[1:]), collections.Counter(r[2] for r in arows[1:])
    want_out = ["commit,lines,asserts"] + ["%s,%d,%d" % (c, lines[c], asserts[c]) for c in order if lines[c]]
    assert stdout.splitlines() == want_out
    return rows


def test_blame_head_and_older_revision(repo, tmp_path):
    check(repo, str(tmp_path), "HEAD", "--find-renames", "50")
    older = git(repo, "rev-parse", "HEAD~6").decode().strip()
    check(repo, str(tmp_path), older, min_asserts=0)        # before the move (no rename) and the assertion lines


def test_blame_windows(repo, tmp_path):
    for n in (1, 3, 6):                                     # the window of 6 commits holds the move
        rows = check(repo, str(tmp_path), "HEAD", "--find-renames", "50", "--max-commits", str(n), window=n)
        assert any(r[6] == "1" for r in rows[1:]) and any(r[6] == "0" for r in rows[1:])


def test_blame_small_batches_and_packed(repo, tmp_path):
    want = run_blame(repo, str(tmp_path), "--find-renames", "50")
    assert run_blame(repo, str(tmp_path), "--find-renames", "50", "--batch-bytes", "1") == want
    check(repo, str(tmp_path), "HEAD", "--find-renames", "50", "--batch-bytes", "1")
    check(repo, str(tmp_path), "HEAD", "--find-renames", "50", "--max-commits", "4", "--batch-bytes", "300", window=4)
    git(repo, "gc", "-q", "--aggressive")
    assert run_blame(repo, str(tmp_path), "--find-renames", "50") == want
