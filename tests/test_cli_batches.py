"""The batch loops of `tosem-scan`.  Scans: on the C1 test files (tests/golden/c1_testfiles.npz) in nine roots, `scan`, `body` and
`releases` give byte-identical stdout and files with the default batch size and with a `--batch-bytes` that cuts the tree into
dozens of batches (counters and walk order carried across batches, one context per command); and every command prints its empty
result for a tree with no selected file.  Revision pairs: `history` and `diff` with every output and rename pairing give the same
bytes whether their pairs go in one batch, a few or one per batch, and a history of more than 65 535 commits gives the same
assertion churn when its batches are cut at the group limit as when they are cut every few hundred commits."""
import csv
import os
import shutil
import subprocess
import tarfile

import pytest

import corpus_util as cu
import test_history_cases
import test_history_renames
from test_history import git

pytestmark = pytest.mark.gpu
needs_git = pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
SMALL = "200000"                                           # C1 is 10.55 MB: about 55 batches


def write(root, files):
    for rel, data in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(data)


@pytest.fixture(scope="module")
def c1():
    names = cu.load_fixture_names(os.path.join(GOLD, "c1_testfiles.npz"))
    files, _, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    return dict(zip(names, files))


@pytest.fixture(scope="module")
def c1_roots(tmp_path_factory, c1):
    """One root per project of C1 (nine), so that the count table has a group per root."""
    top = str(tmp_path_factory.mktemp("c1"))
    write(top, c1)
    return [os.path.join(top, p) for p in sorted({n.split("/")[0] for n in c1})]


def run(args, outs):
    """stdout, the last stderr line and the bytes of every output file of one CLI call."""
    p = subprocess.run([CLI] + args, capture_output=True)
    assert p.returncode == 0, p.stderr.decode()
    return p.stdout, p.stderr.decode().strip().split("\n")[-1], [open(o, "rb").read() for o in outs]


def default_and_small(tmp_path, cmd, args, flags, sizes=(SMALL,)):
    """One run with the default batch size and one per `--batch-bytes` of `sizes`: all give the same bytes."""
    got = []
    for tag, extra in [("default", [])] + [("b%s" % s, ["--batch-bytes", s]) for s in sizes]:
        outs = [str(tmp_path / ("%s_%s.csv" % (tag, f.lstrip("-")))) for f in flags]
        opts = [x for f, o in zip(flags, outs) for x in (f, o)]
        got.append(run([cmd] + args + opts + extra, outs))
    for g in got[1:]:
        assert g == got[0]
    return got[0]


def test_scan_batches(tmp_path, c1_roots):
    stdout, summary, (rows, summ) = default_and_small(tmp_path, "scan", c1_roots, ["--rows", "--summary"])
    assert summary.startswith("tosem-scan: lines=") and summ.count(b"\r\n") == 1779 + 1 and rows.count(b"\r\n") > 1779


def test_body_batches(tmp_path, c1_roots):
    stdout, _, (out,) = default_and_small(tmp_path, "body", c1_roots, ["--out"])
    files, cases, stmts = (int(x) for x in stdout.decode().split("\r\n")[1].split(","))
    assert files == 1779 and cases > 1000 and out.count(b"\r\n") >= 1 + cases + stmts


def test_releases_batches(tmp_path, c1):
    """Three snapshots of C1: v2 moves every 7th file and edits every 5th, v3 drops every 11th, moves and edits every 13th and adds
    files; identities by path, by content and by base name must not depend on where the batches are cut."""
    names = sorted(c1)
    v1 = dict(c1)
    v2 = {}
    for i, n in enumerate(names):
        data = c1[n] + (b"\nassert edited_%d\n" % i if i % 5 == 0 else b"")
        v2["moved/" + n if i % 7 == 0 else n] = data
    v3 = {}
    for i, (n, data) in enumerate(sorted(v2.items())):
        if i % 11 == 0:
            continue
        v3["later/" + n.replace("/", "_") if i % 13 == 0 else n] = data + (b"    assert later\n" if i % 13 == 0 else b"")
    v3.update({"new_tests/test_%d.py" % k: b"def test_k():\n    assert %d == %d\n" % (k, k) for k in range(40)})
    specs = []
    for tag, snap in (("v1", v1), ("v2", v2), ("v3", v3)):
        write(str(tmp_path / tag), snap)
        specs.append("%s=%s" % (tmp_path / tag, tag))
    stdout, _, (out,) = default_and_small(tmp_path, "releases", specs, ["--out"])
    ids = int(stdout.decode().split("\r\n")[1].split(",")[0])
    assert ids > len(names) and out.count(b"\r\n") == 1 + ids


@pytest.fixture
def empty(tmp_path):
    """A tree without a selected file: no `test` in the path, or no scannable extension."""
    root = tmp_path / "proj"
    write(str(root), {"src/main.py": b"assert False\n", "tests/data.json": b'{"assert": 1}\n'})
    return str(root)


def test_empty_selection(tmp_path, empty):
    rows, summ, out = str(tmp_path / "rows.csv"), str(tmp_path / "sum.csv"), str(tmp_path / "out.csv")
    stdout, summary, files = run(["scan", empty, "--rows", rows, "--summary", summ], [rows, summ])
    assert stdout == b"category,count\r\n"
    assert summary == "tosem-scan: lines=0 assertion_lines=0 headers=0 fixture_headers=0 on 1 GPU(s), shares 0..0 bytes"
    assert files == [b"fileName,extension,test_name,method,statement,counts,category\r\n", b"Id,FileName,total assert,assertion\r\n"]
    stdout, _, files = run(["body", empty, "--out", out], [out])
    assert stdout == b"files,cases,statements\r\n0,0,0\r\n" and files == [b"Index,text,Category,cases,File_ID,Component\r\n"]
    stdout, _, files = run(["releases", empty + "=v1", "--out", out], [out])
    assert stdout == b"identities,snapshots\r\n0,1\r\n" and files == [b"Id,FileName,v1,total assert,assertion\r\n"]
    stdout, _, files = run(["clones", empty, "--out", out], [out])
    assert stdout == (b"repository,files,lines,duplicated_lines,assertion_lines,duplicated_assertion_lines,classes\r\n"
                      b"proj,0,0,0,0,0,0\r\n<all>,0,0,0,0,0,0\r\n")
    assert files == [b"class,repository,fileName,first_line,last_line\r\n"]


PAIR_FLAGS = ["--out", "--asserts", "--assert-churn", "--cases"]
PAIR_SIZES = ("1", "3000")                                 # one pair per batch; a few pairs per batch


@pytest.fixture(scope="module", params=["renames", "cases"])
def history_repo(request, tmp_path_factory):
    """The repositories of test_history_renames.py (pure, edited and base-name moves) and test_history_cases.py (cases added,
    deleted, edited and moved)."""
    build = {"renames": test_history_renames.build, "cases": test_history_cases.build}[request.param]
    return build(tmp_path_factory.mktemp(request.param))


@needs_git
def test_history_pair_batches(tmp_path, history_repo):
    stdout, last, files = default_and_small(tmp_path, "history", [str(history_repo), "--find-renames", "50"], PAIR_FLAGS, PAIR_SIZES)
    assert stdout.count(b"\r\n") == 1 + len(git(history_repo, "rev-list", "HEAD").split())
    assert last.startswith("tosem-scan: ") and "rename(s) found at 50%" in last
    assert all(f.count(b"\r\n") > 1 for f in files[:3])     # (the renames repository has no test case headers)


@needs_git
def test_diff_pair_batches(tmp_path, history_repo):
    """`diff` of `git archive` checkouts of the first and the last commit."""
    revs = git(history_repo, "rev-list", "--first-parent", "--reverse", "HEAD").split()
    roots = []
    for rev in (revs[0], revs[-1]):
        d = tmp_path / ("tree_" + rev[:8])
        os.makedirs(d)
        tar = tmp_path / ("t_%s.tar" % rev[:8])
        tar.write_bytes(git(history_repo, "archive", "--format=tar", rev, text=False))
        with tarfile.open(tar) as t:
            t.extractall(d, filter="data")
        roots.append(str(d))
    stdout, last, files = default_and_small(tmp_path, "diff", roots + ["--find-renames", "50"], PAIR_FLAGS, PAIR_SIZES)
    assert stdout.startswith(b"cloc,added,removed\r\n") and "rename(s) found (" in last
    assert all(f.count(b"\r\n") > 1 for f in files[:3])


@needs_git
def test_history_past_the_group_limit(tmp_path):
    """65 540 commits, each rewriting the assertion line of one test file: the default batch size cuts the history at 65 535
    commits (a batch's assertion tables have u16 groups), --batch-bytes 100000 every 300 or so.  The churn must not depend on the
    cuts and must have the row of every commit."""
    n = 65540
    repo = tmp_path / "repo"
    os.makedirs(repo)
    git(repo, "init", "-q", ".")
    stream = []
    for i in range(n):
        data = b"def test_a(self):\n    self.assertEqual(x, %d)\n" % i
        stream.append(b"commit refs/heads/t\ncommitter c <c@example.org> %d +0000\ndata 1\nc\nM 100644 inline tests/test_a.py\n"
                      b"data %d\n%s\n" % (1600000000 + i, len(data), data))
    subprocess.run(["git", "-C", str(repo), "fast-import", "--quiet"], input=b"".join(stream), capture_output=True, check=True,
                   env=dict(os.environ, GIT_CONFIG_NOSYSTEM="1", HOME=str(repo)))
    git(repo, "symbolic-ref", "HEAD", "refs/heads/t")
    got = []
    for extra in ([], ["--batch-bytes", "100000"]):
        churn, out = tmp_path / ("churn%d.csv" % len(extra)), tmp_path / ("out%d.csv" % len(extra))
        got.append(run(["history", str(repo), "--assert-churn", str(churn), "--out", str(out)] + extra, [churn, out]))
    assert got[0] == got[1]
    stdout, _, (churn, _) = got[0]
    commits = [row.split(",")[0] for row in stdout.decode().split("\r\n")[1:] if row]
    assert len(commits) == n
    assert [r[0] for r in csv.reader(churn.decode().split("\r\n")[1:]) if r] == commits   # one category per commit
