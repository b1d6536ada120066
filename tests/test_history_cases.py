"""`tosem-scan history --cases` and `diff --cases` (docs/SPEC.md section 16) on a repository built here: every row equals
case_ref.py_case_churn over the `git cat-file` blobs of each commit, the scenario commits give their known rows, `git gc
--aggressive` changes nothing, `diff` of two `git archive` checkouts gives the commit's rows, `--find-renames 50` turns an
edited move into M rows, and every other output is byte-identical with and without `--cases`."""
import csv
import os
import shutil
import subprocess
import tarfile

import pytest

import case_ref
from test_history import CLI, EMPTY_TREE, git

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

EXT = {"py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}
HEAD = ["commit", "parent", "time", "fileName", "case", "change", "line", "oldLine", "lines", "oldLines", "asserts", "oldAsserts",
        "insertedLines", "deletedLines", "insertedAsserts", "deletedAsserts"]


def ext_of(path):
    name = path.rsplit("/", 1)[-1]
    return EXT.get(name.rsplit(".", 1)[-1], 0) if "." in name else 0


def selected(path):
    return "test" in path.lower() and ext_of(path) != 0


def py_case(name, n, asserts=(), body=b"v"):
    out = [b"def %s(self):\n" % name] + [b"    %s_%s_%d = %d\n" % (body, name, i, i) for i in range(n - 1)]
    for k in asserts:
        out[k] = b"    assert %s_%d\n" % (name, k)
    return out


def build(root):
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
        for nm, ls in files.items():
            os.makedirs(os.path.dirname(repo / nm), exist_ok=True)
            (repo / nm).write_bytes(b"".join(ls))
        git(repo, "add", "-A")
        git(repo, "commit", "-q", "--allow-empty", "-m", msg)

    files["tests/test_a.py"] = [b"import os\n"] + py_case(b"test_one", 5, (3,)) + py_case(b"test_two", 4) + py_case(b"test_three", 9, (2, 7))
    files["tests/test_b.cc"] = [b"#include <x>\n", b"TEST(S, A) {\n", b"  EXPECT_EQ(1, 1);\n", b"}\n", b"TEST(S, B) {\n", b"  int b;\n",
                                b"}\n"]
    files["tests/test_move.py"] = py_case(b"test_m1", 12, (4,)) + py_case(b"test_m2", 12, (5,))
    files["src/helper.py"] = py_case(b"test_zz", 3)
    commit("initial")
    a = files["tests/test_a.py"]
    one, two, three = a[1:6], a[6:10], a[10:19]
    one = one[:3] + [b"    assert changed\n"] + one[4:]                     # test_one: one assertion line replaced
    three = three[:4] + [b"def test_split(self):\n"] + three[4:]             # a header inserted inside test_three
    files["tests/test_a.py"] = [b"import sys\n"] + one + three + py_case(b"test_four", 3, (1,))   # test_two deleted, test_four added
    b = files["tests/test_b.cc"]
    files["tests/test_b.cc"] = b[:1] + [b"TEST_F(F, A) {\n"] + b[2:4] + b[5:]  # A rewritten (same name), B's header deleted
    commit("edit cases")
    m = files.pop("tests/test_move.py")
    files["tests/moved/test_move.py"] = m[:6] + [b"    assert moved\n"] + m[7:]   # an edited move
    files["tests/test_new.java"] = [b"class NewTest {\n", b"  @Test public void testX() {\n", b"    assertTrue(x);\n", b"  }\n", b"}\n"]
    commit("move and add")
    files.pop("tests/test_b.cc")
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
    """Rows of case_ref.py_case_churn over the blobs of every changed selected file (no renames), per commit in path order."""
    out = []
    for commit, parent, time in commits(repo):
        names = git(repo, "diff", "--name-only", "--no-renames", "-z", parent or EMPTY_TREE, commit).split("\0")
        for path in sorted(n for n in names if n and selected(n)):
            rows = case_ref.py_case_churn(blob(repo, parent, path), blob(repo, commit, path), ext_of(path), ext_of(path))
            for r in rows:
                c = cells(r)
                out.append([commit, parent, time, path] + c)
    return out


def run(*args):
    r = subprocess.run([CLI] + [str(a) for a in args], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return r


def read(path):
    return list(csv.reader(open(path, newline="", encoding="latin-1")))


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    return build(tmp_path_factory.mktemp("cases"))


def test_history_cases_equal_the_reference(repo, tmp_path):
    out = tmp_path / "c.csv"
    run("history", repo, "--cases", out)
    table = read(out)
    assert table[0] == HEAD
    want = want_rows(repo)
    assert table[1:] == want
    c = commits(repo)
    rows = {(r[0], r[3], r[4], r[5]): r[6:] for r in table[1:]}
    edit = c[1][0]
    assert rows[(edit, "tests/test_a.py", "test_two", "D")] == ["", "7", "", "4", "", "0", "", "4", "", "0"]
    assert rows[(edit, "tests/test_a.py", "test_one", "M")] == ["2", "2", "5", "5", "1", "1", "1", "1", "1", "1"]
    assert rows[(edit, "tests/test_a.py", "test_four", "A")] == ["17", "", "3", "", "1", "", "3", "", "1", ""]
    assert rows[(edit, "tests/test_a.py", "test_three", "M")] == ["7", "11", "4", "9", "1", "2", "0", "0", "0", "0"]
    assert rows[(edit, "tests/test_a.py", "test_split", "A")][:3] == ["11", "", "6"]
    assert rows[(edit, "tests/test_b.cc", "A", "M")][:2] == ["2", "2"]            # matched by name
    assert rows[(edit, "tests/test_b.cc", "B", "D")][:2] == ["", "5"]             # its body merged into A
    move = c[2][0]
    assert (move, "tests/test_move.py", "test_m1", "D") in rows and (move, "tests/moved/test_move.py", "test_m1", "A") in rows
    assert not any(r[3].startswith("src/") for r in table[1:])
    # the same after one pack with delta chains
    git(repo, "gc", "-q", "--aggressive")
    out2 = tmp_path / "c2.csv"
    run("history", repo, "--cases", out2)
    assert open(out2, "rb").read() == open(out, "rb").read()


def test_find_renames_gives_m_rows_for_an_edited_move(repo, tmp_path):
    out = tmp_path / "r.csv"
    run("history", repo, "--cases", out, "--find-renames", "50")
    table = read(out)
    assert table[0] == HEAD + ["oldFileName"]
    move = commits(repo)[2][0]
    mine = [r for r in table[1:] if r[0] == move and "move" in r[3]]
    assert mine == [[move, commits(repo)[1][0], commits(repo)[2][2], "tests/moved/test_move.py", "test_m1", "M", "1", "1", "12", "12",
                     "2", "1", "1", "1", "1", "0", "tests/test_move.py"]]
    plain = {tuple(r[:16]) for r in read(tmp_path / "r.csv")[1:] if "move" not in r[3]}
    assert plain == {tuple(r) for r in want_rows(repo) if "move" not in r[3]}


def test_outputs_are_byte_identical_with_and_without_cases(repo, tmp_path):
    for extra in ([], ["--find-renames", "50"]):
        a = {k: tmp_path / ("a_%s%d.csv" % (k, len(extra))) for k in ("out", "asserts", "churn", "cases")}
        b = {k: tmp_path / ("b_%s%d.csv" % (k, len(extra))) for k in ("out", "asserts", "churn")}
        ra = run("history", repo, "--out", a["out"], "--asserts", a["asserts"], "--assert-churn", a["churn"], "--cases", a["cases"], *extra)
        rb = run("history", repo, "--out", b["out"], "--asserts", b["asserts"], "--assert-churn", b["churn"], *extra)
        assert ra.stdout == rb.stdout
        for k in b:
            assert open(a[k], "rb").read() == open(b[k], "rb").read(), k
        alone = tmp_path / ("alone%d.csv" % len(extra))
        rc = run("history", repo, "--cases", alone, *extra)
        assert rc.stdout == rb.stdout and open(alone, "rb").read() == open(a["cases"], "rb").read()


def test_diff_of_archives_gives_the_commit_rows(repo, tmp_path):
    c = commits(repo)
    hist = tmp_path / "h.csv"
    run("history", repo, "--cases", hist)
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
    a = run("diff", roots[c[0][0]], roots[c[1][0]], "--cases", out)
    got = read(out)
    assert got[0] == HEAD[3:]
    want = [r[3:] for r in table[1:] if r[0] == c[1][0]]
    assert got[1:] == want and len(want) >= 6
    b = run("diff", roots[c[0][0]], roots[c[1][0]])
    assert a.stdout == b.stdout
