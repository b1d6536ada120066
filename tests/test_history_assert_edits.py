"""`tosem-scan history --assert-edits` and `diff --assert-edits` (docs/SPEC.md section 17) on a repository built here: every row
equals edit_ref.py_assert_edits over the `git cat-file` blobs of each commit, also after `git gc --aggressive`; the hunks equal
those of `git diff --minimal -U0` on these unambiguous edits; `diff` of two `git archive` checkouts gives the commit's rows; an
edited move pairs its lines under `--find-renames 50`; every other output is byte-identical with and without the option."""
import csv
import os
import re
import shutil
import subprocess
import tarfile

import pytest

import edit_ref
import spec_ref
from test_history import CLI, EMPTY_TREE, git
from test_history_asserts import category_cell

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

EXT = {"py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}
HEAD = ["commit", "parent", "time", "fileName", "oldLine", "line", "similarity", "oldStatement", "statement", "oldCategory", "category"]


def ext_of(path):
    name = path.rsplit("/", 1)[-1]
    return EXT.get(name.rsplit(".", 1)[-1], 0) if "." in name else 0


def selected(path):
    return "test" in path.lower() and ext_of(path) != 0


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

    body = [b"class T(unittest.TestCase):\n", b"    def test_a(self):\n", b"        x = f(1)\n", b"        self.assertEqual(x, 1)\n",
            b"        y = g(2)\n", b"        assert y == 2\n", b"        assert y > 0\n", b"    def test_b(self):\n", b"        z = 3\n",
            b"        self.assertTrue(z)\n", b"        w = 4\n", b"        assert w == 4\n", b"        assert w != 5\n"]
    files["tests/test_a.py"] = list(body)
    files["tests/test_m.py"] = [b"def test_m():\n"] + [b"    v%d = %d\n" % (i, i) for i in range(12)] + [b"    assert v3 == 3\n"]
    files["tests/test_c.cc"] = [b"TEST(S, A) {\n", b"  EXPECT_EQ(a, 1);\n", b"  EXPECT_TRUE(b);\n", b"}\n"]
    files["src/helper.py"] = [b"assert helper\n"]
    commit("initial")
    a = files["tests/test_a.py"]
    a[3] = b"        self.assertAlmostEqual(x, 1)\n"                             # exact becomes approximate
    files["tests/test_c.cc"][1] = b"  EXPECT_NEAR(a, 1, 1e-6);\n"
    files["src/helper.py"] = [b"assert helper2\n"]                              # not a test file
    commit("exact to approximate")
    a = files["tests/test_a.py"]
    files["tests/test_a.py"] = a[:7] + [b"    " + l for l in a[7:]]            # re-indent test_b's block
    commit("re-indent")
    a = files["tests/test_a.py"]
    files["tests/test_a.py"] = a[:5] + [b"        assert y == 3\n", b"        assert y >= 0\n", b"        assert y < 9\n"] + a[7:]   # 2 -> 3
    commit("two assertions become three")
    a = files["tests/test_a.py"]
    a[3] = b"        self.assertAlmostEqual(x, 2)\n"                             # two hunks in one file
    a[-1] = b"            assert w != 6\n"
    commit("two hunks")
    a = files["tests/test_a.py"]
    files["tests/test_a.py"] = [l for l in a if b"assert y" not in l]           # deletions only
    commit("delete assertions")
    m = files.pop("tests/test_m.py")
    files["tests/moved/test_m.py"] = m[:-1] + [b"    assert v3 == 4\n"]        # an edited move
    commit("move")
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


def edit_cells(old, new, xo, xn):
    """The row cells after fileName of every edit of one pair, from edit_ref."""
    lo, ln = spec_ref.py_lines(old), spec_ref.py_lines(new)
    out = []
    for i, j, sc in edit_ref.py_assert_edits(old, new, xo, xn):
        so, sn = spec_ref.py_statement(lo[i]), spec_ref.py_statement(ln[j])
        out.append([str(i + 1), str(j + 1), str(sc // 600), so.decode("latin-1"), sn.decode("latin-1"), category_cell(so)[1],
                    category_cell(sn)[1]])
    return out


def want_rows(repo):
    out = []
    for commit, parent, time in commits(repo):
        names = git(repo, "diff", "--name-only", "--no-renames", "-z", parent or EMPTY_TREE, commit).split("\0")
        for path in sorted(n for n in names if n and selected(n)):
            for c in edit_cells(blob(repo, parent, path), blob(repo, commit, path), ext_of(path), ext_of(path)):
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
    return build(tmp_path_factory.mktemp("edits"))


def test_history_assert_edits_equal_the_reference(repo, tmp_path):
    out = tmp_path / "e.csv"
    run("history", repo, "--assert-edits", out)
    table = read(out)
    assert table[0] == HEAD
    assert table[1:] == want_rows(repo)
    c = [x[0] for x in commits(repo)]
    rows = {}
    for r in table[1:]:
        rows.setdefault((r[0], r[3]), []).append(r[4:])
    assert [r[:5] for r in rows[(c[1], "tests/test_a.py")]] == [["4", "4", str(120000 * 22 // 50 // 600), "self.assertEqual",
                                                                 "self.assertAlmostEqual"]]
    assert [r[3:5] for r in rows[(c[1], "tests/test_c.cc")]] == [["EXPECT_EQ", "EXPECT_NEAR"]]
    assert {r[2] for r in rows[(c[2], "tests/test_a.py")]} == {"100"} and len(rows[(c[2], "tests/test_a.py")]) == 3
    assert len(rows[(c[3], "tests/test_a.py")]) == 2                            # 2 deleted, 3 inserted: one left over
    assert [r[:2] for r in rows[(c[4], "tests/test_a.py")]] == [["4", "4"], ["14", "14"]]
    assert (c[5], "tests/test_a.py") not in rows
    assert not any(r[3].startswith("src/") for r in table[1:])
    git(repo, "gc", "-q", "--aggressive")
    out2 = tmp_path / "e2.csv"
    run("history", repo, "--assert-edits", out2)
    assert open(out2, "rb").read() == open(out, "rb").read()


def test_hunks_equal_git_diff_minimal(repo):
    """On these edits the hunks of section 17 (with assertion lines on both sides) are hunks of `git diff --minimal -U0`."""
    for commit, parent, _ in commits(repo)[1:]:
        for path in ("tests/test_a.py",):
            old, new = blob(repo, parent, path), blob(repo, commit, path)
            if not old or not new or old == new:
                continue
            d = git(repo, "diff", "--minimal", "-U0", "--no-renames", parent, commit, "--", path)
            git_hunks = []
            for m in re.finditer(r"^@@ -(\d+)(?:,(\d+))? \+(\d+)(?:,(\d+))? @@", d, re.M):
                a0, an = int(m.group(1)), int(m.group(2) or 1)
                b0, bn = int(m.group(3)), int(m.group(4) or 1)
                git_hunks.append((set(range(a0 - 1, a0 - 1 + an)), set(range(b0 - 1, b0 - 1 + bn))))
            for dels, ins in edit_ref.py_hunks(old, new, 1, 1):
                assert any(set(dels) <= g[0] and set(ins) <= g[1] for g in git_hunks), (commit, dels, ins)


def test_find_renames_pairs_an_edited_move(repo, tmp_path):
    out = tmp_path / "r.csv"
    run("history", repo, "--assert-edits", out, "--find-renames", "50")
    table = read(out)
    assert table[0] == HEAD + ["oldFileName"]
    move = commits(repo)[-1][0]
    mine = [r for r in table[1:] if r[0] == move]
    assert [r[3:] for r in mine] == [["tests/moved/test_m.py", "14", "14", str(120000 * 13 // 28 // 600), "assert v3 == 3", "assert v3 == 4",
                                      mine[0][9], mine[0][10], "tests/test_m.py"]]
    assert [r[:11] for r in table[1:] if r[0] != move] == [r for r in want_rows(repo) if r[0] != move]


def test_outputs_are_byte_identical_with_and_without_assert_edits(repo, tmp_path):
    for extra in ([], ["--find-renames", "50"]):
        a = {k: tmp_path / ("a_%s%d.csv" % (k, len(extra))) for k in ("out", "asserts", "churn", "cases", "edits")}
        b = {k: tmp_path / ("b_%s%d.csv" % (k, len(extra))) for k in ("out", "asserts", "churn", "cases")}
        ra = run("history", repo, "--out", a["out"], "--asserts", a["asserts"], "--assert-churn", a["churn"], "--cases", a["cases"],
                 "--assert-edits", a["edits"], *extra)
        rb = run("history", repo, "--out", b["out"], "--asserts", b["asserts"], "--assert-churn", b["churn"], "--cases", b["cases"], *extra)
        assert ra.stdout == rb.stdout
        for k in b:
            assert open(a[k], "rb").read() == open(b[k], "rb").read(), k
        alone = tmp_path / ("alone%d.csv" % len(extra))
        rc = run("history", repo, "--assert-edits", alone, *extra)
        assert rc.stdout == rb.stdout and open(alone, "rb").read() == open(a["edits"], "rb").read()


def test_diff_of_archives_gives_the_commit_rows(repo, tmp_path):
    c = commits(repo)
    hist = tmp_path / "h.csv"
    run("history", repo, "--assert-edits", hist)
    table = read(hist)
    roots = {}
    for rev in (c[3][0], c[4][0]):
        d = tmp_path / ("tree_%s" % rev[:8])
        os.makedirs(d)
        tar = tmp_path / ("t_%s.tar" % rev[:8])
        tar.write_bytes(git(repo, "archive", "--format=tar", rev, text=False))
        with tarfile.open(tar) as t:
            t.extractall(d, filter="data")
        roots[rev] = str(d)
    out = tmp_path / "d.csv"
    a = run("diff", roots[c[3][0]], roots[c[4][0]], "--assert-edits", out)
    got = read(out)
    assert got[0] == HEAD[3:]
    want = [r[3:] for r in table[1:] if r[0] == c[4][0]]
    assert got[1:] == want and len(want) == 2
    b = run("diff", roots[c[3][0]], roots[c[4][0]])
    assert a.stdout == b.stdout
