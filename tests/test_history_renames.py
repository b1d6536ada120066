"""`tosem-scan history --find-renames` and `diff --find-renames` (docs/SPEC.md section 13) against `git diff -M` on a
repository built here: pure moves, moves with 10 / 30 / 45 / 55 % of their lines replaced, identical files moved to
different base names, a moved empty file, the base-name step at 80 % / 95 % and at 70 %, and a move out of the test-file
selection.  Every line is shorter than 64 bytes and unique in its file, so git's span hashing equals the line hashing of
section 13 and git's minimal script equals the canonical one of section 8."""
import collections
import csv
import os
import random
import re
import shutil
import subprocess
import tarfile

import pytest

import spec_ref
import tosemscan as ts
from test_history import CLI, EMPTY_TREE, git

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

EXTS = {"py", "cc", "cpp", "java", "c", "h"}


def selected(path):
    """S0 / S1: the path contains `test` and has a tagged extension."""
    return "test" in path.lower() and path.rsplit(".", 1)[-1] in EXTS and "." in path.rsplit("/", 1)[-1]


def lines(tag, n, asserts=()):
    out = [b"v_%s_%03d = %d\n" % (tag, i, i) for i in range(n)]
    for k in asserts:
        out[k] = b"    self.assertEqual(%s_%03d, 1)\n" % (tag, k)
    return out


def replaced(src, frac, tag, seed):
    """src with round(frac * len) lines replaced by new unique lines of the same length (assertion lines stay assertions)."""
    rng = random.Random(seed)
    out = list(src)
    for i in sorted(rng.sample(range(len(out)), int(round(frac * len(out))))):
        old = out[i]
        new = (b"    self.assertTrue(%s_%03d)" % (tag, i)) if b"assert" in old else (b"w_%s_%03d = 0" % (tag, i))
        out[i] = new.ljust(len(old) - 1, b" ")[:len(old) - 1] + b"\n" if len(new) < len(old) else new + b"\n"
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

    files["tests/test_pure.py"] = lines(b"pu", 30, (3, 17))
    for pct in (10, 30, 45, 55):
        files["tests/test_e%d.py" % pct] = lines(b"e%d" % pct, 40, (2, 9, 21, 33))
    files["tests/test_twin1.py"] = lines(b"tw", 12, (4,))
    files["tests/test_twin2.py"] = lines(b"tw", 12, (4,))
    files["tests/test_empty.py"] = []
    files["a/x_test.py"] = lines(b"xx", 20, (5,))
    files["c/x_test.py"] = lines(b"xc", 20, (5,))
    files["tests/test_gone.py"] = lines(b"go", 15, (1,))
    files["tests/test_stay.py"] = lines(b"st", 10)
    commit("initial")
    # pure moves, edited moves, identical twins to new base names, a moved empty file
    files["tests/moved/test_pure.py"] = files.pop("tests/test_pure.py")
    for pct in (10, 30, 45, 55):
        files["tests/moved/test_e%d.py" % pct] = replaced(files.pop("tests/test_e%d.py" % pct), pct / 100, b"e%d" % pct, pct)
    files["tests/moved/test_twin_a.py"] = files.pop("tests/test_twin1.py")
    files["tests/moved/test_twin_b.py"] = files.pop("tests/test_twin2.py")
    files["tests/moved/test_empty.py"] = files.pop("tests/test_empty.py")
    files["tests/test_stay.py"] = files["tests/test_stay.py"] + [b"v_more = 1\n"]
    commit("moves")
    # base-name step: a/x_test.py is 80 % similar to b/x_test.py and 95 % similar to b/y_test.py
    x = files.pop("a/x_test.py")
    files["b/x_test.py"] = replaced(x, 0.20, b"bx", 1)
    files["b/y_test.py"] = replaced(x, 0.05, b"by", 2)
    commit("base name 80")
    # the same at 70 %
    x = files.pop("c/x_test.py")
    files["d/x_test.py"] = replaced(x, 0.30, b"dx", 3)
    files["d/y_test.py"] = replaced(x, 0.05, b"dy", 4)
    commit("base name 70")
    # a move out of the selection: only the deletion is a row
    files["src/gone.py"] = files.pop("tests/test_gone.py")
    commit("out of selection")
    return repo


def commits(repo):
    out = []
    for entry in filter(None, git(repo, "log", "--first-parent", "--reverse", "--format=%H %P").split("\n")):
        parts = entry.split()
        out.append((parts[0], parts[1] if len(parts) > 1 else ""))
    return out


def selected_paths(repo, parent, commit):
    names = git(repo, "diff", "--name-only", "--no-renames", "-z", parent or EMPTY_TREE, commit).split("\0")
    return [n for n in names if n and selected(n)]


def git_rows(repo, pct):
    """{(commit, old path or '', path): (added, removed, similarity or '')} of `git diff --minimal -M<pct>%` on the selected
    files (the pathspec limits the files before git pairs them, as the selection does)."""
    rows = {}
    for commit, parent in commits(repo):
        paths = selected_paths(repo, parent, commit)
        if not paths:
            continue
        base = [parent or EMPTY_TREE, commit, "--"] + paths
        num = git(repo, "diff", "--minimal", "-M%d%%" % pct, "--numstat", "-z", *base).split("\0")
        st = git(repo, "diff", "-M%d%%" % pct, "--name-status", "-z", *base).split("\0")
        sim = {}
        i = 0
        while i < len(st) and st[i]:
            if st[i].startswith("R"):
                sim[(st[i + 1], st[i + 2])] = str(int(st[i][1:]))
                i += 3
            else:
                i += 2
        i = 0
        while i < len(num) and num[i]:
            a, r, p = num[i].split("\t")
            if p:
                rows[(commit, "", p)] = (a, r, "")
                i += 1
            else:
                old, new = num[i + 1], num[i + 2]
                rows[(commit, old, new)] = (a, r, sim[(old, new)])
                i += 3
    return rows


def run_history(repo, tmp, pct, *extra):
    out = tmp / ("h%d.csv" % pct)
    r = subprocess.run([CLI, "history", str(repo), "--out", str(out), "--find-renames", str(pct)] + list(extra),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return list(csv.reader(open(out, newline=""))), r


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    return build(tmp_path_factory.mktemp("renames"))


@pytest.mark.parametrize("pct", [50, 80, 70])
def test_rows_equal_git_diff_find_renames(repo, tmp_path, pct):
    table, r = run_history(repo, tmp_path, pct)
    head = table[0]
    assert head[-2:] == ["oldFileName", "similarity"] and len(head) == 14
    got = {(row[0], row[12], row[3]): (row[5], row[6], row[13]) for row in table[1:]}
    assert len(got) == len(table) - 1
    want = git_rows(repo, pct)
    assert got == want
    renames = [k for k, v in want.items() if v[2]]
    if pct == 50:
        assert len(renames) == 9 and "9 rename(s) found at 50% (4 exact, 5 inexact)" in r.stderr
        by_new = {k[2]: (k[1], v[2]) for k, v in want.items() if v[2]}
        assert by_new["b/x_test.py"][0] == "a/x_test.py" and by_new["d/y_test.py"] == ("c/x_test.py", "95")
        assert by_new["tests/moved/test_empty.py"] == ("tests/test_empty.py", "100")
        assert "tests/moved/test_e55.py" not in by_new and "tests/test_gone.py" not in {k[1] for k in renames}
    if pct == 70:
        by_new = {k[2]: (k[1], v[2]) for k, v in want.items() if v[2]}
        assert by_new["b/y_test.py"] == ("a/x_test.py", "95")


def test_files_column_counts_a_pair_once_and_plain_output_is_unchanged(repo, tmp_path):
    _, r = run_history(repo, tmp_path, 50)
    plain = subprocess.run([CLI, "history", str(repo)], capture_output=True, text=True)
    assert plain.returncode == 0
    files = {ln.split(",")[0]: int(ln.split(",")[1]) for ln in r.stdout.splitlines()[1:] if ln}
    files0 = {ln.split(",")[0]: int(ln.split(",")[1]) for ln in plain.stdout.splitlines()[1:] if ln}
    moves = commits(repo)[1][0]
    assert files0[moves] == files[moves] + 7                 # 7 selected pairs of the commit were two rows each
    out = tmp_path / "plain.csv"
    subprocess.run([CLI, "history", str(repo), "--out", str(out)], check=True, capture_output=True)
    assert open(out, newline="").readline().rstrip("\r\n").split(",")[-1] == "removed_assert"


def git_assert_rows(repo, pct):
    rows, churn = [], collections.defaultdict(lambda: [0, 0])
    for commit, parent in commits(repo):
        paths = selected_paths(repo, parent, commit)
        if not paths:
            continue
        diff = git(repo, "diff", "--minimal", "-M%d%%" % pct, "-U0", "--no-color", parent or EMPTY_TREE, commit, "--", *paths,
                   text=False)
        old = new = None
        lo = ln = 0
        for line in diff.split(b"\n"):
            if line.startswith(b"diff --git"):
                old = new = None
                continue
            if line.startswith(b"--- "):
                old = None if line[4:] == b"/dev/null" else line[6:].decode()
                continue
            if line.startswith(b"+++ "):
                new = None if line[4:] == b"/dev/null" else line[6:].decode()
                continue
            m = re.match(rb"@@ -(\d+)(?:,\d+)? \+(\d+)(?:,\d+)? @@", line)
            if m:
                lo, ln = int(m.group(1)), int(m.group(2))
                continue
            if line[:1] in (b"+", b"-"):
                minus = line[:1] == b"-"
                num = lo if minus else ln
                if minus:
                    lo += 1
                else:
                    ln += 1
                if not spec_ref.py_is_assert_line(line[1:], 1):
                    continue
                stmt = spec_ref.py_statement(line[1:])
                cat = spec_ref.py_category(stmt)
                rows.append((commit, old if minus else new, line[:1].decode(), str(num), stmt.decode(), ts.category_name(cat)))
                churn[(commit, ts.category_name(cat))][1 if minus else 0] += 1
    return rows, churn


def test_assert_rows_of_renamed_files(repo, tmp_path):
    ar, cr = tmp_path / "a.csv", tmp_path / "c.csv"
    _, r = run_history(repo, tmp_path, 50, "--asserts", str(ar), "--assert-churn", str(cr))
    got = [(x[0], x[3], x[4], x[5], x[6], x[7]) for x in list(csv.reader(open(ar, newline="")))[1:]]
    want, churn = git_assert_rows(repo, 50)
    assert sorted(got) == sorted(want)
    moves = commits(repo)[1][0]
    touched = {(x[1], x[2]) for x in got if x[0] == moves}
    assert not any("pure" in p or "twin" in p or "empty" in p for p, _ in touched)      # pure moves: no rows
    assert ("tests/test_e30.py", "-") in touched and ("tests/moved/test_e30.py", "+") in touched
    got_churn = {(c[0], c[1]): (int(c[2]), int(c[3])) for c in list(csv.reader(open(cr, newline="")))[1:]}
    assert got_churn == {k: tuple(v) for k, v in churn.items()}


def read_rows(path):
    return list(csv.reader(open(path, newline="")))


def test_diff_of_archives_gives_the_history_rows(repo, tmp_path):
    """`diff` of two archives equals `history` at that commit with the commit columns removed, with and without renames:
    --out rows (those that change a line or pair a rename: `history` also lists a changed file whose diff changes no
    line), --asserts and --assert-churn."""
    roots = {}
    for k in (1, 2):                                         # the commits whose changed files are all test files
        commit, parent = commits(repo)[k]
        for rev in (parent, commit):
            if rev in roots:
                continue
            d = tmp_path / ("tree_%s" % rev[:8])
            os.makedirs(d)
            tar = tmp_path / ("t_%s.tar" % rev[:8])
            tar.write_bytes(git(repo, "archive", "--format=tar", rev, text=False))
            with tarfile.open(tar) as t:
                t.extractall(d, filter="data")
            roots[rev] = str(d)
    for renames in (["--find-renames", "50"], []):
        check_diff_against_history(repo, tmp_path / ("r" if renames else "p"), roots, renames)


def check_diff_against_history(repo, tmp, roots, renames):
    os.makedirs(tmp)
    hist = {p: tmp / ("h_%s.csv" % p) for p in ("out", "asserts", "churn")}
    r = subprocess.run([CLI, "history", str(repo), "--out", str(hist["out"]), "--asserts", str(hist["asserts"]),
                        "--assert-churn", str(hist["churn"])] + renames, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    table = read_rows(hist["out"])
    for k in (1, 2):
        commit, parent = commits(repo)[k]
        mine = {p: tmp / ("d%d_%s.csv" % (k, p)) for p in ("out", "asserts", "churn")}
        r = subprocess.run([CLI, "diff", roots[parent], roots[commit], "--out", str(mine["out"]), "--asserts", str(mine["asserts"]),
                            "--assert-churn", str(mine["churn"])] + renames, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        got = read_rows(mine["out"])
        assert got[0] == table[0][3:]
        want = [x[3:] for x in table[1:] if x[0] == commit and (x[5] != "0" or x[6] != "0" or (renames and x[-1]))]
        assert sorted(got[1:]) == sorted(want) and len(want) >= 2
        got = read_rows(mine["asserts"])
        want = read_rows(hist["asserts"])
        assert got[0] == want[0][3:]
        assert sorted(got[1:]) == sorted(x[3:] for x in want[1:] if x[0] == commit) and len(got) > 1
        got = read_rows(mine["churn"])
        want = read_rows(hist["churn"])
        assert got[0] == want[0][1:]
        assert got[1:] == [x[1:] for x in want[1:] if x[0] == commit] and len(got) > 1
