"""`tosem-scan history --links` and `diff --links` (docs/SPEC.md section 28) on a repository built in the test, whose commits play the
worked examples of section 28 (a call added to a test, a signature edit, a deleted definition, a second definition elsewhere, a
rename of the test file), with a commit that touches no source file and one that edits the C++ source of a header/source pair.
Checks: the rows equal a restatement over `git ls-tree` / `git cat-file` of every revision (tests/link_churn_ref.py), with and
without `--find-renames`, over a `--max-commits` window, and after `git gc --aggressive`; `diff --links` of two `git archive`
checkouts gives the commit's rows without the lead columns; every other output is byte-identical with and without `--links`; and
`--dry-run --links` is refused."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import case_ref
import link_churn_ref as ref
import link_ref as lr
import test_link_churn_ref as ex
from spec_ref import py_lines
from test_history import CLI, git
from test_history_clones import EXT, binary, checkout, commit, commits, read, run, write

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")]

HEAD = ["fileName", "test", "change", "line", "oldLine", "callee", "event", "cause", "calls", "oldCalls", "definitions",
        "oldDefinitions", "defFile", "defLine", "oldDefFile", "oldDefLine"]


@pytest.fixture(scope="module")
def repo(tmp_path_factory):
    r = str(tmp_path_factory.mktemp("links") / "repo")
    os.makedirs(r)
    git(r, "init", "-q", ".")
    for p, d in ex.REVS[0].items():
        write(r, p, d)
    for p, d in ex.CJ_OLD.items():
        write(r, p, d)
    commit(r, "root")
    for k, msg in ((1, "call add from test_sub"), (2, "edit the signature of add"), (3, "delete sub"), (4, "define add in ops.py")):
        for p, d in ex.REVS[k].items():
            write(r, p, d)
        commit(r, msg)
    write(r, "NOTES.txt", b"no source file\n")
    commit(r, "touch no source file")
    write(r, "w/widget.cc", ex.CJ_NEW["w/widget.cc"])
    commit(r, "edit the C++ source of size()")
    git(r, "mv", "tests/test_calc.py", "tests/test_math.py")
    commit(r, "rename the test file")
    return r


def selected(path):
    ext = path.rsplit(".", 1)[-1] if "." in path.rsplit("/", 1)[-1] else ""
    return ext in EXT


def revision(repo, rev):
    if not rev:
        return [], {}
    paths = [p for p in git(repo, "ls-tree", "-r", "--name-only", rev).split("\n") if p and selected(p)]
    paths.sort(key=lambda p: p.split("/"))
    return paths, {p: git(repo, "cat-file", "blob", "%s:%s" % (rev, p), text=False) for p in paths}


def changes(repo, parent, child, renames):
    args = ["diff-tree", "-r", "--no-commit-id", "--name-status"] + (["-M50%"] if renames else []) + [parent or "--root", child]
    out = []
    for line in filter(None, git(repo, *args).split("\n")):
        f = line.split("\t")
        k = f[0][0]
        out.append((f[1], f[2]) if k == "R" else (f[1], None) if k == "D" else (None, f[1]) if k == "A" else (f[1], f[1]))
    return [(o, n) for o, n in out if (o is None or selected(o)) and (n is None or selected(n))]


def as_rev(paths, files):
    role = np.array([lr.is_test_path(p) for p in paths], np.uint8)
    return ([files[p] for p in paths], np.array([EXT[p.rsplit(".", 1)[1]] for p in paths], np.uint8), role, lr.focal_stems(paths, role))


def step_rows(repo, parent, child, renames):
    """The rows of one commit without the lead columns, from the restatement."""
    po_, po = revision(repo, parent)
    pn_, pn = revision(repo, child)
    pairs = []
    for o, nw in changes(repo, parent, child, renames):
        a, b = (po_.index(o) if o else -1), (pn_.index(nw) if nw else -1)
        if a >= 0 and b >= 0 and (binary(po[o]) or binary(pn[nw])):
            pairs += [(a, -1), (-1, b)]
        else:
            pairs.append((a, b))
    old, new = as_rev(po_, po), as_rev(pn_, pn)
    res = ref.churn(old, new, [a for a, _ in pairs], [b for _, b in pairs])
    sides = {"old": (old, po_), "new": (new, pn_)}
    num = lambda v: "" if v < 0 else str(v)

    def name_of(s, j):
        d = res[s]["defs"][int(res[s]["links"][j]["name_def"])]
        return sides[s][0][0][int(d["file"])][int(d["name_off"]):int(d["name_off"]) + int(d["name_len"])].decode("latin-1")

    def target(s, j):
        t = int(res[s]["links"][j]["target"]) if j >= 0 else -1
        if t < 0:
            return ["", ""]
        d = res[s]["defs"][t]
        return [sides[s][1][int(d["file"])], str(int(d["line"]) + 1)]
    rows = []
    for e in res["events"]:
        ev, cause, a, b, jo, jn, ocl, ncl, od, nd = (int(x) for x in e)
        s, t = ("new", b) if b >= 0 else ("old", a)
        (files, exts, _, _), paths = sides[s]
        tr = res[s]["tests"][t]
        f, line = int(tr["file"]), int(tr["line"])
        row = [paths[f], case_ref.py_case_name(py_lines(files[f])[line], int(exts[f])).decode("latin-1"), chr(res[s]["change"][t]),
               str(int(res["new"]["tests"][b]["line"]) + 1) if b >= 0 else "", str(int(res["old"]["tests"][a]["line"]) + 1) if a >= 0 else ""]
        if ev >= ref.EAGER_IN:
            row += ["", ref.EVENTS[ev]] + [""] * 9
        else:
            row += [name_of("new", jn) if jn >= 0 else name_of("old", jo), ref.EVENTS[ev], ref.CAUSES[cause] if cause >= 0 else "",
                    num(ncl), num(ocl), str(nd), str(od)] + target("new", jn) + target("old", jo)
        if renames:
            row.append(po_[int(res["old"]["tests"][a]["file"])] if a >= 0 else "")
        rows.append(row)
    return rows


def want(repo, chain, renames):
    rows = []
    for c, p, t in chain:
        rows += [[c, p, t] + r for r in step_rows(repo, p, c, renames)]
    return rows


@pytest.mark.parametrize("renames", [False, True])
def test_history_rows_equal_the_restatement(repo, tmp_path, renames):
    out = tmp_path / "l.csv"
    run("history", repo, "--links", out, *(["--find-renames", 50] if renames else []))
    got = read(out)
    assert got[0] == ["commit", "parent", "time"] + HEAD + (["oldFileName"] if renames else [])
    rows = want(repo, commits(repo), renames)
    assert got[1:] == rows
    events = {(r[5], r[9]) for r in rows}
    assert {("=", "redefined"), ("M", "added"), ("=", "removed"), ("=", "lazy_introduced")} <= events
    assert any(r[8] == "size" and r[9] == "redefined" for r in rows)          # the C++ source edit, the header unchanged
    assert ("=", "retargeted") in events if renames else ("D", "removed") in events


def test_max_commits_window_and_gc(repo, tmp_path):
    out = tmp_path / "w.csv"
    run("history", repo, "--links", out, "--max-commits", 3)
    chain = commits(repo)
    assert read(out)[1:] == want(repo, chain[-3:], False)
    full = tmp_path / "full.csv"
    run("history", repo, "--links", full, "--find-renames", 50)
    packed = str(tmp_path / "packed")
    shutil.copytree(repo, packed)
    git(packed, "gc", "-q", "--aggressive")
    again = tmp_path / "gc.csv"
    run("history", packed, "--links", again, "--find-renames", 50)
    assert open(full, "rb").read() == open(again, "rb").read()


def test_diff_equals_the_commit_rows(repo, tmp_path):
    hist = tmp_path / "h.csv"
    run("history", repo, "--links", hist, "--find-renames", 50)
    table = read(hist)[1:]
    for c, p, _ in commits(repo)[1:]:
        checkout(repo, p, tmp_path / ("o_" + c))
        checkout(repo, c, tmp_path / ("n_" + c))
        out = tmp_path / ("d_%s.csv" % c)
        run("diff", tmp_path / ("o_" + c), tmp_path / ("n_" + c), "--links", out, "--find-renames", 50)
        got = read(out)
        assert got[0] == HEAD + ["oldFileName"]
        assert got[1:] == [r[3:] for r in table if r[0] == c], c


def test_other_outputs_are_unchanged(repo, tmp_path):
    outs = ["--out", "--asserts", "--assert-churn", "--cases", "--assert-edits", "--smells", "--moves", "--clones", "--similar-tests"]

    def history(tag, *extra):
        args = [a for o in outs for a in (o, tmp_path / (tag + o.strip("-") + ".csv"))]
        return run("history", repo, *args, "--find-renames", 50, *extra)
    r1 = history("a")
    r2 = history("b", "--links", tmp_path / "links.csv")
    assert r1.stdout == r2.stdout
    for o in outs:
        name = o.strip("-") + ".csv"
        assert open(tmp_path / ("a" + name), "rb").read() == open(tmp_path / ("b" + name), "rb").read(), o
    c, p, _ = commits(repo)[2]
    checkout(repo, p, tmp_path / "o")
    checkout(repo, c, tmp_path / "n")
    d1 = run("diff", tmp_path / "o", tmp_path / "n", "--out", tmp_path / "d1.csv")
    d2 = run("diff", tmp_path / "o", tmp_path / "n", "--out", tmp_path / "d2.csv", "--links", tmp_path / "dl.csv")
    assert d1.stdout == d2.stdout and open(tmp_path / "d1.csv", "rb").read() == open(tmp_path / "d2.csv", "rb").read()
    assert len(read(tmp_path / "dl.csv")) == 3                               # the signature edit: two redefined rows


def test_dry_run_with_links_is_refused(repo, tmp_path):
    r = subprocess.run([CLI, "history", repo, "--dry-run", "--links", str(tmp_path / "x.csv")], capture_output=True)
    assert r.returncode != 0 and b"--links" in r.stderr
