"""`tosem-scan links` (docs/SPEC.md section 27): stdout, --out and --defs equal a restatement over the plain-Python reference
link_ref for two roots (roles from the S0 path rule, stems from the naming convention, files of tag 0 left out), and --git equals
the root form on a `git archive` checkout of the same revision."""
import csv
import io
import os
import shutil
import subprocess

import numpy as np
import pytest

import link_ref as lk
from case_ref import py_case_name
from spec_ref import py_lines

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CLI = os.path.join(os.path.dirname(HERE), "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
KIND = {1: "function", 2: "class"}


def read_csv(data: bytes):
    text = data.decode("latin-1")
    assert "\r\n" in text
    return list(csv.reader(io.StringIO(text, newline="")))


def make_roots(tmp_path):
    """Two roots: the hand-written repositories 0 and 1 under `repoA`, repository 2 (with a tag-0 file) under `repoB`."""
    roots = []
    for name, groups in (("repoA", (0, 1)), ("repoB", (2,))):
        files = []
        for g, rel, ext, data in lk.HAND:
            if g in groups:
                p = tmp_path / name / rel
                p.parent.mkdir(parents=True, exist_ok=True)
                p.write_bytes(data)
                files.append((rel, ext, data))
        roots.append((name, sorted(files)))
    return roots


def expected(roots):
    rels, exts, data, grp, names = [], [], [], [], []
    for g, (name, files) in enumerate(roots):
        names.append(name)
        for rel, ext, d in files:
            if ext:
                rels.append(rel); exts.append(ext); data.append(d); grp.append(g)
    role = np.array([lk.is_test_path(r) for r in rels], np.uint8)
    stem = lk.focal_stems(rels, role)
    grp = np.array(grp, np.uint16)
    r = lk.py_links(data, np.array(exts, np.uint8), role, stem, grp)
    tests, links, defs = r["tests"], r["links"], r["defs"]
    tot = np.zeros((len(names) + 1, 10), np.int64)

    def add(g, k, v):
        tot[g, k] += v
        tot[-1, k] += v
    for f in range(len(rels)):
        add(grp[f], 0 if role[f] else 1, 1)
    for t in tests:
        g = grp[t["file"]]
        add(g, 2, 1); add(g, 3, t["links"] > 0); add(g, 8, t["flags"] & 1); add(g, 9, t["flags"] >> 1 & 1)
    for d in defs:
        add(grp[d["file"]], 4, 1); add(grp[d["file"]], 5, d["tests_by_name"] > 0)
    for lnk in links:
        g = grp[tests[lnk["test"]]["file"]]
        add(g, 6, 1); add(g, 7, lnk["target"] < 0)
    rows = [["repository", "test_files", "production_files", "tests", "linked_tests", "definitions", "linked_definitions", "links",
             "ambiguous_links", "eager", "lazy"]]
    rows += [[n] + [str(int(v)) for v in tot[g]] for g, n in enumerate(names + ["<all>"])]

    def name_of(d):
        return data[d["file"]][d["name_off"]:d["name_off"] + d["name_len"]].decode("latin-1")
    out = [["repository", "fileName", "test", "line", "callee", "kind", "calls", "definitions", "defFile", "defLine", "focal"]]
    for lnk in links:
        t = tests[lnk["test"]]
        f = t["file"]
        case = py_case_name(py_lines(data[f])[t["line"]], exts[f]).decode("latin-1")
        nd = defs[lnk["name_def"]]
        td = defs[lnk["target"]] if lnk["target"] >= 0 else None
        focal = td is not None and stem[f] >= 0 and stem[td["file"]] == stem[f]
        out.append([names[grp[f]], rels[f], case, str(lnk["line"] + 1), name_of(nd), KIND[int((td if td is not None else nd)["kind"])],
                    str(lnk["calls"]), str(lnk["n_defs"]), rels[td["file"]] if td is not None else "",
                    str(td["line"] + 1) if td is not None else "", "1" if focal else "0"])
    dout = [["repository", "fileName", "line", "name", "kind", "tests", "tests_by_name", "calls"]]
    for d in defs:
        dout.append([names[grp[d["file"]]], rels[d["file"]], str(d["line"] + 1), name_of(d), KIND[int(d["kind"])], str(d["tests"]),
                     str(d["tests_by_name"]), str(d["calls"])])
    return rows, out, dout


def test_cli_links_roots_and_git(tmp_path):
    roots = make_roots(tmp_path)
    paths = [str(tmp_path / name) for name, _ in roots]
    outp, defp = str(tmp_path / "links.csv"), str(tmp_path / "defs.csv")
    p = subprocess.run([CLI, "links"] + paths + ["--out", outp, "--defs", defp], capture_output=True, check=True)
    rows, out, dout = expected(roots)
    assert read_csv(p.stdout) == rows
    assert read_csv(open(outp, "rb").read()) == out and read_csv(open(defp, "rb").read()) == dout
    assert int(rows[-1][7]) > 10 and int(rows[-1][9]) > 0 and int(rows[-1][10]) > 0
    if shutil.which("git") is None:
        pytest.skip("git is not installed")
    repo = tmp_path / "g" / "repoA"
    shutil.copytree(tmp_path / "repoA", repo)
    env = dict(os.environ, GIT_AUTHOR_NAME="t", GIT_AUTHOR_EMAIL="t@t", GIT_COMMITTER_NAME="t", GIT_COMMITTER_EMAIL="t@t")
    for cmd in (["init", "-q"], ["add", "-A"], ["commit", "-q", "-m", "c1"]):
        subprocess.run(["git", "-C", str(repo)] + cmd, check=True, env=env)
    (repo / "calc" / "later_test.py").write_bytes(lk.PYTEST_TEST)
    subprocess.run(["git", "-C", str(repo), "add", "-A"], check=True, env=env)
    subprocess.run(["git", "-C", str(repo), "commit", "-q", "-m", "later"], check=True, env=env)
    first = subprocess.run(["git", "-C", str(repo), "rev-parse", "HEAD~1"], capture_output=True, check=True).stdout.decode().strip()
    arch = tmp_path / "arch" / "repoA"
    arch.mkdir(parents=True)
    tar = subprocess.run(["git", "-C", str(repo), "archive", first], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", str(arch)], input=tar, check=True)
    g = subprocess.run([CLI, "links", "--git", str(repo), "--rev", first, "--out", str(tmp_path / "g.csv"), "--defs",
                        str(tmp_path / "gd.csv")], capture_output=True, check=True)
    r = subprocess.run([CLI, "links", str(arch), "--out", str(tmp_path / "r.csv"), "--defs", str(tmp_path / "rd.csv")],
                       capture_output=True, check=True)
    assert g.stdout == r.stdout and read_csv(g.stdout)[1][0] == "repoA"
    assert open(tmp_path / "g.csv", "rb").read() == open(tmp_path / "r.csv", "rb").read()
    assert open(tmp_path / "gd.csv", "rb").read() == open(tmp_path / "rd.csv", "rb").read()
    head = subprocess.run([CLI, "links", "--git", str(repo)], capture_output=True, check=True)
    assert read_csv(head.stdout)[1][1] == str(int(read_csv(r.stdout)[1][1]) + 1)   # HEAD adds one test file
