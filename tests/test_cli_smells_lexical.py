"""`tosem-scan smells --lexical` (docs/SPEC.md section 25): stdout and --out equal a restatement over the plain-Python references
(smell_ref for the nine smells of section 18, lexsmell_ref for the five of section 25) for two roots, many small batches give the
same bytes as one, --git equals the root form on a checkout of the same revision, and without --lexical the output is that of
section 18 alone."""
import csv
import io
import os
import shutil
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import lexsmell_ref as lr
import smell_ref as sr

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CLI = os.path.join(os.path.dirname(HERE), "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
SUFFIX = {1: ".py", 2: ".cc", 3: ".cpp", 4: ".java", 5: ".c", 6: ".h"}
ORDER = {s: k for k, s in enumerate(list(sr.SMELLS) + list(lr.LSMELLS))}


def read_csv(data: bytes):
    text = data.decode("latin-1")
    assert "\r\n" in text
    return list(csv.reader(io.StringIO(text, newline="")))


def make_roots(tmp_path):
    """Two roots: the hand-written files, and 300 C1 test files; every file under a `test` path with its tag's suffix."""
    c1, exts, _, _ = cu.load_fixture(os.path.join(HERE, "golden", "c1_testfiles.npz"))
    groups = [[(d, e) for _, e, d in lr.HAND if e], list(zip(c1[:300], exts[:300].tolist()))]
    roots = []
    for g, items in enumerate(groups):
        name = "repo%d" % g
        files = []
        for i, (data, ext) in enumerate(items):
            rel = "tests/f%04d_test%s" % (i, SUFFIX[int(ext)])
            p = tmp_path / name / rel
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_bytes(data)
            files.append((rel, data, int(ext)))
        roots.append((name, sorted(files)))
    return roots


def expected(roots, lexical):
    smells = list(sr.SMELLS) + (list(lr.LSMELLS) if lexical else [])
    rows = [["repository", "files", "tests"] + smells]
    out = [["repository", "fileName", "test", "line", "smell", "smellLine", "statement"]]
    tot = np.zeros(2 + len(smells), np.int64)
    for name, files in roots:
        data, exts, rels = [f[1] for f in files], [f[2] for f in files], [f[0] for f in files]
        tests, _ = sr.py_smells(data, exts)
        lex = lr.py_lexsmells(data, exts)["lex"]
        v = [len(files), len(tests)] + [sum(1 for t in tests if t[4] >> k & 1) for k in range(len(sr.SMELLS))]
        if lexical:
            v += [int((lex["smells"] >> k & 1).sum()) for k in range(len(lr.LSMELLS))]
        tot += np.array(v)
        rows.append([name] + [str(int(x)) for x in v])
        got = sr.py_smell_rows(data, exts, rels) + (lr.py_lexsmell_rows(data, exts, rels) if lexical else [])
        got.sort(key=lambda r: (rels.index(r[0]), r[2], r[4], ORDER[r[3]]))
        for fn, test, line, smell, sline, st in got:
            out.append([name, fn, test.decode("latin-1"), str(line), smell, str(sline), st.decode("latin-1")])
    rows.append(["<all>"] + [str(int(x)) for x in tot])
    return rows, out


def test_cli_lexical_roots_batches_and_git(tmp_path):
    roots = make_roots(tmp_path)
    paths = [str(tmp_path / name) for name, _ in roots]
    plain = str(tmp_path / "plain.csv")
    p = subprocess.run([CLI, "smells"] + paths + ["--out", plain], capture_output=True, check=True)
    want_rows, want_out = expected(roots, False)
    assert read_csv(p.stdout) == want_rows and read_csv(open(plain, "rb").read()) == want_out
    want_rows, want_out = expected(roots, True)
    assert all(int(x) > 0 for x in want_rows[-1][-5:])
    outp = str(tmp_path / "lexical.csv")
    p = subprocess.run([CLI, "smells"] + paths + ["--lexical", "--out", outp], capture_output=True, check=True)
    assert read_csv(p.stdout) == want_rows
    assert read_csv(open(outp, "rb").read()) == want_out
    small = str(tmp_path / "small.csv")                    # many batches: the same bytes
    q = subprocess.run([CLI, "smells", "--lexical"] + paths + ["--batch-bytes", "4096", "--out", small], capture_output=True, check=True)
    assert q.stdout == p.stdout and open(small, "rb").read() == open(outp, "rb").read()
    if shutil.which("git") is None:
        pytest.skip("git is not installed")
    repo = tmp_path / "g" / "repo1"
    shutil.copytree(tmp_path / "repo1", repo)
    env = dict(os.environ, GIT_AUTHOR_NAME="t", GIT_AUTHOR_EMAIL="t@t", GIT_COMMITTER_NAME="t", GIT_COMMITTER_EMAIL="t@t")
    for cmd in (["init", "-q"], ["add", "-A"], ["commit", "-q", "-m", "c1"]):
        subprocess.run(["git", "-C", str(repo)] + cmd, check=True, env=env)
    (repo / "tests" / "later_test.py").write_bytes(lr.HAND[0][2])
    subprocess.run(["git", "-C", str(repo), "add", "-A"], check=True, env=env)
    subprocess.run(["git", "-C", str(repo), "commit", "-q", "-m", "later"], check=True, env=env)
    first = subprocess.run(["git", "-C", str(repo), "rev-parse", "HEAD~1"], capture_output=True, check=True).stdout.decode().strip()
    arch = tmp_path / "arch" / "repo1"
    arch.mkdir(parents=True)
    tar = subprocess.run(["git", "-C", str(repo), "archive", first], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", str(arch)], input=tar, check=True)
    gout, rout = str(tmp_path / "g.csv"), str(tmp_path / "r.csv")
    g = subprocess.run([CLI, "smells", "--git", str(repo), "--rev", first, "--lexical", "--out", gout], capture_output=True, check=True)
    r = subprocess.run([CLI, "smells", str(arch), "--lexical", "--out", rout], capture_output=True, check=True)
    assert g.stdout == r.stdout and open(gout, "rb").read() == open(rout, "rb").read()
    assert read_csv(g.stdout)[1][0] == "repo1" and len(read_csv(g.stdout)[0]) == 3 + 9 + 5
