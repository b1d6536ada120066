"""`tosem-scan similar-tests` (docs/SPEC.md section 23): stdout, --out and --classes equal a restatement over the references
(tests/simtest_ref.py) on two roots whose tests pair within and across roots, and --git equals the root form on a checkout of
the same revision."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import simtest_ref as sr
import smell_ref
from test_cli_smells import CLI, HERE, SUFFIX, read_csv
from test_similar_tests_ref import EXAMPLE

pytestmark = pytest.mark.gpu


def make_roots(tmp_path):
    """repo0: the hand-written smell files and the worked example; repo1: 300 C1 test files and the worked example again."""
    c1, exts, _, _ = cu.load_fixture(os.path.join(HERE, "golden", "c1_testfiles.npz"))
    groups = [[(d, e) for _, e, d in smell_ref.HAND if e] + [(EXAMPLE, 1)], list(zip(c1[:300], exts[:300].tolist())) + [(EXAMPLE, 1)]]
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


def expected(roots, min_lines, P):
    allf = [(name, rel, data, ext) for name, files in roots for rel, data, ext in files]
    tests, seqs = sr.py_sequences([f[2] for f in allf], [f[3] for f in allf])
    pairs = sr.c_similar(seqs, min_lines, P)
    base, member = sr.classes(pairs, len(seqs))
    names = []
    for f, b, _ in tests:
        lines = smell_ref.py_lines(allf[f][2])
        names.append(smell_ref.py_case_name(lines[b], allf[f][3]).decode("latin-1"))
    root = [allf[f][0] for f, _, _ in tests]
    roots_n = [name for name, _ in roots] + ["<all>"]
    tot = {r: [0] * 6 for r in roots_n}
    for name, files in roots:
        tot[name][0] = len(files)
        tot["<all>"][0] += len(files)
    linked = set(member.tolist())
    for t, s in enumerate(seqs):
        for r in (root[t], "<all>"):
            tot[r][1] += 1
            tot[r][2] += len(s) >= min_lines
            tot[r][3] += t in linked
    out = [["repository", "fileName", "test", "line", "otherRepository", "otherFileName", "otherTest", "otherLine", "keptLines",
            "otherKeptLines", "lcs", "similarity"]]
    for a, b, l, sc in pairs:
        for r in {root[a], root[b], "<all>"}:
            tot[r][4] += 1
        fa, fb = tests[a][0], tests[b][0]
        out.append([root[a], allf[fa][1], names[a], str(tests[a][1] + 1), root[b], allf[fb][1], names[b], str(tests[b][1] + 1),
                    str(len(seqs[a])), str(len(seqs[b])), str(l), str(sc // 600)])
    cls = [["class", "repository", "fileName", "test", "line", "last_line", "keptLines"]]
    for k in range(len(base) - 1):
        ms = member[base[k]:base[k + 1]].tolist()
        for r in {root[t] for t in ms} | {"<all>"}:
            tot[r][5] += 1
        for t in ms:
            f, b, n = tests[t]
            cls.append([str(k + 1), root[t], allf[f][1], names[t], str(b + 1), str(b + n), str(len(seqs[t]))])
    rows = [["repository", "files", "tests", "compared_tests", "similar_tests", "pairs", "classes"]]
    rows += [[r] + [str(v) for v in tot[r]] for r in roots_n]
    return rows, out, cls


@pytest.mark.parametrize("min_lines,P", [(5, 70), (3, 90)])
def test_cli_roots(tmp_path, min_lines, P):
    roots = make_roots(tmp_path)
    want_rows, want_out, want_cls = expected(roots, min_lines, P)
    assert any(r[0] != r[4] for r in want_out[1:]), "a pair across the two roots"
    paths = [str(tmp_path / name) for name, _ in roots]
    outp, clsp = str(tmp_path / "pairs.csv"), str(tmp_path / "classes.csv")
    p = subprocess.run([CLI, "similar-tests"] + paths + ["--min-lines", str(min_lines), "--similarity", str(P), "--out", outp,
                                                         "--classes", clsp], capture_output=True, check=True)
    assert read_csv(p.stdout) == want_rows
    assert read_csv(open(outp, "rb").read()) == want_out
    assert read_csv(open(clsp, "rb").read()) == want_cls


def test_cli_git_equals_checkout(tmp_path):
    roots = make_roots(tmp_path)
    if shutil.which("git") is None:
        pytest.skip("git is not installed")
    repo = tmp_path / "g" / "repo1"
    shutil.copytree(tmp_path / "repo1", repo)
    env = dict(os.environ, GIT_AUTHOR_NAME="t", GIT_AUTHOR_EMAIL="t@t", GIT_COMMITTER_NAME="t", GIT_COMMITTER_EMAIL="t@t")
    for cmd in (["init", "-q"], ["add", "-A"], ["commit", "-q", "-m", "c1"]):
        subprocess.run(["git", "-C", str(repo)] + cmd, check=True, env=env)
    (repo / "tests" / "later_test.py").write_bytes(EXAMPLE)
    subprocess.run(["git", "-C", str(repo), "add", "-A"], check=True, env=env)
    subprocess.run(["git", "-C", str(repo), "commit", "-q", "-m", "later"], check=True, env=env)
    first = subprocess.run(["git", "-C", str(repo), "rev-parse", "HEAD~1"], capture_output=True, check=True).stdout.decode().strip()
    arch = tmp_path / "arch" / "repo1"
    arch.mkdir(parents=True)
    tar = subprocess.run(["git", "-C", str(repo), "archive", first], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", str(arch)], input=tar, check=True)
    res = {}
    for key, args in (("git", ["--git", str(repo), "--rev", first]), ("root", [str(arch)])):
        o, c = str(tmp_path / (key + "_p.csv")), str(tmp_path / (key + "_c.csv"))
        r = subprocess.run([CLI, "similar-tests"] + args + ["--out", o, "--classes", c], capture_output=True, check=True)
        res[key] = (r.stdout, open(o, "rb").read(), open(c, "rb").read())
    assert res["git"] == res["root"]
    assert read_csv(res["git"][0])[1][0] == "repo1" and int(read_csv(res["git"][0])[1][5]) > 0
