"""The batch loop every file-scanning command of `tosem-scan` shares: on the C1 test files (tests/golden/c1_testfiles.npz) in nine
roots, `scan`, `body` and `releases` give byte-identical stdout and files with the default batch size and with a `--batch-bytes`
that cuts the tree into dozens of batches (counters and walk order carried across batches, one context per command); and every
command prints its empty result for a tree with no selected file."""
import os
import subprocess

import pytest

import corpus_util as cu

pytestmark = pytest.mark.gpu

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


def default_and_small(tmp_path, cmd, args, flags):
    got = []
    for tag, extra in (("default", []), ("small", ["--batch-bytes", SMALL])):
        outs = [str(tmp_path / ("%s_%s.csv" % (tag, f.lstrip("-")))) for f in flags]
        opts = [x for f, o in zip(flags, outs) for x in (f, o)]
        got.append(run([cmd] + args + opts + extra, outs))
    assert got[0] == got[1]
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
