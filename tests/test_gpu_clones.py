"""`tsm_clones` / `Scanner.clones` (docs/SPEC.md section 15) bit for bit against the serial C reference orc_clones, every
output array: the C1 test files at windows of 3, 5 and 10 lines, a C4-scale corpus with planted copies, a class of more
fragments than one CTA sorts in shared memory, two copies of a 60 000-line file, a corpus without duplication and an empty
one; the capacity retry, the argument checks, repeated calls and a non-blocking stream; and `tosem-scan clones` over a tree
and over a git revision."""
import csv
import ctypes as C
import io
import os
import shutil
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import orc_clones as ocl
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
SMEM_FRAGMENTS = 4096                                      # SIM_SMEM_LINES: larger classes take the tiled sort


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def c1():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    return files, exts


def check(s, corpus, n, **kw):
    got = s.clones(corpus, n, **kw)
    ocl.assert_equal(got, ocl.clones(corpus, n))
    return got


@pytest.mark.parametrize("n", [3, 5, 10])
def test_c1(scanner, c1, n):
    got = check(scanner, ts.pack(*c1), n)
    assert len(got["class_len"]) > 1000
    ms = scanner.clones_last_ms()
    assert len(ms) == 3 and all(m > 0 for m in ms)


def test_c4_scale_planted_copies(scanner):
    files, exts = ocl.c4_planted(0x7053454D0C4, 100000)
    c = ts.pack(files, exts)
    got = check(scanner, c, 5)
    sizes = np.diff(got["class_base"])
    assert len(sizes) > 10000 and sizes.max() > 2 and got["file_dup"].sum() > 0


def test_classes_beyond_shared_memory(scanner):
    header = b"".join(b"# licence line %d\n" % i for i in range(12))
    other = b"".join(b"// shared block %d\n" % i for i in range(7))
    files = [header + (other if i % 5 == 0 else b"") + b"def test_%d():\n    assert f(%d)\n" % (i, i) for i in range(SMEM_FRAGMENTS + 900)]
    got = check(scanner, ts.pack(files, [1] * len(files)), 5)
    sizes = np.diff(got["class_base"])
    assert sizes.max() > SMEM_FRAGMENTS and 32 < sizes.min() <= SMEM_FRAGMENTS   # the tiled sort and the shared-memory sort


def test_two_copies_of_a_long_file(scanner):
    big = b"".join(b"line %d\n" % i for i in range(60000))
    got = check(scanner, ts.pack([b"x\n", big, b"y\n", big], [1, 1, 1, 1]), 5)
    assert got["class_len"].tolist() == [60000] and got["member"].tolist() == [1, 60002]


def test_no_duplication_and_empty_corpus(scanner):
    files = [b"".join(b"f%d l%d\n" % (f, i) for i in range(50)) for f in range(100)]
    got = check(scanner, ts.pack(files, [1] * 100), 3)
    assert len(got["member"]) == 0 and got["class_base"].tolist() == [0] and got["file_dup"].sum() == 0
    got = check(scanner, ts.pack([], []), 3)
    assert got["line_base"].tolist() == [0] and len(got["member"]) == 0
    got = check(scanner, ts.pack([b"", b""], [1, 1]), 1)
    assert got["line_base"].tolist() == [0, 0, 0]


def test_capacity_retry_and_arguments(scanner, c1):
    c = ts.pack(*c1)
    want = ocl.clones(c, 5)
    ocl.assert_equal(scanner.clones(c, 5, cap=1), want)
    cs = c.c_struct()
    r = ts._CloneResult(None, None, None, None, None, 0, -1, None, 0, -1)
    assert ts.lib().tsm_clones(scanner._ctx, C.byref(cs), 5, C.byref(r), None) == 0      # no output asked: no capacity needed
    assert (r.n_classes, r.n_members) == (len(want["class_len"]), len(want["member"]))
    base = np.zeros(1, np.int64)
    r = ts._CloneResult(None, None, None, ts._p(base), None, 0, -1, None, 0, -1)
    assert ts.lib().tsm_clones(scanner._ctx, C.byref(cs), 5, C.byref(r), None) == ts.TSM_E_CAPACITY
    assert (r.n_classes, r.n_members) == (len(want["class_len"]), len(want["member"]))
    for n in (0, 1025, -1):
        with pytest.raises(ts.TsmError) as e:
            scanner.clones(c, n)
        assert e.value.status == -1


def test_repeated_calls_and_a_nonblocking_stream(scanner, c1):
    torch = pytest.importorskip("torch")
    c = ts.pack(*c1)
    first = scanner.clones(c, 5)
    launches = scanner.last_launch_count()
    ocl.assert_equal(scanner.clones(c, 5), first)
    assert scanner.last_launch_count() == launches > 0
    s = torch.cuda.Stream()
    ocl.assert_equal(scanner.clones(c, 5, stream=C.c_void_p(s.cuda_stream)), first)


def write_tree(root, names, files):
    for name, data in zip(names, files):
        p = os.path.join(root, name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as fh:
            fh.write(data)


def expected_cli(roots, n):
    """stdout and --out of `tosem-scan clones` from the C reference: roots = [(name, [(rel, bytes, ext)])] in walk order."""
    files, exts, where = [], [], []
    for g, (name, entries) in enumerate(roots):
        for rel, data, ext in sorted(entries):
            files.append(data); exts.append(ext); where.append((g, rel))
    r = ocl.clones(ts.pack(files, exts), n)
    base = r["line_base"]
    fid = np.searchsorted(base, r["member"], side="right") - 1
    out = [["class", "repository", "fileName", "first_line", "last_line"]]
    per_root_classes = [set() for _ in roots]
    for c in range(len(r["class_len"])):
        for j in range(r["class_base"][c], r["class_base"][c + 1]):
            f = int(fid[j]); g, rel = where[f]
            first = int(r["member"][j] - base[f]) + 1
            out.append([str(c + 1), roots[g][0], rel, str(first), str(first + int(r["class_len"][c]) - 1)])
            per_root_classes[g].add(c)
    lines = np.diff(base)
    rows = [["repository", "files", "lines", "duplicated_lines", "assertion_lines", "duplicated_assertion_lines", "classes"]]
    tot = np.zeros(5, np.int64)
    for g, (name, _) in enumerate(roots):
        sel = [i for i, w in enumerate(where) if w[0] == g]
        alines = sum(sum(1 for ln in cu_lines(files[i]) if exts[i] and (b"assert" in ln.lower() or b"EXPECT_" in ln)) for i in sel)
        v = np.array([len(sel), lines[sel].sum(), r["file_dup"][sel].sum(), alines, r["file_dup_assert"][sel].sum()], np.int64)
        tot += v
        rows.append([name] + [str(int(x)) for x in v] + [str(len(per_root_classes[g]))])
    rows.append(["<all>"] + [str(int(x)) for x in tot] + [str(len(r["class_len"]))])
    return rows, out


def cu_lines(data):
    import spec_ref
    return spec_ref.py_lines(data)


def read_csv(text):
    assert "\r\n" in text or not text
    return [row for row in csv.reader(io.StringIO(text, newline=""))]


def test_cli_roots_and_git(tmp_path, c1):
    files, exts = c1
    names = cu.load_fixture_names(os.path.join(GOLD, "c1_testfiles.npz"))
    half = len(files) // 2
    roots = []
    for g, (lo, hi) in enumerate([(0, half), (half, len(files))]):
        name = "repo%d" % g
        rels = ["%s_test/%s" % (g, names[i].replace("/", "_")) for i in range(lo, hi)]
        write_tree(str(tmp_path / "a" / name), rels, files[lo:hi])
        roots.append((name, [(rel, files[i], int(exts[i])) for rel, i in zip(rels, range(lo, hi))]))
    want_rows, want_out = expected_cli(roots, 5)
    outp = str(tmp_path / "frag.csv")
    p = subprocess.run([CLI, "clones", str(tmp_path / "a" / "repo0"), str(tmp_path / "a" / "repo1"), "--out", outp],
                       capture_output=True, check=True)
    assert read_csv(p.stdout.decode()) == want_rows
    assert read_csv(open(outp, newline="").read()) == want_out
    # --git on a repository of one root's tree equals the root form on a checkout of that revision
    if shutil.which("git") is None:
        pytest.skip("git is not installed")
    repo = tmp_path / "g" / "repo0"
    shutil.copytree(tmp_path / "a" / "repo0", repo)
    env = dict(os.environ, GIT_AUTHOR_NAME="t", GIT_AUTHOR_EMAIL="t@t", GIT_COMMITTER_NAME="t", GIT_COMMITTER_EMAIL="t@t")
    for cmd in (["init", "-q"], ["add", "-A"], ["commit", "-q", "-m", "c1"]):
        subprocess.run(["git", "-C", str(repo)] + cmd, check=True, env=env)
    (repo / "later_test.py").write_bytes(files[0])
    subprocess.run(["git", "-C", str(repo), "add", "-A"], check=True, env=env)
    subprocess.run(["git", "-C", str(repo), "commit", "-q", "-m", "later"], check=True, env=env)
    gout = str(tmp_path / "gfrag.csv")
    first = subprocess.run(["git", "-C", str(repo), "rev-parse", "HEAD~1"], capture_output=True, check=True).stdout.decode().strip()
    g = subprocess.run([CLI, "clones", "--git", str(repo), "--rev", first, "--min-lines", "3", "--out", gout], capture_output=True, check=True)
    rout = str(tmp_path / "rfrag.csv")
    r = subprocess.run([CLI, "clones", str(tmp_path / "a" / "repo0"), "--min-lines", "3", "--out", rout], capture_output=True, check=True)
    assert g.stdout == r.stdout and open(gout, "rb").read() == open(rout, "rb").read()
    assert read_csv(g.stdout.decode())[1][0] == "repo0"
