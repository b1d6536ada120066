"""`tsm_clones_blind` / `Scanner.clones(..., blind=True)` (docs/SPEC.md section 21) bit for bit against the serial C reference
(tests/orc_blind.c), every output array: the C1 test files at windows of 1, 3, 5 and 10 kept lines with the pinned counts, the
hazard files (2 061-byte lines, CRLF, no trailing LF, non-UTF-8), a C4-scale corpus with planted Type-2 copies, the line-state
scan under stress (a 60 000-line block comment and docstring, states that flip on every line, many files that open a comment on
their first line), lines of 16 KiB, a corpus without a kept line and an empty one; the raw ABI (argument checks, each output
NULL, each cap exact and short) and a non-blocking stream while the legacy stream is busy; and `tosem-scan clones --blind` over
a tree and over a git revision."""
import ctypes as C
import csv
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import blind_ref as br
import corpus_util as cu
import orc_blind as ob
import spec_ref
import tosemscan as ts
from test_clones_blind_ref import C1_KEPT, C1_PINNED

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tosem-2021-replication_b200", "tosemscan", "tosem-scan")


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 28, max_files=1 << 17, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def c1():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    return files, exts


def check(s, corpus, n, **kw):
    got = s.clones(corpus, n, blind=True, **kw)
    br.assert_equal(got, ob.clones_blind(corpus, n))
    return got


@pytest.mark.parametrize("n", [1, 3, 5, 10])
def test_c1(scanner, c1, n):
    got = check(scanner, ts.pack(*c1), n)
    assert len(got["kept_line"]) == C1_KEPT
    if n in C1_PINNED:
        assert (len(got["class_len"]), len(got["member"]), int(got["file_dup"].sum()), int(got["file_dup_assert"].sum())) == C1_PINNED[n]
    ms = scanner.clones_blind_last_ms()
    assert len(ms) == 4 and all(m > 0 for m in ms)


def test_hazard_files(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_hazard_files.npz"))
    check(scanner, ts.pack(files, exts), 5)


KEYWORDS = br.PY_KEYWORDS | br.CJ_KEYWORDS | br.PY_LITERALS | br.CJ_LITERALS


def type2_copy(data, ext, rng):
    """A Type-2 copy: identifiers renamed, numbers changed, every line re-indented, a comment line after every fifth."""
    def rename(m):
        w = m.group(0)
        return w if w in KEYWORDS else w + b"_copy"
    out = []
    for k, line in enumerate(data.split(b"\n")):
        line = re.sub(rb"[A-Za-z_][A-Za-z0-9_]*", rename, line)
        line = re.sub(rb"\b[0-9]+\b", lambda m: b"%d" % rng.integers(0, 1000), line)
        out.append(b"    " + line if line else line)
        if k % 5 == 4 and ext:
            out.append(b"    # copied" if ext == 1 else b"    // copied")
    return b"\n".join(out)


def test_c4_scale_planted_type2_copies(scanner):
    n_files = 100000
    c = ts.gen_corpus(0x7053454D0C4B, n_files, size_law=1, pinned=False)
    files = [c.file_bytes(i) for i in range(n_files)]
    rng = np.random.default_rng(21)
    for i in range(4, n_files, 4):
        j = int(rng.integers(0, i))
        files[i] = type2_copy(files[j], int(c.ext[j]), rng)
        c.ext[i] = c.ext[j]
    got = check(scanner, ts.pack(files, c.ext), 5)
    assert len(got["class_len"]) > 10000 and got["file_dup"][4::4].sum() > 0.5 * (np.diff(got["kept_base"])[4::4].sum())


def test_line_state_scan_stress(scanner):
    long_comment = b"/* opens on line 0\n" + b"".join(b"int x%d = %d;\n" % (i, i) for i in range(59998)) + b"*/ done();\n"
    long_doc = b'"""opens on line 0\n' + b"".join(b"x%d = %d\n" % (i, i) for i in range(59998)) + b'""" + done()\n'
    flip_c = b"".join(b"a%d = 1; /* x\n*/ b%d = 2;\n" % (i, i) for i in range(3000))
    flip_py = b"".join(b"a%d = '''x\n''' + b%d\n" % (i, i) for i in range(3000))
    openers = [b"/* never closed\nint x = 1;\nint y = 2;\n", b"int x = 1;\nint y = 2;\nint z = 3;\n"] * 2000
    files = [long_comment, long_doc, flip_c, flip_py, flip_c, flip_py, long_comment] + openers
    exts = [3, 1, 3, 1, 4, 1, 5] + [3, 3] * 2000
    got = check(scanner, ts.pack(files, exts), 2)
    kb = got["kept_base"]
    assert kb[1] - kb[0] == 1 and kb[2] - kb[1] == 2 and kb[3] - kb[2] == 6000 and kb[8] - kb[7] == 0 and kb[9] - kb[8] == 3


def test_lines_of_16_kib(scanner):
    long_code = b"x = " + b" + ".join(b"v%d" % i for i in range(3000))[:16380] + b"\n"
    long_str = b's = "' + b"a # b " * 2730 + b'"\n'
    long_cmt = b"int a; /* " + b"x " * 8190 + b"*/ int b;\n"
    assert min(len(long_code), len(long_str), len(long_cmt)) >= 16380
    files = [long_code + long_str, long_cmt * 3, long_code + long_str + b"y = 1\n", long_cmt * 2]
    got = check(scanner, ts.pack(files, [1, 3, 1, 4]), 2)
    assert len(got["class_len"]) >= 2


def test_no_kept_line_and_empty_corpus(scanner):
    files = [b"# c\n\n   \n", b"// a\n/* b\n c */\n", b""]
    got = check(scanner, ts.pack(files, [1, 3, 2]), 1)
    assert got["kept_base"].tolist() == [0, 0, 0, 0] and len(got["member"]) == 0 and got["line_base"].tolist() == [0, 3, 6, 6]
    got = check(scanner, ts.pack([], []), 3)
    assert got["line_base"].tolist() == [0] and got["kept_base"].tolist() == [0] and len(got["kept_line"]) == 0


def raw(scanner, c, n, kept_cap, class_cap, member_cap, drop=()):
    """One raw tsm_clones_blind call with every output of the given caps, the names in `drop` passed as NULL."""
    nf = c.n_files
    a = {"line_base": np.zeros(nf + 1, np.int64), "file_dup": np.zeros(nf, np.uint32), "file_dup_assert": np.zeros(nf, np.uint32),
         "class_base": np.zeros(class_cap + 1, np.int64), "class_len": np.zeros(max(class_cap, 1), np.uint32),
         "member": np.zeros(max(member_cap, 1), np.int64), "kept_base": np.zeros(nf + 1, np.int64),
         "kept_line": np.zeros(max(kept_cap, 1), np.int64), "blind_hash": np.zeros(max(kept_cap, 1), np.uint64),
         "file_kept_assert": np.zeros(nf, np.uint32)}
    p = {k: (None if k in drop else ts._p(v)) for k, v in a.items()}
    r = ts._CloneResult(p["line_base"], p["file_dup"], p["file_dup_assert"], p["class_base"], p["class_len"], class_cap, -1,
                        p["member"], member_cap, -1)
    b = ts._BlindResult(p["kept_base"], p["kept_line"], p["blind_hash"], p["file_kept_assert"], kept_cap, -1)
    cs = c.c_struct()
    rc = ts.lib().tsm_clones_blind(scanner._ctx, C.byref(cs), n, C.byref(b), C.byref(r), None)
    return rc, a, (b.n_kept, r.n_classes, r.n_members)


def test_raw_abi(scanner, c1):
    c = ts.pack(*c1)
    want = ob.clones_blind(c, 5)
    counts = (len(want["kept_line"]), len(want["class_len"]), len(want["member"]))
    rc, a, got = raw(scanner, c, 5, *counts)                          # every cap exact
    assert rc == 0 and got == counts
    a["class_base"], a["class_len"], a["member"] = a["class_base"][:counts[1] + 1], a["class_len"][:counts[1]], a["member"][:counts[2]]
    br.assert_equal(a, want)
    for k in br.KEYS:                                                 # each output NULL: the others are still filled
        rc, a, got = raw(scanner, c, 5, *counts, drop=(k,))
        assert rc == 0 and got == counts
        assert all(np.array_equal(a[j][:len(want[j])], want[j]) for j in br.KEYS if j != k), k
    for i in range(3):                                                # each cap one short
        caps = list(counts)
        caps[i] -= 1
        rc, _, got = raw(scanner, c, 5, *caps)
        assert rc == ts.TSM_E_CAPACITY and got == counts, i
    rc, _, got = raw(scanner, c, 5, 0, 0, 0, drop=("kept_line", "blind_hash", "class_base", "class_len", "member"))
    assert rc == 0 and got == counts                                  # no array asked for: no capacity needed
    cs = c.c_struct()
    for n, kc, cc in ((0, 0, 0), (1025, 0, 0), (5, -1, 0), (5, 0, -1)):
        r = ts._CloneResult(None, None, None, None, None, cc, 0, None, 0, 0)
        b = ts._BlindResult(None, None, None, None, kc, 0)
        assert ts.lib().tsm_clones_blind(scanner._ctx, C.byref(cs), n, C.byref(b), C.byref(r), None) == -1
    r = ts._CloneResult(None, None, None, None, None, 0, 0, None, 0, 0)
    assert ts.lib().tsm_clones_blind(scanner._ctx, C.byref(cs), 5, None, C.byref(r), None) == 0   # blind may be NULL
    assert ts.lib().tsm_clones_blind(scanner._ctx, C.byref(cs), 5, None, None, None) == -1


def test_repeated_calls_and_a_nonblocking_stream_with_the_legacy_stream_busy(scanner, c1):
    torch = pytest.importorskip("torch")
    c = ts.pack(*c1)
    first = check(scanner, c, 5)
    launches = scanner.last_launch_count()
    br.assert_equal(scanner.clones(c, 5, blind=True), first)
    assert scanner.last_launch_count() == launches > 0
    s = torch.cuda.Stream()
    legacy = torch.cuda.default_stream()
    with torch.cuda.stream(legacy):
        torch.cuda._sleep(50_000_000)                                  # a bounded spin (well under a second)
    br.assert_equal(scanner.clones(c, 5, blind=True, stream=C.c_void_p(s.cuda_stream)), first)
    legacy.synchronize()
    s.synchronize()


def write_tree(root, names, files):
    for name, data in zip(names, files):
        p = os.path.join(root, name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as fh:
            fh.write(data)


def expected_cli(roots, n):
    """stdout and --out of `tosem-scan clones --blind` from the C reference: roots = [(name, [(rel, bytes, ext)])] in walk order."""
    files, exts, where = [], [], []
    for g, (name, entries) in enumerate(roots):
        for rel, data, ext in sorted(entries):
            files.append(data); exts.append(ext); where.append((g, rel))
    r = ob.clones_blind(ts.pack(files, exts), n)
    base, kb, kl = r["line_base"], r["kept_base"], r["kept_line"]
    fid = np.searchsorted(kb, r["member"], side="right") - 1
    out = [["class", "repository", "fileName", "first_line", "last_line"]]
    per_root_classes = [set() for _ in roots]
    for c in range(len(r["class_len"])):
        for j in range(r["class_base"][c], r["class_base"][c + 1]):
            f = int(fid[j]); g, rel = where[f]
            at = int(r["member"][j])
            first, last = int(kl[at] - base[f]) + 1, int(kl[at + int(r["class_len"][c]) - 1] - base[f]) + 1
            out.append([str(c + 1), roots[g][0], rel, str(first), str(last)])
            per_root_classes[g].add(c)
    lines = np.diff(kb)
    rows = [["repository", "files", "lines", "duplicated_lines", "assertion_lines", "duplicated_assertion_lines", "classes"]]
    tot = np.zeros(5, np.int64)
    for g, (name, _) in enumerate(roots):
        sel = [i for i, w in enumerate(where) if w[0] == g]
        v = np.array([len(sel), lines[sel].sum(), r["file_dup"][sel].sum(), r["file_kept_assert"][sel].sum(), r["file_dup_assert"][sel].sum()],
                     np.int64)
        tot += v
        rows.append([name] + [str(int(x)) for x in v] + [str(len(per_root_classes[g]))])
    rows.append(["<all>"] + [str(int(x)) for x in tot] + [str(len(r["class_len"]))])
    return rows, out


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
    p = subprocess.run([CLI, "clones", str(tmp_path / "a" / "repo0"), str(tmp_path / "a" / "repo1"), "--blind", "--out", outp],
                       capture_output=True, check=True)
    assert read_csv(p.stdout.decode()) == want_rows
    assert read_csv(open(outp, newline="").read()) == want_out
    rows = read_csv(p.stdout.decode())
    assert all(int(r[3]) <= int(r[2]) for r in rows[1:])              # duplicated_lines <= lines
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
    first = subprocess.run(["git", "-C", str(repo), "rev-parse", "HEAD~1"], capture_output=True, check=True).stdout.decode().strip()
    gout, rout = str(tmp_path / "gfrag.csv"), str(tmp_path / "rfrag.csv")
    g = subprocess.run([CLI, "clones", "--git", str(repo), "--rev", first, "--blind", "--min-lines", "3", "--out", gout],
                       capture_output=True, check=True)
    r = subprocess.run([CLI, "clones", str(tmp_path / "a" / "repo0"), "--blind", "--min-lines", "3", "--out", rout], capture_output=True,
                       check=True)
    assert g.stdout == r.stdout and open(gout, "rb").read() == open(rout, "rb").read()
    plain = subprocess.run([CLI, "clones", str(tmp_path / "a" / "repo0"), "--min-lines", "3"], capture_output=True, check=True)
    assert plain.stdout != r.stdout and read_csv(r.stdout.decode())[1][0] == "repo0"


def test_blind_hash_matches_the_blind_form(scanner):
    text = b'def test_x(self):\n    """doc\n    more"""\n    self.assertEqual(f(1), "a")  # c\n'
    got = check(scanner, ts.pack([text], [1]), 1)
    assert got["blind_hash"].tolist() == [spec_ref.py_bytes_hash(f) for f in br.blind_lines(text, 1) if f]
