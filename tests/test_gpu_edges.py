"""GPU edge tests: device paths the parity fuzz reaches rarely or never - Mersenne-61 line hashes of non-ASCII bytes, long
n-gram windows, the category table, k_classify's global histogram and full deferral queue, saturated statement fields and
corpora denser in events than a context's default lists.  Where the SPEC allows, the device is compared with the
plain-Python restatements of tests/spec_ref.py (pinned to the oracle by tests/test_spec_ref.py), otherwise with the
oracle; every field of every line or event is compared exactly."""
import json
import os
import random
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import orc
import spec_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu

FLAGS = ts.SCAN_ASSERT_EVENTS | ts.SCAN_HEADER_EVENTS
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "tosem-2021-replication_b200", "tosemscan", "tosem-scan")


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 30, max_files=1 << 18, max_groups=4096)
    yield s
    s.close()


def check_against_oracle(scanner, c, flags=FLAGS, rev_b=False):
    want = orc.scan(c.arena, c.off, c.len, c.ext, c.grp, c.n_groups, rev_b=rev_b)
    got = scanner.scan(c, flags | (ts.SCAN_REV_B if rev_b else 0))
    for f in ("n_lines", "n_assert", "n_headers", "n_fixture", "digest"):
        bad = np.nonzero(got["stats"][f] != want["stats"][f])[0]
        assert bad.size == 0, (f, bad[:10], got["stats"][bad[:5]], want["stats"][bad[:5]])
    assert np.array_equal(got["group_counts"], want["group_counts"])
    assert np.array_equal(got["global_counts"], want["global_counts"])
    for k in ("assert_events", "header_events"):
        if k in got:
            a, b = got[k], want[k]
            assert len(a) == len(b), (k, len(a), len(b))
            for f in a.dtype.names:
                bad = np.nonzero(a[f] != b[f])[0]
                assert bad.size == 0, (k, f, bad[:5], a[bad[:5]], b[bad[:5]])
    return got


class LineRef:
    """py_line_records per file, memoised per line (the filler lines repeat)."""

    def __init__(self):
        self.memo = {}

    def file(self, data, ext):
        out, pos = [], 0
        for line in sr.py_lines(data):
            key = (line, ext)
            if key not in self.memo:
                self.memo[key] = sr.py_line_records(line + b"\n", ext)[0]
            h, e, fl = self.memo[key]
            out.append((h, pos + e, fl))
            pos += len(line) + 1
        return out


def check_line_records_against_python(scanner, files, exts, ngrams=()):
    c = ts.pack(files, exts)
    gb, gh, ge, gf = scanner.line_hashes(c)
    ref = LineRef()
    want_h, want_e, want_f, want_b = [], [], [], [0]
    for f, e in zip(files, exts):
        recs = ref.file(f, e)
        want_h += [r[0] for r in recs]
        want_e += [r[1] for r in recs]
        want_f += [r[2] for r in recs]
        want_b.append(want_b[-1] + len(recs))
    assert gb.tolist() == want_b
    for name, a, b, dt in (("hash", gh, want_h, np.uint64), ("end", ge, want_e, np.uint32), ("flag", gf, want_f, np.uint8)):
        bad = np.nonzero(a != np.array(b, dt))[0]
        assert bad.size == 0, (name, bad[:8], a[bad[:4]], [b[i] for i in bad[:4]])
    st = scanner.scan(c, 0)["stats"]
    assert st["n_lines"].tolist() == np.diff(want_b).tolist()
    dig = [sum(want_h[want_b[i]:want_b[i + 1]]) & sr.MASK for i in range(len(files))]
    assert [int(x) for x in st["digest"]] == dig
    for n in ngrams:
        ng = scanner.line_hashes(c, ngram=n)[4]
        for i in range(len(files)):
            a, b = want_b[i], want_b[i + 1]
            assert [int(x) for x in ng[a:b]] == sr.py_ngrams(want_h[a:b], n), (n, i)
    return gh


def filler(n):
    """n bytes of short lines ending in LF (nothing for n = 0)."""
    q, r = divmod(n, 64)
    return (b"a" * 63 + b"\n") * q + (b"b" * (r - 1) + b"\n" if r else b"")


# ---------------------------------------------------------------------------------------- 1. hash arithmetic
def test_hash_arithmetic_behind_every_pad(scanner):
    """Each hash-edge content (0xFF runs, multiples of 2^61 - 1, wrapping CR steps, zeros, bare CRs) behind pads of
    0..150 bytes: every position in a word, a stripe (136 B) and a 4-word checkpoint group."""
    files = [b"#" * (pad - 1) + b"\n" + c + b"\nz" if pad else c + b"\n" for c in cu.hash_edge_contents() for pad in range(151)]
    check_line_records_against_python(scanner, files, [1] * len(files))


def test_hash_arithmetic_at_chunk_and_lookahead_edges(scanner):
    """The same contents ending at 4096 +- 8 (the chunk edge) and 4096 + 240 +- 8 (the end of the look-ahead), long
    contents across a chunk edge (the long-line slow path), and as unterminated last lines."""
    rng = random.Random(17)
    contents = cu.hash_edge_contents()
    files = []
    for c in contents:
        for end in list(range(4088, 4105)) + list(range(4328, 4345)):
            if end >= len(c):
                files.append(filler(end - len(c)) + c + b"\n" + b"y" * 9)
        files.append(b"x\n" + c)
        files.append(c)
    longs = [b"\xff" * n for n in (300, 301, 555, 4100, 9000)] + [cu.cr_wrap_content(rng, n) + b"\r" for n in (300, 333, 511, 1000, 5000)]
    longs += [((k * cu.M61) << (8 * 300)).to_bytes(320, "little") for k in (1, 2, 3)]   # value 0 mod p, 300 zero bytes in front
    for c in longs:
        for start in (4096 - 1, 4096 - 8, 4096 - 37, 4096 - 59, 4096 - 100, 2 * 4096 - 3):
            files.append(filler(start) + c + b"\n" + b"w" * 5)
            files.append(filler(start) + c)
    check_line_records_against_python(scanner, files, [1] * len(files))


def test_binary_fuzz_line_records(scanner):
    files, exts, _ = cu.fuzz_corpus(501, 300, 20000, long_lines=True, binary=True)
    check_line_records_against_python(scanner, files, [int(e) for e in exts], ngrams=(3,))
    check_against_oracle(scanner, ts.pack(files, exts))


# ---------------------------------------------------------------------------------------- 2. n-gram windows
@pytest.mark.parametrize("n", [1, 4, 5, 6, 7, 8, 13, 47, 48, 60, 61, 62, 200])
def test_ngram_windows(scanner, n):
    """Files of 0, 1, n-1, n and n+1 lines with empty files between them, against the big-integer windows."""
    rng = random.Random(n)
    contents = cu.hash_edge_contents()
    files = [b""]
    for k in (0, 1, n - 1, n, n + 1):
        lines = [rng.choice(contents) if rng.random() < 0.5 else b"line %d" % rng.randrange(1000) for _ in range(k)]
        files += [b"".join(l + b"\n" for l in lines), b"", b""]
    check_line_records_against_python(scanner, files, [1] * len(files), ngrams=(n,))


# ---------------------------------------------------------------------------------------- 3. the category table
def g4_rows():
    return json.load(open(os.path.join(GOLD, "g4_statement_category.json")))


def event_category_strings(files, ev):
    out = []
    for e in ev:
        if int(e["cat"]) == sr.OTHER:
            f = files[int(e["file"])]
            out.append(f[int(e["ident_off"]):int(e["ident_off"]) + int(e["ident_len"])].decode("latin-1"))
        else:
            out.append(sr.CATEGORY_NAMES.get(int(e["cat"]), ""))
    return out


@pytest.mark.parametrize("ext", [1, 2])
def test_g4_statements_through_k_classify(scanner, ext):
    """Every G4 statement S as the line `    S(assert_x)` (T stays S): the event categories equal py_category(S), and
    re-scoring the sheet rows from the device's events gives 11 954 / 11 981 with exactly the ledger's misses."""
    rows = g4_rows()
    stmts = [r["statement"].encode("utf-8") for r in rows]
    for s in stmts:
        assert b"(" not in s and b"\n" not in s and s == s.strip(sr.W)
    per = 400
    files = [b"".join(b"    " + s + b"(assert_x)\n" for s in stmts[i:i + per]) for i in range(0, len(stmts), per)]
    got = check_against_oracle(scanner, ts.pack(files, [ext] * len(files)))
    ev = got["assert_events"]
    assert len(ev) == len(stmts)
    assert [int(c) for c in ev["cat"]] == [sr.py_category(s) for s in stmts]
    assert [int(h) for h in ev["stmt_hash"]] == [sr.py_bytes_hash(s) for s in stmts]
    cells = event_category_strings(files, ev)
    ledger = json.load(open(os.path.join(GOLD, "ledger.json")))["G4"]
    hit = sum(r["rows"] for r, c in zip(rows, cells) if c == r["category"])
    misses = {(r["statement"], r["category"]) for r, c in zip(rows, cells) if c != r["category"]}
    assert [hit, sum(r["rows"] for r in rows)] == [11954, 11981]
    assert misses == {(m["statement"], m["sheet_says"]) for m in ledger["misses"]}


@pytest.mark.parametrize("rev_b", [False, True], ids=["rev_a", "rev_b"])
def test_table_names_and_near_misses(scanner, rev_b):
    """Every table name as `self.<name>(` and its near misses, at every indentation mod 8 (the FNV perfect hash over
    8-byte loads and the exact compare).  Rev B too: rules 1b / 2b do not apply to `self.` statements."""
    names = [n.encode() for n in sr.CATEGORY_NAMES.values()]
    variants = cu.table_name_variants(names)
    lines = [b" " * (i % 8) + b"self." + v + b"(a, b)\n" for i, v in enumerate(variants)]
    files = [b"".join(lines[i:i + 500]) for i in range(0, len(lines), 500)]
    for ext in (1, 3):
        got = check_against_oracle(scanner, ts.pack(files, [ext] * len(files)), rev_b=rev_b)
        ev = got["assert_events"]
        want = [sr.py_category(b"self." + v) for v, l in zip(variants, lines) if sr.py_is_assert_line(l, ext)]
        assert len(want) > 0.8 * len(variants) and [int(c) for c in ev["cat"]] == want


# ---------------------------------------------------------------------------------------- 4. k_classify paths
@pytest.mark.parametrize("rev_b", [False, True], ids=["rev_a", "rev_b"])
@pytest.mark.parametrize("n_groups", [1, 16, 17, 100, 4096])
def test_group_counts_at_every_histogram_size(scanner, n_groups, rev_b):
    """n_groups <= 16: the shared-memory histogram; more: global atomics on the group row and the global row."""
    files, exts, _ = cu.fuzz_corpus(31, 600, 3000)
    rng = np.random.default_rng(n_groups)
    for grp in (rng.integers(0, n_groups, len(files)), rng.integers(max(n_groups - 3, 0), n_groups, len(files))):
        got = check_against_oracle(scanner, ts.pack(files, exts, grp.astype(np.uint16), n_groups), rev_b=rev_b)
        assert np.array_equal(got["group_counts"].sum(axis=0), got["global_counts"])
        assert int(got["global_counts"].sum()) == int(got["totals"][1]) > 0


BARE = [b"assert not a", b"assert a not in b", b"assert x is not None", b"assert x == True", b"assert a == b",
        b"assert a != b", b"assert a <= b", b"assert a >= b", b"assert a < b", b"assert a > b", b"assert ok",
        b"assert b'not in' in x", b"assert not_a", b"assert x and True", b"assert  not a"]
OTHER_ASSERTS = [b"self.assertEqual(a, b)", b"EXPECT_EQ(a, b);", b"assert", b"x.assert_called_with(1)"]


def test_full_deferral_queue(scanner):
    """1.6 M assertion lines, 95 % bare `assert <expr>` over every operator of SPEC section 6 rule 2: more than
    BQ_CAP = 1 024 deferrals per block of k_classify's grid (at most 132 x 8 blocks of 256 threads), so every block
    decides some inline after its queue is full."""
    rng = np.random.default_rng(7)
    pool = BARE + OTHER_ASSERTS
    p = np.array([0.95 / len(BARE)] * len(BARE) + [0.05 / len(OTHER_ASSERTS)] * len(OTHER_ASSERTS))
    pick = rng.choice(len(pool), size=1_600_000, p=p / p.sum())
    lines = [pool[i] + b"\n" for i in pick]
    files = [b"".join(lines[i:i + 50000]) for i in range(0, len(lines), 50000)]
    got = check_against_oracle(scanner, ts.pack(files, [1, 3] * (len(files) // 2)))
    assert len(got["assert_events"]) == 1_600_000
    assert int(np.isin(pick, range(len(BARE))).sum()) > 4 * 132 * 8 * 256


# ---------------------------------------------------------------------------------------- 5. long lines and statements
def test_saturated_statement_fields_and_full_statement_hash(scanner):
    """stmt_len / ident_len saturate at 65 535 while stmt_hash covers the whole T; a '(' as the last byte of a file."""
    files = [b"    assert " + b"x" * 70000 + b"\n", b"self.assert" + b"y" * 70000 + b"(q)\n"]
    files += [b"  self.assert" + b"z" * (65535 - 11 + d) + b"(q)\n" for d in (-1, 0, 1)]
    files += [b"  assert " + b"k" * (65535 - 7 + d) + b"\n" for d in (-1, 0, 1)]
    files += [b"assert x(", b"  self.assertEqual(", b"x\nEXPECT_EQ(", b"assert ("]
    for ext in (1, 2):
        got = check_against_oracle(scanner, ts.pack(files, [ext] * len(files)))
        ev = got["assert_events"]
        assert len(ev) == len(files)
        for e in ev:
            f = files[int(e["file"])]
            line = f[int(e["line_off"]):].split(b"\n", 1)[0]
            t = sr.py_statement(line)
            s, n = sr.py_ident(t)
            assert int(e["stmt_len"]) == min(len(t), 65535) and int(e["ident_len"]) == min(n, 65535)
            assert int(e["stmt_hash"]) == sr.py_bytes_hash(t) and int(e["cat"]) == sr.py_category(t)
    assert [min(len(sr.py_statement(f.split(b"\n")[0])), 65535) for f in files[:2]] == [65535, 65535]


@pytest.mark.parametrize("rev_b", [False, True], ids=["rev_a", "rev_b"])
def test_triggers_inside_lines_longer_than_the_lookahead(scanner, rev_b):
    """Rev-A and Rev-B triggers at every offset mod 8 inside lines that start in one chunk and end more than 240 B
    into the next (long_line, the automaton walked from HBM), before, on and behind the chunk edge."""
    trig = [b"assert", b"EXPECT_", b"_CHECK", b"TESTEQUAL", b"FAIL"]
    files = []
    for t in trig:
        for at in (4000, 4090, 4096, 4101, 4200, 4330, 4336, 4400, 5000):
            for k in range(8):
                start = 3990 - k
                body = b"q" * (at + k - start) + t + b" x == 1(r)" + b"w" * 500
                files.append(filler(start) + body + b"\n" + b"assert tail\n")
    got = check_against_oracle(scanner, ts.pack(files, [1, 2] * (len(files) // 2) + [3] * (len(files) % 2)), rev_b=rev_b)
    if not rev_b:
        for e in got["assert_events"]:
            f = files[int(e["file"])]
            t = sr.py_statement(f[int(e["line_off"]):].split(b"\n", 1)[0])
            assert int(e["stmt_hash"]) == sr.py_bytes_hash(t) and int(e["cat"]) == sr.py_category(t)


LONG_HEADS = [b"class Foo(Base):", b"class", b"def test_x(self):", b"TEST_F(Fix, Name) {", b"TEST_F(Fix, Name)",
              b"test_case(int x) {", b"void helper(int x) {"]


@pytest.mark.parametrize("rev_b", [False, True], ids=["rev_a", "rev_b"])
@pytest.mark.parametrize("ext", [1, 2, 4, 0], ids=["py", "cc", "java", "none"])
def test_header_rules_on_lines_longer_than_the_lookahead(scanner, ext, rev_b):
    """Header and fixture-header lines (`class` + blank + text, `class` + only blanks, `def`, `TEST_F(` with and
    without `{`, `test ... {`, `void ... {`) that start in one chunk at every offset mod 8 and end more than 240 B
    into the next (long_line reads them from HBM): behind 0-20 blanks of indentation (runs of spaces, with and
    without tabs), ended by LF, by CR LF, or unterminated at the end of the file."""
    indents = [b" " * n for n in range(21)] + [b"\t", b" \t", b"\t" * 9 + b" ", b" " * 7 + b"\t" + b" " * 7,
                                               b"\t " * 10, b" " * 15 + b"\t"]
    files = []
    for h, head in enumerate(LONG_HEADS):
        pad = b" " * 500 + b"\t" if head == b"class" else b" " + b"z" * 500
        for i, ind in enumerate(indents):
            for k in range(8):
                end = (b"\n", b"\r\n", b"")[(h + i + k) % 3]
                files.append(filler(4000 + k) + ind + head + pad + end + (b"def tail():\n" if end else b""))
    c = ts.pack(files, [ext] * len(files))
    got = check_against_oracle(scanner, c, rev_b=rev_b)
    if ext:
        assert int(got["stats"]["n_headers"].sum()) > len(files) // 4 and (ext == 1) == (int(got["stats"]["n_fixture"].sum()) == 0)
    if not rev_b:                                        # (line records are Rev A's)
        want = orc.line_records(c.arena, c.off, c.len, c.ext)
        for a, b in zip(scanner.line_hashes(c), want):
            assert np.array_equal(a, b)


# ---------------------------------------------------------------------------------------- 6. dense events
DENSE = [(b"assert\n", 1, False), (b"def\n", 1, False), (b"{test\n", 2, False), (b"FAIL\n", 2, True)]


def cli_sized_scanner(c):
    """A context sized the way `tosem-scan scan` sizes its own: the batch's arena + 4 KiB, default event lists."""
    return ts.Scanner(device=0, max_arena_bytes=int(c.off[-1]) + 4096, max_files=max(c.n_files, 16), max_groups=1, max_events=0)


@pytest.mark.parametrize("line,ext,rev_b", DENSE, ids=["assert", "def", "brace_test", "FAIL_rev_b"])
def test_dense_event_corpora(line, ext, rev_b):
    """2 MB of one short assertion or header line: 8x more events than the default lists (arena / 32) and more than
    the default host arrays (bytes / 8).  Through tsm_scan and through upload / scan_resident / download."""
    data = line * ((2 << 20) // len(line))
    c = ts.pack([b"x\n", data], [ext, ext])
    want = orc.scan(c.arena, c.off, c.len, c.ext, c.grp, 1, rev_b=rev_b)
    flags = FLAGS | (ts.SCAN_REV_B if rev_b else 0)
    n_ev = len(want["assert_events"]) + len(want["header_events"])
    assert n_ev > 4 * ((int(c.off[-1]) + 4096) // 32 + 16) and n_ev > c.source_bytes // 8 + 16
    s = cli_sized_scanner(c)
    outs = [s.scan(c, flags)]
    s.close()
    s = cli_sized_scanner(c)
    s.upload(c)
    s.scan_resident(flags)
    outs.append(s.download(flags))
    s.scan_resident(flags)                               # the grown lists are kept: no rerun, the same results
    outs.append(s.download(flags))
    s.close()
    for got in outs:
        assert np.array_equal(got["stats"], want["stats"])
        assert np.array_equal(got["group_counts"], want["group_counts"]) and np.array_equal(got["global_counts"], want["global_counts"])
        assert np.array_equal(got["assert_events"], want["assert_events"])
        assert np.array_equal(got["header_events"], want["header_events"])


def dense_tree(tmp_path, line):
    """A project whose only file, tests/test_dense.py, is 2 MB of `line`; returns the number of lines."""
    n = (2 << 20) // len(line)
    p = tmp_path / "proj" / "tests" / "test_dense.py"
    p.parent.mkdir(parents=True)
    p.write_bytes(line * n)
    return n


def test_dense_events_through_the_cli(tmp_path):
    """`tosem-scan scan` over a tree whose only file is 2 MB of `assert\\n`."""
    n = dense_tree(tmp_path, b"assert\n")
    sum_p = str(tmp_path / "summary.csv")
    out = subprocess.run([CLI, "scan", str(tmp_path / "proj"), "--summary", sum_p], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    agg = dict(l.split(",") for l in out.stdout.replace("\r\n", "\n").strip().split("\n")[1:])
    assert {k: int(v) for k, v in agg.items() if int(v)} == {"assertTrue": n}
    rows = open(sum_p, "rb").read().decode().split("\r\n")
    assert rows[1].split(",")[1:3] == ["tests/test_dense.py", str(n)]


@pytest.mark.parametrize("cmd", ["body", "releases"])
def test_dense_events_through_body_and_releases(tmp_path, cmd):
    """`tosem-scan body` over 2 MB of `def\\n` and `releases` over 2 MB of `assert\\n`: more events than the host arrays of
    bytes / 8 + 1024 both commands start with, as for `scan` above."""
    n = dense_tree(tmp_path, b"def\n" if cmd == "body" else b"assert\n")
    outp = str(tmp_path / "out.csv")
    proj = str(tmp_path / "proj")
    out = subprocess.run([CLI, "body", proj, "--out", outp] if cmd == "body" else [CLI, "releases", proj + "=v1", "--out", outp],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = open(outp, "rb").read().decode().split("\r\n")
    if cmd == "body":
        assert orc.header_kind(1, b"def")                   # every line starts a case; a case header is no statement
        assert out.stdout.replace("\r\n", "\n").strip().split("\n") == ["files,cases,statements", "1,%d,0" % n]
        assert len(rows) == n + 2 and rows[-2].split(",")[::3] == [str(n), str(n)]
    else:
        assert rows[1].split(",") == ["1", "tests/test_dense.py", "tests/test_dense.py", str(n), "%d:assertTrue" % n]
