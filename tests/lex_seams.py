"""Crafted corpora for the lexical test smells (docs/SPEC.md section 25: k_lex_body, k_lex_lines and k_lex_tests in
csrc/tsm_lexsmell_kernels.cuh, driven by lex_stage in csrc/tsm_api.cu), built to sit on the seams of those kernels, and the host
facts that show each corpus reaches its seams.  TEST INFRASTRUCTURE ONLY.

* The names: `kernel_names` reads every name the kernels compare an identifier with (lx_name("...") and lx_is_long(..., "..."))
  out of the kernel source; `name_corpus` places each, and its one-byte variants, in a call or code line on the load grid of
  front_seams (every line start and name start modulo 8).
* The walk: `cap_corpus` puts the token that decides a statement (its message or its magic number) 62 to 65 lines below the
  assertion line, and the body end 63 to 65 lines below it.
* The token automata: `automaton_corpus` writes every short token sequence as the argument or expression of every statement form,
  and every short code line, one per test.
* The name sets: `nameset_corpus` holds the name whose hash is the empty-slot key, names whose home slot is the last one, 32 copies
  of a name in one round, 300 names on one line and more tests than the launch has warps.
* The body scan: `body_corpus` puts header statements, docstrings and test starts on both sides of 32-line rounds.

Each builder returns (files, exts, reach): `reach` holds what the corpus reaches, computed from its bytes, and the tests assert it.
"""
import itertools
import os
import random
import re

import front_seams as fs
import lexsmell_ref as lr
import spec_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEX_KERNELS = os.path.join(ROOT, "tosem-2021-replication_b200", "csrc", "tsm_lexsmell_kernels.cuh")
M64 = (1 << 64) - 1
SET_SLOTS = 512                                       # LEX_SET_SLOTS: the shared set of a test of up to 256 names
# An identifier whose section-3 hash is 2^64 - 1, the key of an empty slot (py_bytes_hash inverted through the mix finaliser)
SENTINEL = b"\xf8Y5\xa9Jqr\xa1c\xc3\xb7\xfe\x82\xb5\xac\xcbYr\xd6\xa5AEoX"


# -------------------------------------------------------------------------------------------------------------------- names
def kernel_names():
    """Every name of lx_name("...") and lx_is_long(..., "...") in the kernel source."""
    src = open(LEX_KERNELS).read()
    return {w.encode() for pair in re.findall(r'lx_name\("([^"]*)"\)|lx_is_long\([^")]*"([^"]*)"\)', src) for w in pair if w}


# Names the reference compares with in its code rather than in a table (keywords, the call prefixes, the keyword arguments)
REF_CODE_NAMES = {b"assert", b"static_assert", b"is", b"in", b"not", b"assert_", b"EXPECT_", b"ASSERT_", b"msg", b"err_msg",
                  b"isinstance", b"equals"}


def reference_names():
    """The names of lexsmell_ref's tables and of REF_CODE_NAMES."""
    tables = (lr.PY_ARITY1, lr.PY_ARITY3, lr.PY_UNCOUNTED, lr.PY_UNCOUNTED_EXACT, lr.MOCK_PREFIXES, lr.MOCK_EXACT, lr.J_ARITY1,
              lr.SUB_BOOL, lr.SUB_EQ, lr.PY_GUEST_CALLS, lr.CJ_GUEST_CALLS, lr.CJ_GUEST_NAMES)
    return set().union(*map(set, tables)) | REF_CODE_NAMES


def swap(c):
    """Another identifier byte for byte c (a case flip's neighbour: 'd' -> 'e')."""
    x = c ^ 1
    return x if chr(x).isalnum() else ord("x") if c != ord("x") else ord("y")


def variants(name):
    """The name, its last byte changed, its byte 16 changed (names longer than 16 bytes), its last byte dropped, a byte added."""
    out = [name, name[:-1] + bytes([swap(name[-1])]), name[:-1], name + b"x"]
    if len(name) > 16:
        out.append(name[:16] + bytes([swap(name[16])]) + name[17:])
    return [w for w in out if w]


def templates(name):
    """[(ext, head, tail)]: the lines in which the name is compared - a call of every family whose names it may start, the
    keyword argument, isinstance and equals trackers, the Mystery Guest calls and names, and the keywords' statements."""
    if name in (b"msg", b"err_msg"):
        return [(1, b"np.testing.assert_allclose(a, b, ", b"='m')"), (1, b"self.assertEqual(a, b, ", b"='m')")]
    if name == b"isinstance":
        return [(1, b"self.assertTrue(", b"(x, int))")]
    if name == b"equals":
        return [(4, b"assertTrue(a.", b"(b));")]
    if name in lr.PY_GUEST_CALLS:
        out = [(1, b"v = ", b"(f)")]
        return out + ([(3, b"auto v = ", b"(f);")] if name in lr.CJ_GUEST_CALLS else [])
    if name in lr.CJ_GUEST_CALLS:
        return [(3, b"auto v = ", b"(f);"), (4, b"Object v = ", b"(f);")]
    if name in lr.CJ_GUEST_NAMES:
        return [(3, b"", b" v;"), (4, b"", b" v = g();")]
    if name in (b"assert", b"static_assert"):
        return [(1, b"", b" x == 1"), (3, b"", b"(x == 1);"), (4, b"", b" x == 1;")]
    if name in (b"is", b"in", b"not"):
        return [(1, b"assert a ", b" 1")]
    if name.startswith((b"EXPECT_", b"ASSERT_")):
        return [(3, b"", b"(a, 1);")]
    return [(1, b"self.", b"(a, 1)"), (1, b"", b"(a, 1)"), (4, b"", b"(a, 1);")]


# `assert` (in any case) or `EXPECT_` inside a longer identifier, at every position
ASSERT_CORES = [b"assert", b"ASSERT", b"Assert", b"asSErT", b"EXPECT_", b"expect_", b"EXPECT", b"assrt"]


def embedded_words():
    return [b"q" * p + core + b"z" * (12 - p) for core in ASSERT_CORES for p in range(13)]


class FastGrid(fs.Grid):
    """front_seams.Grid that keeps its length as it grows (the name corpus has some 50 000 lines)."""

    def __init__(self):
        super().__init__()
        self.n = 0

    def pos(self):
        return self.n

    def add(self, line):
        super().add(line)
        self.n += len(line) + 1


HEADS = {1: b"def test_names():", 2: b"void test_names() {", 3: b"TEST(S, Names) {", 4: b"  public void testNames() {"}
ENDS = {1: None, 2: b"}", 3: b"}", 4: b"  }"}


def name_corpus():
    """Every kernel name, its variants and the embedded `assert` / `EXPECT_` words in every template that applies, at every line
    start and name start modulo 8, one test per ext.  reach: (ext, head, word) -> placements; `marks`: (file, line, head, word)
    of every placed line."""
    words = []
    for n in sorted(kernel_names()):
        words += [(w, n) for w in variants(n)]
    by_ext = {}
    seen = set()
    for w, n in words:
        for ext, head, tail in templates(n):
            if (ext, head, w) not in seen:
                seen.add((ext, head, w))
                by_ext.setdefault(ext, []).append((w, head, tail))
    for w in embedded_words():
        for ext, head, tail in ((1, b"self.", b"(a, 1)"), (3, b"", b"(a, 1);"), (4, b"", b"(a, 1);")):
            by_ext.setdefault(ext, []).append((w, head, tail))
    files, exts, reach, marks = [], [], {}, []
    for ext in sorted(by_ext):
        g = FastGrid()
        g.add(HEADS[ext])
        for w, head, tail in by_ext[ext]:
            for a in range(8):
                for o in range(8):
                    g.place((ext, head, w), a, b"    " + b" " * o + head, w, tail)
        if ENDS[ext]:
            g.add(ENDS[ext])
        reach.update(g.reach())
        marks += [(len(files), ln, name[1], name[2]) for name, ln, _, _ in g.marks]
        files.append(g.data())
        exts.append(ext)
    reach = {"grid": reach, "marks": marks, "words": {w for w, _ in words}}
    return files, exts, reach


def long_name_misses():
    """Variants of the kernel's names longer than 16 bytes that share the name's first 16 bytes (assert_not_callee)."""
    out = set()
    for n in kernel_names():
        if len(n) > 16:
            out |= {w for w in variants(n) if w != n and len(w) == len(n) and w[:16] == n[:16]}
    return out


# ----------------------------------------------------------------------------------------------------------------- the walk
# (name, ext, first line, filler, token line, decides): the statement opens on its first line, filler lines follow and the token
# that decides it comes on its own line; decides: "msg" (explained when seen) or "magic" (a magic number when seen)
CAP_FORMS = [
    ("unittest_msg", 1, b"self.assertEqual(a,", b"# c", b"b, 'm')", "msg"),
    ("unittest_magic", 1, b"self.assertEqual(a,", b"# c", b"5)", "magic"),
    ("numpy_msg", 1, b"np.testing.assert_allclose(a, b,", b"# c", b"msg='m')", "msg"),
    ("py_backslash", 1, b"assert x \\", b"\\", b", 'm'", "msg"),
    ("py_bracket", 1, b"assert (x", b"# c", b"), 'm'", "msg"),
    ("gtest_after", 3, b"EXPECT_EQ(a,", b"// c", b'b) << "m";', "msg"),
    ("static_second", 3, b"static_assert(x,", b"// c", b'"m");', "msg"),
    ("junit_lead", 4, b"assertEquals(", b"// c", b'"m", a, b);', "msg"),
    ("java_assert", 4, b"assert x", b"// c", b': "m";', "msg"),
]
CAP_HEADS = {1: b"def test_cap():", 3: b"TEST(S, Cap) {", 4: b"  public void testCap() {"}


def cap_test(form, d, end):
    """One test: the form's statement on its first body line, the token line at offset d from it; end: the body ends at that
    offset (None: it runs on behind the token)."""
    _, ext, first, filler, token, _ = form
    py, ind = ext == 1, b"    "
    lines = [CAP_HEADS[ext], ind + first]
    after = ind + (b"x = 1" if py else b"x = 1;")
    # with an end, the byte count of brackets (PY) or braces (C family) is 0 behind line end - 1, so that line `end` (PY: at
    # column 0) ends the body
    close = b"# )" if py else b"// }"
    while len(lines) - 1 < (d if end is None or d < end else end - 1):
        lines.append(ind + filler)
    if end is None:
        lines += [ind + token, after] + ([] if py else [b"}"])
    elif d < end:
        lines += [ind + token + (b"" if py else b" " + close), after.lstrip() if py else after]
    else:
        lines += [ind + close, token if py else ind + token]
    return lines


def cap_corpus():
    """Per form: the token at offset 62, 63, 64 and 65 from the assertion line, and the body end at offset 63, 64 and 65 with
    the token on the last body line or on the body-end line; one test each.  reach: [(form, ext, offset of the token, offset of
    the body end or None, seen)] in test order, with seen = the token lies inside the walk of LEX_STMT_LINES lines."""
    files, exts, cases = [], [], []
    for form in CAP_FORMS:
        lines = []
        for d, end in [(d, None) for d in (62, 63, 64, 65)] + [(e - 1, e) for e in (63, 64, 65)] + [(e, e) for e in (63, 64, 65)]:
            t = cap_test(form, d, end)
            b = len(lines)
            lines += t
            pl = spec_ref.py_lines(b"\n".join(t) + b"\n")
            assert form[4] in pl[1 + d]
            cases.append((form[0], form[1], d, end, d < lr.LEX_STMT_LINES and (end is None or d < end), b))
        files.append(b"\n".join(lines) + b"\n")
        exts.append(form[1])
    return files, exts, {"cases": cases, "forms": {f[0]: f[5] for f in CAP_FORMS}}


# ------------------------------------------------------------------------------------------------------------ token automata
def statement_alphabet(ext):
    """The tokens of the statement sequences: number, signs, comparison bytes, is / not / in, an identifier, the literal name,
    a string, brackets, comma, dot, equals and isinstance."""
    lit = {1: b"None", 2: b"NULL", 3: b"nullptr", 4: b"null"}[ext]
    return [b"1", b"-", b"+", b"=", b"!", b"<", b">", b"is", b"not", b"in", b"x", lit, b"'s'" if ext == 1 else b'"s"', b"(", b")",
            b",", b".", b"equals", b"isinstance"]


# (ext, head, tail): the sequence is the argument list, the expression, or the tokens after a gtest call
STATEMENT_FORMS = [
    (1, b"self.assertTrue(", b")"), (1, b"self.assertEqual(a, ", b")"), (1, b"assert ", b""),
    (1, b"np.testing.assert_allclose(", b")"),
    (2, b"assert(", b");"), (3, b"static_assert(", b");"), (3, b"EXPECT_EQ(", b");"), (3, b"EXPECT_TRUE(a) ", b";"),
    (4, b"assertTrue(", b");"), (4, b"assertEquals(", b");"), (4, b"assert ", b";"),
]
CODE_ALPHABET = [b"x", b"y", b",", b"=", b"(", b")", b"[", b".", b"1", b"+", b"!", b"<", b"open", b"File"]
CODE_EXTS = (1, 3, 4)


def sequences(alphabet, lengths, sample=None, seed=0):
    """Every sequence of the given lengths over the alphabet (sample: that many of them, seeded)."""
    out = [s for n in lengths for s in itertools.product(alphabet, repeat=n)]
    if sample is not None and sample < len(out):
        out = random.Random(seed).sample(out, sample)
    return out


def automaton_corpus(lengths=(1, 2, 3), sample=None):
    """One test per (statement form, sequence) and per (code ext, code sequence): the sequence's tokens joined by spaces as
    the argument list, the expression or the gtest trailer of one statement, or as one code line.  One file per form.  reach:
    per form the number of tests."""
    files, exts, reach = [], [], {}
    for k, (ext, head, tail) in enumerate(STATEMENT_FORMS):
        seqs = sequences(statement_alphabet(ext), lengths, sample, seed=k)
        files.append(_one_line_tests(ext, [head + b" ".join(s) + tail for s in seqs]))
        exts.append(ext)
        reach[("stmt", ext, head)] = len(seqs)
    for k, ext in enumerate(CODE_EXTS):
        seqs = sequences(CODE_ALPHABET + ([b"fopen"] if ext != 1 else []), lengths, sample, seed=100 + k)
        files.append(_one_line_tests(ext, [b" ".join(s) for s in seqs]))
        exts.append(ext)
        reach[("code", ext)] = len(seqs)
    return files, exts, reach


def _one_line_tests(ext, lines):
    if ext == 1:
        return b"".join(b"def test_%d():\n    %s\n" % (i, x) for i, x in enumerate(lines))
    if ext == 4:
        return b"class T {\n" + b"".join(b"  public void test%d() {\n    %s\n  }\n" % (i, x) for i, x in enumerate(lines)) + b"}\n"
    return b"".join(b"TEST(S, T%d) {\n  %s\n}\n" % (i, x) for i, x in enumerate(lines))


# --------------------------------------------------------------------------------------------------------------- name sets
def home(h, slots):
    return (h * slots) >> 64


def insert_wraps(hashes, slots):
    """Insert the hashes in order into an open-addressing set of `slots` slots (the kernel's probe; the sentinel hash stays
    outside): (distinct count with the sentinel counted once, probes that wrap from slot slots - 1 to 0)."""
    tab, wraps, sent = [None] * slots, 0, False
    for h in hashes:
        if h == M64:
            sent = True
            continue
        q = home(h, slots)
        while tab[q] is not None and tab[q] != h:
            if q == slots - 1:
                wraps += 1
            q = (q + 1) % slots
        tab[q] = h
    return sum(x is not None for x in tab) + sent, wraps


def last_slot_names(slots, k, prefix=b"w"):
    """k identifiers whose home slot in a set of `slots` slots is the last one."""
    out, i = [], 0
    while len(out) < k:
        w = prefix + b"%d" % i
        if home(spec_ref.py_bytes_hash(w), slots) == slots - 1:
            out.append(w)
        i += 1
    return out


def py_test(name, body):
    return b"def %s():\n" % name + b"".join(b"    " + x + b"\n" for x in body)


def nameset_corpus(n_tests=18000, sms=132):
    """The sentinel name alone, repeated, among other names, in a C-family test and in a test of more than 256 names; names
    whose home is the last slot in a shared set and in a global one; 32 copies of one name in the first round; 300 names on one
    tuple line; the local-name and Assertion Roulette thresholds; then n_tests tests of 0 to 20 distinct names v0 .. (the same
    names in every test), every thirteenth one with 257 to 300 names on one line, for a launch of min(ceil(n_tests / 8), sms * 8)
    blocks of 8 warps.  reach: the tests' names in order, the simulated wraps per test, and the warps that meet a shared, a
    global and a shared set in turn."""
    S = SENTINEL
    tests = []                                         # (name, body, ext)
    tests.append((b"test_sentinel_alone", [S + b" = 1"], 1))
    tests.append((b"test_sentinel_repeated", [S + b" = 1", S + b" = 2", S + b", " + S + b" = f()"], 1))
    tests.append((b"test_sentinel_among", [b"a, " + S + b", b = f()", b"c = 1", S + b" = 3", b"d = a"], 1))
    big = [b"v%d" % i for i in range(299)]
    tests.append((b"test_sentinel_global", [b", ".join(big[:150] + [S] + big[150:]) + b" = t", S + b" = 1"], 1))
    tests.append((b"test_sentinel_cj", None, 3))
    shared = last_slot_names(SET_SLOTS, 4)
    tests.append((b"test_wrap_shared", [w + b" = 1" for w in shared] + [b"z = 1"], 1))
    n_glob = 300
    glob = last_slot_names(2 * n_glob, 4, b"g")
    fill = [b"f%d" % i for i in range(n_glob - len(glob))]
    tests.append((b"test_wrap_global", [b", ".join(fill + glob) + b" = t"], 1))
    tests.append((b"test_round_copies", [b"dup = %d" % i for i in range(32)] + [b"other = 1"], 1))
    tests.append((b"test_tuple_copies", [b", ".join([b"dup"] * 32) + b" = t"], 1))
    tests.append((b"test_tuple_300", [b", ".join(b"n%d" % i for i in range(300)) + b" = t"], 1))
    for n in (10, 11):
        tests.append((b"test_locals_%d" % n, [b"v%d = 0" % i for i in range(n)] + [b"v0 = 1"], 1))
    for n in (1, 2):
        tests.append((b"test_unexplained_%d" % n, [b"assert x%d" % i for i in range(n)] + [b"assert y, 'm'"], 1))
    py = b"".join(py_test(n, b) for n, b, e in tests if e == 1)
    cj = b"TEST(S, Sentinel) {\n  int " + S + b" = 1;\n  int a = 2;\n  auto " + S + b" = 3;\n}\n"
    warps = []
    for t in range(n_tests):
        k = 257 + (t // 13) % 44 if t % 13 == 5 else t % 21
        warps.append(b"def test_w%d():\n" % t + (b"    %s = t\n" % b", ".join(b"v%d" % i for i in range(k)) if k else b"    pass\n"))
    many = b"".join(warps)
    files = [py, b"", cj, b"x = 1\n", many]
    exts = [1, 1, 3, 0, 1]
    names = []
    for data, ext in zip(files, exts):
        if not ext:
            continue
        toks = lr.file_tokens(data, ext)
        lines = spec_ref.py_lines(data)
        for b, bend, hend, code in lr.bodies(lines, ext):
            names.append([spec_ref.py_bytes_hash(n) for l in code for n in lr.local_names(toks[l], ext)])
    wraps = [insert_wraps(h, SET_SLOTS if len(h) <= SET_SLOTS // 2 else 2 * len(h))[1] for h in names]
    nt = len(names)
    W = min((nt + 7) // 8, sms * 8) * 8
    first = nt - n_tests
    kinds = [len(h) > SET_SLOTS // 2 for h in names]
    alternating = sum(1 for w in range(W) if any(not kinds[t] and kinds[t + W] and t + 2 * W < nt and not kinds[t + 2 * W]
                                                 for t in range(w, nt - 2 * W, W)))
    reach = {"names": names, "wraps": wraps, "warps": W, "alternating_warps": alternating, "first_warp_test": first,
             "sentinel_tests": [i for i, h in enumerate(names) if M64 in h]}
    return files, exts, reach


# ---------------------------------------------------------------------------------------------------------------- body scan
def body_corpus():
    """Header statements of 30 to 34 continuation lines (keyword arguments that assign names and assertion calls on them, an
    assertion on the first body line); docstrings opened on lane 31 of the body scan and closed 1 to 3 rounds later, with
    assertions and assignments inside and after; PY and C-family tests whose body ends at every lane of the last round of
    k_lex_body's and k_lex_tests' scans (body_lines 2 to 41); empty and tag-0 files between.  reach: the lane and round of
    each long header statement's end counted from the search start, the lane and round of each docstring's opening and
    closing lines counted from the header, and per ext the lanes (body_lines modulo 32) at which bodies end."""
    py = []
    for n in range(30, 35):
        py.append(b"def test_head_%d(\n" % n + b"".join(b"    k%d=self.assertEqual(a, %d),\n" % (i, i) if i % 3 == 0 else
                                                       b"    k%d=%d,\n" % (i, i) for i in range(n - 1)) +
                  b"):\n    self.assertEqual(b, 7)\n    v = 1\n")
    for r in (1, 2, 3):
        for q in (b'"""', b"'''"):
            body = [b"    x%d = %d" % (i, i) for i in range(30)] + [b"    " + q] + \
                   [b"    assert d%d == %d\n    d%d = 1" % (i, i, i) for i in range(16 * r - 8)] + [b"    " + q]
            body += [b"    assert after == 1", b"    after = 2", b"    assert after"]
            py.append(b"def test_doc_%d_%d():\n" % (r, len(q)) + b"\n".join(body) + b"\n")
    lanes = []
    for k in range(40):
        lanes.append(b"def test_lane_%d():\n" % k + b"".join(b"    assert v%d == %d\n" % (i, i) for i in range(k + 1)))
    cc = b"".join(b"TEST(S, L%d) {\n" % k + b"".join(b"  EXPECT_EQ(v, %d);\n" % i for i in range(k)) + b"}\n" for k in range(40))
    files = [b"".join(py), b"", b"x = 1\nassert 2\n", b"".join(lanes), b"", cc, b"def test_tag0():\n    assert 1\n"]
    exts = [1, 1, 0, 1, 2, 3, 0]
    reach = {"head_end": [], "doc": [], "end_lanes": {}}
    for data, ext in zip(files, exts):
        if not ext:
            continue
        lines = spec_ref.py_lines(data)
        for b, bend, hend, code in lr.bodies(lines, ext):
            reach["end_lanes"].setdefault(ext, set()).add((bend - b) % 32)
            if hend - b > 2:
                reach["head_end"].append((hend - b - 1, fs.lane_round(hend, b + 1)))
            qs = [l for l in range(hend, bend) if lines[l].strip() in (b'"""', b"'''")]
            if qs:
                reach["doc"].append((fs.lane_round(qs[0], b), fs.lane_round(qs[1], b)))
    return files, exts, reach
