"""Crafted corpora for the per-line front of the smell parser (k_smell_lines, k_smell_tests in csrc/tsm_smell_kernels.cuh) and
the blind lexer (k_blind_state, k_blind_scan, k_blind_lines, k_blind_files in csrc/tsm_blind_kernels.cuh), built to sit on the
seams of those kernels, and the host facts that show each corpus reaches its seams.  TEST INFRASTRUCTURE ONLY.

* The load grid: the kernels read each line as 8-byte words from `start & ~7`, and files start 128-byte aligned (ts.pack,
  orc.pack), so a byte's offset modulo 8 in its file is its offset modulo 8 in its word.  `Grid` places a construct at every line
  start and every construct offset modulo 8, and records where it put it.
* The scans: k_blind_scan and k_smell_tests take 32 lines per round; `lane_round` is the lane and round of a line counted from
  the first line of the scan.
* The keyword table of k_blind_lines: `keyword_table` reads the four TSM_BLIND_* lists out of the kernel source and inserts
  them in the C order with blind_kw_home; `probe` walks it the way the kernel's lookup does.

Each builder returns (files, exts, reach): `reach` holds what the corpus reaches, computed from its bytes, and the tests assert it.
"""
import os
import re

import blind_ref as br
import spec_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLIND_KERNELS = os.path.join(ROOT, "tosem-2021-replication_b200", "csrc", "tsm_blind_kernels.cuh")
SLOTS = 512
M64 = (1 << 64) - 1
ALL8 = {(a, o) for a in range(8) for o in range(8)}


# ---------------------------------------------------------------------------------------------------------------- geometry
def line_spans(data):
    """(start, end) in the file of every section-2 line, the LF not included."""
    out, pos = [], 0
    for line in spec_ref.py_lines(data):
        out.append((pos, pos + len(line)))
        pos += len(line) + 1
    return out


def lane_round(line, first=0):
    """Lane and round of `line` in a warp scan of 32 lines per round that starts at line `first`."""
    return (line - first) % 32, (line - first) // 32


class Grid:
    """Lines of one file, with constructs placed at chosen line starts and offsets modulo 8."""

    def __init__(self):
        self.lines, self.marks = [], []             # marks: (name, line index, offset of the construct in the line, length)

    def pos(self):
        return sum(len(x) + 1 for x in self.lines)

    def add(self, line):
        self.lines.append(line)

    def align(self, a):
        """A blank filler line (spaces, or empty) so that the next line starts at a modulo 8."""
        self.add(b" " * ((a - self.pos() - 1) % 8))

    def place(self, name, a, head, construct, tail=b""):
        """A line that starts at a modulo 8 and holds `construct` behind `head`."""
        self.align(a)
        self.marks.append((name, len(self.lines), len(head), len(construct)))
        self.add(head + construct + tail)

    def data(self, final_lf=True):
        return b"\n".join(self.lines) + (b"\n" if final_lf else b"")

    def reach(self):
        """name -> set of (line start, construct start) modulo 8, from the bytes of the file."""
        spans = line_spans(self.data())
        out = {}
        for name, ln, off, n in self.marks:
            s, e = spans[ln]
            assert s + off + n <= e
            out.setdefault(name, set()).add((s % 8, (s + off) % 8))
        return out


def on_the_grid(reach):
    """Every construct of `reach` was placed at every line start and construct start modulo 8."""
    return {name: got == ALL8 for name, got in reach.items()}


# --------------------------------------------------------------------------------------------------------- keyword table
def kernel_keyword_lists():
    """The TSM_BLIND_PY_KEYWORDS, _CJ_KEYWORDS, _PY_LITERALS and _CJ_LITERALS lists of the kernel source, in its order."""
    src = open(BLIND_KERNELS).read()
    out = []
    for name in ("PY_KEYWORDS", "CJ_KEYWORDS", "PY_LITERALS", "CJ_LITERALS"):
        m = re.search(r"#define TSM_BLIND_%s((?:[^\n]*\\\n)*[^\n]*)" % name, src)
        out.append([w.encode() for w in " ".join(re.findall(r'"([^"]*)"', m.group(1))).split()])
    return out


def kw_key(word):
    w = word[:16].ljust(16, b"\0")
    return int.from_bytes(w[:8], "little"), int.from_bytes(w[8:], "little")


def kw_home(word):
    """blind_kw_home of the word's first 16 bytes."""
    lo, hi = kw_key(word)
    return (((lo ^ ((hi * 0x9E3779B97F4A7C15) & M64)) * 0xBF58476D1CE4E5B9) & M64) >> 55


def keyword_table():
    """The kernel's table: slots[512] (the name in each slot or None), inserted in the C order by blind_keyword_table."""
    slots = [None] * SLOTS
    for names in kernel_keyword_lists():
        for w in names:
            s = kw_home(w)
            while slots[s] is not None and slots[s] != w:
                s = (s + 1) % SLOTS
            slots[s] = w
    return slots


def probe(slots, word):
    """The occupied slots the kernel's lookup of `word` reads before it stops (at its name or at an empty slot), and whether
    it wraps from slot 511 to slot 0.  Words longer than 16 bytes are not looked up."""
    if len(word) > 16:
        return [], False
    s, seen, key = kw_home(word), [], kw_key(word)
    while slots[s] is not None:
        seen.append(s)
        if kw_key(slots[s]) == key:
            break
        s = (s + 1) % SLOTS
    return seen, any(a == SLOTS - 1 and b == 0 for a, b in zip(seen, seen[1:]))


def chains(slots):
    """Maximal runs of two or more occupied slots (a run may wrap from 511 to 0), as lists of slots."""
    occ = [x is not None for x in slots]
    start = next(i for i in range(SLOTS) if not occ[i])
    out, run = [], []
    for k in range(1, SLOTS + 1):
        i = (start + k) % SLOTS
        if occ[i]:
            run.append(i)
        else:
            if len(run) >= 2:
                out.append(run)
            run = []
    return out


def keyword_words(slots):
    """The words of the keyword corpus: every name, each with one byte added and one removed, identifiers of 8, 9, 16 and 17
    bytes, and identifiers (found by search) whose home slot is a displaced name's home or lies inside a chain, plus one
    whose lookup wraps from slot 511 to slot 0.  Returns (words, searched)."""
    names = [w for lst in kernel_keyword_lists() for w in lst]
    words = list(names) + [w + b"x" for w in names] + [w[:-1] for w in names if len(w) > 1]
    words += [b"abcdefgh", b"abcdefghi", b"abcdefghijklmnop", b"abcdefghijklmnopq", b"reinterpret_cast", b"reinterpret_castX",
              b"_Static_assertXY", b"_Static_assertXYZ", b"synchronizedABCD", b"synchronizedABCDE"]
    where = {w: i for i, w in enumerate(slots) if w is not None}
    targets = {kw_home(w) for w in names if where[w] != kw_home(w)} | {s for c in chains(slots) for s in c}
    searched, wrap, k = {}, None, 0
    while targets - set(searched) or wrap is None:
        w = b"k%d" % k
        k += 1
        h = kw_home(w)
        if h in targets and h not in searched:
            searched[h] = w
        if wrap is None and probe(slots, w)[1]:
            wrap = w
    found = sorted(set(searched.values()) | {wrap})
    return words + found, found


def keyword_lines(words, per_line=7):
    return [b" ".join(words[i:i + per_line]) for i in range(0, len(words), per_line)]


# ------------------------------------------------------------------------------------------------------------- blind lexer
# (name, lines before, construct, lines after): the construct goes on a line of its own, behind `=` bytes; the lines around it
# set up and close the cross-line state it needs.
PY_CONSTRUCTS = [
    ("tq_dq", [], b'"""d"""', []), ("tq_sq", [], b"'''d'''", []),
    ("tq_dq_open", [], b'"""', [b'"""']), ("tq_sq_open", [], b"'''", [b"'''"]),
    ("tq_dq_close", [b'x = """'], b'"""', []), ("tq_sq_close", [b"x = '''"], b"'''", []),
    ("esc_dq", [], b'"a\\"b"', []), ("esc_sq", [], b"'a\\'b'", []),
    ("backslash_last_str", [], b'"ab\\', []), ("backslash_last_tq", [], b'"""ab\\', [b'"""']),
    ("esc_in_tq", [b"x = '''"], b"a\\'''b'''", []),
] + [("prefix_" + p.decode(), [], p + b'"x"', []) for p in (b"r", b"b", b"u", b"f", b"rb", b"bR", b"Rb", b"fr", b"rf", b"ur")] + [
    ("prefix_tq_rb", [], b"rb'''x", [b"'''"]), ("prefix_long_rbx", [], b'rbx"x"', []),
    ("num_exp", [], b"1e+5", []), ("num_hexp", [], b"0x1p-3", []), ("num_dot", [], b".5", []), ("num_hexe", [], b"0xE+1", []),
    ("hash_comment", [], b"# c \"\"\" '''", []), ("dollar_ident", [], b"a$b", []), ("high_ident", [], b"caf\xc3\xa9x", []),
]
CJ_CONSTRUCTS = [
    ("block", [], b"/* c */", []), ("block_open", [], b"/*", [b"*/"]), ("block_close", [b"/*"], b"*/", []),
    ("esc_dq", [], b'"a\\"b"', []), ("esc_sq", [], b"'\\''", []), ("backslash_last_str", [], b'"ab\\', []),
] + [("prefix_" + p.decode(), [], p + b'"x"', []) for p in (b"L", b"u", b"U", b"u8", b"R", b"LR", b"uR", b"UR", b"u8R")] + [
    ("prefix_long_u8Rx", [], b'u8Rx"x"', []),
    ("num_exp", [], b"1e+5", []), ("num_hexp", [], b"0x1p-3", []), ("num_dot", [], b".5", []), ("num_sep", [], b"1'000'000", []),
    ("num_hexe", [], b"0xE+1", []),
    ("line_comment", [], b"// c /* x", []), ("dollar_ident", [], b"a$b", []), ("high_ident", [], b"caf\xc3\xa9x", []),
]


def blind_grid(fam):
    """Every construct of the family at every line start and construct start modulo 8, once at the line's end and once
    followed by ` y` (its lookahead then reads a byte of the line)."""
    g = Grid()
    for name, before, construct, after in (PY_CONSTRUCTS if fam == br.PY else CJ_CONSTRUCTS):
        for tail in (b"", b" y"):
            for a in range(8):
                for o in range(8):
                    for x in before:
                        g.add(x)
                    g.place(name, a, b"=" * o, construct, tail)
                    for x in after:
                        g.add(x)
    return g


def blind_grid_corpus():
    """The grids of both families (the C-family one as a C++ and as a Java file).  reach: (family, construct) -> placements."""
    gp, gc = blind_grid(br.PY), blind_grid(br.CJ)
    reach = {("py",) + (k,): v for k, v in gp.reach().items()}
    reach.update({("cj",) + (k,): v for k, v in gc.reach().items()})
    return [gp.data(), gc.data(), gc.data()], [1, 3, 4], reach


def filter_corpus():
    """k_blind_state's SWAR filter: lines whose only quote run (PY) or only '*' (CJ) has a byte at line byte 0, 7, 8 or the
    last byte, at every line start modulo 8; and short lines without one whose first or last load word holds a neighbour
    line's quote.  reach: construct -> line starts modulo 8; and the neighbour cases found."""
    py, cj = Grid(), Grid()
    for a in range(8):
        py.place("byte0", a, b"", b'"""', b" x")
        py.add(b'"""')
        py.place("byte7", a, b"x = 10 ", b'"""')
        py.add(b'"""')
        py.place("byte8", a, b"x = 100 ", b'"""')
        py.add(b'"""')
        py.place("last", a, b"x = ", b"'''")
        py.add(b"'''")
        cj.add(b"/* c")
        cj.place("byte0", a, b"", b"*/", b" x;")
        cj.place("byte7", a, b"x = 1 ", b"/*")
        cj.add(b"*/")
        cj.place("byte8", a, b"x = 10 ", b"/*", b" c")
        cj.add(b"*/")
        cj.place("last", a, b"int a; ", b"/*")
        cj.add(b"*/")
    for k in range(1, 7):                              # short lines between quote lines
        for a in range(8):
            py.align(a)
            py.add(b"q = 'a'")
            py.add(b"b" * k)
            py.add(b"'c'")
            cj.align(a)
            cj.add(b"p = a * b;")
            cj.add(b"c" * k)
            cj.add(b"*d = e;")
    reach = {}
    for fam, g, qs in (("py", py, b"\"'"), ("cj", cj, b"*")):
        data = g.data()
        spans = line_spans(data)
        for name, ln, off, n in g.marks:
            s, e = spans[ln]
            q = [i for i in range(s, e) if data[i] in qs]
            at = {"byte0": 0, "byte7": 7, "byte8": 8, "last": e - s - 1}[name]
            assert at in [i - s for i in q] and q == list(range(q[0], q[0] + len(q))), (fam, name)
            reach.setdefault((fam, name), set()).add(s % 8)
        for s, e in spans:
            if s == e or any(data[i] in qs for i in range(s, e)):
                continue
            if any(data[i] in qs for i in range(s & ~7, s)):
                reach.setdefault((fam, "neighbour_before"), set()).add(s % 8)
            if any(data[i] in qs for i in range(e, min(len(data), ((e - 1) | 7) + 1))):
                reach.setdefault((fam, "neighbour_after"), set()).add(e % 8)
    return [py.data(), cj.data()], [1, 3], reach


def keyword_corpus():
    """Every keyword-table word in a PY file and in a C-family file.  reach: the searched identifiers' probes."""
    slots = keyword_table()
    words, searched = keyword_words(slots)
    lines = keyword_lines(words)
    data = b"\n".join(lines) + b"\n"
    probes = {w: probe(slots, w) for w in words}
    reach = {"searched_walk": all(len(probes[w][0]) >= 1 for w in searched), "wraps": [w for w in words if probes[w][1]],
             "displaced_found": sorted({w for w in words if len(probes[w][0]) > 1 and slots[probes[w][0][-1]] == w})}
    return [data, data], [1, 3], reach


# Transfer functions over the PY states (code, inside \"\"\", inside ''') and the C-family ones (code, inside /* */).
PY_CHANGERS = [b"''' \"\"\"", b'"""', b"'''", b'x = """ a', b"y = ''' b"]   # a 3-cycle; the two swaps, bare and in code
CJ_CHANGERS = [b"/*/", b"/* a", b"b */", b"*/ c /* d"]                       # swap, constant 1, constant 0, constant 1


def transfer(line, fam):
    """(state after the line from each state) under blind_ref's lexer."""
    return tuple(br.lex_line(line, fam, s)[1] for s in ((0, 1, 2) if fam == br.PY else (0, 1)))


def scan_corpus():
    """k_blind_scan across rounds: PY and C-family files of 31, 32, 33, 64 and 65 lines whose lines at lanes 0, 1, 30 and 31
    (and a few others) change the state, the changers alternating between functions that do not commute; then an empty file
    and a tag-0 file between C-family files whose last line leaves a comment open.  reach: per family file its length and the
    (lane, round) of its changing lines, the number of neighbour lines whose functions do not commute, and whether a line
    sends the three PY states to three different states."""
    files, exts = [], []
    for fam, ext, changers in ((br.PY, 1, PY_CHANGERS), (br.CJ, 3, CJ_CHANGERS)):
        for n in (31, 32, 33, 64, 65):
            lines, k = [], 0
            for i in range(n):
                if i % 32 in (0, 1, 30, 31) or i % 7 == 3:
                    lines.append(changers[k % len(changers)])
                    k += 1
                else:
                    lines.append(b"v%d = %d" % (i, i))
            files.append(b"\n".join(lines) + b"\n")
            exts.append(ext)
    files += [b"int a;\n/* open at the end", b"", b"x = 1\n", b"int b;\n", b"/* open\n", b"  ", b"int c; /*"]
    exts += [3, 3, 0, 3, 4, 0, 3]
    reach = {"lanes": [], "noncommuting_neighbours": 0, "permutation": False}
    for data, ext in zip(files, exts):
        fam = br.family(ext)
        if fam == br.NONE:
            continue
        fns = [transfer(x, fam) for x in spec_ref.py_lines(data)]
        ident = tuple(range(3 if fam == br.PY else 2))
        reach["lanes"].append((ext, len(fns), sorted({lane_round(i) for i, f in enumerate(fns) if f != ident})))
        for f, g in zip(fns, fns[1:]):
            if tuple(g[s] for s in f) != tuple(f[s] for s in g):
                reach["noncommuting_neighbours"] += 1
        reach["permutation"] |= any(len(set(f)) == 3 for f in fns)
    return files, exts, reach


def files_corpus():
    """k_blind_files: files with 0, 1, 32, 33 and 100 kept assertion lines (among other kept lines and unkept comment lines),
    then files without a kept line at the end of the corpus."""
    files, exts = [], []
    for n, ext in ((0, 1), (1, 3), (32, 1), (33, 3), (100, 1), (100, 4)):
        rows = []
        for i in range(n):
            rows.append(b"assert x == %d" % i if ext == 1 else b"EXPECT_EQ(x, %d);" % i)
            if i % 5 == 0:
                rows.append(b"# c" if ext == 1 else b"// c")
                rows.append(b"y = %d" % i)
        files.append(b"\n".join(rows + [b"z = 1"]) + b"\n")
        exts.append(ext)
    files += [b"# only a comment\n", b"", b"// c\n/* d\n e */\n"]
    exts += [1, 1, 3]
    return files, exts, {"asserts": [0, 1, 32, 33, 100, 100, 0, 0, 0]}


# ------------------------------------------------------------------------------------------------------------ smell parser
REDUNDANT_BIT, SLEEP, PRINT = 1 << 3, 1 << 6, 1 << 7          # smell_ref.BIT
# (name, statement, smell bits of the line): each pattern with and without what it must have in front of it, and lines where a
# rejected match comes before an accepted one (the System forms use println, which holds no `print(`)
SMELL_PATTERNS = [
    ("print", b"print(x)", PRINT), ("pprint", b"pprint(x)", PRINT), ("xpprint", b"xpprint(x)", 0), ("_print", b"_print(x)", 0),
    ("printf", b'printf("%d", x);', PRINT), ("puts", b"puts(x);", PRINT), ("cout", b"cout << x;", PRINT),
    ("cerr", b"cerr << x;", PRINT), ("std_cout", b"std::cout << x;", PRINT), ("xcout", b"xcout << x;", 0),
    ("sleep", b"sleep(1);", SLEEP), ("time_sleep", b"time.sleep(1)", SLEEP), ("sleep_for", b"sleep_for(1ms);", SLEEP),
    ("sleep_until", b"sleep_until(t);", SLEEP), ("_for", b"_for(1);", 0), ("_until", b"_until(t);", 0),
    ("leep_for", b"leep_for(1);", 0), ("leep_until", b"leep_until(t);", 0),
    ("system_out", b"System.out.println(x);", PRINT), ("system_err", b"System.err.println(x);", PRINT),
    ("ystem_out", b"ystem.out.println(x);", 0), ("out_println", b"out.println(x);", 0), ("ystem_err", b"ystem.err.println(x);", 0),
    ("out_print", b"out.print(x);", PRINT),
    ("two_print", b"xprint(a); print(b)", PRINT), ("two_pprint", b"xpprint(a); pprint(b)", PRINT),
    ("two_sleep_for", b"_for(1); sleep_for(2);", SLEEP), ("two_sleep_until", b"leep_until(1); sleep_until(2);", SLEEP),
    ("two_system", b"ystem.out.println(1); System.out.println(2);", PRINT),
]


def grid_tests(specs, bodies, mask):
    """One test per body form (ext, header line, indent, closing line or None) holding every statement of specs
    [(name, statement, smell bits)] at every line start and statement start modulo 8.  Returns (files, exts, reach, want):
    want = [(file, line, mask, smell bits under mask)] for every placed line."""
    files, exts, reach, want = [], [], {}, []
    bits = {n: b for n, _, b in specs}
    for ext, head, indent, end in bodies:
        g = Grid()
        g.add(head)
        for name, text, _ in specs:
            for a in range(8):
                for o in range(8):
                    g.place(name, a, indent + b" " * o, text)
        if end:
            g.add(end)
        files.append(g.data())
        exts.append(ext)
        reach.update({(ext, k): v for k, v in g.reach().items()})
        want += [(len(files) - 1, ln, mask, bits[name]) for name, ln, _, _ in g.marks]
    return files, exts, reach, want


def pattern_corpus():
    """Every pattern in a gtest body from column 0 (the prefix checks count from the line start, so they meet equality
    there), in a JUnit body and in a PY body from column 1."""
    return grid_tests(SMELL_PATTERNS, [(3, b"TEST(S, Grid) {", b"", b"}"), (4, b"  public void testGrid() {", b"", b"  }"),
                                       (1, b"def test_grid():", b" ", None)], PRINT | SLEEP)


COND, EXC = 1 << 4, 1 << 5
# (statement, smell bits): first tokens of 8 bytes and longer ones that start with a keyword, '}' and W bytes in front (each
# '}' balanced by a '{', so that the C-family bodies run to the end)
FIRST_TOKENS = [
    (b"ifghijkl = 1", 0), (b"forghijk = 1", 0), (b"switchxy = 1", 0), (b"exceptxy = 1", 0), (b"if_something_long = 1", 0),
    (b"format_all(x)", 0), (b"tryhard(x)", 0), (b"switcheroo(x)", 0), (b"throws(x)", 0), (b"elif", COND), (b"raise", EXC),
    (b"if (x) y();", COND), (b"switch (x) y();", COND), (b"while (x) y();", COND), (b"try:", EXC), (b"except:", EXC),
    (b"}else if (x) {", 0), (b"} catch (E e) {", EXC), (b"}if (x) {", COND), (b"}}  for (;;) {{", COND),
    (b"\t\x0b\x0cif (x) y();", COND), (b"\x0c\tthrow x;", EXC), (b"} \x0b catch (E e) {", EXC),
]


def token_corpus():
    """First tokens in a PY test, a gtest and a JUnit test."""
    specs = [("t%d" % k, text, bits) for k, (text, bits) in enumerate(FIRST_TOKENS)]
    return grid_tests(specs, [(1, b"def test_tokens():", b"    ", None), (3, b"TEST(S, Tokens) {", b"  ", b"}"),
                              (4, b"  public void testTokens() {", b"    ", b"  }")], COND | EXC)


# (body statements, empty): `pass` with and without other bytes, lines of only {}();: bytes
EMPTY_BODIES = [([b"pass"], True), ([b"pass;"], False), ([b"pass  # c"], False), ([b"  pass \t"], True), ([b"passx"], False),
                ([b"();:"], True), ([b"{}"], True), ([b"(;)", b"pass"], True), ([b"(x)"], False)]
# quote runs of 3 to 7 of one kind, both kinds on one line, and a run of 2; each followed by a line the docstring state decides
QUOTE_LINES = [b'x = ' + q * n for q in (b'"', b"'") for n in (2, 3, 4, 5, 6, 7)] + [b"x = \"\"\" '''", b"x = ''' \"\"\" '''",
                                                                                       b'x = """""" + """ """']


def facts_corpus():
    """Tests of one statement each for the empty smell, and a PY test whose quote-run lines each precede an `if` line."""
    py, cc = [], []
    for k, (body, _) in enumerate(EMPTY_BODIES):
        py.append(b"def test_empty_%d():\n" % k + b"".join(b"    " + x + b"\n" for x in body))
        cc.append(b"TEST(S, Empty%d) {\n" % k + b"".join(b"  " + x + b"\n" for x in body) + b"}\n")
    doc = [b"def test_quotes():"]
    for a in range(2):
        for q in QUOTE_LINES:
            doc += [b"    " * (1 + a) + q, b"    if y:", b"        z = 1"]
    return [b"".join(py), b"".join(cc), b"\n".join(doc) + b"\n"], [1, 3, 1]


REDUNDANT = [
    (b"assert True", True), (b"assert\tTrue ", True), (b"assert \x0b None\t", True), (b"assert  1", True), (b"assert(1)", True),
    (b"assert True, 'x'", False), (b"assertTrue", False), (b"assert x", False),
    (b"self.assertEqual(x, x)", True), (b"self.assertEqual( x ,x )", True), (b"self.assertEqual(x,x)", True),
    (b"self.assertEqual((a, (b, c)), (a, (b, c)))", True), (b"self.assertEqual([a, b], [a, b])", True),
    (b"self.assertEqual(a, b, a)", False), (b"self.assertEqual(a, a, a)", False), (b"self.assertEqual()", False),
    (b"self.assertTrue( )", False), (b"assert x) == (x", False), (b"self.assertEqual(f(a, b), f(a, b)", False),
    (b"self.assertEqual(, )", False), (b"EXPECT_EQ(x, x);", True), (b"ASSERT_TRUE( true );", True), (b"EXPECT_TRUE(NULL);", True),
]


def redundant_corpus():
    """Every redundant form in a PY test and a gtest."""
    specs = [("r%d" % k, text, REDUNDANT_BIT if r else 0) for k, (text, r) in enumerate(REDUNDANT)]
    return grid_tests(specs, [(1, b"def test_redundant():", b"    ", None), (3, b"TEST(S, Redundant) {", b"  ", b"}")],
                      REDUNDANT_BIT)


def scan_smell_corpus():
    """k_smell_tests' scans across rounds: PY header statements of 31, 32, 33 and 40 continuation lines; PY bodies whose first
    dedented line is on lane 31 or lane 0 of the body scan, behind a column-0 comment or a continuation line; JUnit bodies
    whose `{` comes on a later line at lane 31 or 32; `{}` on the header line; a `}` ahead of the first `{` at lanes 31 and
    32; a docstring that opens on lane 31 and closes two rounds later."""
    py, java, cc = [], [], []
    for n in (31, 32, 33, 40):
        py.append(b"def test_head_%d(\n" % n + b"".join(b"    a%d,\n" % i for i in range(n - 2)) + b"    b=assert_that,\n):\n"
                  b"    if x:\n        assert a0\n")
    for n in (31, 32, 63, 64):
        for before in ([b"# column-0 comment"], [b"    y = f(", b"1)"]):
            body = [b"    x%d = %d" % (i, i) for i in range(n - len(before))] + before
            py.append(b"def test_body_%d():\n" % n + b"\n".join(body) + b"\nif z:\n    pass\n")
    for n in (31, 32):
        java.append(b"  public void testAllman%d()\n" % n + b"".join(b"      // throws %d\n" % i for i in range(n - 1)) +
                    b"  {\n    if (x) y();\n  }\n    if (z) w();\n")
        java.append(b"  public void testClose%d()\n" % n + b"".join(b"    x%d();\n" % i for i in range(n - 1)) +
                    b"  }\n  {\n    if (x) y();\n  }\n    if (z) w();\n")
    cc.append(b"TEST(S, OneLine) {}\n  if (x) y();\nTEST(S, Next) { }\n  if (x) y();\n")
    py.append(b"def test_doc():\n" + b"    x = 1\n" * 30 + b'    """\n' + b"    if a:\n" * 63 + b'    """\n' + b"    if b:\n" * 3)
    files = [b"".join(py), b"class T {\n" + b"".join(java) + b"}\n", b"".join(cc)]
    return files, [1, 4, 3]


def scan_facts(data, ext):
    """(header, end of the header statement, body end, first line holding '{') of every test of a file, by smell_ref's rules."""
    import smell_ref as sr
    lines = spec_ref.py_lines(data)
    kinds = sr.py_kinds(lines)
    ends = dict(sr.py_cases(lines, ext))
    out = []
    for b, n, *_ in sr.py_file_smells(data, ext)[0]:
        hs = b + 1
        while hs < ends[b] and kinds[hs] == 2:
            hs += 1
        brace = next((l for l in range(b, len(lines)) if b"{" in lines[l]), None)
        out.append((b, hs, b + n, brace))
    return out


def header_corpus():
    """Decorators and headers: '@' lines up to the file's first line (behind a file whose last line is a skip decorator), an
    '@' line cut off by another line or by a header, skip / @Ignore / @Disabled / DISABLED_ on headers and decorators of each
    family, the async forms, each gtest and Boost macro and each with one byte changed, and headers on a file's last line with
    and without a final LF."""
    files, exts = [], []
    files += [b"x = 1\n@pytest.mark.skip", b"@pytest.mark.skip\n@other\ndef test_first():\n    pass\n",
              b"@other\ndef test_not_skipped():\n    pass\n",
              b"@pytest.mark.skip\n# c\ndef test_cut():\n    pass\n@pytest.mark.skip\n\ndef test_blank():\n    pass\n"
              b"@pytest.mark.skip\ndef helper():\n    pass\ndef test_after_header():\n    pass\n"
              b"@pytest.mark.skip(reason='undefined')\ndef test_deco_is_header():\n    pass\n"
              b"def test_skip_in_header():\n    pass\n@Ignore\ndef test_ignore_deco():\n    pass\n"
              b"def test_DISABLED_x():\n    pass\n@Disabled\ndef test_disabled_deco():\n    pass\n"
              b"async def test_a():\n    pass\nasync  def\ttest_b():\n    pass\nasyncdef test_c():\n    pass\n"
              b"def  test_d():\n    pass\nasync\tdef test_e():\n    pass\ndef test_f ():\n    pass\n"]
    exts += [1, 1, 1, 1]
    java = (b"@Ignore\n@Test\npublic void testFirst() {\n}\n@Test @Ignore public void testOnHeader() {\n}\n"
            b"@Disabled(\"x\")\n  @Test\n  public void testDisabled() {\n  }\n@Ignore\n  // c\n  public void testCut() {\n  }\n"
            b"  @pytest.mark.skip\n  public void testSkipDeco() {\n  }\n  public void testDISABLED_x() {\n  }\n"
            b"  @Disabled public void testDisabledOnHeader() {\n  }\n")
    files.append(java)
    exts.append(4)
    macros = [b"TEST(", b"TEST_F(", b"TEST_P(", b"TYPED_TEST(", b"TYPED_TEST_P(", b"BOOST_AUTO_TEST_CASE(",
              b"BOOST_FIXTURE_TEST_CASE(", b"BOOST_DATA_TEST_CASE("]
    cc = []
    for m in macros:
        for k in (None, 0, len(m) - 2, len(m) - 1):
            h = m if k is None else m[:k] + (b"X" if m[k:k + 1] != b"X" else b"Y") + m[k + 1:]
            cc.append(h + b"S, Case) {\n  if (x) y();\n}\n")
    cc.append(b"@Ignore\nTEST(S, DISABLED_Off) {\n  if (x) y();\n}\n@DISABLED_\nTEST(S, On) {\n  if (x) y();\n}\n"
              b"@skip\nTEST(S, Skip) {\n}\n")
    files.append(b"".join(cc))
    exts.append(3)
    files += [b"x = 1\ndef test_last():", b"x = 1\ndef test_last():\n", b"int x;\nTEST(S, Last) {", b"int x;\nTEST(S, Last) {\n"]
    exts += [1, 1, 3, 3]
    return files, exts
