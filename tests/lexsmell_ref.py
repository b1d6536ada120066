"""Plain-Python restatement of the lexical test smells of docs/SPEC.md section 25 (test infrastructure): the section-21 tokens
*seen* (kind and bytes), the section-18 tests, bodies and line kinds, the assertion call of every counted assertion line and its
argument list, and the five smells.  Written from the SPEC text on blind_ref.py (its literal, comment and number rules), spec_ref.py
and smell_ref.py; no shared code with the kernels.

* `lex_tokens(line, fam, state)`: the tokens that begin on one line, as (kind, bytes), and the state after it; blinding them
  gives exactly `blind_ref.lex_line`;
* `file_lexsmells(data, ext)`: the tests of one file with their records, and the lexical smell bits of every line;
* `py_lexsmells(files, exts)`: the same over a corpus, as the arrays of `tosemscan.Scanner.smells_lexical`.
"""
import numpy as np

import blind_ref as br
import corpus_util as cu
import smell_ref as sr
from case_ref import py_case_name, py_cases
from spec_ref import W, py_bytes_hash, py_is_assert_line, py_lines

LSMELLS = ("assertion_roulette", "magic_number", "suboptimal_assert", "mystery_guest", "obscure_setup")
LBIT = {s: 1 << i for i, s in enumerate(LSMELLS)}
LEX_STMT_LINES = 64
OBSCURE_LOCALS = 10

IDENT, KEYWORD, LITNAME, NUMBER, STRING, PUNCT = "I", "K", "L", "N", "S", "P"

PY_ARITY1 = {b"assertTrue", b"assertFalse", b"assertIsNone", b"assertIsNotNone", b"assert_"}
PY_ARITY3 = {b"assertAlmostEqual", b"assertNotAlmostEqual", b"assertAlmostEquals", b"assertNotAlmostEquals"}
PY_UNCOUNTED = (b"assertRaises", b"assertWarns")
PY_UNCOUNTED_EXACT = {b"assertLogs", b"assertNoLogs"}
MOCK_PREFIXES = (b"assert_called", b"assert_awaited")
MOCK_EXACT = {b"assert_any_call", b"assert_has_calls", b"assert_not_called"}
J_ARITY1 = {b"assertTrue", b"assertFalse", b"assertNull", b"assertNotNull"}
SUB_BOOL = {b"assertTrue", b"assertFalse", b"assert_", b"EXPECT_TRUE", b"EXPECT_FALSE", b"ASSERT_TRUE", b"ASSERT_FALSE"}
SUB_EQ = {b"assertEqual", b"assertEquals", b"assertNotEqual", b"assertNotEquals", b"assertIs", b"assertIsNot", b"EXPECT_EQ",
          b"EXPECT_NE", b"ASSERT_EQ", b"ASSERT_NE"}
PY_GUEST_CALLS = {b"open", b"urlopen", b"connect", b"read_csv", b"read_excel", b"read_json", b"read_parquet", b"loadtxt",
                  b"genfromtxt", b"imread", b"listdir"}
CJ_GUEST_CALLS = {b"fopen", b"freopen", b"open", b"getConnection"}
CJ_GUEST_NAMES = {b"ifstream", b"ofstream", b"fstream", b"File", b"FileReader", b"FileWriter", b"FileInputStream",
                  b"FileOutputStream", b"RandomAccessFile", b"Files"}
NOT_LONE_BEFORE = set(b"=!<>+-*/%&|^")


def lex_tokens(line, fam, state):
    """(tokens as (kind, bytes) that begin on the line, state at its end): section 21's lexer, seeing."""
    toks, i, n = [], 0, len(line)
    if state != br.CODE:
        i = br._close(line, 0, fam, state)
        if i is None:
            return toks, state
    kw, lit = (br.PY_KEYWORDS, br.PY_LITERALS) if fam == br.PY else (br.CJ_KEYWORDS, br.CJ_LITERALS)
    while i < n:
        c = line[i]
        nx = line[i + 1] if i + 1 < n else -1
        if c in W:
            i += 1
        elif fam == br.PY and c == 0x23:
            break
        elif fam == br.CJ and c == 0x2F and nx == 0x2F:
            break
        elif fam == br.CJ and c == 0x2F and nx == 0x2A:
            i = br._close(line, i + 2, fam, 1)
            if i is None:
                return toks, 1
        elif c in br.DIGITS or (c == 0x2E and nx in br.DIGITS):
            j = br._number(line, i, fam)
            toks.append((NUMBER, line[i:j]))
            i = j
        elif br._ident_byte(c):
            j = i
            while j < n and br._ident_byte(line[j]):
                j += 1
            word = line[i:j]
            if j < n and line[j] in b"\"'" and br._is_prefix(word, fam):
                k, st = br._string(line, j, fam)
                toks.append((STRING, line[i:k]))
                if st != br.CODE:
                    return toks, st
                i = k
                continue
            toks.append((KEYWORD if word in kw else LITNAME if word in lit else IDENT, word))
            i = j
        elif c in b"\"'":
            k, st = br._string(line, i, fam)
            toks.append((STRING, line[i:k]))
            if st != br.CODE:
                return toks, st
            i = k
        else:
            toks.append((PUNCT, bytes([c])))
            i += 1
    return toks, br.CODE


def blind(tok):
    k, b = tok
    return b"N" if k in (NUMBER, LITNAME) else b"S" if k == STRING else b"I" if k == IDENT else b


def file_tokens(data, ext):
    """The seen tokens of every line of a file (empty lists for tag 0)."""
    fam, state, out = br.family(int(ext)), br.CODE, []
    for line in py_lines(data):
        if fam == br.NONE:
            out.append([])
            continue
        toks, state = lex_tokens(line, fam, state)
        out.append(toks)
    return out


def bodies(lines, ext):
    """Section 18: per test (header line, body end, header-statement end, code lines), 0-based, in header order."""
    fam = sr.family(ext)
    if not fam:
        return []
    kinds = sr.py_kinds(lines)
    out = []
    for b, e in py_cases(lines, ext):
        if not sr.is_test_header(lines[b], ext):
            continue
        hs = b + 1
        while hs < e and kinds[hs] == 2:
            hs += 1
        bend = e
        if fam == "py":
            ind = sr.indent(lines[b])
            for l in range(hs, e):
                if kinds[l] == 1 and not sr.is_comment(lines[l].strip(W), fam) and sr.indent(lines[l]) <= ind:
                    bend = l
                    break
        else:
            run, opened = 0, False
            for l in range(b, e):
                run += lines[l].count(b"{") - lines[l].count(b"}")
                opened = opened or b"{" in lines[l]
                if opened and run <= 0:
                    bend = l + 1
                    break
        hend = min(hs, bend)
        code, dq, sq = [], 0, 0
        for l in range(hend, bend):
            s = lines[l].strip(W)
            doc = False
            if fam == "py":
                doc = dq % 2 == 1 or sq % 2 == 1 or s.startswith((b'"""', b"'''"))
                dq += lines[l].count(b'"""')
                sq += lines[l].count(b"'''")
            if s and not sr.is_comment(s, fam) and not doc:
                code.append(l)
        out.append((b, bend, hend, code))
    return out


# ------------------------------------------------------------------------------------------------------- the assertion call
def find_call(toks, ext):
    """(index of the assertion call's token, its kind) on one line, or None.  Kinds: 'pyassert', 'jassert' (statements), or
    'call' (the token after it is the list's '(')."""
    py = ext == 1
    for j, (k, b) in enumerate(toks):
        nxt = toks[j + 1] if j + 1 < len(toks) else None
        paren = nxt == (PUNCT, b"(")
        if k == KEYWORD and b == b"assert":
            if py:
                return j, "pyassert"
            if ext == 4:
                return j, "jassert"
            if paren:
                return j, "call"
        elif k == KEYWORD and b == b"static_assert" and not py and paren:
            return j, "call"
        elif k == IDENT and paren and (b"assert" in b.lower() or (not py and b"EXPECT_" in b)):
            return j, "call"
    return None


def call_kind(toks, j, ext):
    """(counting kind, arity) of the call whose name is toks[j]: 'unittest', 'numpy', 'gtest', 'cassert', 'static', 'jcall'
    or None (not counted)."""
    name = toks[j][1]
    dot = j > 0 and toks[j - 1] == (PUNCT, b".")
    if ext == 1:
        if name.startswith(b"assert_") and len(name) > 7:
            if name.startswith(MOCK_PREFIXES) or name in MOCK_EXACT:
                return None, 0
            return "numpy", 0
        if dot and name.startswith(b"assert"):
            if name.startswith(PY_UNCOUNTED) or name in PY_UNCOUNTED_EXACT:
                return None, 0
            return "unittest", 1 if name in PY_ARITY1 else 3 if name in PY_ARITY3 else 2
        return None, 0
    if toks[j][0] == KEYWORD:
        return ("static", 0) if name == b"static_assert" else ("cassert", 0)
    if name.startswith((b"EXPECT_", b"ASSERT_")):
        return "gtest", 0
    if ext == 4 and name.startswith(b"assert"):
        return "jcall", 1 if name in J_ARITY1 else 2
    return None, 0


def depth_step(tok, d):
    if tok[0] == PUNCT and tok[1] in (b"(", b"[", b"{"):
        return d + 1
    if tok[0] == PUNCT and tok[1] in (b")", b"]", b"}"):
        return d - 1
    return d


def split_top(toks, sep):
    """Pieces of toks split at the depth-0 tokens for which sep(i) holds (the separators dropped)."""
    out, cur, d = [], [], 0
    for i, t in enumerate(toks):
        if d == 0 and sep(i):
            out.append(cur)
            cur = []
        else:
            cur.append(t)
        d = depth_step(t, d)
    out.append(cur)
    return out


def is_sep_cmp(toks, i, py):
    k, b = toks[i]
    if k == PUNCT and b in (b"<", b">", b"="):
        return True
    if k == PUNCT and b == b"!" and i + 1 < len(toks) and toks[i + 1] == (PUNCT, b"="):
        return True
    if py and k == KEYWORD and b in (b"is", b"in"):
        return True
    if py and k == KEYWORD and b == b"not" and ((i > 0 and toks[i - 1] == (KEYWORD, b"is")) or
                                                (i + 1 < len(toks) and toks[i + 1] == (KEYWORD, b"in"))):
        return True
    return False


def has_magic(expr, py):
    for op in split_top(expr, lambda i: is_sep_cmp(expr, i, py)):
        if len(op) == 1 and op[0][0] == NUMBER:
            return True
        if len(op) == 2 and op[0] in ((PUNCT, b"-"), (PUNCT, b"+")) and op[1][0] == NUMBER:
            return True
    return False


def is_kwarg(arg):
    return len(arg) >= 2 and arg[0][0] == IDENT and arg[1] == (PUNCT, b"=") and (len(arg) < 3 or arg[2] != (PUNCT, b"="))


def close_of(toks, i):
    """Index of the token that closes the bracket opened at toks[i], or None."""
    d = 0
    for k in range(i, len(toks)):
        d = depth_step(toks[k], d)
        if d == 0:
            return k
    return None


def bool_suboptimal(arg, ext):
    py, d = ext == 1, 0
    for i, (k, b) in enumerate(arg):
        if d == 0:
            if k == PUNCT and b == b"=" and i > 0 and arg[i - 1][0] == PUNCT and arg[i - 1][1] in (b"=", b"!", b"<", b">"):
                return True
            if py and ((k == PUNCT and b in (b"<", b">")) or (k == KEYWORD and b in (b"is", b"in"))):
                return True
        d = depth_step((k, b), d)
    if py and len(arg) >= 3 and arg[0] == (IDENT, b"isinstance") and arg[1] == (PUNCT, b"(") and close_of(arg, 1) == len(arg) - 1:
        return True
    if ext == 4 and arg and arg[-1] == (PUNCT, b")"):
        for o in range(len(arg) - 1):
            if arg[o] == (PUNCT, b"(") and close_of(arg, o) == len(arg) - 1:
                return o >= 2 and arg[o - 1] == (IDENT, b"equals") and arg[o - 2] == (PUNCT, b".")
    return False


def statement(lines_toks, l, lim, ext):
    """The assertion statement of line l (tokens of the file's lines in lines_toks; the walk may use lines l .. lim - 1):
    None when the line has no assertion call, else (counted, unexplained, magic, suboptimal)."""
    py = ext == 1
    toks = lines_toks[l]
    fc = find_call(toks, ext)
    if fc is None:
        return None
    j, form = fc
    stream, ends = list(toks[j + 1:]), []                # ends[k]: the stream length at the end of line l + k
    ends.append(len(stream))
    for m in range(l + 1, lim):
        stream += lines_toks[m]
        ends.append(len(stream))
    if form in ("pyassert", "jassert"):
        if form == "pyassert":
            # the logical line: up to the first line end at depth 0 whose line does not end in a backslash token
            d, cut, pos = 0, None, 0
            for m, e in enumerate(ends):
                for t in stream[pos:e]:
                    d = depth_step(t, d)
                pos = e
                line_toks = lines_toks[l + m]
                if d == 0 and not (line_toks and line_toks[-1] == (PUNCT, b"\\")):
                    cut = e
                    break
            expr = stream[:cut] if cut is not None else stream
            parts = split_top(expr, lambda i: expr[i] == (PUNCT, b","))
        else:
            d, cut = 0, None
            for i, t in enumerate(stream):
                if d == 0 and t == (PUNCT, b";"):
                    cut = i
                    break
                d = depth_step(t, d)
            expr = stream[:cut] if cut is not None else stream
            parts = split_top(expr, lambda i: expr[i] == (PUNCT, b":"))
        return True, len(parts) == 1, has_magic(parts[0], py), False
    kind, arity = call_kind(toks, j, ext)
    close = close_of(stream, 0)
    lst = stream[1:close] if close is not None else stream[1:]
    args = [a for a in split_top(lst, lambda i: lst[i] == (PUNCT, b",")) if a]
    pos = [a for a in args if not (py and is_kwarg(a))]
    kws = [a[0][1] for a in args if py and is_kwarg(a)]
    magic = any(has_magic(a, py) for a in pos)
    name = toks[j][1]
    sub = False
    if name in SUB_BOOL and args:
        sub = bool_suboptimal(args[0], ext)
    if name in SUB_EQ:
        sub = sub or any(len(a) == 1 and a[0][0] == LITNAME for a in pos)
    if kind is None:
        return False, False, magic, sub
    if kind == "unittest":
        expl = len(pos) > arity or b"msg" in kws
    elif kind == "numpy":
        expl = b"msg" in kws or b"err_msg" in kws
    elif kind == "gtest":
        expl = close is not None and stream[close + 1:close + 3] == [(PUNCT, b"<"), (PUNCT, b"<")]
    elif kind == "cassert":
        expl = False
    elif kind == "static":
        expl = len(args) >= 2
    else:
        one_str = lambda a: len(a) == 1 and a[0][0] == STRING   # noqa: E731
        expl = len(args) > arity and (one_str(args[0]) or one_str(args[-1]))
    return True, not expl, magic, sub


# -------------------------------------------------------------------------------------------------------------- code lines
def mystery(toks, ext):
    for j, (k, b) in enumerate(toks):
        if k != IDENT:
            continue
        paren = j + 1 < len(toks) and toks[j + 1] == (PUNCT, b"(")
        if ext == 1 and paren and b in PY_GUEST_CALLS:
            return True
        if ext != 1 and ((paren and b in CJ_GUEST_CALLS) or b in CJ_GUEST_NAMES):
            return True
    return False


def local_names(toks, ext):
    """The local names a code line assigns (section 25), in order."""
    if ext == 1:
        names, i = [], 0
        while i < len(toks) and toks[i][0] == IDENT:
            names.append(toks[i][1])
            if i + 1 < len(toks) and toks[i + 1] == (PUNCT, b","):
                i += 2
                continue
            if i + 1 < len(toks) and toks[i + 1] == (PUNCT, b"=") and (i + 2 >= len(toks) or toks[i + 2] != (PUNCT, b"=")):
                return names
            break
        return []
    d = 0
    for k, t in enumerate(toks):
        if d == 0 and t == (PUNCT, b"=") and not (k > 0 and toks[k - 1][0] == PUNCT and toks[k - 1][1][0] in NOT_LONE_BEFORE) \
                and not (k + 1 < len(toks) and toks[k + 1] == (PUNCT, b"=")):
            if k >= 2 and toks[k - 1][0] == IDENT and not any(x[0] == PUNCT and x[1] in (b"(", b".", b"[") for x in toks[:k]):
                return [toks[k - 1][1]]
            return []
        d = depth_step(t, d)
    return []


# ------------------------------------------------------------------------------------------------------------------ tests
def file_lexsmells(data, ext):
    """(tests, line_lsmell): tests as (header line, body_lines, n_stmts, n_unexplained, n_magic, n_locals, smells, n_instances,
    [(line, bit), ...]) with 0-based lines, and the lexical smell bits of every line of the file."""
    ext = int(ext)
    lines = py_lines(data)
    lsm = [0] * len(lines)
    tests = []
    if not sr.family(ext):
        return tests, lsm
    lt = file_tokens(data, ext)
    for b, bend, hend, code in bodies(lines, ext):
        counted = list(range(b, hend)) + code
        n_st = n_un = n_mg = 0
        un, inst = [], []
        for l in counted:
            if not py_is_assert_line(lines[l], ext):
                continue
            r = statement(lt, l, min(bend, l + LEX_STMT_LINES), ext)
            if r is None:
                continue
            cnt, unexpl, magic, sub = r
            n_st += 1
            if cnt and unexpl:
                n_un += 1
                un.append(l)
            if magic:
                n_mg += 1
                inst.append((l, LBIT["magic_number"]))
            if sub:
                inst.append((l, LBIT["suboptimal_assert"]))
        names = set()
        for l in code:
            if mystery(lt[l], ext):
                inst.append((l, LBIT["mystery_guest"]))
            names.update(py_bytes_hash(n) for n in local_names(lt[l], ext))
        if n_un >= 2:
            inst += [(l, LBIT["assertion_roulette"]) for l in un]
        if len(names) > OBSCURE_LOCALS:
            inst.append((b, LBIT["obscure_setup"]))
        smells = 0
        for l, bit in inst:
            lsm[l] |= bit
            smells |= bit
        inst.sort()
        tests.append((b, bend - b, n_st, n_un, n_mg, len(names), smells, len(inst), inst))
    return tests, lsm


LEX_TEST = np.dtype([("n_stmts", "<i4"), ("n_unexplained", "<i4"), ("n_magic", "<i4"), ("n_locals", "<i4"), ("smells", "<u4"),
                     ("n_instances", "<i4")])


def py_lexsmells(files, exts):
    """Section 25 over a corpus: line_base, line_lsmell (u8 per line) and lex (LEX_TEST per test, in global line order)."""
    base, lsm, lex = [0], [], []
    for data, e in zip(files, exts):
        t, ls = file_lexsmells(data, e)
        lex += [x[2:8] for x in t]
        lsm += ls
        base.append(len(lsm))
    return {"line_base": np.array(base, np.int64), "line_lsmell": np.array(lsm, np.uint8),
            "lex": np.array(lex, LEX_TEST) if lex else np.zeros(0, LEX_TEST)}


def py_lexsmell_rows(files, exts, names=None):
    """The --out rows of the five smells: (fileName, test, line, smell, smellLine, statement), lines 1-based, in file, header
    line, instance line and smell order; `statement` is empty for obscure_setup (a test-level smell)."""
    rows = []
    for f, (data, ext) in enumerate(zip(files, exts)):
        lines = py_lines(data)
        for t in file_lexsmells(data, int(ext))[0]:
            b = t[0]
            name = py_case_name(lines[b], int(ext))
            for l, bit in t[8]:
                smell = LSMELLS[bit.bit_length() - 1]
                st = b"" if bit == LBIT["obscure_setup"] else lines[l].strip(W)
                rows.append((names[f] if names else f, name, b + 1, smell, l + 1, st))
    return rows


# Hand-written files with known answers (tests/test_lexsmells_ref.py pins them): (name, ext, bytes).
UNITTEST = b'''import unittest


class T(unittest.TestCase):
    def test_roulette(self):
        self.assertEqual(a, b)
        self.assertEqual(a, b, "m")
        self.assertTrue(x)
        self.assertTrue(x, msg="m")
        self.assertAlmostEqual(a, b, 3)
        self.assertAlmostEqual(a, b, 3, "m")
        self.assertRaises(E, f)
        x = self.assertEqual
'''

PYTEST = b'''def test_plain():
    assert x == 5
    assert x == 5, "m"
    assert y
    assert (
        z == -3
    )
    assert f(1e-5) == 0x1F
    assert x1 == True
    assert .5 is None
    assert a, "commas, (parens) and # inside"
    # assert 7
'''

NUMPY = b'''def test_np(self):
    np.testing.assert_allclose(a, b)
    np.testing.assert_allclose(a, b, err_msg="m")
    assert_array_equal(a, b, 2)
    m.assert_called_once_with(1)
    m.assert_not_called()
    self.assertEqual(x, None)
    self.assertTrue(isinstance(x, int))
    self.assertTrue(a in b)
    self.assertFalse(a < b)
    self.assertTrue(f(a == b))
    self.assertIsNone(x, "m")
'''

GTEST = b'''TEST(Suite, Gtest) {
  EXPECT_EQ(a, 5) << "m";
  EXPECT_EQ(a, b);
  EXPECT_TRUE(a == b);
  EXPECT_TRUE(std::is_same<A, B>::value);
  ASSERT_EQ(p, nullptr)
      << "multi";
  EXPECT_EQ(s, "a,b(<<");  // comment, (
  assert(x);
  static_assert(sizeof(int) == 4, "m");
  static_assert(sizeof(int) == 4);
  std::ifstream in("data.txt");
  FILE* f = fopen("x", "r");
  int v = 3;
  x = 5;
  EXPECT_TRUE(a /* , b */);
}
'''

JUNIT = b'''public class JTest {
  @Test public void testJ() {
    assertEquals(1.0, x, 0.01);
    assertEquals("m", a, b);
    assertTrue("m", ok);
    assertTrue(ok);
    assertTrue(a.equals(b));
    assertEquals(a, b, "m");
    assert x > 0 : "m";
    assert x > 0;
    File f = new File("a");
    Files.readAllLines(p);
    assertNull(null);
  }
}
'''

HAND = [("unittest.py", 1, UNITTEST), ("pytest_style.py", 1, PYTEST), ("numpy_mock.py", 1, NUMPY), ("gtest.cc", 3, GTEST),
        ("JTest.java", 4, JUNIT)] + [(n, e, d) for n, e, d in sr.HAND if n != "other.txt"]


def planted_file(rng, n_tests, ext):
    """A test file of n_tests tests drawn from templates of every section-25 rule (seeded), for corpora at scale."""
    py = ext == 1
    pool = ([b"self.assertEqual(a, %d)", b"self.assertEqual(a, b, 'm')", b"self.assertTrue(x == y)", b"assert x == %d",
             b"assert x, 'm'", b"np.testing.assert_allclose(a, b, err_msg='m')", b"self.assertIsNone(x)", b"self.assertEqual(\n"
             b"        a,\n        b)", b"with open('f%d') as fh:", b"v%d = f()", b"a, b%d = g()", b"m.assert_called_with(%d)",
             b"# assert %d", b"self.assertTrue(isinstance(x, int))"] if py else
            [b"EXPECT_EQ(a, %d);", b"EXPECT_EQ(a, b) << \"m\";", b"ASSERT_TRUE(a != b);", b"assert(x > %d);",
             b"static_assert(N == %d, \"m\");", b"EXPECT_EQ(p, nullptr);", b"EXPECT_EQ(a,\n            b);", b"FILE* f = fopen(\"x\");",
             b"int v%d = 0;", b"std::ifstream in%d;", b"// EXPECT_EQ(a, %d);", b"EXPECT_TRUE(x)\n      << \"m\";"])
    out = [b"import os\n\n"] if py else [b"#include <x.h>\n\n"]
    for t in range(n_tests):
        body = []
        for _ in range(rng.randrange(0, 10) if rng.random() < 0.9 else rng.randrange(20, 60)):
            s = rng.choice(pool)
            body.append(s % rng.randrange(20) if b"%d" in s else s)
        if py:
            out.append(b"def test_%d():\n" % t + b"".join(b"    " + x + b"\n" for x in body) + (b"" if body else b"    pass\n") + b"\n")
        else:
            out.append(b"TEST(S, t%d) {\n" % t + b"".join(b"  " + x + b"\n" for x in body) + b"}\n\n")
    return b"".join(out)


def planted_corpus(seed, n_files):
    """n_files planted test files (PY and C++), most with a few tests, some with many."""
    import random
    rng = random.Random(seed)
    files, exts = [], []
    for _ in range(n_files):
        ext = rng.choice([1, 1, 3, 2])
        n = rng.randrange(0, 6) if rng.random() < 0.95 else rng.randrange(20, 80)
        files.append(planted_file(rng, n, ext))
        exts.append(ext)
    return files, np.array(exts, np.uint8)


def fuzz_with_calls(seed, long_lines=False, binary=False):
    """A fuzz corpus with test headers, open assertion calls, assignments and guest calls planted in every third file."""
    files, exts, _ = cu.fuzz_corpus(seed, 300, 20000, long_lines=long_lines, binary=binary)
    rng = np.random.default_rng(seed)
    heads = [b"def test_a():", b"    def test_b(self):", b"TEST(A, B) {", b"  public void testX() {", b"    self.assertEqual(a, 1,",
             b"  EXPECT_EQ(x, 2)", b"    assert x == 3, (", b"  assertEquals(\"m\", a,", b"    v = open(f)", b"  int k = 4;"]
    for i in range(0, len(files), 3):
        lines = files[i].split(b"\n")
        for _ in range(max(1, len(lines) // 10)):
            lines.insert(int(rng.integers(0, len(lines) + 1)), heads[int(rng.integers(0, len(heads)))])
        files[i] = b"\n".join(lines)
    return files, exts
