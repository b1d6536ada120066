"""Plain-Python restatement of the test-to-code links of docs/SPEC.md section 27 (test infrastructure): the section-21 tokens seen
with their positions, the section-18 tests and code lines of lexsmell_ref, the definitions of production lines, the calls of test
code lines, the naming convention and the resolution.  Written from the SPEC text; no shared code with the kernels.

* `focal_stems(paths, role)`: the stem ids of `tosemscan.focal_stems`;
* `py_links(files, exts, role, stem, grp)`: the arrays of `tosemscan.Scanner.test_links`.
"""
import numpy as np

import blind_ref as br
import lexsmell_ref as lr
from spec_ref import W, py_bytes_hash, py_lines

KEYWORD, IDENT = lr.KEYWORD, lr.IDENT
NOT_BEFORE_DEF = {b"return", b"new", b"delete", b"throw", b"else", b"case", b"goto", b"sizeof", b"typeid", b"alignof", b"decltype",
                  b"co_return", b"co_yield", b"co_await"}
MODIFIERS = {b"public", b"protected", b"private", b"static", b"final", b"abstract", b"export"}
SUFFIXES = (b"_test", b"_tests", b"_unittest", b"Test", b"Tests")
PREFIXES = (b"test_", b"test")
FUNCTION, CLASS = 1, 2
EAGER, LAZY = 1, 2

LINK_TEST = np.dtype([("file", "<i4"), ("line", "<i4"), ("calls", "<i4"), ("linked_calls", "<i4"), ("links", "<i4"),
                      ("function_links", "<i4"), ("focal_links", "<i4"), ("flags", "<u4")])
LINK = np.dtype([("test", "<i4"), ("name_def", "<i4"), ("target", "<i4"), ("n_defs", "<i4"), ("calls", "<i4"), ("line", "<i4"),
                 ("byte", "<i4")])
LINK_DEF = np.dtype([("file", "<i4"), ("line", "<i4"), ("name_off", "<i4"), ("name_len", "<i4"), ("kind", "<i4"), ("tests", "<i4"),
                     ("tests_by_name", "<i4"), ("calls", "<i4")])


def is_test_path(path):
    """S0: a path that contains `test`, compared case-insensitively."""
    return b"test" in (path.encode() if isinstance(path, str) else path).lower()


def base_stem(path):
    b = path.encode() if isinstance(path, str) else bytes(path)
    b = b.rsplit(b"/", 1)[-1]
    dot = b.rfind(b".")
    return b[:dot] if dot > 0 else b


def focal_stem(path):
    """The focal stem of a test file's path, or None when it is empty."""
    b = base_stem(path)
    for s in SUFFIXES:
        if b.endswith(s):
            b = b[:-len(s)]
            break
    else:
        for p in PREFIXES:
            if b.startswith(p):
                b = b[len(p):]
                break
    return b or None


def focal_stems(paths, role):
    ids, out = {}, []
    for p, r in zip(paths, role):
        s = focal_stem(p) if r else base_stem(p)
        out.append(-1 if s is None else ids.setdefault(s, len(ids)))
    return np.array(out, np.int32)


def lex_at(line, fam, state):
    """lexsmell_ref.lex_tokens with the byte of each token in the line: ([(kind, bytes, start)], state at the end)."""
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
        elif (fam == br.PY and c == 0x23) or (fam == br.CJ and c == 0x2F and nx == 0x2F):
            break
        elif fam == br.CJ and c == 0x2F and nx == 0x2A:
            i = br._close(line, i + 2, fam, 1)
            if i is None:
                return toks, 1
        elif c in br.DIGITS or (c == 0x2E and nx in br.DIGITS):
            j = br._number(line, i, fam)
            toks.append((lr.NUMBER, line[i:j], i))
            i = j
        elif br._ident_byte(c):
            j = i
            while j < n and br._ident_byte(line[j]):
                j += 1
            word = line[i:j]
            if j < n and line[j] in b"\"'" and br._is_prefix(word, fam):
                k, st = br._string(line, j, fam)
                toks.append((lr.STRING, line[i:k], i))
                if st != br.CODE:
                    return toks, st
                i = k
                continue
            toks.append((KEYWORD if word in kw else lr.LITNAME if word in lit else IDENT, word, i))
            i = j
        elif c in b"\"'":
            k, st = br._string(line, i, fam)
            toks.append((lr.STRING, line[i:k], i))
            if st != br.CODE:
                return toks, st
            i = k
        else:
            toks.append((lr.PUNCT, bytes([c]), i))
            i += 1
    return toks, br.CODE


def file_tokens(lines, ext):
    fam, state, out = br.family(int(ext)), br.CODE, []
    for line in lines:
        if fam == br.NONE:
            out.append([])
            continue
        toks, state = lex_at(line, fam, state)
        out.append(toks)
    return out


def definition(toks, fam):
    """(kind, name, byte) of the definition a production line holds, or None."""
    kinds = [k for k, _, _ in toks]
    words = [b for _, b, _ in toks]
    if fam == br.PY:
        j = 1 if words[:2] == [b"async", b"def"] and kinds[0] == KEYWORD else 0
        if len(toks) > j + 1 and kinds[j] == KEYWORD and words[j] in (b"def", b"class") and kinds[j + 1] == IDENT:
            if j == 0 or words[j] == b"def":
                return (FUNCTION if words[j] == b"def" else CLASS, words[j + 1], toks[j + 1][2])
        return None
    # the class rule
    j = 0
    while j < len(toks) and kinds[j] == KEYWORD and words[j] in MODIFIERS:
        j += 1
    if j < len(toks) and kinds[j] == KEYWORD and words[j] in (b"class", b"struct", b"interface", b"enum"):
        m = j + 1
        if words[j] == b"enum" and m < len(toks) and kinds[m] == KEYWORD and words[m] in (b"class", b"struct"):
            m += 1
        if m < len(toks) and kinds[m] == IDENT and not (m + 1 < len(toks) and toks[m + 1][1] == b";" and kinds[m + 1] == lr.PUNCT):
            return (CLASS, words[m], toks[m][2])
    # the function rule
    depth = 0
    for i, (k, b, pos) in enumerate(toks):
        if k == IDENT and depth == 0 and i + 1 < len(toks) and toks[i + 1][0] == lr.PUNCT and toks[i + 1][1] == b"(":
            if i == 0:
                return None
            pk, pb, _ = toks[i - 1]
            ok = pk == IDENT or (pk == KEYWORD and pb not in NOT_BEFORE_DEF) or (pk == lr.PUNCT and pb in (b"*", b"&", b">")) or \
                (pk == lr.PUNCT and pb == b":" and i >= 2 and toks[i - 2][0] == lr.PUNCT and toks[i - 2][1] == b":")
            ok = ok and not any(t[0] == lr.PUNCT and t[1] == b"=" for t in toks[:i])
            ok = ok and not (toks[-1][0] == lr.PUNCT and toks[-1][1] == b";")
            return (FUNCTION, b, pos) if ok else None
        if k == lr.PUNCT and b in (b"(", b"[", b"{"):
            depth += 1
        elif k == lr.PUNCT and b in (b")", b"]", b"}"):
            depth -= 1
    return None


def calls(toks, fam):
    """(name, byte) of every call on a test code line."""
    out = []
    for i, (k, b, pos) in enumerate(toks):
        if k != IDENT or i + 1 >= len(toks) or toks[i + 1][:2] != (lr.PUNCT, b"("):
            continue
        if fam == br.PY and i > 0 and toks[i - 1][0] == KEYWORD and toks[i - 1][1] in (b"def", b"class"):
            continue
        out.append((b, pos))
    return out


def py_links(files, exts, role, stem=None, grp=None):
    n = len(files)
    stem = np.full(n, -1, np.int32) if stem is None else np.asarray(stem)
    grp = np.zeros(n, np.int64) if grp is None else np.asarray(grp)
    defs, tests, test_calls = [], [], []                  # defs: (file, line, off, len, kind, key); tests: (file, header line)
    for f, (data, ext) in enumerate(zip(files, exts)):
        fam = br.family(int(ext))
        if fam == br.NONE:
            continue
        lines = py_lines(data)
        starts = np.cumsum([0] + [len(x) + 1 for x in lines]).tolist()
        toks = file_tokens(lines, ext)
        if role[f]:
            for b, _, _, code in lr.bodies(lines, int(ext)):
                tests.append((f, b))
                test_calls.append([(py_bytes_hash(nm), l, starts[l] + pos) for l in code for nm, pos in calls(toks[l], fam)])
        else:
            for l, t in enumerate(toks):
                d = definition(t, fam)
                if d:
                    defs.append((f, l, starts[l] + d[2], len(d[1]), d[0], py_bytes_hash(d[1])))
    by_name, by_focal = {}, {}
    for i, (f, _, _, _, _, key) in enumerate(defs):
        by_name.setdefault((int(grp[f]), key), []).append(i)
        if stem[f] >= 0:
            by_focal.setdefault((int(grp[f]), int(stem[f]), key), []).append(i)
    links = []                                             # (test, key, calls, line, byte)
    for t, cl in enumerate(test_calls):
        f = tests[t][0]
        seen = {}
        for key, l, byte in cl:
            if (int(grp[f]), key) not in by_name:
                continue
            if key in seen:
                seen[key][2] += 1
            else:
                seen[key] = [t, key, 1, l, byte]
                links.append(seen[key])
    file_name_tests = {}
    for t, key, *_ in links:
        file_name_tests[(tests[t][0], key)] = file_name_tests.get((tests[t][0], key), 0) + 1
    name_tests = {}
    for t, key, *_ in links:
        g = (int(grp[tests[t][0]]), key)
        name_tests[g] = name_tests.get(g, 0) + 1
    out_links = np.zeros(len(links), LINK)
    d_tests, d_calls = np.zeros(len(defs), np.int64), np.zeros(len(defs), np.int64)
    t_rec = np.zeros(len(tests), LINK_TEST)
    for t, (f, b) in enumerate(tests):
        t_rec[t]["file"], t_rec[t]["line"], t_rec[t]["calls"] = f, b, len(test_calls[t])
    for j, (t, key, nc, l, byte) in enumerate(links):
        f = tests[t][0]
        ds = by_name[(int(grp[f]), key)]
        focal = by_focal.get((int(grp[f]), int(stem[f]), key)) if stem[f] >= 0 else None
        target = ds[0] if len(ds) == 1 else focal[0] if focal else -1
        func = any(defs[d][4] == FUNCTION for d in ds)
        out_links[j] = (t, ds[0], target, len(ds), nc, l, byte)
        if target >= 0:
            d_tests[target] += 1
            d_calls[target] += nc
        r = t_rec[t]
        r["linked_calls"] += nc
        r["links"] += 1
        r["function_links"] += func
        r["focal_links"] += focal is not None
        if func and file_name_tests[(f, key)] >= 2:
            r["flags"] |= LAZY
    t_rec["flags"] |= np.where(t_rec["function_links"] >= 2, EAGER, 0).astype(np.uint32)
    out_defs = np.zeros(len(defs), LINK_DEF)
    for i, (f, l, off, ln, kind, key) in enumerate(defs):
        out_defs[i] = (f, l, off, ln, kind, d_tests[i], name_tests.get((int(grp[f]), key), 0), d_calls[i])
    return {"tests": t_rec, "links": out_links, "defs": out_defs}


# ------------------------------------------------------------------------------------------------------- hand-written repositories
UNITTEST_SRC = b'''import os


class Calculator:
    """def not_a_def(): inside a docstring"""

    def add(self, a, b):
        return a + b

    async def fetch(self):
        return 1


def helper(x):  # helper(1) in a comment
    return x


def add(a, b):
    return a + b
'''
UNITTEST_TEST = b'''import unittest
from calc import Calculator, helper


class TestCalculator(unittest.TestCase):
    def test_add(self):
        c = Calculator()
        self.assertEqual(c.add(1, 2), 3)
        self.assertEqual(helper(c.add(2, 2)), 4)

    def test_strings(self):
        s = "helper(1) Calculator()"
        """fetch()"""
        # helper(2)
        self.assertTrue(s)

    def test_nested(self):
        def helper(y):
            return y
        self.assertEqual(helper(3), 3)
        assert Calculator ()
'''
PYTEST_TEST = b'''def test_fetch():
    c = Calculator()
    assert c.fetch() == 1

def test_unknown():
    assert unknown(1) == missing()
'''
GTEST_H = b'''#pragma once
class Widget {
 public:
  Widget(int x);
  int size() const;
};
int make_widget(int n);
enum class Color { Red };
struct Point;
'''
GTEST_CC = b'''#include "widget.h"
Widget::Widget(int x) : x_(x) {
}
int Widget::size() const {
  return x_;
}
int make_widget(int n)
{
  return helper_internal(n);
}
static int helper_internal(int n) {
  int y = compute(n);
  if (y) return y;
  return 0;
}
'''
GTEST_TEST = b'''#include "widget.h"
TEST(WidgetTest, Size) {
  Widget w(3);
  EXPECT_EQ(w.size(), 3);
  EXPECT_EQ(make_widget(2), 2);  // size() in a comment
  /* make_widget(9) */
}
TEST(WidgetTest, Make) {
  EXPECT_EQ(make_widget(1), 1);
}
'''
JAVA_SRC = b'''package demo;
public class Stack {
    private int n;
    public void push(int x) {
        n = n + 1;
    }
    public int size() {
        return n;
    }
}
interface Sized
{
}
'''
JAVA_TEST = b'''package demo;
import org.junit.Test;
public class StackTest {
    @Test
    public void testPush() {
        Stack s = new Stack();
        s.push(1);
        assertEquals(1, s.size());
    }
    @Test
    public void testEmpty() {
        assertEquals(0, new Stack().size());
    }
}
'''
# every definition and non-definition example of section 27, one per line
CJ_DEFS = b'''int add(int a, int b) {
Foo::Foo(int x) : a_(x) {
std::vector<int> get() const
public void run() {
long wide(int a,
return add(1, 2);
x = add(
int decl(int, int);
Foo f(1);
class Fwd;
enum Kind { A };
template <typename T> T* make() {
'''
HAND = [  # (repository, path, ext, data)
    (0, "calc/calc.py", 1, UNITTEST_SRC), (0, "calc/test_calc.py", 1, UNITTEST_TEST), (0, "calc/calc_test.py", 1, PYTEST_TEST),
    (1, "w/widget.h", 6, GTEST_H), (1, "w/widget.cc", 2, GTEST_CC), (1, "w/widget_unittest.cc", 2, GTEST_TEST),
    (2, "j/Stack.java", 4, JAVA_SRC), (2, "j/StackTest.java", 4, JAVA_TEST), (2, "j/defs.cc", 2, CJ_DEFS),
    (2, "j/notes.txt", 0, b"def add(a):\n"),
]


def hand():
    """The hand-written repositories as (files, exts, role, stem, grp, paths)."""
    paths = [p for _, p, _, _ in HAND]
    role = np.array([is_test_path(p) for p in paths], np.uint8)
    return ([d for _, _, _, d in HAND], np.array([e for _, _, e, _ in HAND], np.uint8), role, focal_stems(paths, role),
            np.array([g for g, _, _, _ in HAND], np.uint16), paths)


def planted_repos(seed, n_files, n_repos=3, n_names=400):
    """Repositories of production and test files (a third of them tests) whose tests call Zipf-distributed names, some defined
    in several files, some in the focal file, some nowhere; python, C++ and Java."""
    rng = np.random.default_rng(seed)
    names = [b"fn_%d" % i if i % 7 else b"a_rather_long_function_name_%d" % i for i in range(n_names)]
    zipf = 1.0 / np.arange(1, n_names + 1)
    zipf /= zipf.sum()
    files, exts, paths, grp = [], [], [], []
    for i in range(n_files):
        g = int(rng.integers(n_repos))
        ext = int(rng.choice([1, 2, 4]))
        stem = b"mod%d" % int(rng.integers(max(1, n_files // 6)))
        suffix = {1: b".py", 2: b".cc", 4: b".java"}[ext]
        test = i % 3 == 0
        out = []
        if test:
            for t in range(int(rng.integers(1, 5))):
                body = [b"x%d = %s(%d)" % (j, names[rng.choice(n_names, p=zipf)], j) for j in range(int(rng.integers(1, 6)))]
                if ext == 1:
                    out.append(b"def test_%d_%d(self):\n" % (i, t) + b"".join(b"    " + x + b"\n" for x in body))
                else:
                    out.append(b"TEST(S%d, T%d) {\n" % (i, t) + b"".join(b"  auto " + x + b";\n" for x in body) + b"}\n"
                               if ext == 2 else b"@Test\npublic void test%d() {\n" % t + b"".join(b"  int " + x + b";\n" for x in body)
                               + b"}\n")
            if ext == 4:
                out = [b"public class T%d {\n" % i] + out + [b"}\n"]
            path = b"r%d/test_%s%s" % (g, stem, suffix) if ext == 1 else b"r%d/%sTest%s" % (g, stem, suffix)
        else:
            for k in range(int(rng.integers(1, 8))):
                nm = names[rng.choice(n_names, p=zipf)]
                if ext == 1:
                    out.append(b"def %s(a):\n    return other(a)\n" % nm if k % 4 else b"class %s:\n    pass\n" % nm)
                else:
                    out.append(b"int %s(int a) {\n  return other(a);\n}\n" % nm if k % 4 else b"class %s {\n};\n" % nm)
            path = b"r%d/%s%s" % (g, stem, suffix)
        files.append(b"".join(out))
        exts.append(ext)
        paths.append(path)
        grp.append(g)
    role = np.array([is_test_path(p) for p in paths], np.uint8)
    return files, np.array(exts, np.uint8), role, focal_stems(paths, role), np.array(grp, np.uint16), paths
