"""Plain-Python restatement of the test smells of docs/SPEC.md section 18 (test infrastructure): tests, bodies, line kinds and
the nine smells, straight from the bytes of one file.  Written from the SPEC text on spec_ref.py and case_ref.py; no shared
code with the kernels or tests/orc_smells.c."""
from spec_ref import W, _ident, py_bytes_hash, py_is_assert_line, py_lines
from case_ref import py_case_name, py_cases

SMELLS = ("empty", "assertion_free", "duplicate_assert", "redundant_assert", "conditional_logic", "exception_handling",
          "sleepy", "print", "ignored")
BIT = {s: 1 << i for i, s in enumerate(SMELLS)}
TEST_LEVEL = BIT["empty"] | BIT["assertion_free"]      # reported on the header line, with an empty statement

C_PREFIXES = (b"TEST(", b"TEST_F(", b"TEST_P(", b"TYPED_TEST(", b"TYPED_TEST_P(", b"BOOST_AUTO_TEST_CASE(",
              b"BOOST_FIXTURE_TEST_CASE(", b"BOOST_DATA_TEST_CASE(")
CONSTANTS = (b"True", b"False", b"true", b"false", b"None", b"nullptr", b"NULL", b"0", b"1")
COND = (b"if", b"elif", b"for", b"while", b"switch")
EXC = (b"try", b"except", b"catch", b"raise", b"throw")
BRACKETS = set(b"{}();:") | set(W)


def py_kinds(lines):
    """SPEC section 10 line kinds: 0 blank, 1 first line of a statement, 2 continuation."""
    out, d = [], 0
    for ln in lines:
        if not ln.strip(W):
            out.append(0)
            continue
        out.append(1 if d == 0 else 2)
        d = max(0, d + ln.count(b"(") - ln.count(b")"))
    return out


def family(ext: int) -> str:
    return "py" if ext == 1 else ("java" if ext == 4 else ("c" if ext in (2, 3, 5, 6) else ""))


def is_test_header(line: bytes, ext: int) -> bool:
    """SPEC section 18: does a section-5 header line open a test?"""
    s, fam = line.strip(W), family(ext)
    if fam == "py":
        i = 0
        if s.startswith(b"async"):
            i = 5
            j = i
            while j < len(s) and s[j] in W:
                j += 1
            if j == i:
                return False
            i = j
        if not s.startswith(b"def", i):
            return False
        i += 3
        j = i
        while j < len(s) and s[j] in W:
            j += 1
        return j > i and s.startswith(b"test", j)
    if fam == "c":
        return s.startswith(C_PREFIXES)
    if fam == "java":
        return b"void" in line and b"(" in line
    return False


def indent(line: bytes) -> int:
    n = 0
    while n < len(line) and line[n] in (0x20, 0x09):
        n += 1
    return n


def is_comment(s: bytes, fam: str) -> bool:
    return s.startswith(b"#") if fam == "py" else s.startswith((b"//", b"/*", b"*"))


def first_token(s: bytes) -> bytes:
    i = 0
    while i < len(s) and (s[i] in W or s[i] == 0x7D):
        i += 1
    j = i
    while j < len(s) and _ident(s[j]):
        j += 1
    return s[i:j]


def tq_count(line: bytes, q: bytes) -> int:
    """Non-overlapping occurrences of q (three quotes), left to right."""
    return line.count(q)


def is_redundant(s: bytes) -> bool:
    """SPEC section 18 redundant assertion, on a stripped assertion line."""
    for c in CONSTANTS:
        if s.startswith(b"assert") and len(s) > 6 and s[6] in W and s[6:].strip(W) == c:
            return True
    a, b = s.find(b"("), s.rfind(b")")
    if a < 0 or b <= a:
        return False
    x = s[a + 1:b].strip(W)
    if x in CONSTANTS:
        return True
    parts, depth, start = [], 0, 0
    for i, c in enumerate(x):
        if c in b"([{":
            depth += 1
        elif c in b")]}":
            depth -= 1
        elif c == 0x2C and depth == 0:
            parts.append(x[start:i])
            start = i + 1
    parts.append(x[start:])
    if len(parts) != 2:
        return False
    p, q = parts[0].strip(W), parts[1].strip(W)
    return p != b"" and p == q


def has_print(s: bytes) -> bool:
    if b"System.out.print" in s or b"System.err.print" in s:
        return True
    for pat in (b"print(", b"pprint(", b"printf(", b"puts(", b"cout", b"cerr"):
        i = s.find(pat)
        while i >= 0:
            if i == 0 or not _ident(s[i - 1]):
                return True
            i = s.find(pat, i + 1)
    return False


def py_file_smells(data: bytes, ext: int):
    """The tests of one file: a list of (header line, body_lines, n_assert, smells, n_instances, [(line, bit), ...]) with
    0-based lines, and the smell bits of every line of the file."""
    lines = py_lines(data)
    fam = family(ext)
    line_smell = [0] * len(lines)
    tests = []
    if not fam:
        return tests, line_smell
    kinds = py_kinds(lines)
    heads = set(h for h, _ in py_cases(lines, ext))
    for b, e in py_cases(lines, ext):
        if not is_test_header(lines[b], ext):
            continue
        hs = b + 1
        while hs < e and kinds[hs] == 2:
            hs += 1
        bend = e
        if fam == "py":
            ind = indent(lines[b])
            for l in range(hs, e):
                if kinds[l] == 1 and not is_comment(lines[l].strip(W), fam) and indent(lines[l]) <= ind:
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
        code = []
        dq = sq = 0
        for l in range(hend, bend):
            s = lines[l].strip(W)
            doc = False
            if fam == "py":
                doc = dq % 2 == 1 or sq % 2 == 1 or s.startswith((b'"""', b"'''"))
                dq += tq_count(lines[l], b'"""')
                sq += tq_count(lines[l], b"'''")
            if s and not is_comment(s, fam) and not doc:
                code.append(l)
        asserts = [l for l in list(range(b, hend)) + code if py_is_assert_line(lines[l], ext)]
        inst = []
        seen = set()
        for l in asserts:
            s = lines[l].strip(W)
            h = py_bytes_hash(s)
            if h in seen:
                inst.append((l, BIT["duplicate_assert"]))
            seen.add(h)
            if is_redundant(s):
                inst.append((l, BIT["redundant_assert"]))
        for l in code:
            s = lines[l].strip(W)
            t = first_token(s)
            if t in COND:
                inst.append((l, BIT["conditional_logic"]))
            if t in EXC:
                inst.append((l, BIT["exception_handling"]))
            if b"sleep(" in s or b"sleep_for(" in s or b"sleep_until(" in s:
                inst.append((l, BIT["sleepy"]))
            if has_print(s):
                inst.append((l, BIT["print"]))
            if fam == "py" and s.startswith((b"self.skipTest(", b"pytest.skip(")):
                inst.append((l, BIT["ignored"]))
        deco = []
        a = b - 1
        while a >= 0 and a not in heads and lines[a].strip(W).startswith(b"@"):
            deco.append(lines[a])
            a -= 1
        ignored = False
        if fam == "py":
            ignored = any(b"skip" in d for d in deco)
        elif fam == "java":
            ignored = any(b"@Ignore" in d or b"@Disabled" in d for d in deco + [lines[b]])
        else:
            ignored = b"DISABLED_" in lines[b]
        if ignored:
            inst.append((b, BIT["ignored"]))
        if not asserts:
            inst.append((b, BIT["assertion_free"]))
            if all(lines[l].strip(W) == b"pass" or all(c in BRACKETS for c in lines[l]) for l in code):
                inst.append((b, BIT["empty"]))
        smells = 0
        for l, bit in inst:
            line_smell[l] |= bit
            smells |= bit
        inst.sort(key=lambda t: (t[0], t[1]))
        tests.append((b, bend - b, len(asserts), smells, len(inst), inst))
    return tests, line_smell


def py_smells(files, exts):
    """SPEC section 18 over a corpus: (tests, line_smell) with tests as (file, header line, body_lines, n_assert, smells,
    n_instances) in global line order and line_smell the smell bits of every line, files in order."""
    tests, smell = [], []
    for f, (data, ext) in enumerate(zip(files, exts)):
        t, ls = py_file_smells(data, int(ext))
        tests += [(f, b, n, a, s, k) for b, n, a, s, k, _ in t]
        smell += ls
    return tests, smell


def py_smell_rows(files, exts, names=None):
    """The --out rows of SPEC section 18 without the repository column: (fileName, test, line, smell, smellLine, statement),
    lines 1-based, in file, header line, instance line and smell order."""
    rows = []
    for f, (data, ext) in enumerate(zip(files, exts)):
        lines = py_lines(data)
        for b, _, _, _, _, inst in py_file_smells(data, int(ext))[0]:
            name = py_case_name(lines[b], int(ext))
            for l, bit in inst:
                smell = SMELLS[bit.bit_length() - 1]
                st = b"" if bit & TEST_LEVEL else lines[l].strip(W)
                rows.append((names[f] if names else f, name, b + 1, smell, l + 1, st))
    return rows


# Hand-written files with known answers (tests/test_smells_ref.py pins them): (name, ext, bytes).
HAND = [
    ("unittest.py", 1, b'''import unittest, time


class TestThing(unittest.TestCase):
    def setUp(self):
        self.x = 1

    def test_free(self):
        x = compute()
        print(x)

    def test_dup(self):
        self.assertEqual(a, b)
        self.assertEqual(a, b)
        self.assertEqual(a, a)
        self.assertTrue(True)

    def test_logic(self):
        if x:
            self.assertTrue(x)
        for i in range(3):
            pass
        try:
            time.sleep(1)
        except ValueError:
            raise
        # time.sleep(1)
        y = sprintf(x) + fingerprint(y)
        pprint(y)

    def test_skip(self):
        self.skipTest("later")
        assert x

    def test_empty(self):
        pass

    def test_doc(self):
        """Assert that "if" in here is no code.
        if x:
        """
        s = """
        x""" """
        if y:
        """
        assert s
'''),
    ("pytest_style.py", 1, b'''import pytest


@pytest.mark.skip(reason="x")
@pytest.mark.parametrize("a", [1])
def test_skipped(a):
    assert a == 1


async def test_async():
    assert await f()


def test_black(
    a,
    b,
):
    x = a
# a column-0 comment
    assert x == b
    assert x == b


def helper():
    assert 1


def test_last():
    assert 1
    assert f(a, b) == f(a, b)
    self.assertEqual(f(a, b), f(a, b))


if __name__ == "__main__":
    main()
'''),
    ("crlf.py", 1, b"def test_crlf():\r\n    assert x\r\n\tassert x\r\n    assert  x\r\n    while True:\r\n        break\r\ndef test_tail():\r\n    pass"),
    ("gtest.cc", 3, b'''#include <gtest/gtest.h>

TEST(Suite, Plain) {
  EXPECT_EQ(a, b);
  EXPECT_EQ(a, b);
  if (x) {
    std::cout << x;
  }
}

TEST_F(Fixture, DISABLED_Later) {
  ASSERT_TRUE(true);
  std::this_thread::sleep_for(1s);
  printf("%d", x);
}

TEST(Suite, OneLiner) { foo(); }
int helper_test() { return 1; }

TEST(Suite, Empty) {
}

TEST(Suite, void_never_opens)
  ASSERT_EQ(1, 1);

TEST(Suite, Negative) }} {
  try { x(); } catch (...) { throw; }
  EXPECT_TRUE(1);
}
'''),
    ("boost.cpp", 2, b'''BOOST_AUTO_TEST_CASE(first_test) {
  BOOST_CHECK(x);
  // assert(x) in a comment
  BOOST_CHECK(x);
  while (y) { usleep(10); }
}
BOOST_FIXTURE_TEST_CASE(second_test, F) {
  puts("x");
  fputs("y", f);
}
'''),
    ("Junit4Test.java", 4, b'''public class Junit4Test {
  @Ignore
  @Test public void testIgnored() {
    assertEquals(1, 1);
  }
  @Test public void testPrint() {
    System.out.println("x");
    for (int i = 0; i < 2; i++) { }
    assertTrue(x);
  }
  @Disabled @Test public void testDisabled() { }
}
'''),
    ("Junit3Test.java", 4, b'''public class Junit3Test extends TestCase {
  public void testOne() throws Exception {
    Thread.sleep(10);
    /* assert nothing */
    * not code
    assertEquals(a, b);
    assertEquals(a, b);
  }
}
'''),
    ("headerless.py", 1, b"x = 1\nprint(x)\n"),
    ("empty.py", 1, b""),
    ("other.txt", 0, b"def test_x():\n    pass\n"),
]


def planted_file(rng, n_tests: int, ext: int) -> bytes:
    """A test file of n_tests tests drawn from smelly and clean templates (seeded), for corpora at scale."""
    py = ext == 1
    out = [b"import os\n\n"] if py else [b"#include <x.h>\n\n"]
    for t in range(n_tests):
        body = []
        for _ in range(rng.randrange(0, 8)):
            r = rng.random()
            if r < 0.35:
                body.append(b"assert x == %d" % rng.randrange(3) if py else b"EXPECT_EQ(x, %d);" % rng.randrange(3))
            elif r < 0.45:
                body.append(b"if x:" if py else b"if (x) { y(); }")
            elif r < 0.5:
                body.append(b"time.sleep(0.1)" if py else b"sleep(1);")
            elif r < 0.55:
                body.append(b"print(x)" if py else b"std::cout << x;")
            elif r < 0.6:
                body.append(b"self.assertEqual(a, a)" if py else b"ASSERT_TRUE(true);")
            elif r < 0.65:
                body.append(b"# assert x" if py else b"// EXPECT_EQ(a, b);")
            elif r < 0.7:
                body.append(b"raise ValueError()" if py else b"throw 1;")
            else:
                body.append(b"y = f(%d)" % rng.randrange(10) if py else b"y = f(%d);" % rng.randrange(10))
        if py:
            deco = b"@pytest.mark.skip\n" if rng.random() < 0.05 else b""
            out.append(deco + b"def test_%d():\n" % t + b"".join(b"    " + x + b"\n" for x in body) + (b"" if body else b"    pass\n") + b"\n")
        else:
            name = b"DISABLED_t%d" % t if rng.random() < 0.05 else b"t%d" % t
            out.append(b"TEST(S, " + name + b") {\n" + b"".join(b"  " + x + b"\n" for x in body) + b"}\n\n")
    return b"".join(out)


def planted_corpus(seed: int, n_files: int):
    """n_files planted test files (PY and C++), most with a few tests, some with many."""
    import random
    import numpy as np
    rng = random.Random(seed)
    files, exts = [], []
    for _ in range(n_files):
        ext = rng.choice([1, 1, 3, 2])
        n = rng.randrange(0, 6) if rng.random() < 0.95 else rng.randrange(20, 80)
        files.append(planted_file(rng, n, ext))
        exts.append(ext)
    return files, np.array(exts, np.uint8)
