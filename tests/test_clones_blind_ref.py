"""The blind clones of docs/SPEC.md section 21 on the CPU: the serial C reference (tests/orc_blind.c) and the plain-Python
restatement (tests/blind_ref.py) agree line by line (kept flag and blind hash) and class by class, on the lexer's hazards (comment
and string openers inside literals, escapes, unterminated literals, string prefixes, docstrings and block comments that span lines,
pp-numbers, keywords against identifiers, literal names, non-ASCII identifier bytes, tag-0 files, CRLF, empty and all-comment
files), on the section's worked examples, on the C1 counts pinned in the section, and on the crafted seam corpora of
tests/front_seams.py, which reach the seams they name (the keyword table the kernel builds, its chains and its wrap included)."""
import os
import types

import numpy as np
import pytest

import blind_ref as br
import corpus_util as cu
import front_seams as fs
import orc
import orc_blind as ob
import spec_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def corpus(files, exts):
    arena, off, length = orc.pack(files)
    return types.SimpleNamespace(arena=arena, off=off, len=length, ext=np.asarray(exts, np.uint8))


def both(files, exts, n):
    """The two references on one corpus: per line, then the classes.  Returns the C reference's dict."""
    c = corpus(files, exts)
    base, kept, bhash, _ = ob.blind_lines(c)
    forms = [f for data, e in zip(files, exts) for f in br.blind_lines(data, e)]
    assert len(forms) == len(kept) == base[-1]
    assert kept.tolist() == [bool(f) for f in forms]
    assert bhash.tolist() == [br.blind_hash(f) if f else 0 for f in forms]
    got = ob.clones_blind(c, n)
    br.assert_equal(got, br.py_blind_clones(files, exts, n))
    return got


def forms(text, ext):
    got = br.blind_lines(text, ext)
    both([text], [ext], 1)
    return got


PY_CASES = [
    (b'x = "a # b"  # c\n', [b"I = S"]),
    (b'y = \'it\\\'s\' + "q\\"x"\n', [b"I = S + S"]),
    (b'z = "open\nw = 1 \'\n', [b"I = S", b"I = N S"]),
    (b'a = rb"x#" + f\'{b}\' + Rb\'\' + br"" + u"u" + ab"x" + rbf"y"\n', [b"I = S + S + S + S + S + I S + I S"]),
    (b'"""doc""" ; x = 1\n', [b"S ; I = N"]),
    (b's = """first\ninner # not a comment\n\nend""" + x\n', [b"I = S", b"", b"", b"+ I"]),
    (b"t = '''a \"\"\" b\n''' \"\"\"c\\\"\"\" d\"\"\"\n", [b"I = S", b"S"]),
    (b'"""\\"""" x\n', [b"S I"]),
    (b"1e+5 0x1F .5 1. 1_000 1e-3j x.y\n", [b"N N N N N N I . I"]),
    (b"iffy if import_ True None False Nonesuch\n", [b"I if I N N N I"]),
    (b"caf\xc3\xa9 = 1\n\xff\xfe = 2\n$x = _\n", [b"I = N", b"I = N", b"I = I"]),
    (b"match x:\n    case _: pass\n", [b"I I :", b"I I : pass"]),
    (b"# only a comment\n    # another\n\n  \t \n", [b"", b"", b"", b""]),
    (b"x = 1\r\n\r\ny = 2", [b"I = N", b"", b"I = N"]),
    (b'u = "tail\\', [b"I = S"]),
]
CJ_CASES = [
    (b's = "a // b"; // c\n', [b"I = S ;"]),
    (b"c = '/*'; d = \"*/\";\n", [b"I = S ; I = S ;"]),
    (b"u8\"x\" L'y' u\"z\" U\"w\" R\"(r)\" LR\"a\" uR\"b\" UR\"c\" u8R\"d\" Lx\"e\"\n", [b"S S S S S S S S S I S"]),
    (b"/* a */ int x = 0; /* b\nstill */ y++;\n/*/ still\n*/ z;\n", [b"int I = N ;", b"I + + ;", b"", b"I ;"]),
    (b"1'000 0x1F 1e+5 .5 1. 0x1p-3 1'f' x'y'\n", [b"N N N N N N N S I S"]),
    (b"nullptr true null NULL false\n", [b"N N N I N"]),
    (b"if (x) return; else iffy; reinterpret_cast<int>(y);\n", [b"if ( I ) return ; else I ; reinterpret_cast < int > ( I ) ;"]),
    (b'String s = """\n  hello\n  """;\n', [b"I I = S S", b"I", b"S S"]),
    (b"int a; /* open to the end\n x = 1;\n", [b"int I ;", b""]),
    (b"// a\n/* b */\n", [b"", b""]),
    (b"a = '\\\\'; b = '\\'';\r\n", [b"I = S ; I = S ;"]),
]


@pytest.mark.parametrize("text,want", PY_CASES)
def test_python_lexer(text, want):
    assert forms(text, 1) == want


@pytest.mark.parametrize("text,want", CJ_CASES)
def test_c_family_lexer(text, want):
    for ext in (2, 3, 4, 5, 6):
        assert forms(text, ext) == want


def test_tag0_files_drop_whitespace_only():
    assert forms(b"  a b\t# c \r\n\r\n\"x\"  /* y */\n", 0) == [b"ab#c", b"", b"\"x\"/*y*/"]


def test_state_does_not_leak_across_files():
    files = [b'"""open\nx = 1\n', b"x = 1\n", b"/* open\nx = 1;\n", b"x = 1;\n"]
    got = both(files, [1, 1, 3, 3], 1)
    assert got["kept_base"].tolist() == [0, 1, 2, 2, 3] and got["kept_line"].tolist() == [0, 2, 5]


def test_empty_files_and_all_comment_files():
    got = both([b"", b"# a\n# b\n", b"", b"// x\n/* y\n z */\n"], [1, 1, 3, 3], 3)
    assert got["kept_base"].tolist() == [0, 0, 0, 0, 0] and len(got["member"]) == 0 and got["line_base"].tolist() == [0, 0, 2, 2, 5]
    got = both([], [], 5)
    assert got["line_base"].tolist() == [0] and got["kept_base"].tolist() == [0]


# The worked examples of section 21.
TEST_ADD = b"""class TestAdd(unittest.TestCase):
    def test_add_1(self):
        self.assertEqual(add(1, 1), 2)

    def test_add_2(self):
        # the same check, other values
        self.assertEqual(add(2, 3), 5)
"""
MOVED = b"""def test_add_3(self):
    self.assertEqual(add(4, 4), 8)
"""


def test_worked_examples():
    a = b"def test_add_2(self): self.assertEqual(add(2, 3), 5)\n"
    b = b"def test_add_1(self): self.assertEqual(add(1, 1), 2)\n"
    assert br.blind_lines(a, 1) == br.blind_lines(b, 1) == [b"def I ( I ) : I . I ( I ( N , N ) , N )"]
    got = both([TEST_ADD, MOVED], [1, 1], 2)
    # kept lines: 0 class, 1 def, 2 assert, 3 def, 4 assert (line 5 is a comment), 5 def, 6 assert
    assert got["kept_line"].tolist() == [0, 1, 2, 4, 6, 7, 8]
    assert got["class_len"].tolist() == [2] and got["member"].tolist() == [1, 3, 5]
    first_last = [(int(got["kept_line"][m]), int(got["kept_line"][m + 1])) for m in got["member"]]
    assert first_last == [(1, 2), (4, 6), (7, 8)]                 # the spans differ: 2 lines, 3 lines (comment inside), 2 lines
    assert got["file_dup"].tolist() == [4, 2] and got["file_dup_assert"].tolist() == [2, 1] and got["file_kept_assert"].tolist() == [2, 1]
    over = both([b"x = f(x)\n", b"y = g(z)\n"], [1, 1], 1)
    assert over["class_len"].tolist() == [1] and over["member"].tolist() == [0, 1]   # blind renaming is not consistent renaming


def test_planted_type2_copies():
    rng = np.random.default_rng(21)
    body = [b"def test_case_%d(self):", b"    value = compute(%d, 'x%d')", b"    # check it", b"    self.assertEqual(value, %d)",
            b"    self.assertTrue(value > %d)", b'    """done %d"""']
    files, exts = [], []
    for i in range(40):
        lines = [ln % ((int(rng.integers(0, 99)),) * ln.count(b"%d")) for ln in body]
        if i % 3 == 0:
            lines = [b"    " + ln for ln in lines]
        if i % 4 == 0:
            lines.insert(2, b"")
        files.append(b"\n".join(lines) + b"\n")
        exts.append(1)
    got = both(files, exts, 3)
    assert len(got["class_len"]) >= 1 and int(np.diff(got["class_base"]).max()) >= 26


def test_hazard_files_agree():
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_hazard_files.npz"))
    small = [(f, e) for f, e in zip(files, exts) if len(f) < 200000]
    both([f for f, _ in small], [e for _, e in small], 5)


# C1 counts pinned in section 21: (classes, fragments, duplicated kept lines, duplicated kept assertion lines) at n = 3 / 5 / 10.
C1_KEPT, C1_KEPT_ASSERT = 201747, 25181
C1_PINNED = {3: (16494, 91326, 155678, 18666), 5: (9501, 43951, 123501, 14611), 10: (3411, 13322, 80972, 9162)}


@pytest.mark.parametrize("n", [3, 5, 10])
def test_c1_pinned_counts(n):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    got = both(files, exts, n)
    assert len(got["kept_line"]) == C1_KEPT and int(got["file_kept_assert"].sum()) == C1_KEPT_ASSERT
    assert (len(got["class_len"]), len(got["member"]), int(got["file_dup"].sum()), int(got["file_dup_assert"].sum())) == C1_PINNED[n]
    assert int(got["file_dup"].sum()) <= C1_KEPT


def test_blind_hash_is_section3_bytes_hash():
    assert br.blind_hash(b"I = N") == spec_ref.py_bytes_hash(b"I = N")


# The crafted corpora of tests/front_seams.py, on which tests/test_gpu_clones_blind_seams.py runs the kernels: the two references
# agree on each, and each reaches the seams it names.
def test_kernel_keyword_lists_are_the_reference_sets():
    py, cj, py_lit, cj_lit = fs.kernel_keyword_lists()
    assert (set(py), set(cj), set(py_lit), set(cj_lit)) == (br.PY_KEYWORDS, br.CJ_KEYWORDS, br.PY_LITERALS, br.CJ_LITERALS)
    assert len(py + cj + py_lit + cj_lit) == len(set(py + cj + py_lit + cj_lit)) + len(br.PY_KEYWORDS & br.CJ_KEYWORDS)


def test_keyword_table_chains_and_wrap():
    slots = fs.keyword_table()
    names = br.PY_KEYWORDS | br.CJ_KEYWORDS | br.PY_LITERALS | br.CJ_LITERALS
    assert sorted(w for w in slots if w) == sorted(names) and len(names) == 143
    shift = {w: (i - fs.kw_home(w)) % fs.SLOTS for i, w in enumerate(slots) if w}
    assert sum(1 for v in shift.values() if v) == 12 and max(shift.values()) == 3
    assert slots[511] == b"bitor" and slots[0] == b"decltype"         # a chain that wraps from the last slot to slot 0
    for i, w in enumerate(slots):                                      # every name is found where the kernel put it
        if w:
            assert fs.probe(slots, w)[0][-1] == i


def test_keyword_corpus_walks_chains_and_wraps():
    files, exts, reach = fs.keyword_corpus()
    assert reach["searched_walk"] and reach["wraps"] and len(reach["displaced_found"]) == 12
    words = files[0].split()
    assert {b"reinterpret_cast", b"reinterpret_castX", b"abcdefghijklmnop", b"abcdefghijklmnopq"} <= set(words)
    assert br.lex_line(b"reinterpret_cast reinterpret_castX", br.CJ, 0)[0] == [b"reinterpret_cast", b"I"]
    both(files, exts, 1)


def test_blind_grid_corpus():
    files, exts, reach = fs.blind_grid_corpus()
    assert all(fs.on_the_grid(reach).values()) and len(reach) == len(fs.PY_CONSTRUCTS) + len(fs.CJ_CONSTRUCTS)
    both(files, exts, 2)


def test_filter_corpus():
    files, exts, reach = fs.filter_corpus()
    for fam in ("py", "cj"):
        assert all(reach[(fam, k)] == set(range(8)) for k in ("byte0", "byte7", "byte8", "last"))
        assert reach[(fam, "neighbour_before")] and reach[(fam, "neighbour_after")]
    both(files, exts, 2)


def test_scan_corpus():
    files, exts, reach = fs.scan_corpus()
    for ext, n, lanes in reach["lanes"][:10]:
        assert {(l, r) for l in (0, 1, 30, 31) for r in range(n // 32 + 1) if 32 * r + l < n} <= set(lanes), (ext, n)
    assert reach["permutation"] and reach["noncommuting_neighbours"] >= 20
    got = both(files, exts, 1)
    kb = got["kept_base"]
    assert kb[11] - kb[10] == 1 and kb[12] == kb[11] and kb[14] - kb[13] == 1    # the open comment does not leak into int b;


def test_files_corpus():
    files, exts, reach = fs.files_corpus()
    got = both(files, exts, 1)
    assert got["file_kept_assert"].tolist() == reach["asserts"]
    assert got["kept_base"][-4:].tolist() == [got["kept_base"][-1]] * 4      # no kept line in the last three files
