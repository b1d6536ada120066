"""The plain-Python restatement of docs/SPEC.md section 27 (link_ref) on hand-written repositories whose answers are known, every
definition and non-definition example of the section, and the naming convention against the library's tsm_focal_stems (a host
function: no GPU)."""
import numpy as np
import pytest

import link_ref as lk
import tosemscan as ts


@pytest.fixture(scope="module")
def hand():
    files, exts, role, stem, grp, paths = lk.hand()
    return paths, files, lk.py_links(files, exts, role, stem, grp)


def name_of(files, d):
    return files[d["file"]][d["name_off"]:d["name_off"] + d["name_len"]]


def test_definitions_of_the_section(hand):
    paths, files, got = hand
    defs = got["defs"][got["defs"]["file"] == paths.index("j/defs.cc")]
    # lines 5-9 are `return add(1, 2);`, `x = add(`, `int decl(int, int);`, `Foo f(1);` and `class Fwd;`
    assert [(int(d["line"]), name_of(files, d), int(d["kind"])) for d in defs] == [
        (0, b"add", 1), (1, b"Foo", 1), (2, b"get", 1), (3, b"run", 1), (4, b"wide", 1), (10, b"Kind", 2), (11, b"make", 1)]


def test_python_definitions(hand):
    paths, files, got = hand
    defs = got["defs"][got["defs"]["file"] == paths.index("calc/calc.py")]
    # the docstring's `def` and the comment's call are no definitions; `async def` is one
    assert [(int(d["line"]), name_of(files, d), int(d["kind"])) for d in defs] == [
        (3, b"Calculator", 2), (6, b"add", 1), (9, b"fetch", 1), (13, b"helper", 1), (17, b"add", 1)]


def test_unittest_links(hand):
    paths, files, got = hand
    t, links, defs = got["tests"], got["links"], got["defs"]
    assert [paths[f] for f in t["file"]] == ["calc/test_calc.py"] * 3 + ["calc/calc_test.py"] * 2 + ["w/widget_unittest.cc"] * 2 + \
        ["j/StackTest.java"] * 2
    # test_add calls Calculator, assertEqual (twice), add (twice) and helper.  add is defined twice in calc.py, the focal file
    # of test_calc.py, so its target is the first of them in line order, the method.
    add = links[(links["test"] == 0)]
    names = [name_of(files, defs[x["name_def"]]) for x in add]
    assert names == [b"Calculator", b"add", b"helper"]
    assert list(add["calls"]) == [1, 2, 1] and list(add["n_defs"]) == [1, 2, 1]
    assert list(add["target"]) == [0, 1, 3]
    assert tuple(t[0][["calls", "linked_calls", "links", "function_links", "focal_links"]]) == (6, 4, 3, 2, 3)
    assert t[0]["flags"] == lk.EAGER
    # names inside strings, docstrings and comments are no calls
    assert (t[1]["calls"], t[1]["links"]) == (1, 0)
    # a nested def ends the test's case (section 16): its calls are outside the test
    assert t[2]["calls"] == 0


def test_gtest_focal_header_and_source(hand):
    paths, files, got = hand
    t, links, defs = got["tests"], got["links"], got["defs"]
    size = [x for x in links if x["test"] == 5 and name_of(files, defs[x["name_def"]]) == b"size"][0]
    assert size["n_defs"] == 1 and name_of(files, defs[size["target"]]) == b"size"
    # both gtest tests call make_widget: Lazy Test; the first also calls size: Eager Test
    assert t[5]["flags"] == lk.EAGER | lk.LAZY and t[6]["flags"] == lk.LAZY
    w = [d for d in defs if name_of(files, d) == b"Widget"]
    assert [paths[d["file"]] for d in w] == ["w/widget.h", "w/widget.cc"] and all(d["tests"] == 0 for d in w)


def test_junit_new(hand):
    paths, files, got = hand
    links, defs = got["links"], got["defs"]
    named = [(int(x["test"]), name_of(files, defs[x["name_def"]]), int(x["calls"])) for x in links if x["test"] >= 7]
    assert named == [(7, b"Stack", 1), (7, b"push", 1), (7, b"size", 1), (8, b"Stack", 1), (8, b"size", 1)]
    stack = [d for d in defs if name_of(files, d) == b"Stack"][0]
    assert (stack["tests"], stack["tests_by_name"], stack["calls"]) == (2, 2, 2)


def test_names_defined_twice_with_and_without_focal():
    prod_a = b"def run(x):\n    return x\n"
    prod_b = b"def run(y):\n    return y\n"
    test = b"def test_run():\n    assert run(1)\n"
    paths = ["a.py", "b.py", "test_b.py", "test_c.py"]
    role = np.array([0, 0, 1, 1], np.uint8)
    stem = lk.focal_stems(paths, role)
    got = lk.py_links([prod_a, prod_b, test, test], np.ones(4, np.uint8), role, stem)
    # test_b.py has b.py as its focal file; test_c.py has none: ambiguous
    assert list(got["links"]["target"]) == [1, -1] and list(got["links"]["n_defs"]) == [2, 2]
    assert list(got["links"]["name_def"]) == [0, 0]
    assert list(got["defs"]["tests"]) == [0, 1] and list(got["defs"]["tests_by_name"]) == [2, 2]


def test_two_repositories_and_long_names():
    name = b"a_name_much_longer_than_sixteen_bytes"
    prod = b"def %s():\n    pass\n" % name
    test = b"def test_x():\n    %s()\n    %s()\n" % (name, name)
    grp = np.array([0, 1, 1, 2], np.uint16)
    got = lk.py_links([prod, prod, test, test], np.ones(4, np.uint8), np.array([0, 0, 1, 1], np.uint8), None, grp)
    # each repository resolves only its own definitions; repository 2 defines nothing
    assert len(got["links"]) == 1 and tuple(got["links"][0][["test", "target", "n_defs", "calls"]]) == (0, 1, 1, 2)
    assert list(got["defs"]["tests"]) == [0, 1]


@pytest.mark.parametrize("path,role,want", [
    ("x/test_foo.py", 1, b"foo"), ("FooTest.java", 1, b"Foo"), ("FooTests.java", 1, b"Foo"), ("foo_unittest.cc", 1, b"foo"),
    ("foo_test.go", 1, b"foo"), ("foo_tests.py", 1, b"foo"), ("testfoo.py", 1, b"foo"), ("test.py", 1, None), ("Test.java", 1, None),
    ("tests/conftest.py", 1, b"conftest"), ("test_foo_test.py", 1, b"test_foo"), ("src/foo.py", 0, b"foo"), ("a.b/c", 0, b"c"),
    (".hidden", 0, b".hidden"), ("foo.tar.gz", 0, b"foo.tar")])
def test_focal_stem_rules(path, role, want):
    assert (lk.focal_stem(path) if role else lk.base_stem(path)) == want


def test_focal_stems_library_equals_reference():
    paths = ["r/test_foo.py", "r/foo.py", "FooTest.java", "Foo.java", "foo_unittest.cc", "foo.cc", "foo.h", "test.py", "x/tests.py",
             "a_very_long_module_name_test.py", "a_very_long_module_name.py", "dir.with.dots/bar_tests.py", "bar.py", "Test.java"]
    role = np.array([lk.is_test_path(p) for p in paths], np.uint8)
    assert list(ts.focal_stems(paths, role)) == list(lk.focal_stems(paths, role))
    assert list(ts.focal_stems([], np.zeros(0, np.uint8))) == []


def test_is_test_path():
    assert lk.is_test_path("src/Tests/x.py") and lk.is_test_path("FooTEST.java") and not lk.is_test_path("src/tst.py")
