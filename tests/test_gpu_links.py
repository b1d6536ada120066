"""`tsm_test_links` / `Scanner.test_links` (docs/SPEC.md section 27) against the plain-Python reference link_ref.py_links, every
output array: the hand-written repositories, the C1 test files (no production files: no links) with their pinned call count, the
hazard files, planted repositories, fuzz corpora, one name defined 100 000 times and called 1 M times, one test of 20 000 linked
names, more tests than the launch has warps, no production files, no tests and an empty corpus; the raw ABI's caps and NULL
outputs, repeated calls and a non-blocking stream while the legacy stream is busy."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import corpus_util as cu
import lexsmell_ref as lr
import link_ref as lk
import tosemscan as ts

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 26, max_files=1 << 16, max_groups=8)
    yield s
    s.close()


def check(s, files, exts, role, stem=None, grp=None, **kw):
    c = ts.pack(files, exts, grps=grp, n_groups=int(grp.max()) + 1 if len(grp) else 1) if grp is not None \
        else ts.pack(files, exts)
    got = s.test_links(c, role, stem, **kw)
    want = lk.py_links(files, exts, role, stem, grp)
    for k, dt in (("tests", ts.LINK_TEST), ("links", ts.LINK), ("defs", ts.LINK_DEF)):
        assert got[k].dtype == dt and np.array_equal(got[k], want[k].astype(dt)), k
    return got


def test_hand(scanner):
    files, exts, role, stem, grp, _ = lk.hand()
    got = check(scanner, files, exts, role, stem, grp)
    assert len(got["links"]) > 10 and (got["tests"]["flags"] == 3).any()
    ms = scanner.test_links_last_ms()
    assert len(ms) == 4 and all(m > 0 for m in ms)


def test_c1_counts(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    got = check(scanner, files, exts, np.ones(len(files), np.uint8))
    assert (len(got["tests"]), int(got["tests"]["calls"].sum()), len(got["links"]), len(got["defs"])) == (6239, 73897, 0, 0)


def test_hazard_files(scanner):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_hazard_files.npz"))
    role = (np.arange(len(files)) % 2).astype(np.uint8)
    check(scanner, files, exts, role, None, (np.arange(len(files)) % 3).astype(np.uint16))


def test_planted_repositories(scanner):
    files, exts, role, stem, grp, _ = lk.planted_repos(0x27, 3000)
    got = check(scanner, files, exts, role, stem, grp)
    t, links = got["tests"], got["links"]
    assert (t["flags"] & 1).any() and (t["flags"] & 2).any() and (links["target"] < 0).any() and (t["focal_links"] > 0).any()
    # the link order comes from a scan of the calls, which holds because the tests own disjoint line ranges in test order: the
    # links are sorted by test, then by first call, and each test's links are contiguous
    key = links["test"].astype(np.int64) << 32 | links["line"].astype(np.int64)
    assert (np.diff(links["test"]) >= 0).all() and (np.diff(key) >= 0).all()
    assert (np.bincount(links["test"], minlength=len(t)) == t["links"]).all()


@pytest.mark.parametrize("n", [1023, 1024, 1025, 100000])
def test_many_calls_on_one_line(scanner, n):
    # far more calls than lines: the scans over the calls need their own block sums (ceil(n / 1024) of them, for a 3-line corpus)
    prod = b"def f(x):\n    return x\n"
    test = b"def test_one_line():\n    " + b"f(1);" * n + b"\n"
    got = check(scanner, [prod, test], np.ones(2, np.uint8), np.array([0, 1], np.uint8))
    assert got["tests"][0]["calls"] == n and got["links"][0]["calls"] == n and got["defs"][0]["calls"] == n


@pytest.mark.parametrize("long_lines,binary", [(False, False), (True, False), (False, True)])
def test_fuzz(scanner, long_lines, binary):
    files, exts = lr.fuzz_with_calls(0x2701 + 7 * long_lines + 3 * binary, long_lines, binary)
    role = (np.arange(len(files)) % 3 == 0).astype(np.uint8)
    check(scanner, files, exts, role, None, (np.arange(len(files)) % 2).astype(np.uint16))


def test_hot_name(scanner):
    # one name defined 100 000 times (in 10 production files) and called 1 000 000 times (in 1 000 tests)
    prod = b"".join(b"def hot(x%d):\n    pass\n" % i for i in range(10000))
    test = b"".join(b"def test_%d():\n" % i + b"    hot(1); hot(2); hot(3); hot(4); hot(5)\n" * 200 for i in range(100))
    files = [prod] * 10 + [test] * 10
    role = np.array([0] * 10 + [1] * 10, np.uint8)
    got = check(scanner, files, np.ones(20, np.uint8), role)
    assert len(got["defs"]) == 100000 and int(got["tests"]["calls"].sum()) == 1000000
    assert (got["links"]["n_defs"] == 100000).all() and (got["links"]["target"] == -1).all()
    assert (got["tests"]["flags"] == lk.LAZY).all()


def test_many_names_in_one_test(scanner):
    n = 20000
    prod = b"".join(b"int f%d(int a) {\n  return a;\n}\n" % i for i in range(n))
    test = b"TEST(A, B) {\n" + b"".join(b"  f%d(%d);\n" % (i, i) for i in range(n)) + b"}\n"
    got = check(scanner, [prod, test], np.array([2, 2], np.uint8), np.array([0, 1], np.uint8))
    assert len(got["links"]) == n and got["tests"][0]["flags"] == lk.EAGER and (got["defs"]["tests"] == 1).all()


def test_more_tests_than_warps(scanner):
    prod = b"def f(x):\n    return x\n\ndef g(x):\n    return x\n"
    tests = [b"".join(b"def test_%d():\n    assert f(%d) == g(1)\n" % (i, i) for i in range(3000)) for _ in range(4)]
    got = check(scanner, [prod] + tests, np.ones(5, np.uint8), np.array([0, 1, 1, 1, 1], np.uint8))
    assert len(got["tests"]) == 12000 > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 8
    assert (got["tests"]["flags"] == 3).all()


def test_no_production_no_tests_and_empty(scanner):
    got = check(scanner, [b"def test_a():\n    f()\n"], np.ones(1, np.uint8), np.ones(1, np.uint8))
    assert len(got["links"]) == 0 and len(got["defs"]) == 0 and got["tests"][0]["calls"] == 1
    got = check(scanner, [b"def f():\n    pass\n", b"x = f()\n"], np.ones(2, np.uint8), np.array([0, 1], np.uint8))
    assert len(got["tests"]) == 0 and len(got["defs"]) == 1 and got["defs"][0]["tests"] == 0
    got = scanner.test_links(ts.pack([], np.zeros(0, np.uint8)), np.zeros(0, np.uint8))
    assert all(len(got[k]) == 0 for k in ("tests", "links", "defs"))


def test_raw_caps_and_null_outputs(scanner):
    files, exts, role, stem, grp, _ = lk.hand()
    c = ts.pack(files, exts, grps=grp, n_groups=3)
    cs = c.c_struct()
    want = scanner.test_links(c, role, stem)
    T, K, D = len(want["tests"]), len(want["links"]), len(want["defs"])
    lib = ts.lib()

    def call(tests, tcap, links, kcap, defs, dcap):
        r = ts._LinksResult(tests=ts._p(tests), test_cap=tcap, links=ts._p(links), link_cap=kcap, defs=ts._p(defs), def_cap=dcap)
        rc = lib.tsm_test_links(scanner._ctx, C.byref(cs), ts._p(role), ts._p(stem), C.byref(r), None)
        return rc, (r.n_tests, r.n_links, r.n_defs)

    def arrays():
        return np.zeros(T, ts.LINK_TEST), np.zeros(K, ts.LINK), np.zeros(D, ts.LINK_DEF)

    t, k, d = arrays()
    assert call(t, T, k, K, d, D) == (0, (T, K, D))
    assert np.array_equal(t, want["tests"]) and np.array_equal(k, want["links"]) and np.array_equal(d, want["defs"])
    assert call(t, T - 1, k, K, d, D) == (ts.TSM_E_CAPACITY, (T, K, D))
    assert call(t, T, k, K - 1, d, D) == (ts.TSM_E_CAPACITY, (T, K, D))
    assert call(t, T, k, K, d, D - 1) == (ts.TSM_E_CAPACITY, (T, K, D))
    assert call(None, 0, None, 0, None, 0) == (0, (T, K, D))
    for i, key in enumerate(("tests", "links", "defs")):
        outs = [None] * 3
        outs[i] = arrays()[i]
        caps = [0, 0, 0]
        caps[i] = len(want[key])
        assert call(outs[0], caps[0], outs[1], caps[1], outs[2], caps[2]) == (0, (T, K, D)) and np.array_equal(outs[i], want[key])
    r = ts._LinksResult()
    assert lib.tsm_test_links(scanner._ctx, C.byref(cs), None, None, C.byref(r), None) == -1
    bad = np.full(len(files), -2, np.int32)
    assert lib.tsm_test_links(scanner._ctx, C.byref(cs), ts._p(role), ts._p(bad), C.byref(r), None) == -1


def test_repeated_calls_and_stream(scanner):
    files, exts, role, stem, grp, _ = lk.planted_repos(0x2702, 600)
    c = ts.pack(files, exts, grps=grp, n_groups=3)
    first = scanner.test_links(c, role, stem)
    for _ in range(3):
        again = scanner.test_links(c, role, stem)
        assert all(np.array_equal(first[k], again[k]) for k in first)
    busy = torch.empty(1 << 26, device="cuda:0")
    st = torch.cuda.Stream(device=0)                      # (created non-blocking by torch)
    for _ in range(20):
        busy.mul_(1.0001)                                  # the legacy stream is busy while the call runs on st
    got = scanner.test_links(c, role, stem, stream=st.cuda_stream)
    torch.cuda.synchronize()
    assert all(np.array_equal(first[k], got[k]) for k in first)
