"""GPU tests of the clone classes (docs/SPEC.md section 15) at the seams tests/test_gpu_clones.py does not reach: the hand-made
cases of tests/test_clones_ref.py; windows whose keys are crafted (tests/orc_clones.py window_with_key) to hit the hash table's
key-0 side slot, a probe chain that wraps from the last slot into slot 0, many keys on one home slot and two contents with
one key; classes of every size around the warp sort, the shared-memory sort and the tiled sort, and more large classes than
the k_clone_sort_cta grid; class lengths around the 32-flag ballots of k_clone_length and more classes than its warps; files
without lines around the file search; and the raw C ABI one output at a time.  Every output array is compared with the serial
C reference orc_clones, and every test asserts from the host-side keys, sizes and counts that its input reaches the seam it
names."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import corpus_util as cu
import orc_clones as ocl
import spec_ref
import tosemscan as ts
from test_clones_ref import HAND_MADE, planted

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WARP_MAX = 32                                              # CLONE_WARP_MAX: larger classes are sorted by k_clone_sort_cta
SMEM = 4096                                                # SIM_SMEM_LINES: larger classes take the tiled sort
BLOCK = 256                                                # threads of a k_clone_scatter block (one per line)


@pytest.fixture(scope="module")
def sc():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 14, max_groups=4)
    yield s
    s.close()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def run(sc, files, n, exts=None, py=False):
    """tsm_clones against orc_clones (and against the content-equality reference py_clones with py); (result, corpus)."""
    exts = [1] * len(files) if exts is None else exts
    c = ts.pack(files, exts)
    got = sc.clones(c, n)
    ocl.assert_equal(got, ocl.clones(c, n))
    if py:
        ocl.assert_equal(got, ocl.py_clones(files, exts, n))
    return got, c


def sizes(r):
    return np.diff(r["class_base"])


def class_of(r, start):
    """The class whose representative (first fragment) starts at global line `start`, or None."""
    hit = np.nonzero(r["member"][r["class_base"][:-1]] == start)[0] if len(r["member"]) else []
    return int(hit[0]) if len(hit) else None


def home(keys, mask):
    return keys & np.uint64(mask)


# ---------------------------------------------------------------------------------------------- the reference's own cases
@pytest.mark.parametrize("name", sorted(HAND_MADE))
def test_hand_made_cases(sc, name):
    files, n = HAND_MADE[name]
    got, c = run(sc, files, n, py=True)
    assert got["line_base"][-1] == sum(len(spec_ref.py_lines(f)) for f in files)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_planted_copies(sc, n):
    files = planted(0xC10E + n, 300)
    got, _ = run(sc, files, n, [(i % 7) for i in range(len(files))], py=True)
    assert len(got["class_len"]) > 10 and got["file_dup_assert"].sum() > 0


def test_c1_windows_of_one_line(sc):
    files, exts, _, _ = cu.load_fixture(os.path.join(GOLD, "c1_testfiles.npz"))
    got, _ = run(sc, files, 1, exts)
    assert len(got["class_len"]) > 10000 and sizes(got).max() > WARP_MAX


def test_windows_of_1024_lines_around_the_file_length(sc):
    """Files of 1 023 lines have no window of 1 024, files of 1 024 one, files of 1 025 two."""
    block = {m: b"".join(b"L%d_%d\n" % (m, i) for i in range(m)) for m in (1023, 1024, 1025)}
    files = [block[1023], block[1024], block[1025], block[1023], block[1024], block[1025]]
    got, c = run(sc, files, 1024, py=True)
    g = ocl.window_groups(c, 1024)
    assert [int(g["valid"][b:e].sum()) for b, e in zip(g["line_base"][:3], g["line_base"][1:4])] == [0, 1, 2]
    assert got["class_len"].tolist() == [1024, 1025]


# ---------------------------------------------------------------------------------------------- the key-0 side slot
@pytest.mark.parametrize("n", [5, 13])
@pytest.mark.parametrize("case", ["head", "middle", "once", "wide"])
def test_key0_side_slot(sc, case, n):
    files, mask = ocl.key0_corpus(case, n, 0xC10E0 + n)
    got, c = run(sc, [ocl.text(f) for f in files], n, py=True)
    g = ocl.window_groups(c, n)
    z = np.nonzero(g["valid"] & (g["key"] == 0))[0]
    assert mask == ocl.table_mask(int(g["line_base"][-1]))
    # slot 0 holds keys of other groups (homed there), so that a key-0 window merged into slot 0 changes the groups
    homed0 = (home(g["keys"], mask) == 0) & (g["keys"] != 0)
    assert homed0.sum() == ocl.SLOT0_KEYS and (g["counts"][homed0] == ocl.SLOT0_COPIES).all()
    if case == "head":
        # a key-0 group heads a class that extends to the right: the next group's predecessor slot is the side slot
        # (pred_lo == pred_hi == mask + 1), and no key that can sit in slot 0 has the count of the key-0 group
        assert len(z) == 3 and (g["count"][z] == 3).all() and not g["ext"][z].any()
        assert g["ext"][z + 1].all() and (g["count"][z + 1] == 3).all()
        k = class_of(got, z[0])
        assert k is not None and got["class_len"][k] > n and sizes(got)[k] == 3
        reach = ocl.keys_that_can_reach(g["keys"], mask, 0)
        counts = dict(zip(g["keys"].tolist(), g["counts"].tolist()))
        assert reach and all(counts[key] != 3 for key in reach)
    elif case == "middle":
        # the key-0 group is left-extendable, and the predecessor of the next group
        assert len(z) == 2 and (g["count"][z] == 2).all() and g["ext"][z].all() and g["ext"][z + 1].all()
        assert class_of(got, z[0]) is None and class_of(got, z[0] - 3) is not None
    elif case == "once":
        # one key-0 window (the side slot's count is 1) between windows that occur twice
        assert len(z) == 1 and g["count"][z[0]] == 1 and g["count"][z[0] - 1] == 2 and g["count"][z[0] + 1] == 2
    else:
        # a key-0 class of more than 32 fragments: sorted by k_clone_sort_cta
        assert len(z) == 40 > WARP_MAX and not g["ext"][z].any()
        k = class_of(got, z[0])
        assert k is not None and got["member"][got["class_base"][k]:got["class_base"][k + 1]].tolist() == z.tolist()


# ---------------------------------------------------------------------------------------------- probe chains
@pytest.mark.parametrize("extra", [0, 1])
def test_probe_chain_wraps_into_slot_0(sc, extra):
    files, mask = ocl.probe_corpus(extra, 0x9B0BE + extra)
    got, c = run(sc, [ocl.text(f) for f in files], 3)
    g = ocl.window_groups(c, 3)
    T = int(g["line_base"][-1])
    assert T == 4096 + extra and mask + 1 == (2 * T if extra == 0 else 4 * T - 4)   # 2T a power of two, or one line more
    keys, counts, h = g["keys"], g["counts"], home(g["keys"], mask)
    assert ((h == mask) & (counts >= 2)).sum() >= 512 and ((h == mask) & (counts == 1)).sum() >= 20
    assert all(((h == s) & (counts >= 2)).any() for s in range(40))            # homes 0 .. 39: they collide with the chain
    occ = ocl.occupied_slots(keys, mask)
    assert occ[mask] and int(np.argmin(occ)) >= 512                           # the chain from slot mask fills 0 .. 511+
    # the collision pair: two contents, one key homed at mask; the key decides (one group, one class)
    pair = [i for i, f in enumerate(files) if f and f[1].startswith(b"p")]
    starts = [int(g["line_base"][i]) for i in pair]
    assert files[pair[0]] != files[pair[1]] and g["key"][starts[0]] == g["key"][starts[1]]
    assert int(g["key"][starts[0]]) & mask == mask
    k = class_of(got, starts[0])
    assert k is not None and got["member"][got["class_base"][k]:got["class_base"][k + 1]].tolist() == starts


# ---------------------------------------------------------------------------------------------- sort boundaries
SORT_SIZES = [2, 31, 32, 33, 4095, 4096, 4097, 8192, 8193, 16385, 100003]


def runs_corpus(class_sizes, n, seed, chunk=7):
    """Class c is a run of the line r<c>: its m fragments cut into files of 1 .. chunk windows (m_i + n - 1 lines), the
    files of all classes interleaved so that each class's fragments lie in many k_clone_scatter blocks."""
    rng = random.Random(seed)
    parts = []
    for c, m in enumerate(class_sizes):
        cuts = []
        while m:
            k = min(m, rng.randint(1, chunk))
            cuts.append(b"r%d\n" % c * (k + n - 1))
            m -= k
        parts.append(cuts)
    files = []
    for j in range(max(len(p) for p in parts)):
        files += [p[j] for p in parts if j < len(p)]
    return files


def test_sort_boundaries(sc):
    n = 5
    got, _ = run(sc, runs_corpus(SORT_SIZES, n, 0x5027), n)
    sz = sizes(got)
    assert sorted(sz.tolist()) == SORT_SIZES and (got["class_len"] == n).all()
    assert 1 << int(sz.max() - 1).bit_length() >= 16 * SMEM                   # the tiled sort: merge stages 2 .. 32 tiles
    for k in np.nonzero(sz > WARP_MAX)[0]:                                     # every CTA-sorted class is scattered from
        frag = got["member"][got["class_base"][k]:got["class_base"][k + 1]]  # many blocks
        assert len(np.unique(frag // BLOCK)) >= 3


def test_more_large_classes_than_the_cta_grid(sc, sms):
    """More classes of over 32 fragments than k_clone_sort_cta has CTAs (2 x SMs): its grid-stride loop runs."""
    n = 3
    big = [33 + c % 9 for c in range(2 * sms + 37)]
    got, _ = run(sc, runs_corpus(big + [2, 5, 32], n, 0xC7A, chunk=1), n)
    assert (sizes(got) > WARP_MAX).sum() == len(big) > 2 * sms


# ---------------------------------------------------------------------------------------------- k_clone_length
BALLOT_R = [0, 1, 30, 31, 32, 33, 63, 64, 65, 1000]


def test_ballot_edges(sc):
    n = 5
    blocks = {r: [b"k%d_%d" % (r, i) for i in range(n + r)] for r in BALLOT_R}
    files = [[b"ua%d" % r] + blocks[r] + [b"va%d" % r] for r in BALLOT_R]
    files += [[b"ub%d" % r] + blocks[r] + [b"vb%d" % r] for r in BALLOT_R]
    # a copy that ends at a file's end while the next file goes on with the same lines as the other copy: two classes
    B, Cc = [b"B%d" % i for i in range(n + 2)], [b"C%d" % i for i in range(n + 3)]
    files += [B, Cc, [b"mid"], B, Cc]
    # the last file: a run whose representative lies within 32 lines of the corpus' end, then a copy of E on the last line
    E = [b"E%d" % i for i in range(n + 1)]
    files += [[b"e0"] + E + [b"e1"], [b"w"] + [b"z"] * (n + 3) + E]
    got, c = run(sc, [ocl.text(f) for f in files], n, py=True)
    T = int(got["line_base"][-1])
    lens = got["class_len"].tolist()
    assert all(lens.count(n + r) >= 1 for r in BALLOT_R)
    assert len(B) in lens and len(Cc) in lens and len(B) + len(Cc) not in lens
    reps = got["member"][got["class_base"][:-1]]
    assert reps.max() > T - 32                                 # its ballot's lanes reach past the last line
    assert any(int(got["member"][j]) + len(E) == T for j in range(len(got["member"])))       # a fragment ends on it


def test_more_classes_than_length_warps(sc, sms):
    """More classes than k_clone_length has warps (8 x SMs blocks of 8), with run lengths of 0 .. 66 flags."""
    n = 5
    K = 64 * sms + 301
    rng = random.Random(0x1E7)
    blocks = [[b"c%d_%d" % (c, i) for i in range(n + c % 67)] for c in range(K)]
    order_b = list(range(K))
    rng.shuffle(order_b)
    files = []
    for copy, order in ((b"a", range(K)), (b"b", order_b)):
        cur = []
        for j, c in enumerate(order):
            cur += [b"%s%d" % (copy, c)] + blocks[c]
            if j % 200 == 199:
                files.append(cur)
                cur = []
        files.append(cur)
    got, _ = run(sc, [ocl.text(f) for f in files], n)
    assert len(got["class_len"]) == K > 64 * sms
    assert sorted(got["class_len"].tolist()) == sorted(n + c % 67 for c in range(K))


# ---------------------------------------------------------------------------------------------- file search and coverage
def test_files_without_lines_and_ext_0(sc):
    X = b"".join(b"    assert check(%d) == %d\n" % (i, i) if i % 2 else b"x%d = make()\n" % i for i in range(8))
    data = [b""] * 3000 + [X] + [b""] * 2500 + [X] + [b""] * 1500 + [b"first\n" + X] + [b""] * 3000
    exts = [1] * len(data)
    x0, x1, x2 = [i for i, f in enumerate(data) if f]
    exts[x1] = 0
    got, _ = run(sc, data, 5, exts, py=True)
    assert (x0, x1 - x0, x2 - x1, len(data) - x2) == (3000, 2501, 1501, 3001)
    assert got["file_dup"][x0] == got["file_dup"][x1] == 8 and got["file_dup"].sum() == 24
    assert got["file_dup_assert"][x1] == 0 and got["file_dup_assert"][x0] == got["file_dup_assert"][x2] == 4


# ---------------------------------------------------------------------------------------------- the raw ABI
FIELDS = ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len", "member")
SENTINEL = 0x5EB7


def raw(sc, c, n, omit=(), class_cap=None, member_cap=None, want=None):
    """tsm_clones with arrays one entry longer than asked, filled with SENTINEL; (status, result struct, arrays)."""
    nf = c.n_files
    nc, nm = len(want["class_len"]), len(want["member"])
    class_cap = nc if class_cap is None else class_cap
    member_cap = nm if member_cap is None else member_cap
    size = {"line_base": nf + 1, "file_dup": nf, "file_dup_assert": nf, "class_base": class_cap + 1, "class_len": class_cap,
            "member": member_cap}
    out = {k: np.full(size[k] + 1, SENTINEL, want[k].dtype) for k in FIELDS if k not in omit}
    p = {k: (ts._p(out[k]) if k in out else None) for k in FIELDS}
    r = ts._CloneResult(p["line_base"], p["file_dup"], p["file_dup_assert"], p["class_base"], p["class_len"], class_cap, -1,
                        p["member"], member_cap, -1)
    cs = c.c_struct()
    rc = ts.lib().tsm_clones(sc._ctx, C.byref(cs), n, C.byref(r), None)
    return rc, r, out


@pytest.fixture(scope="module")
def abi_case():
    files = planted(0xAB1, 300)
    c = ts.pack(files, [(i % 7) for i in range(len(files))])
    want = ocl.clones(c, 3)
    assert len(want["class_len"]) > 10 and len(want["member"]) > len(want["class_len"])
    return c, want


@pytest.mark.parametrize("omit", FIELDS)
def test_raw_abi_one_output_null(sc, abi_case, omit):
    """Each output NULL on its own; the others are the reference's, exactly as long as the counts (caps exact:
    class_base[n_classes] written, nothing after the last entry of any array)."""
    c, want = abi_case
    rc, r, out = raw(sc, c, 3, omit=(omit,), want=want)
    assert rc == 0 and (r.n_classes, r.n_members) == (len(want["class_len"]), len(want["member"]))
    assert r.class_cap == r.n_classes and r.member_cap == r.n_members
    for k, a in out.items():
        assert np.array_equal(a[:-1], want[k]) and a[-1] == SENTINEL, k


def test_raw_abi_short_caps_and_retry(sc, abi_case):
    c, want = abi_case
    nc, nm = len(want["class_len"]), len(want["member"])
    for caps in ((nc - 1, nm), (nc, nm - 1), (0, nm), (nc, 0)):
        rc, r, _ = raw(sc, c, 3, class_cap=caps[0], member_cap=caps[1], want=want)
        assert rc == ts.TSM_E_CAPACITY and (r.n_classes, r.n_members) == (nc, nm), caps
    rc, r, _ = raw(sc, c, 3, omit=("class_base", "class_len"), class_cap=0, want=want)   # no class output: no class cap
    assert rc == 0 and r.n_classes == nc
    rc, r, _ = raw(sc, c, 3, omit=("member",), member_cap=0, want=want)
    assert rc == 0 and r.n_members == nm
    for _ in range(2):                                          # the retry after the capacity error is the full result
        rc, r, out = raw(sc, c, 3, want=want)
        assert rc == 0
        for k, a in out.items():
            assert np.array_equal(a[:-1], want[k]) and a[-1] == SENTINEL, k


def test_last_ms_of_an_empty_corpus(sc, abi_case):
    sc.clones(abi_case[0], 3)
    assert all(m > 0 for m in sc.clones_last_ms())
    got = sc.clones(ts.pack([], []), 3)
    assert got["line_base"].tolist() == [0] and sc.clones_last_ms() == [0.0, 0.0, 0.0]
    got = sc.clones(ts.pack([b""] * 5, [1] * 5), 3)
    assert got["line_base"].tolist() == [0] * 6 and sc.clones_last_ms()[1:] == [0.0, 0.0]
