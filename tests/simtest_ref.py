"""References of the similar tests of docs/SPEC.md section 23.  TEST INFRASTRUCTURE ONLY.

* `py_sequences(files, exts)`: the plain-Python restatement of the tests and their sequences: tests and bodies from
  `smell_ref.py_file_smells`, kept lines and blind hashes from `blind_ref.blind_lines`;
* `c_sequences(corpus)`: the same from the serial C references (`orc_smells`, `orc_blind`), for corpora at scale;
* `py_similar(seqs, min_lines, P)`: every pair by brute force with an O(nm) LCS table, no filter at all;
* `c_similar(seqs, min_lines, P)`: the serial C brute force of tests/orc_simtest.c (only the exact size filter);
* `prefix_candidates(seqs, min_lines, P)`: a model of the device's exact prefix filter (tokens, rare-first order, prefixes,
  posting lists, the first-common-token rule), which must keep every pair that passes;
* `classes(pairs, nt)`: single-linkage classes by a union-find;
* `reference(corpus, min_lines, P)`: the dict of `tosemscan.Scanner.similar_tests` from the C references;
* `c_lcs_pairs(seqs, a, b)`: the LCS of many pairs by the serial C code;

and the builders of tests/test_gpu_similar_tests_seams.py (each checked on the CPU by tests/test_similar_tests_ref.py):

* `punct(n)` / `py_file(seqs)`: one PY file with a test per sequence of line ids, each id a line of its own blind form;
* `tight_cases(P)`: pairs whose shorter test is exactly the size-filter minimum and shares one token of the other's prefix;
* `repeat_cases(P)`: pairs whose only shared lines are one line repeated, the line common in the rest of the corpus;
* `copies(n, n_copies, P, seed)`: copies of one base of n lines with chosen positions replaced, lcs in closed form;
* `generated(seed, n_tests)`: the seeded corpus of tools/bench_similar_tests.py with its planted Type-3 copies;
* `filler(n_tests, first_id)`: tests of unique lines, which share only their header with anything.
"""
import ctypes as C
import hashlib
import math
import os
import random
import subprocess
import tempfile
import threading
from collections import Counter, defaultdict

import numpy as np

import blind_ref as br
import orc
import orc_blind
import orc_smells
import smell_ref

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orc_simtest.c")
_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(open(SRC, "rb").read()).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_simtest_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-o", tmp, SRC])
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_similar.restype = C.c_int
            L.orc_similar.argtypes = [C.c_void_p] * 3 + [C.c_int32] * 3 + [C.c_void_p] * 3 + [C.c_int64, C.c_void_p]
            L.orc_similar_row.restype = C.c_int64
            L.orc_similar_row.argtypes = [C.c_void_p] * 3 + [C.c_int32] * 4 + [C.c_void_p, C.c_int64]
            L.orc_lcs_pairs.restype = C.c_int
            L.orc_lcs_pairs.argtypes = [C.c_void_p] * 5 + [C.c_int64, C.c_void_p]
            _lib = L
    return _lib


def py_sequences(files, exts):
    """(tests, seqs): tests as (file, header line, body_lines) in global line order, seqs[t] the blind hashes of t's kept lines."""
    tests, seqs = [], []
    for f, (data, ext) in enumerate(zip(files, exts)):
        forms = br.blind_lines(data, int(ext))
        for b, n, *_ in smell_ref.py_file_smells(data, int(ext))[0]:
            tests.append((f, b, n))
            seqs.append([br.blind_hash(x) for x in forms[b:b + n] if x])
    return tests, seqs


def c_sequences(corpus):
    """(SMELL_TEST records, seqs) from the C references."""
    tests = orc_smells.smells(corpus)["tests"]
    base, kept, bhash, _ = orc_blind.blind_lines(corpus)
    seqs = []
    for t in tests:
        l0 = int(base[t["file"]]) + int(t["line"])
        sl = slice(l0, l0 + int(t["body_lines"]))
        seqs.append(bhash[sl][kept[sl]].tolist())
    return tests, seqs


def lcs(a, b):
    prev = [0] * (len(b) + 1)
    for x in a:
        cur = [0]
        for j, y in enumerate(b):
            cur.append(prev[j] + 1 if x == y else max(prev[j + 1], cur[j]))
        prev = cur
    return prev[-1]


def passes(l, ka, kb, P):
    return 200 * l >= P * (ka + kb)


def score(l, ka, kb):
    return 120000 * l // (ka + kb)


def py_similar(seqs, min_lines, P):
    """[(a, b, lcs, score)] over every pair of compared tests, ascending."""
    out = []
    for a in range(len(seqs)):
        if len(seqs[a]) < min_lines:
            continue
        for b in range(a + 1, len(seqs)):
            if len(seqs[b]) < min_lines:
                continue
            l = lcs(seqs[a], seqs[b])
            if passes(l, len(seqs[a]), len(seqs[b]), P):
                out.append((a, b, l, score(l, len(seqs[a]), len(seqs[b]))))
    return out


def c_similar(seqs, min_lines, P):
    k = np.array([len(s) for s in seqs], np.uint32)
    beg = np.concatenate([[0], np.cumsum(k, dtype=np.int64)]).astype(np.int64)
    flat = np.array([h for s in seqs for h in s], np.uint64)
    if flat.size == 0:
        flat = np.zeros(1, np.uint64)
    p = orc._p
    cap = 1 << 16
    for _ in range(2):
        pa, pb, pl = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.uint32)
        n = C.c_int64()
        rc = lib().orc_similar(p(flat), p(beg), p(k), len(seqs), int(min_lines), int(P), p(pa), p(pb), p(pl), cap, C.byref(n))
        if rc == -3:
            cap = n.value
            continue
        if rc:
            raise ValueError("orc_similar failed")
        n = n.value
        return [(int(a), int(b), int(l), score(int(l), int(k[a]), int(k[b]))) for a, b, l in zip(pa[:n], pb[:n], pl[:n])]
    raise ValueError("orc_similar: capacity")


def flatten(seqs):
    """(flat, beg, k) of the C references; pass it instead of seqs to call them many times on one large corpus."""
    if isinstance(seqs, tuple):
        return seqs
    k = np.array([len(s) for s in seqs], np.uint32)
    beg = np.concatenate([[0], np.cumsum(k, dtype=np.int64)]).astype(np.int64)
    flat = np.fromiter((h for s in seqs for h in s), np.uint64, int(k.sum(dtype=np.int64)))
    return (flat if flat.size else np.zeros(1, np.uint64)), beg, k


def c_partners(seqs, a, min_lines, P):
    """The tests that pair with test a, by brute force over the whole corpus (ascending); seqs may be flatten(seqs)."""
    flat, beg, k = flatten(seqs)
    other = np.zeros(len(k), np.int32)
    n = lib().orc_similar_row(orc._p(flat), orc._p(beg), orc._p(k), len(k), int(a), int(min_lines), int(P), orc._p(other), len(k))
    if n < 0:
        raise ValueError("orc_similar_row failed")
    return other[:n].tolist()


def c_lcs_pairs(seqs, a, b):
    """lcs(seqs[a[i]], seqs[b[i]]) for every i, by the serial C LCS; seqs may be flatten(seqs)."""
    flat, beg, k = flatten(seqs)
    a, b = np.ascontiguousarray(a, np.int32), np.ascontiguousarray(b, np.int32)
    out = np.zeros(len(a), np.uint32)
    if lib().orc_lcs_pairs(orc._p(flat), orc._p(beg), orc._p(k), orc._p(a), orc._p(b), len(a), orc._p(out)):
        raise ValueError("orc_lcs_pairs failed")
    return out


def tokens(seq):
    seen = Counter()
    out = []
    for h in seq:
        out.append((h, seen[h]))
        seen[h] += 1
    return out


def prefix_candidates(seqs, min_lines, P, short=0):
    """The candidate pairs of the device's filter: each compared test's tokens (h, j) in the order (count of h over the compared
    tests, h, j), its prefix of k - ceil(P k / (200 - P)) + 1 tokens, the posting lists of prefix tokens, and per list every pair
    that passes the size filter and whose first common prefix token is the list's token.  short: prefixes that many tokens
    shorter (a wrong filter, for the checks of the builders)."""
    cmp = [t for t, s in enumerate(seqs) if len(s) >= min_lines]
    cnt = Counter(h for t in cmp for h in seqs[t])
    order = lambda tok: (cnt[tok[0]], tok[0], tok[1])
    pref, lists = {}, defaultdict(list)
    for t in cmp:
        k = len(seqs[t])
        alpha = -(-P * k // (200 - P))
        pref[t] = sorted(tokens(seqs[t]), key=order)[:k - alpha + 1 - short]
        for tok in pref[t]:
            lists[tok].append(t)
    out = set()
    for tok, mem in lists.items():
        for i in range(len(mem)):
            for j in range(i + 1, len(mem)):
                a, b = min(mem[i], mem[j]), max(mem[i], mem[j])
                ka, kb = len(seqs[a]), len(seqs[b])
                if 200 * min(ka, kb) < P * (ka + kb):
                    continue
                pb = set(pref[b])
                first = next((x for x in pref[a] if x in pb), None)
                if first == tok:
                    assert (a, b) not in out
                    out.add((a, b))
    return out


def classes(pairs, nt):
    """(class_base, member): the components of at least two tests, by smallest member, members ascending."""
    root = list(range(nt))

    def find(x):
        while root[x] != x:
            root[x] = root[root[x]]
            x = root[x]
        return x
    linked = set()
    for a, b, *_ in pairs:
        ra, rb = find(a), find(b)
        root[max(ra, rb)] = min(ra, rb)
        linked.update((a, b))
    groups = defaultdict(list)
    for t in sorted(linked):
        groups[find(t)].append(t)
    base, member = [0], []
    for r in sorted(groups):
        member += groups[r]
        base.append(len(member))
    return np.array(base, np.int64), np.array(member, np.int32)


def reference(corpus, min_lines, P):
    tests, seqs = c_sequences(corpus)
    pairs = c_similar(seqs, min_lines, P)
    base, member = classes(pairs, len(seqs))
    return {"tests": tests, "test_kept": np.array([len(s) for s in seqs], np.uint32),
            "pairs": np.array(pairs, [("a", "<i4"), ("b", "<i4"), ("lcs", "<u4"), ("score", "<u4")]),
            "class_base": base, "member": member}


def assert_equal(got, want):
    for key in ("tests", "test_kept", "pairs", "class_base", "member"):
        g, w = got[key], want[key]
        assert len(g) == len(w), (key, len(g), len(w))
        assert np.array_equal(g.view(np.uint8) if g.dtype.names else g, np.asarray(w, g.dtype).view(np.uint8) if g.dtype.names else w), key


# ---------------------------------------------------------------------------------------------- builders
PUNCT = ":+/=|*.>"


def punct(n):
    """A PY line whose blind form spells n >= 0 in octal over the operators PUNCT (no '#', quote or digit): `x` and one operator
    and `x` per digit, lowest first; the line grows by 2 bytes per octal digit.  Distinct n give distinct blind forms and, for
    n < 2^19, distinct blind hashes: the line hash folds the bytes mod 2^61 - 1, under which most such alphabets collide early
    (with "+-*/%&|^" at n = 69 and 327); this one was chosen for that range."""
    s = "x"
    while True:
        s += PUNCT[n & 7] + "x"
        n >>= 3
        if not n:
            return s


def py_file(seqs):
    """One PY file with test i for seqs[i]: its header, then the line punct(e) per element e.  Every header has the same blind
    form, so the sequence of test i is [header] + seqs[i] with one blind form per id."""
    return "".join("def test_%d():\n" % i + "".join("    %s\n" % punct(e) for e in s) for i, s in enumerate(seqs)).encode()


def alpha(P, k):
    return -(-P * k // (200 - P))


TIGHT_KA = (5, 7, 12, 33, 64, 65, 130)


def tight_cases(P):
    """(seqs, cases) for py_file at similarity P (min_lines 1).  A case (a, b, b2, eq) is three tests: a of k_a kept lines (the
    header, k_a - α lines of its own, then α - 1 lines S, α = α(a)), b = the header and S (k_b = α(a), the least k that can pass
    against a), and b2 = b without its last line (None when α = 1).  The header and S are a's α most frequent tokens, the last
    line of S the rarest of them (count 2, the rest of S 3), so a's prefix of k_a - α + 1 tokens holds exactly one token b has:
    that line; a-b passes with lcs = k_b and a-b2 fails the size filter.  eq: 200 k_b == P (k_a + k_b), the size filter's
    equality.  k_a: TIGHT_KA and the least k_a >= 5 on the equality.  The cases alternate between a first and a last."""
    step = (200 - P) // math.gcd(P, 200)                  # the equality holds when step divides k_a
    seqs, cases, nid = [], [], 0
    for n, ka in enumerate(TIGHT_KA + (step * -(-5 // step),)):
        al = alpha(P, ka)
        own, S = list(range(nid, nid + ka - al)), list(range(nid + ka - al, nid + ka - 1))
        nid += ka - 1
        group = [own + S, S] + ([S[:-1]] if al > 1 else [])
        order = list(range(len(group)))[::-1 if n % 2 else 1]
        at = {g: len(seqs) + i for i, g in enumerate(order)}
        seqs += [group[g] for g in order]
        cases.append((at[0], at[1], at.get(2), 200 * al == P * (ka + al)))
    return seqs, cases


def repeat_cases(P, n_fill=400):
    """(seqs, cases) for py_file at similarity P (min_lines 1): pairs whose only shared lines are the header and one line R
    repeated.  n_fill filler tests of the header and four lines of their own, every second one with R as well (R then counts
    about n_fill / 2 plus the cases' occurrences: common, but rarer than the header).  A case (a, b, c, c2): b is the header and
    c2 lines R, a is the header, lines of its own and c >= c2 lines R, with as many own lines as k_b = α(a) allows (the least
    partner size).  a's prefix then ends inside the run of R's tokens, at (R, c - c2); the lcs is k_b."""
    seqs, cases = [], []
    R, nid = 0, 1
    for i in range(n_fill):
        seqs.append(list(range(nid, nid + 2)) + ([R] if i % 2 == 0 else []) + list(range(nid + 2, nid + 4)))
        nid += 4
    for c in (3, 4, 6):
        for c2 in range(1, c + 1):
            m = -1
            while alpha(P, 2 + m + c) <= c2 + 1:            # the most own lines with α(a) = c2 + 1
                m += 1
            if m < 0 or alpha(P, 1 + m + c) != c2 + 1:
                continue
            cases.append((len(seqs), len(seqs) + 1, c, c2))
            seqs += [list(range(nid, nid + m)) + [R] * c, [R] * c2]
            nid += m
    return seqs, cases


def copies(n, n_copies, P, seed):
    """(seqs, sets): n_copies copies of a base of n distinct lines, copy i with the positions in sets[i] replaced by lines of its
    own.  With the header every copy has k = n + 1, and lcs(i, j) = 1 + n - |sets[i] | sets[j]| (the base lines outside both
    sets, in order, and the header).  P (n + 1) must be a multiple of 100, so that the pair passes exactly when the union holds
    at most T = (n + 1)(100 - P) / 100 positions.  The sets are random subsets of 4 T positions, of 0.45 T to 0.62 T each, so
    that the unions spread around T."""
    assert P * (n + 1) % 100 == 0
    T = (n + 1) * (100 - P) // 100
    rng = random.Random(seed)
    pool = rng.sample(range(n), 4 * T)
    sets = [frozenset(rng.sample(pool, rng.randint(45 * T // 100, 62 * T // 100))) for _ in range(n_copies)]
    seqs, nid = [], n
    for s in sets:
        seqs.append([nid + p if p in s else p for p in range(n)])
        nid += n
    return seqs, sets


def copies_pairs(n, sets, P):
    """The pairs of copies() in closed form, ascending: (a, b, lcs, score)."""
    out = []
    for a in range(len(sets)):
        for b in range(a + 1, len(sets)):
            l = 1 + n - len(sets[a] | sets[b])
            if passes(l, n + 1, n + 1, P):
                out.append((a, b, l, score(l, n + 1, n + 1)))
    return out


def shape(v):
    return "x" + "".join("[x]" if (v >> b) & 1 else "(x)" for b in range(16))


def generated(seed, n_tests, pinned=False):
    """(corpus, planted): PY tests of 4 to 20 lines drawn from 65 536 distinct blind line shapes, a fifth of the lines from 16
    common shapes (the assertion and set-up lines every suite repeats), 100 tests per file; every tenth test is a Type-3 copy of
    an earlier one with one or two lines inserted, deleted or changed.  planted: (copy, original) test indices."""
    import tosemscan as ts
    rng = np.random.default_rng(seed)
    shapes = [shape(v) for v in range(1 << 16)]
    klen = rng.integers(4, 21, n_tests)
    common = rng.random(int(klen.sum())) < 0.2
    ids = np.where(common, rng.integers(0, 16, common.size), rng.integers(16, 1 << 16, common.size))
    bodies, planted, at = [], [], 0
    prng = random.Random(seed)
    for t in range(n_tests):
        b = ids[at:at + klen[t]].tolist()
        at += klen[t]
        if t % 10 == 9:
            src = prng.randrange(t)
            planted.append((t, src))
            b = list(bodies[src])
            for _ in range(prng.randint(1, 2)):
                r = prng.random()
                if r < 0.33 and len(b) > 1:
                    b.pop(prng.randrange(len(b)))
                elif r < 0.66:
                    b.insert(prng.randrange(len(b) + 1), prng.randrange(16, 1 << 16))
                else:
                    b[prng.randrange(len(b))] = prng.randrange(16, 1 << 16)
        bodies.append(b)
    files = []
    for f in range(0, n_tests, 100):
        files.append("".join("def test_%d():\n%s" % (t, "".join("    %s\n" % shapes[v] for v in bodies[t]))
                             for t in range(f, min(f + 100, n_tests))).encode())
    return ts.pack(files, np.ones(len(files), np.uint8), pinned=pinned), planted


def filler(n_tests, first_id, per_file=100):
    """Files of n_tests PY tests of 4 to 11 lines punct(first_id), punct(first_id + 1), ...: every line unique, so the tests share
    only their header with anything (and with the shapes of generated(), which have no operator)."""
    files, nid = [], first_id
    for f in range(0, n_tests, per_file):
        tests = []
        for t in range(f, min(f + per_file, n_tests)):
            k = 4 + t % 8
            tests.append("def test_f%d():\n" % t + "".join("    %s\n" % punct(e) for e in range(nid, nid + k)))
            nid += k
        files.append("".join(tests).encode())
    return files
