"""References of the clone classes of docs/SPEC.md section 15.  TEST INFRASTRUCTURE ONLY.

* `clones(corpus, n)`: ctypes binding of tests/orc_clones.c (compiled together with the oracle's orc.c, for the line and
  n-gram hashes, into a library in the temporary directory, so that the tests never write into the tree).
* `py_clones(files, exts, n)`: the same definition in plain Python over line contents (windows are equal when their n
  contents are equal), independent of the hash.
Both return the dict of `tosemscan.Scanner.clones`.
"""
import ctypes as C
import hashlib
import os
import random
import subprocess
import tempfile
import threading

import numpy as np

import orc
import spec_ref

HERE = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(HERE, "orc_clones.c"), os.path.join(orc.ORC_DIR, "orc.c")]
DEPS = SRCS + [os.path.join(orc.ORC_DIR, "orc.h"), os.path.join(orc.ORC_DIR, "orc_categories.inc")]

_lib = None
_lock = threading.Lock()


def lib():
    global _lib
    with _lock:
        if _lib is None:
            key = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
            so = os.path.join(tempfile.gettempdir(), "tosem_orc_clones_%s_%d.so" % (key, os.getuid()))
            if not os.path.exists(so):
                tmp = so + ".%d" % os.getpid()
                subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c99", "-fPIC", "-shared", "-I", orc.ORC_DIR,
                                       "-o", tmp] + SRCS)
                os.replace(tmp, so)
            L = C.CDLL(so)
            L.orc_clones.restype = C.c_int
            L.orc_clones.argtypes = [C.c_void_p] * 4 + [C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int64, C.c_void_p, C.c_void_p,
                                                                                                    C.c_int64, C.c_void_p]
            _lib = L
    return _lib


def clones(corpus, n):
    """corpus: tosemscan.Corpus (or anything with arena, off, len, ext)."""
    arena = np.ascontiguousarray(corpus.arena, np.uint8)
    off = np.ascontiguousarray(corpus.off, np.int32)
    length = np.ascontiguousarray(corpus.len, np.int32)
    ext = np.ascontiguousarray(corpus.ext, np.uint8)
    nf = len(length)
    p = orc._p
    cap = 0
    for _ in range(2):
        out = {"line_base": np.zeros(nf + 1, np.int64), "file_dup": np.zeros(max(nf, 1), np.uint32),
               "file_dup_assert": np.zeros(max(nf, 1), np.uint32), "class_base": np.zeros(cap + 1, np.int64),
               "class_len": np.zeros(max(cap, 1), np.uint32), "member": np.zeros(max(cap, 1), np.int64)}
        nc, nm = C.c_int64(), C.c_int64()
        rc = lib().orc_clones(p(arena), p(off), p(length), p(ext), nf, int(n), p(out["line_base"]), p(out["file_dup"]),
                              p(out["file_dup_assert"]), p(out["class_base"]), p(out["class_len"]), cap, C.byref(nc),
                              p(out["member"]), cap, C.byref(nm))
        if rc == -3:
            cap = max(nc.value, nm.value)
            continue
        if rc != 0:
            raise ValueError("orc_clones failed")
        out["file_dup"], out["file_dup_assert"] = out["file_dup"][:nf], out["file_dup_assert"][:nf]
        out["class_base"], out["class_len"], out["member"] = out["class_base"][:nc.value + 1], out["class_len"][:nc.value], out["member"][:nm.value]
        return out
    raise ValueError("orc_clones: capacity")


def py_clones(files, exts, n):
    """Section 15 over line contents (the line minus one trailing CR)."""
    content, flag, fid, base = [], [], [], [0]
    for f, (data, e) in enumerate(zip(files, exts)):
        for line in spec_ref.py_lines(data):
            content.append(line[:-1] if line.endswith(b"\r") else line)
            flag.append(spec_ref.py_is_assert_line(line, int(e)))
            fid.append(f)
        base.append(len(content))
    T = len(content)
    groups = {}                                              # window contents -> positions, ascending
    key = [None] * T
    for p in range(T):
        if p + n > base[fid[p] + 1] or all(not c for c in content[p:p + n]):
            continue
        key[p] = tuple(content[p:p + n])
        groups.setdefault(key[p], []).append(p)

    def ext_of(g):                                          # left-extendable
        preds = set()
        for q in g:
            if q == base[fid[q]] or key[q - 1] is None:
                return False
            preds.add(key[q - 1])
        return len(preds) == 1 and len(groups[preds.pop()]) == len(g)

    extendable = {k: len(g) >= 2 and ext_of(g) for k, g in groups.items()}
    covered = [False] * T
    class_base, class_len, member = [0], [], []
    for p in range(T):
        k = key[p]
        if k is None or len(groups[k]) < 2:
            continue
        for x in range(p, p + n):
            covered[x] = True
        if extendable[k] or groups[k][0] != p:
            continue
        r = 0
        while p + r + 1 < T and fid[p + r + 1] == fid[p] and key[p + r + 1] is not None and len(groups[key[p + r + 1]]) >= 2 \
                and extendable[key[p + r + 1]]:
            r += 1
        class_len.append(n + r)
        member += groups[k]
        class_base.append(len(member))
    nf = len(files)
    dup = [sum(covered[base[f]:base[f + 1]]) for f in range(nf)]
    dup_a = [sum(1 for x in range(base[f], base[f + 1]) if covered[x] and flag[x]) for f in range(nf)]
    return {"line_base": np.array(base, np.int64), "file_dup": np.array(dup, np.uint32), "file_dup_assert": np.array(dup_a, np.uint32),
            "class_base": np.array(class_base, np.int64), "class_len": np.array(class_len, np.uint32), "member": np.array(member, np.int64)}


KEYS = ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len", "member")


def assert_equal(got, want):
    for k in KEYS:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k


def c4_planted(seed, n_files, share=4):
    """Files of BASELINE config C4's size law (seeded), every `share`-th of them replaced by tsm_gen_edit (lambda = 6) of
    another, earlier file of the corpus: planted partial copies at a realistic scale.  Returns (files, exts)."""
    import tosemscan as ts
    c = ts.gen_corpus(seed, n_files, size_law=1, pinned=False)
    files = [c.file_bytes(i) for i in range(n_files)]
    rng = np.random.default_rng(seed)
    for i in range(share, n_files, share):
        files[i] = ts.gen_edit(seed + i, files[int(rng.integers(0, i))], 6.0)
    return files, c.ext.copy()


# ---------------------------------------------------------------------------------------------- windows with a chosen key
# finalise (SPEC section 3) is a bijection of 64 bits (xor-shifts and odd multiplies) and the n-gram sum is linear in the
# canonical line hashes, so a window's key can be chosen: invert finalise for the window, subtract the n - 1 given trailing
# lines, invert finalise for one length of the first line and solve for its 8 leading bytes.  This reaches what random keys
# reach only by luck: key 0 (the empty marker of the kernels' hash table), a chosen home slot, two contents with one key.
GOLDEN = 0x9E3779B97F4A7C15
FILLER = b"bcdfghjkmnpqrvwxyz0123456789"                  # no "assert", no "EXPECT_", no CR, no LF


def _unxorshift(x, s):
    y = x
    for _ in range(64 // s + 1):
        y = x ^ (y >> s)
    return y


def unmix(x, length):
    """The h61 with spec_ref.mix(h61, length) == x.  Only values below 2^61 - 1 are hashes of something."""
    x = _unxorshift(x, 31)
    x = x * pow(0x94D049BB133111EB, -1, 1 << 64) & spec_ref.MASK
    x = _unxorshift(x, 27)
    x = x * pow(0xBF58476D1CE4E5B9, -1, 1 << 64) & spec_ref.MASK
    x = _unxorshift(x, 30)
    return x ^ (length * GOLDEN & spec_ref.MASK)


def key_reachable(key, n):
    """Some window of n lines has this key (section 15.1)."""
    return unmix(key, n) < spec_ref.M61


def window_with_key(key, n, tail_lines, rng):
    """The n line contents (no LF) of a window whose key is `key`: a crafted first line (8 leading bytes solved for, then a
    filler drawn from rng, a random.Random), then tail_lines, n - 1 given non-empty contents without LF or trailing CR."""
    assert len(tail_lines) == n - 1
    acc = unmix(key, n)
    if acc >= spec_ref.M61:
        raise ValueError("no window of %d lines has the key %#x" % (n, key))
    M61 = spec_ref.M61
    rest = sum((spec_ref.py_bytes_hash(t) % M61) << (13 * k) for k, t in enumerate(tail_lines, 1)) % M61
    c0 = (acc - rest) % M61                                  # the first line's hash, mod 2^61 - 1
    shift = pow(256, 8, M61)
    for _ in range(1000):
        filler = bytes(rng.choice(FILLER) for _ in range(rng.randrange(4, 24)))
        for h in range(c0, 1 << 64, M61):                    # the line hashes that are c0 mod 2^61 - 1
            y = unmix(h, 8 + len(filler))
            if y >= M61:
                continue
            for f in range((y - int.from_bytes(filler, "little") * shift) % M61, 1 << 64, M61):
                head = f.to_bytes(8, "little")
                if b"\n" not in head:
                    return [head + filler] + list(tail_lines)
    raise AssertionError("no first line found")


def key_at_slot(slot, mask, n, rng):
    """A random non-zero key whose home slot (key & mask) is `slot` and that some window of n lines has."""
    while True:
        key = (rng.getrandbits(64) & ~mask) | slot
        if key and key_reachable(key, n):
            return key


def table_mask(total_lines):
    """The host's table size: slots = the smallest power of two >= 2 x the lines, mask = slots - 1 (key 0: slot mask + 1)."""
    slots = 1
    while slots < 2 * total_lines:
        slots <<= 1
    return slots - 1


def window_groups(corpus, n):
    """The grouping state of section 15 from the oracle's line hashes, per global line p: key[p] = ngram_n(p), valid[p] (a
    window starts at p), count[p] (the size of its group, 0 for no window) and ext[p] (its group is left-extendable);
    plus line_base and the distinct keys of the windows with their counts."""
    nf = len(corpus.len)
    res = orc.scan(corpus.arena, corpus.off, corpus.len, corpus.ext, np.zeros(nf, np.uint16), 1, events=False, line_hashes=True)
    base, lh = res["line_base"].astype(np.int64), res["line_hash"]
    T = len(lh)
    key = orc.ngram_hashes(lh, base, n)
    p = np.arange(T)
    fid = np.searchsorted(base, p, side="right") - 1
    nonempty = np.concatenate([[0], np.cumsum(lh != np.uint64(spec_ref.mix(0, 0)))])   # the hash of empty content
    valid = (p + n <= base[fid + 1]) & (nonempty[np.minimum(p + n, T)] > nonempty[p])
    pos = np.nonzero(valid)[0]
    keys, inv, cnt = np.unique(key[pos], return_inverse=True, return_counts=True)
    gid = np.full(T, -1, np.int64)
    gid[pos] = inv
    none = len(keys)                                         # the predecessor of a file's first line or of a non-window
    pred = np.full(T, none, np.int64)
    inner = pos[(pos > base[fid[pos]]) & (gid[np.maximum(pos - 1, 0)] >= 0)]
    pred[inner] = gid[inner - 1]
    lo, hi = np.full(none + 1, none, np.int64), np.full(none + 1, -1, np.int64)
    np.minimum.at(lo, inv, pred[pos])
    np.maximum.at(hi, inv, pred[pos])
    cnt1 = np.concatenate([cnt, [0]])
    ext_g = (cnt1 >= 2) & (lo == hi) & (lo != none) & (cnt1[np.minimum(lo, none)] == cnt1)
    count = np.zeros(T, np.int64)
    count[pos] = cnt[inv]
    ext = np.zeros(T, bool)
    ext[pos] = ext_g[inv]
    return {"line_base": base, "key": key, "valid": valid, "count": count, "ext": ext, "keys": keys, "counts": cnt}


def occupied_slots(keys, mask):
    """The slots that the distinct non-zero keys fill in a linear-probing table of mask + 1 slots.  The set does not depend
    on the insertion order (only which key sits where does)."""
    occ = np.zeros(mask + 1, bool)
    for k in sorted(set(int(k) for k in keys) - {0}):
        s = k & mask
        while occ[s]:
            s = (s + 1) & mask
        occ[s] = True
    return occ


def keys_that_can_reach(keys, mask, slot):
    """The keys that some insertion order places in `slot`: those whose home lies in the run of filled slots that ends at
    `slot` (empty when the slot stays empty)."""
    occ = occupied_slots(keys, mask)
    if not occ[slot]:
        return []
    run, s = {slot}, slot
    while occ[(s - 1) & mask] and (s - 1) & mask != slot:
        s = (s - 1) & mask
        run.add(s)
    return [int(k) for k in keys if k and (int(k) & mask) in run]


def text(lines):
    """File bytes of line contents, every line terminated."""
    return b"".join(ln + b"\n" for ln in lines)


SLOT0_KEYS, SLOT0_COPIES = 3, 4


def key0_corpus(case, n, seed):
    """Files (as line lists) around one content Z of n lines whose window key is 0 (reachable for n = 5, 13, 18, ...):
    'head'    Z + 4 lines three times, after different lines: a key-0 group heads a class that extends to the right, so the
              predecessor slot of the next group is the side slot;
    'middle'  3 lines + Z + 4 lines twice: the key-0 group is left-extendable (and the predecessor of the next group);
    'once'    Z once, between windows that occur twice;
    'wide'    Z in 40 files: a key-0 class of more than 32 fragments.
    After them SLOT0_KEYS keys homed at slot 0, SLOT0_COPIES one-window files each, so that slot 0 holds a key of another
    count.  Returns (files, mask)."""
    rng = random.Random(seed)
    Z = window_with_key(0, n, [b"z%d" % k for k in range(1, n)], rng)

    def u(tag, i, m=1):
        return [b"%s%d_%d" % (tag, i, k) for k in range(m)]
    if case == "head":
        files = [Z + u(b"x", 0, 4), u(b"a", 1) + Z + u(b"x", 0, 4), u(b"a", 2) + Z + u(b"x", 0, 4) + u(b"b", 2)]
    elif case == "middle":
        files = [u(b"a", i) + u(b"y", 0, 3) + Z + u(b"x", 0, 4) + u(b"b", i) for i in range(2)]
    elif case == "once":
        D = u(b"d", 0, n)
        files = [D + Z + u(b"e", 0, n), u(b"r", 0) + D[-1:] + Z[:-1] + u(b"r", 1), u(b"s", 0) + Z[1:] + u(b"e", 0, n)]
    else:
        assert case == "wide"
        files = [u(b"a", i) + Z + u(b"b", i) for i in range(40)]
    mask = table_mask(sum(len(f) for f in files) + SLOT0_KEYS * SLOT0_COPIES * n)
    for j in range(SLOT0_KEYS):
        files += [window_with_key(key_at_slot(0, mask, n, rng), n, [b"h%d_%d" % (j, k) for k in range(1, n)], rng)] * SLOT0_COPIES
    return files, mask


def probe_corpus(extra, seed, collide=True, n=3, chain=520, low=40, single=24):
    """One n-line file per window, so that every window's key is chosen: `chain` keys of two windows and `single` keys of one
    window homed at the last slot (mask), so that their probe chain wraps into slot 0 onward; keys of two windows homed at
    slots 0 .. low - 1, which collide with the wrapped chain; with `collide`, two windows of different content with one key
    homed at mask.  The files in a seeded order, then one file of empty lines (no windows) that pads the corpus to
    4 096 + extra lines: extra = 0 makes 2 x lines a power of two.  Returns (files, mask)."""
    rng = random.Random(seed)
    total = 4096 + extra
    mask = table_mask(total)

    def window(slot, tag):
        return window_with_key(key_at_slot(slot, mask, n, rng), n, [b"%s_%d" % (tag, k) for k in range(1, n)], rng)
    files = []
    for i in range(chain):
        files += [window(mask, b"c%d" % i)] * 2
    for i in range(low):
        files += [window(i, b"l%d" % i)] * 2
    files += [window(mask, b"s%d" % i) for i in range(single)]
    if collide:
        key = key_at_slot(mask, mask, n, rng)
        files += [window_with_key(key, n, [b"p%d_%d" % (j, k) for k in range(1, n)], rng) for j in range(2)]
    rng.shuffle(files)
    files.append([b""] * (total - n * len(files)))
    return files, mask
