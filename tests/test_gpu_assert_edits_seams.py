"""GPU tests of the assertion edits (docs/SPEC.md section 17) where the rest of the suite never reaches: the long path split
over several launches, long patterns with more than one round of 32 candidates, more short patterns than k_edit_score has
warps, carry chains across the 64-bit words of the bit-parallel LCS, every byte value, the exact threshold on the device,
the kept-list retry, batch independence and the raw ABI's edges.

Inputs too large for the O(nm) C reference (tests/orc_assert_edits.c) are built with an LCS known in closed form: b is a
with d interior bytes deleted (lcs = |a| - d), or with k interior bytes replaced by a byte that a does not contain
(lcs = |a| - k), or with k bytes inserted (lcs = |a|).  The `assert ` head and the last byte stay, so that b is still an
assertion line and a's stripped length is its length.  Every test checks `chg` against tsm_diff_pairs_asserts, the events
of the lines it built, and the edits against the closed form or the C reference or both; and it asserts that it reached
its seam (launch counts, entry counts against the grid's warps, exact scores)."""
import ctypes as C

import numpy as np
import pytest

import corpus_util as cu
import orc_assert_edits as oae
import tosemscan as ts
from test_gpu_assert_edits import TSM_E_ARG, sides

pytestmark = pytest.mark.gpu

HEAD = b"assert "
W = b" \t\r\x0b\x0c"
EDIT_SCRATCH = 1 << 25         # kEditScratch of csrc/tsm_api.cu: words of Peq and V slots per launch of the long path
EDIT_SHORT = 4 * 64            # EDIT_SHORT_WORDS * 64 of csrc/tsm_edit_kernels.cuh: longer patterns take the long path
EDIT_WARPS = 4                 # EDIT_WARPS of csrc/tsm_edit_kernels.cuh; k_edit_score runs at most sms * 16 blocks
MIN = 30000                    # EDIT_SCORE_MIN


def score(lcs, la, lb):
    return 120000 * lcs // (la + lb)


def slot_words(m):
    return 288 * ((m + 63) // 64)


def body(rng, n, alphabet):
    return rng.choice(np.frombuffer(alphabet, np.uint8), n).tobytes()


def line(rng, m, alphabet):
    return HEAD + body(rng, m - len(HEAD), alphabet)


def interior(rng, a, k):
    """k distinct interior positions of a: after the head, before the last byte."""
    assert k <= len(a) - len(HEAD) - 1
    return len(HEAD) + rng.choice(len(a) - len(HEAD) - 1, k, replace=False)


def deletion(rng, a, d):
    """(a with d interior bytes deleted, its score against a): lcs = |a| - d."""
    keep = np.ones(len(a), bool)
    keep[interior(rng, a, d)] = False
    return np.frombuffer(a, np.uint8)[keep].tobytes(), score(len(a) - d, len(a), len(a) - d)


def substitution(rng, a, k, z):
    """(a with k interior bytes replaced by z, which a does not contain, its score against a): lcs = |a| - k."""
    assert z not in a and z not in W and z != 10
    b = np.frombuffer(a, np.uint8).copy()
    b[interior(rng, a, k)] = z
    return b.tobytes(), score(len(a) - k, len(a), len(a))


class Batch:
    """Revision pairs built hunk by hunk between unique kept lines, with the events and the edits they must give."""

    def __init__(self):
        self.olds, self.news = [], []
        self.pos = ([], [])          # (pair, line start) of every deleted / inserted assertion line, in event order
        self.want = []               # (rev, aev, score) of every edit, in the greedy's terms

    def add(self, hunks, lead=(b"", b""), end=b"\n"):
        """hunks: [(deleted lines, inserted lines, [(i, j, score)])], every line an assertion line; lead: indentation of the
        old / new lines.  end: the ending of both sides' last line (b"": an unterminated last line, with no kept line
        after the last hunk)."""
        p = len(self.olds)
        out = ([b"p%d_head\n" % p], [b"p%d_head\n" % p])
        at = [len(out[0][0]), len(out[1][0])]
        for h, (dl, il, ed) in enumerate(hunks):
            r0, a0 = len(self.pos[0]), len(self.pos[1])
            last = h == len(hunks) - 1 and end != b"\n"
            for s, lines in ((0, dl), (1, il)):
                for q, x in enumerate(lines):
                    t = lead[s] + x + (end if last and q == len(lines) - 1 else b"\n")
                    self.pos[s].append((p, at[s]))
                    out[s].append(t)
                    at[s] += len(t)
                if not last:
                    k = b"p%d_kept%d\n" % (p, h)
                    out[s].append(k)
                    at[s] += len(k)
            self.want += [(r0 + i, a0 + j, sc) for i, j, sc in ed if sc >= MIN]
        self.olds.append(b"".join(out[0]))
        self.news.append(b"".join(out[1]))

    def packed(self, sel=None):
        sel = range(len(self.olds)) if sel is None else sel
        o, n = [self.olds[i] for i in sel], [self.news[i] for i in sel]
        return ts.pack(o, [1] * len(o)), ts.pack(n, [1] * len(n))

    def edits(self):
        w = sorted(self.want, key=lambda e: e[1])
        out = np.zeros(len(w), ts.ASSERT_EDIT)
        if w:
            out["rev"], out["aev"], out["score"] = zip(*w)
        return out


def run(sc, a, b, dist=None, ref=True):
    """(result of diff_assert_edits, launches of its edit part).  chg equals tsm_diff_pairs_asserts; with ref the edits equal
    the C reference.  The edit part of the launch count is (short patterns ? 1 : 0) + long launches, per attempt: the rest
    of the call is tsm_diff_pairs_asserts' count plus 8 + 1 launches per side (kept ranks, entry index, compaction)."""
    got = sc.diff_assert_edits(a, b)
    n_edits = sc.last_launch_count()
    want = sc.diff_pairs(a, b, asserts=True)
    n_chg = sc.last_launch_count()
    for g, w in zip(got[:7], want):
        assert g.dtype == w.dtype and np.array_equal(g, w)
    if ref:
        r = oae.assert_edits(*sides(a, b), dist)
        assert np.array_equal(got[7], r), (got[7][:5], r[:5])
    return got, n_edits - n_chg - 18


def check_built(got, bt):
    """The lines the batch built are the changed assertion lines of traced pairs (the events), and the edits are the
    closed form's."""
    aev, rev, ed = got[5], got[6], got[7]
    for ev, pos in ((rev, bt.pos[0]), (aev, bt.pos[1])):
        want = np.array(pos, np.int64).reshape(-1, 2)
        assert len(ev) == len(want)
        assert np.array_equal(ev["file"], want[:, 0]) and np.array_equal(ev["line_off"], want[:, 1])
    w = bt.edits()
    assert np.array_equal(ed[["rev", "aev", "score"]], w[["rev", "aev", "score"]]), (ed[:5], w[:5])


# ---------------------------------------------------------------------------------------------- 1. long-path launch split
def test_long_path_launch_split():
    """640 1x1 hunks with 16 KiB patterns: 73 728-word slots, 455 per launch of 2^25 words, so two launches and the slots
    of the second start at 0 again.  Deletions and substitutions on both sides of 30 000, the exact threshold among them;
    the new line of the last pair is the unterminated last line of its arena.  The patterns of the first launch use one
    alphabet, those of the second another, and the second's substitutions put a byte of the first's alphabet into the
    text: Peq bits left in a slot by the first launch would raise those scores."""
    rng = np.random.default_rng(1)
    m, n = 16383, 640
    per = EDIT_SCRATCH // slot_words(m)
    assert slot_words(m) == 73728 and per == 455 and n > per
    xs, ys = b"bcdfghijklmnopqu", b"vwxyz0123456789_=()"
    amounts = [("d", 1), ("d", 3000), ("s", 4000), ("d", 10922), ("d", 10923), ("s", 8191), ("s", 8192), ("d", 12000),
               ("s", 6000), ("d", 16000)]
    bt, small, scores = Batch(), Batch(), []
    sub = (3, 4, n - 1)                                   # the exact threshold, just below it, and the arena's end
    for p in range(n):
        a = line(rng, m, xs if p < per else ys)
        kind, x = amounts[p % len(amounts)]
        b, s = deletion(rng, a, x) if kind == "d" else substitution(rng, a, x, ord("Z") if p < per else xs[p % len(xs)])
        scores.append(s)
        for t in (bt, small) if p in sub else (bt,):
            t.add([([a], [b], [(0, 0, s)])], end=b"" if p == n - 1 else b"\n")
    assert scores[3] == MIN > scores[4] and min(scores) < MIN < max(scores)
    assert not bt.news[-1].endswith(b"\n")
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = bt.packed()
    got, launches = run(sc, a, b, ref=False)
    check_built(got, bt)
    assert launches == -(-n // per) >= 2
    assert sum(s >= MIN for s in scores) == len(got[7]) > n // 2
    a, b = small.packed()                                 # the C reference where it is cheap
    check_built(run(sc, a, b)[0], small)
    sc.close()


# ---------------------------------------------------------------------------------------------- 2. more than 32 candidates
POOL = bytes(c for c in range(1, 256) if c not in b"\n \t\r\x0b\x0casertZ")


def alphabets(k):
    """k disjoint 3-byte alphabets, none with a byte of the head or Z: lines over two of them share the head only."""
    assert 3 * k <= len(POOL)
    return [POOL[3 * i:3 * i + 3] for i in range(k)]


def test_long_patterns_with_more_than_32_candidates():
    """70 x 70 hunks with patterns of 257, 320, 321, 1 024 and 4 097 bytes: three rounds of the warp loop per pattern.
    Inserted line j is a closed-form edit of deleted line pi(j); the deleted lines use disjoint alphabets, so every other
    candidate has lcs 7 (the head), far below 50 %.  And 1 x 70 hunks whose candidates have distinct known scores, the best
    one in the second or third round: the greedy pass takes it."""
    rng = np.random.default_rng(2)
    abcs = alphabets(70)
    bt, small = Batch(), Batch()                          # small: the hunks cheap enough for the C reference
    for m in (257, 320, 321, 1024, 4097):
        olds = [line(rng, m, abcs[i]) for i in range(70)]
        pi = rng.permutation(70)
        news, ed = [], []
        for j in range(70):
            i = int(pi[j])
            x = 1 + (j * 7) % max(2, m // 4)
            b, s = deletion(rng, olds[i], x) if j % 2 else substitution(rng, olds[i], x, ord("Z"))
            assert s >= MIN
            news.append(b)
            ed.append((i, j, s))
        assert score(len(HEAD), m, max(len(x) for x in news)) < MIN     # every other candidate
        for t in (bt, small) if m == 257 else (bt,):
            t.add([(olds, news, ed)])
    for m, best in ((257, 45), (320, 66), (321, 33), (1024, 40), (4097, 69)):
        a = line(rng, m, abcs[0])
        ds = rng.permutation(np.arange(2, 2 + 69 * max(1, m // 100), max(1, m // 100)))[:69]
        ds = np.insert(ds, best, 1)
        news, scs = [], []
        for d in ds.tolist():
            b, s = deletion(rng, a, d)
            news.append(b)
            scs.append(s)
        assert int(np.argmax(scs)) == best and sorted(scs)[-2] < scs[best]
        for t in (bt, small) if m <= 1024 else (bt,):
            t.add([([a], news, [(0, best, scs[best])])])
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = bt.packed()
    got, launches = run(sc, a, b, ref=False)
    check_built(got, bt)
    assert launches == 1 and len(got[7]) == 5 * 70 + 5
    a, b = small.packed()
    check_built(run(sc, a, b)[0], small)
    sc.close()


# ---------------------------------------------------------------------------------------------- 3. persistent-warp reuse
def test_persistent_warps_reuse_their_peq():
    """More than twice as many short patterns as k_edit_score has warps, in 1 x 1 and 1 x 3 hunks: every warp clears and
    refills its Peq for at least two more patterns.  A warp's next pattern (entry t + warps) has another word count and
    the other alphabet, and its text carries bytes of the previous pattern's alphabet (substitutions), so that Peq bits left
    from it would raise the score."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = sms * 16 * EDIT_WARPS
    n_pat = 2 * warps + 700
    rng = np.random.default_rng(3)
    xy = (b"bcdfghij", b"klmnopqu")
    lens = ((12, 64), (65, 128), (129, EDIT_SHORT))
    bt, hunks, n_cand = Batch(), [], 0
    for t in range(n_pat):
        rnd = t // warps
        lo, hi = lens[(t + rnd) % 3]
        own, other = xy[rnd % 2], xy[1 - rnd % 2]
        a = line(rng, int(rng.integers(lo, hi + 1)), own)
        m = len(a)
        z = other[t % 8]
        if t % 4 == 3:                                   # 1 x 3: distinct scores, the best taken
            ks = sorted(rng.choice(np.arange(1, max(4, m // 3)), 3, replace=False).tolist())
            order = rng.permutation(3)
            news = [None] * 3
            for r, k in zip(order.tolist(), ks):
                news[r], s = substitution(rng, a, k, z)
                if k == ks[0]:
                    best = (0, r, s)
            hunks.append(([a], news, [best]))
            n_cand += 3
        else:
            x = int(rng.integers(1, max(2, (m - 8) * 3 // 5)))
            b, s = substitution(rng, a, min(x, m - 8), z) if t % 2 else deletion(rng, a, min(x, m - 8))
            hunks.append(([a], [b], [(0, 0, s)]))
            n_cand += 1
        if len(hunks) == 200:
            bt.add(hunks)
            hunks = []
    bt.add(hunks)
    assert len(bt.pos[0]) == n_pat >= 2 * warps
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = bt.packed()
    got, launches = run(sc, a, b)
    check_built(got, bt)
    assert launches == 1 and len(got[6]) == n_pat and len(got[5]) == n_cand
    assert (got[7]["score"] < 60000).all() and len(got[7]) > n_pat // 2
    sc.close()


# ---------------------------------------------------------------------------------------------- 4. carry chains
def straddling(n):
    """A body of n bytes: b with runs of a over positions 56-72, 120-136 and 184-200 of the line (bits 63/64, 127/128,
    191/192 of the pattern)."""
    x = bytearray(b"b" * n)
    for lo in (56, 120, 184):
        for q in range(lo, lo + 17):
            if len(HEAD) <= q < len(HEAD) + n:
                x[q - len(HEAD)] = ord("a")
    return bytes(x)


STYLES = {"a": lambda n: b"a" * n, "ab": lambda n: (b"ab" * n)[:n], "aab": lambda n: (b"aab" * n)[:n],
          "ba": lambda n: (b"ba" * n)[:n], "straddle": straddling}


def test_carry_chains_across_words():
    """One- and two-letter bodies (the longest add carries) at pattern lengths 64w - 1, 64w, 64w + 1 for w = 1, 2, 4 and
    257, 320, 1 024 on the long path, against texts shorter and longer than the pattern: the C reference."""
    bt = Batch()
    for m in (63, 64, 65, 127, 128, 129, 255, 256, 257, 320, 1024):
        for ps in ("a", "ab", "aab", "straddle"):
            a = HEAD + STYLES[ps](m - len(HEAD))
            for ts_, dn in ((ps, -40), (ps, -1), (ps, 1), (ps, 40), ("a", 3), ("ba", -2), ("straddle", 0), ("aab", 64)):
                n = m + dn
                b = HEAD + STYLES[ts_](n - len(HEAD))
                if n > len(HEAD) and b != a:
                    bt.add([([a], [b], [])])
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = bt.packed()
    got, launches = run(sc, a, b)
    assert launches == 2 and len(got[6]) == len(bt.olds)
    assert len(got[7]) > 0.7 * len(bt.olds) and (got[7]["score"] < 60000).sum() > 0.5 * len(got[7])
    sc.close()


# ---------------------------------------------------------------------------------------------- 5. every byte value
def test_every_byte_value():
    """Bodies of bytes 0x00 - 0xFF (no LF) with interior tab, VT, FF and CR, inside leading and trailing runs that mix all
    five W bytes, with LF, CRLF and unterminated endings: the C reference."""
    rng = np.random.default_rng(5)
    anyb = bytes(c for c in range(256) if c != 10)
    bt = Batch()
    for p in range(240):
        m = [12, 40, 63, 64, 65, 100, 129, 200, 256, 257, 700, 1500][p % 12]
        core = bytearray(line(rng, m, anyb))
        for q in interior(rng, bytes(core), min(4, m - 8)):
            core[q] = b"\t\x0b\x0c\r"[q % 4]
        core[-1] = 0x80 + p % 128                          # not W: the stripped line ends here
        new = bytearray(core)
        for q in interior(rng, bytes(core), max(1, m // 10)):
            new[q] = anyb[int(rng.integers(len(anyb)))]
        if new == core:
            new[len(HEAD)] ^= 1
        runs = [bytes(rng.permutation(np.frombuffer(W * 2, np.uint8))) for _ in range(4)]
        end = (b"\n", b"\r\n", b"")[p % 3]
        bt.add([([runs[0] + bytes(core) + runs[1]], [runs[2] + bytes(new) + runs[3]], [])], end=end)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = bt.packed()
    got, launches = run(sc, a, b)
    assert launches == 2 and len(got[6]) == len(bt.olds) and len(got[7]) > 200
    files = [bt.olds[int(got[6]["file"][e])] for e in got[7]["rev"]]
    assert sum(b"\0" in x for x in files) > 20
    sc.close()


# ---------------------------------------------------------------------------------------------- 6. exact threshold
@pytest.mark.parametrize("m", [63, 64, 126, 128, 255, 256, 258, 1023, 1024])
def test_exact_threshold_on_the_device(m):
    """Deletions with 3d = 2m (score exactly 30 000: kept) and 3d = 2m + 3 (below), substitutions with k = m / 2 and
    m / 2 + 1, on the register paths of 1, 2 and 4 words and the long path."""
    rng = np.random.default_rng(m)
    bt, want = Batch(), []
    a = line(rng, m, b"bcdfghijklmnop")
    if m % 3 == 0:
        for d in (2 * m // 3, (2 * m + 3) // 3):
            b, s = deletion(rng, a, d)
            want.append(s)
            bt.add([([a], [b], [(0, 0, s)])])
    if m % 2 == 0:
        for k in (m // 2, m // 2 + 1):
            b, s = substitution(rng, a, k, ord("Z"))
            want.append(s)
            bt.add([([a], [b], [(0, 0, s)])])
    assert want[0] == MIN and want[1] < MIN and len(want) in (2, 4)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    x, y = bt.packed()
    got, launches = run(sc, x, y)
    check_built(got, bt)
    assert launches == 1
    assert got[7]["score"].tolist() == [MIN] * (len(want) // 2)
    sc.close()


# ---------------------------------------------------------------------------------------------- 7. kept-list retry
def indented(k, text, old=True):
    return [(b"    " if old else b"  ") + text] * k


@pytest.mark.parametrize("shape", ["64x64", "65x64", "short+long"])
def test_kept_list_retry(shape):
    """Hunks of identical assertion lines that differ from the other side only in indentation: every candidate of the same
    text scores 60 000.  The first list holds max(4096, no + nn) = 4096: at 64 x 64 exactly full (no retry), at 65 x 64
    one over (retry); short and long lines together overflow it with both score kernels appending."""
    s_ = b"assert x == 1"
    l_ = b"assert " + b"".join(b"v_%03d == 1 and " % i for i in range(20)) + b"done"
    if shape == "64x64":
        dl, il, per_attempt, nk = indented(64, s_), indented(64, s_, False), 1, 64 * 64
    elif shape == "65x64":
        dl, il, per_attempt, nk = indented(65, s_), indented(64, s_, False), 1, 65 * 64
    else:
        dl = indented(50, s_) + indented(40, l_)
        il = indented(50, s_, False) + indented(40, l_, False)
        per_attempt, nk = 2, 50 * 50 + 40 * 40
        assert len(l_) > EDIT_SHORT >= len(s_) and score(len(s_), len(s_), len(l_)) < MIN
    cap = max(4096, len(dl) + len(il))
    assert (nk == cap) == (shape == "64x64") and nk >= cap
    k = min(len(dl), len(il))
    bt = Batch()
    bt.add([([x.lstrip() for x in dl], [x.lstrip() for x in il], [(i, i, 60000) for i in range(k)])], lead=(b"    ", b"  "))
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = bt.packed()
    got, launches = run(sc, a, b)
    check_built(got, bt)
    assert launches == per_attempt * (1 if nk <= cap else 2)
    sc.close()


# ---------------------------------------------------------------------------------------------- 8. batch independence
def c5_files():
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    return [a.file_bytes(i) for i in range(a.n_files)], [b.file_bytes(i) for i in range(b.n_files)], a.ext.tolist()


def dense(olds, exts):
    """New sides built from the old ones: every assertion line (section 4, Rev A) with 2m - 2 to 2m + 2 bytes inserted
    before the last byte of its stripped text (lcs = m, score 120000 m / (4m + delta): around 30 000)."""
    news = []
    for f, (o, e) in enumerate(zip(olds, exts)):
        out = []
        for q, x in enumerate(o.split(b"\n")):
            s = x.strip(W)
            if e and len(s) > 1 and (b"assert" in x.lower() or b"EXPECT_" in x):
                z = next(c for c in b"~|`^" if c not in s)
                i = x.index(s) + len(s) - 1
                x = x[:i] + bytes([z]) * (2 * len(s) + (f + q) % 5 - 2) + x[i:]
            out.append(x)
        news.append(b"\n".join(out))
    return news


def shifted(got, lo, r0, a0):
    ed = got[7].copy()
    ed["rev"] += r0
    ed["aev"] += a0
    evs = []
    for ev in got[5], got[6]:
        ev = ev.copy()
        ev["file"] += lo
        evs.append(ev)
    return evs[0], evs[1], ed


@pytest.mark.parametrize("corpus", ["c5", "dense"])
def test_batch_independence_and_determinism(corpus):
    """The 50 000 C5 pairs, and the pairs of their old sides with every assertion line edited near 50 %: the same bytes on
    a second call; three uneven batches concatenated equal the whole batch (the first one, 7 001 pairs, also equals the C
    reference on the dense pairs); the pairs in reverse order give the same edits after remapping."""
    olds, news, exts = c5_files()
    if corpus == "dense":
        news = dense(olds, exts)
    n = len(olds)
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    whole, _ = run(sc, a, b, ref=False)
    ed = whole[7]
    if corpus == "dense":
        near = np.abs(ed["score"].astype(np.int64) - MIN) < 300
        assert len(ed) > 20000 and near.sum() > 5000 and (ed["score"] == MIN).sum() > 500
    again = sc.diff_assert_edits(a, b)
    for x, y in zip(again, whole):
        assert x.tobytes() == y.tobytes()
    parts, r0, a0 = [], 0, 0
    for lo, hi in ((0, 7001), (7001, 31000), (31000, n)):
        x, y = ts.pack(olds[lo:hi], exts[lo:hi]), ts.pack(news[lo:hi], exts[lo:hi])
        got = run(sc, x, y, ref=corpus == "dense")[0] if lo == 0 else sc.diff_assert_edits(x, y)
        parts.append(shifted(got, lo, r0, a0))
        r0, a0 = r0 + len(got[6]), a0 + len(got[5])
    for k, want in enumerate((whole[5], whole[6], ed)):
        assert np.array_equal(np.concatenate([p[k] for p in parts]), want)
    back = sc.diff_assert_edits(ts.pack(olds[::-1], exts[::-1]), ts.pack(news[::-1], exts[::-1]))
    maps = []
    for ev_b, ev_w in ((back[6], whole[6]), (back[5], whole[5])):
        ev_b = ev_b.copy()
        ev_b["file"] = n - 1 - ev_b["file"].astype(np.int64)
        key_b = ev_b["file"].astype(np.int64) << 32 | ev_b["line_off"]
        key_w = ev_w["file"].astype(np.int64) << 32 | ev_w["line_off"]
        idx = np.searchsorted(key_w, key_b)                 # whole's events are in (file, line) order
        assert np.array_equal(ev_w[idx], ev_b)
        maps.append(idx)
    red = np.zeros(len(back[7]), ts.ASSERT_EDIT)
    red["rev"], red["aev"], red["score"] = maps[0][back[7]["rev"]], maps[1][back[7]["aev"]], back[7]["score"]
    assert np.array_equal(np.sort(red, order="aev"), ed)
    sc.close()


# ---------------------------------------------------------------------------------------------- 9. raw ABI
def raw(sc, a, b, edits, cap):
    ca, cb = a.c_struct(), b.c_struct()
    n = a.n_files
    big = 1 << 18
    ac, rc_ = np.zeros((1, ts.K), np.int64), np.zeros((1, ts.K), np.int64)
    aev, rev = np.zeros(big, ts.ASSERT_EVENT), np.zeros(big, ts.ASSERT_EVENT)
    r = ts._DiffAsserts(ts._p(ac), ts._p(rc_), ts._p(aev), big, 0, ts._p(rev), big, 0)
    ne = C.c_int64(-7)
    rc = ts.lib().tsm_diff_pairs_assert_edits(sc._ctx, C.byref(ca), C.byref(cb), ts._p(np.zeros(n, np.int64)),
                                              ts._p(np.zeros(n, np.int64)), None, C.byref(r), edits, cap, C.byref(ne), None)
    return rc, r.n_aev, r.n_rev, ne.value


def test_raw_abi_edges():
    """edits NULL with a large enough edit_cap (TSM_E_ARG, after every count is set); a batch whose pairs are all untraced;
    traced pairs with deleted assertion lines and no inserted ones, and the converse (one side has no entry: no scoring)."""
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    a, b = ts.gen_pairs(0x7053454D0005, 2000, pinned=False)
    full = sc.diff_assert_edits(a, b)
    assert len(full[7]) > 0
    assert raw(sc, a, b, None, 1 << 20) == (TSM_E_ARG, len(full[5]), len(full[6]), len(full[7]))
    assert raw(sc, a, b, None, 0)[0] == ts.TSM_E_CAPACITY
    olds, news, dist = [], [], {}
    for i, s in enumerate((((11585,), (11585,)), ((11584,), (11585,)))):
        o, nw, w = cu.block_pair(b"U%d" % i, *s, assert_every=3)
        olds.append(o); news.append(nw)
        dist[i] = len(w[3]) + len(w[4])
    assert sorted(dist.values()) == [23169, 23170]
    got, launches = run(sc, ts.pack(olds, [1, 1]), ts.pack(news, [1, 1]), dist)
    assert (got[2]["added_assert"] == -1).all() and got[5].size == got[6].size == got[7].size == 0 and launches == 0
    olds = [b"k%d\nassert x_%d == 1\nassert y_%d\nz\n" % (i, i, i) for i in range(30)]
    news = [b"k%d\nx_%d = 1\nz\n" % (i, i) for i in range(30)]
    for o, n_, what in ((olds, news, 6), (news, olds, 5)):
        got, launches = run(sc, ts.pack(o, [1] * 30), ts.pack(n_, [1] * 30))
        assert len(got[what]) == 60 and len(got[11 - what]) == 0 and got[7].size == 0 and launches == 0
    sc.close()
