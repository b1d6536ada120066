"""GPU tests of the moved code (docs/SPEC.md section 20): tsm_diff_pairs_moves against tsm_diff_pairs_marks and the numpy
reference tests/orc_moves.py (serial marks, the oracle's hashes) on the C5 pairs in steps of 1, 7 and 50 pairs and in one step,
planted moves inside and across steps, a duplicate-heavy step, runs of 1 to 70 000 lines, untraced pairs, every diff kernel's
shapes and reach ties; then capacity retries, NULL outputs, an empty batch, a bad step and a non-blocking stream."""
import ctypes as C
import random

import numpy as np
import pytest

import corpus_util as cu
import orc_moves as omv
import spec_ref as sr
import tosemscan as ts

pytestmark = pytest.mark.gpu


def stepped(c, steps):
    """Corpus c with the step of every pair as its grp."""
    steps = np.asarray(steps if steps is not None else np.zeros(c.n_files), np.uint16)
    return ts.Corpus(c.arena, c.off, c.len, c.ext, grp=steps, n_groups=int(steps.max()) + 1 if len(steps) else 1, keep=c._keep)


def sides(a, b):
    return (a.arena, a.off, a.len, a.ext), (b.arena, b.off, b.len, b.ext)


def check(sc, a, b, steps=None, dist=None, stream=None, cap=None, marks=None):
    """Every output equals tsm_diff_pairs_marks (bit 0) and the reference; returns the result."""
    a, b = stepped(a, steps), stepped(b, steps)
    r = sc.diff_moves(a, b, stream=stream, cap=cap)
    add, rem, det, bo, bn, dl, ins = sc.diff_marks(a, b)
    assert np.array_equal(r["added"], add) and np.array_equal(r["removed"], rem) and np.array_equal(r["detail"], det)
    assert np.array_equal(r["line_base_old"], bo) and np.array_equal(r["line_base_new"], bn)
    assert np.array_equal(r["dels"] & 1, dl) and np.array_equal(r["ins"] & 1, ins)
    wbo, wbn, wdl, wins, wob, wnb = omv.diff_moves(*sides(a, b), steps, dist, marks)
    for k, want in (("dels", wdl), ("ins", wins), ("old_blocks", wob), ("new_blocks", wnb)):
        got = r[k]
        assert len(got) == len(want), (k, len(got), len(want))
        if k.endswith("blocks"):
            got, want = got.tolist(), want.tolist()
            bad = [i for i, (x, y) in enumerate(zip(got, want)) if x != y]
            assert not bad, "%s differs at %s: %s vs %s" % (k, bad[:3], [got[i] for i in bad[:3]], [want[i] for i in bad[:3]])
        else:
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, "%s differs at %s: %s vs %s" % (k, bad[:3], got[bad[:3]], want[bad[:3]])
    return r


def test_moves_c5_steps():
    """All 50 000 pairs of BASELINE config C5 in steps of 1, 7 and 50 pairs; 3 000 of them in one step (the reference enumerates
    every matching pair of a step, and one step of all 50 000 holds too many for it)."""
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    marks = omv.serial_marks(*sides(a, b))
    for k in (1, 7, 50):
        check(sc, a, b, [i // k for i in range(a.n_files)], marks=marks)
    a, b = ts.gen_pairs(0x7053454D0005, 3_000, pinned=False)
    check(sc, a, b, [0] * a.n_files)
    sc.close()


def test_moves_c5_one_step():
    """All 50 000 C5 pairs in one step, as `diff` puts a whole tree pair (too many matching pairs for the reference): bit 0 of the
    marks equals tsm_diff_pairs_marks, the moved lines are exactly the lines of the blocks, blocks are in line order inside one run
    with at least 20 alphanumerics, and every block line hashes as the partner's line at the same offset."""
    a, b = ts.gen_pairs(0x7053454D0005, 50_000, pinned=False)
    a, b = stepped(a, [0] * a.n_files), stepped(b, [0] * b.n_files)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = sc.diff_moves(a, b)
    _, _, _, bo, bn, dl, ins = sc.diff_marks(a, b)
    assert np.array_equal(r["dels"] & 1, dl) and np.array_equal(r["ins"] & 1, ins)
    hashes = [sc.line_hashes(c)[1] for c in (a, b)]
    alnum = np.zeros(256, np.int64)
    alnum[[c for c in range(256) if chr(c).isalnum() and c < 128]] = 1
    for s, (key, mk) in enumerate((("old_blocks", r["dels"]), ("new_blocks", r["ins"]))):
        blk = r[key]
        assert len(blk) > 0 and np.all(np.diff(blk["line"]) > 0) and np.all(blk["line"][1:] >= blk["line"][:-1] + blk["n_lines"][:-1])
        moved = np.zeros(len(mk), bool)
        at = np.repeat(blk["line"], blk["n_lines"]) + (np.arange(blk["n_lines"].sum()) - np.repeat(np.cumsum(blk["n_lines"]) - blk["n_lines"], blk["n_lines"]))
        moved[at] = True
        assert np.array_equal(moved, (mk & 2) != 0) and np.all(mk[at] == 3)
        other = np.repeat(blk["partner"], blk["n_lines"]) + (at - np.repeat(blk["line"], blk["n_lines"]))
        assert np.array_equal(hashes[s][at], hashes[1 - s][other])
        corp = a if s == 0 else b
        base = bo if s == 0 else bn
        for x, n in zip(blk["line"][:200].tolist(), blk["n_lines"][:200].tolist()):   # alnum >= 20 on a sample
            f = int(np.searchsorted(base, x, "right") - 1)
            lines = corp.file_bytes(f).split(b"\n")[x - base[f]:x - base[f] + n]
            assert sum(int(alnum[list(l)].sum()) if l else 0 for l in lines) >= 20
    sc.close()


def planted(seed, n_pairs, step):
    """C5-like pairs with moves planted between the pairs of each step of `step` pairs: a stretch of a new side cut out and
    put into another pair's new side of the same step, and the same stretch put into a pair of the next step too (where nothing
    deletes it: it must not match)."""
    a, b = ts.gen_pairs(seed, n_pairs, pinned=False)
    olds = [a.file_bytes(i) for i in range(n_pairs)]
    news = [b.file_bytes(i).splitlines(keepends=True) for i in range(n_pairs)]
    rng = random.Random(seed)
    for s0 in range(0, n_pairs - step, step):
        p, q = s0 + rng.randrange(step), s0 + rng.randrange(step)
        if p == q or len(news[p]) < 12:
            continue
        k = rng.randrange(0, len(news[p]) - 10)
        m = rng.choice((1, 2, 3, 5, 8))
        cut = news[p][k:k + m]
        del news[p][k:k + m]
        at = rng.randrange(len(news[q]) + 1)
        news[q][at:at] = cut
        r = s0 + step + rng.randrange(step)
        news[r][:0] = cut
    return olds, [b"".join(n) for n in news], [int(x) for x in a.ext]


def test_moves_planted():
    olds, news, exts = planted(0x7053454D0020, 4_000, 8)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, exts), ts.pack(news, exts), [i // 8 for i in range(len(olds))])
    assert len(r["old_blocks"]) > 100 and len(r["new_blocks"]) > 100
    sc.close()


def test_moves_duplicate_heavy_step():
    """2 000 blank and 2 000 `}` lines per side in one step, among unique lines, every line changed."""
    def side(tag):
        return b"".join(b"%s_%d = compute_%d(x)\n\n}\n" % (tag, i, i) for i in range(2_000))
    olds = [side(b"a"), b"", b"keep\n"]
    news = [b"", side(b"b"), b"keep\n" + side(b"a")[:6000]]
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, [1, 1, 1]), ts.pack(news, [1, 1, 1]))
    assert len(r["new_blocks"]) > 0
    sc.close()


def test_moves_run_lengths():
    """Runs of 1, 31, 32, 33 and 70 000 lines moved between the pairs of one step (the lane walk of k_move_reach ends at 32), a
    70 000-line whole-file move, and a 70 000-line run whose every line matches but no block forms (its walk takes 70 000
    steps)."""
    olds, news = [], []
    for k in (1, 31, 32, 33, 70_000):
        run = [b"moved_%d_line_%d\n" % (k, j) for j in range(k)]
        olds += [b"head_%d\n" % k + b"".join(run) + b"tail_%d\n" % k, b"dst_%d_a\ndst_%d_b\n" % (k, k)]
        news += [b"head_%d\ntail_%d\n" % (k, k), b"dst_%d_a\n" % k + b"".join(run) + b"dst_%d_b\n" % k]
    whole = b"".join(b"    self.assertEqual(value_%d, other_%d)\n" % (j, j) for j in range(70_000))
    olds += [whole, b""]
    news += [b"", whole]
    lines = [b"m%05d\n" % j for j in range(70_000)]
    swapped = [lines[j ^ 1] for j in range(70_000)]
    olds += [b"".join(lines), b""]
    news += [b"", b"".join(swapped)]
    exts = [1] * len(olds)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, exts), ts.pack(news, exts))
    assert {31, 32, 33, 70_000} <= set(r["old_blocks"]["n_lines"].tolist())
    assert (r["new_blocks"]["n_assert"] == 70_000).sum() == 1
    sc.close()


def test_moves_untraced_pairs():
    """Distances 23 169 and 23 170, just above the trace limit, between traced pairs: the whole middle is changed, and lines of it
    move to a traced pair."""
    olds, news, dist = [], [], {}
    for i, (ko, kn) in enumerate(((3, 2), (11585, 11584), (4, 5), (11585, 11585), (2, 2))):
        o, n, _ = cu.block_pair(b"u%d" % i, [ko], [kn])
        olds.append(o); news.append(n)
        dist[i] = ko + kn
    o1 = olds[1].splitlines(keepends=True)
    news[0] = news[0] + b"".join(o1[100:110])
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, [1] * 5), ts.pack(news, [1] * 5), dist={**dist, 0: None})
    assert (r["detail"]["added_assert"] == -1).sum() == 2 and len(r["new_blocks"]) >= 1
    sc.close()


def test_moves_every_kernel():
    """Tie-heavy pairs at every k_diff_small size and left over to k_myers_trace, in steps of 5 pairs."""
    olds, news, exts = cu.tie_heavy_pairs(11, scale=2)
    d = [sum(sr.py_diff_files(o, n, x, x)[:2]) for o, n, x in zip(olds, news, exts)]
    assert max(d) > 127 and any(0 < x <= 31 for x in d)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    check(sc, ts.pack(olds, exts), ts.pack(news, exts), [i // 5 for i in range(len(olds))])
    assert sc.diff_last_ms()[2] > 0
    sc.close()


def test_moves_reach_ties():
    """A deleted run that two inserted runs match equally far, and one that repeats inside one inserted run: the partner is the
    smallest line."""
    blk = [b"    self.assertEqual(tie_value_%d, expected)\n" % j for j in range(3)]
    olds = [b"o0\n" + b"".join(blk) + b"o1\n", b"p0\np1\n", b"q0\nq1\n"]
    news = [b"o0\no1\n", b"p0\n" + b"".join(blk) + b"p1\n", b"q0\n" + b"".join(blk + [b"sep = 1\n"] + blk) + b"q1\n"]
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    r = check(sc, ts.pack(olds, [1] * 3), ts.pack(news, [1] * 3))
    assert r["old_blocks"]["partner"].tolist() == [int(r["line_base_new"][1]) + 1]
    assert len(r["new_blocks"]) == 3 and set(r["new_blocks"]["partner"].tolist()) == {1}
    sc.close()


KEYS = ("dels", "ins", "old_blocks", "new_blocks")


def test_moves_capacity_null_outputs_empty_batch_and_bad_step():
    olds, news, exts = planted(0x7053454D0021, 300, 6)
    steps = [i // 6 for i in range(300)]
    a, b = stepped(ts.pack(olds, exts), steps), stepped(ts.pack(news, exts), steps)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    full = check(sc, ts.pack(olds, exts), ts.pack(news, exts), steps)
    assert len(full["old_blocks"]) > 0 and len(full["new_blocks"]) > 0
    assert all(np.array_equal(sc.diff_moves(a, b, cap=c)[k], full[k]) for c in (1, 10**6) for k in KEYS)
    L = ts.lib()
    n = a.n_files
    add, rem = np.zeros(n, np.int64), np.zeros(n, np.int64)
    ca, cb = a.c_struct(), b.c_struct()

    def call(r, x=ca, y=cb):
        add[:] = 0
        return L.tsm_diff_pairs_moves(sc._ctx, C.byref(x), C.byref(y), ts._p(add), ts._p(rem), None, C.byref(r), None)

    counts = [len(full[k]) for k in KEYS]
    bufs = {k: np.zeros(len(full[k]), full[k].dtype) for k in KEYS}
    bo, bn = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)

    def moves(p, caps):
        return ts._DiffMoves(ts._LineMarks(p.get("bo"), p.get("bn"), p["dels"], caps[0], 0, p["ins"], caps[1], 0),
                             p["old_blocks"], caps[2], 0, p["new_blocks"], caps[3], 0)

    t = moves({k: None for k in KEYS}, [0] * 4)
    assert call(t) == 0 and add.any()                                  # every output NULL: nothing to size
    assert [t.marks.n_old, t.marks.n_new, t.n_old_blocks, t.n_new_blocks] == counts
    ptr = {k: ts._p(bufs[k]) for k in KEYS}
    ptr.update(bo=ts._p(bo), bn=ts._p(bn))
    for short in range(4):                                           # one output one short: counts set, nothing copied
        r = moves(ptr, [c - (i == short) for i, c in enumerate(counts)])
        assert call(r) == ts.TSM_E_CAPACITY
        assert [r.marks.n_old, r.marks.n_new, r.n_old_blocks, r.n_new_blocks] == counts
    r = moves(ptr, counts)                                           # exact caps
    assert call(r) == 0 and all(np.array_equal(bufs[k], full[k]) for k in KEYS)
    assert np.array_equal(bo, full["line_base_old"]) and np.array_equal(bn, full["line_base_new"])
    for skip in KEYS:                                                # each output NULL in turn
        for k in KEYS:
            bufs[k][...] = 0
        p = {k: (None if k == skip else ts._p(bufs[k])) for k in KEYS}
        assert call(moves(p, counts)) == 0
        for k in KEYS:
            assert np.array_equal(bufs[k], full[k]) != (k == skip), (skip, k)
    e = ts.pack([], [])
    assert all(sc.diff_moves(e, e)[k].size == 0 for k in KEYS)
    grp = a.grp.copy()
    grp[5] += 1                                                      # a pair whose two sides are in different steps
    bad = ts.Corpus(a.arena, a.off, a.len, a.ext, grp=grp, n_groups=a.n_groups + 1).c_struct()
    assert call(moves(ptr, counts), bad, cb) == -1
    over = ts.Corpus(b.arena, b.off, b.len, b.ext, grp=b.grp, n_groups=int(b.grp.max())).c_struct()   # a step >= n_groups
    assert call(moves(ptr, counts), ts.Corpus(a.arena, a.off, a.len, a.ext, grp=a.grp, n_groups=int(a.grp.max())).c_struct(), over) == -1
    sc.close()


def test_moves_non_blocking_stream_with_another_busy():
    import torch
    olds, news, exts = planted(0x7053454D0022, 400, 4)
    a, b = ts.pack(olds, exts), ts.pack(news, exts)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    s, legacy = torch.cuda.Stream(), torch.cuda.default_stream()
    assert legacy.cuda_stream == 0
    with torch.cuda.stream(legacy):
        torch.cuda._sleep(50_000_000)
    check(sc, a, b, [i // 4 for i in range(400)], stream=s.cuda_stream)
    legacy.synchronize()
    sc.close()
