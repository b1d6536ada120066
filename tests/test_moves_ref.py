"""The moved code of docs/SPEC.md section 20 on the CPU: the plain-Python restatement (tests/move_ref.py) against git 2.43's
`--color-moved=blocks` on a planted history (tests/move_repo.py), commit by commit, with the known answers of the two cases the
section pins; and the numpy reference (tests/orc_moves.py) against the restatement on that history and on C5 pairs in steps."""
import shutil

import numpy as np
import pytest

import move_ref as mr
import move_repo as rp
import orc
import orc_moves as omv
import tosemscan as ts

needs_git = pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")


@pytest.fixture(scope="module")
def history(tmp_path_factory):
    repo = tmp_path_factory.mktemp("moves") / "repo"
    commits = rp.build(str(repo))
    out = []
    parent = rp.git(repo, "rev-list", "--max-parents=0", "HEAD").strip()
    for name, c in commits:
        paths = rp.changed_paths(repo, parent, c)
        pairs = [(rp.blob(repo, parent, p), rp.blob(repo, c, p), 1, 1) for p in paths]
        out.append((name, repo, parent, c, paths, pairs))
        parent = c
    return out


def by_name(history, name):
    return next(h for h in history if h[0] == name)


@needs_git
def test_moves_ref_equal_git(history):
    for name, repo, parent, c, paths, pairs in history:
        want = rp.git_moved(repo, parent, c, paths)
        got = mr.py_moves(pairs)
        for i, p in enumerate(paths):
            mo, mn, dl, ins = want.get(p, (set(), set(), set(), set()))
            b_o, b_n = got["old"]["base"], got["new"]["base"]
            chg_o = {g - b_o[i] for g in got["old"]["changed"] if b_o[i] <= g < b_o[i + 1]}
            chg_n = {g - b_n[i] for g in got["new"]["changed"] if b_n[i] <= g < b_n[i + 1]}
            assert (chg_o, chg_n) == (dl, ins), (name, p, "the edits must be unambiguous")
            assert set(mr.file_moved(got, "old", i)) == mo, (name, p)
            assert set(mr.file_moved(got, "new", i)) == mn, (name, p)


@needs_git
def test_moves_known_answers(history):
    name, repo, parent, c, paths, pairs = by_name(history, "two files")
    got = mr.py_moves(pairs)
    ia, ib = paths.index("test_a.py"), paths.index("test_b.py")
    assert mr.file_moved(got, "old", ia) == [2, 3, 6, 7]          # test_2 and test_4; `x = 1` (old line 12) is not moved
    assert mr.file_moved(got, "new", ia) == [7, 8]                # test_4 after test_5; `x = 1` (new line 2) is not moved
    assert mr.file_moved(got, "new", ib) == [4, 5]                # test_2 at the end of test_b.py
    name, repo, parent, c, paths, pairs = by_name(history, "rewind")
    got = mr.py_moves(pairs)
    i1, i2 = paths.index("test_r1.py"), paths.index("test_r2.py")
    assert mr.file_moved(got, "old", i1) == [2, 3, 4]            # -cd and both asserts; -ab is not moved
    assert mr.file_moved(got, "new", i2) == [4, 5, 6]            # the second run; +ab, +cd of the first run are not
    b_n = got["new"]["base"]
    (line, partner, n_lines, n_assert), = got["old"]["blocks"]
    assert (partner - b_n[i2], n_lines, n_assert) == (4, 3, 2)


@needs_git
def test_moves_edge_cases(history):
    got = {h[0]: (h[4], mr.py_moves(h[5])) for h in history}
    paths, r = got["20 and 19"]
    assert [b[2] for b in r["old"]["blocks"]] == [1] and mr.file_moved(r, "new", paths.index("test_q.py")) == [1]
    paths, r = got["partner run ends"]
    assert [b[2] for b in r["old"]["blocks"]] == [2] and mr.file_moved(r, "old", paths.index("test_cut_a.py")) == [1, 2]
    paths, r = got["two destinations"]
    assert len(r["new"]["blocks"]) == 2 and r["old"]["blocks"][0][1] == r["new"]["blocks"][0][0]   # the smallest partner
    paths, r = got["blank lines"]
    assert [b[2] for b in r["old"]["blocks"]] == [3]
    paths, r = got["adjacent blocks"]
    assert [(b[0] - r["old"]["base"][paths.index("test_adj_x.py")], b[2]) for b in r["old"]["blocks"]] == [(1, 2), (3, 2)]
    paths, r = got["whole file"]
    assert [b[2] for b in r["old"]["blocks"]] == [6] == [b[2] for b in r["new"]["blocks"]]


def packed(pairs):
    olds = orc.pack([p[0] for p in pairs]) + (np.array([p[2] for p in pairs], np.uint8),)
    news = orc.pack([p[1] for p in pairs]) + (np.array([p[3] for p in pairs], np.uint8),)
    return olds, news


def check_orc(pairs, steps=None):
    want = mr.py_moves(pairs, steps)
    olds, news = packed(pairs)
    bo, bn, dl, ins, ob, nb = omv.diff_moves(olds, news, steps)
    for side, blocks, mark in (("old", ob, dl), ("new", nb, ins)):
        assert [tuple(int(v) for v in b) for b in blocks] == want[side]["blocks"]
        assert set(np.flatnonzero(mark & 2)) == want[side]["moved"]
        assert set(np.flatnonzero(mark)) == want[side]["changed"]


@needs_git
def test_orc_moves_equal_ref_on_history(history):
    for name, repo, parent, c, paths, pairs in history:
        check_orc(pairs)
    every = [p for h in history for p in h[5]]                   # the whole history as one batch, a step per commit
    check_orc(every, [k for k, h in enumerate(history) for _ in h[5]])


def test_orc_moves_equal_ref_on_c5_steps():
    a, b = ts.gen_pairs(0x7053454D0005, 60, pinned=False)
    pairs = [(a.file_bytes(i), b.file_bytes(i), int(a.ext[i]), int(b.ext[i])) for i in range(a.n_files)]
    for k in (1, 7, 60):
        check_orc(pairs, [i // k for i in range(len(pairs))])
