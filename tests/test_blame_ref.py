"""Line provenance (docs/SPEC.md section 14) restated in plain Python, pinned against `git blame --porcelain --first-parent
--minimal` on a repository built here, and the serial edit-mark reference (tests/orc_diff_marks.c) pinned against
spec_ref.py_diff_script.  CPU only; the git tests need the `git` executable."""
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import orc_marks
import spec_ref as sr


def py_marks(old: bytes, new: bytes):
    r = sr.py_diff_files(old, new, 0, 0)
    return r[7], r[8]


def py_blame(commits, window=0):
    """commits: list of (name, {path: bytes}, {new path: old path}) oldest first.  The provenance of every line of every file of
    the last commit over the window commits[window:], with commits[window - 1] as the boundary P0 when window > 0: {path: [(commit,
    origin path, origin line, boundary)]}."""
    state = {}
    if window:
        p0, tree0, _ = commits[window - 1]
        state = {p: [(p0, p, j + 1, 1) for j in range(len(sr.py_lines(f)))] for p, f in tree0.items()}
        prev_tree = tree0
    else:
        prev_tree = {}
    for name, tree, renames in commits[window:]:
        nxt = {}
        for path, new in tree.items():
            src = renames.get(path, path)
            old = prev_tree.get(src)
            if old is None:                                 # an added file: all insertions
                nxt[path] = [(name, path, j + 1, 0) for j in range(len(sr.py_lines(new)))]
                continue
            dels, ins = py_marks(old, new)
            dset, iset = set(dels), set(ins)
            kept = iter([o for i, o in enumerate(state[src]) if i not in dset])
            nxt[path] = [(name, path, j + 1, 0) if j in iset else next(kept) for j in range(len(sr.py_lines(new)))]
        state, prev_tree = nxt, tree
    return state


def git(repo, *args, env=None):
    return subprocess.run(["git", "-C", repo] + list(args), check=True, capture_output=True, env=env).stdout


def git_blame(repo, rev, path, root):
    """(commit, orig filename, orig line, boundary) per line from --line-porcelain."""
    args = ["blame", "--line-porcelain", "--first-parent", "--minimal"] + (["--root"] if root else []) + [rev, "--", path]
    out, rows, cur = git(repo, *args).decode().split("\n"), [], None
    for ln in out:
        if cur is None:
            if not ln:
                continue
            sha, orig = ln.split()[:2]
            cur = [sha, None, int(orig), 0]
        elif ln.startswith("boundary"):
            cur[3] = 1
        elif ln.startswith("filename "):
            cur[1] = ln[len("filename "):]
        elif ln.startswith("\t"):
            rows.append(tuple(cur))
            cur = None
    return rows


def build_history(repo):
    """A repository of unique-line edits: inserts, deletes, replacements, a file deleted and re-added, a move with edits.
    Returns [(sha, tree, renames)], oldest first."""
    rng = random.Random(3)
    uid = iter(range(10**6))

    def lines(k, tag):
        return [b"%s_%d = %d\n" % (tag, next(uid), rng.randrange(10**6)) for _ in range(k)]

    def edit(ls, tag):
        ls = list(ls)
        for _ in range(rng.randrange(1, 4)):
            kind, at = rng.randrange(3), rng.randrange(len(ls) + 1)
            if kind == 0:
                ls[at:at] = lines(rng.randrange(1, 4), tag)
            elif kind == 1 and len(ls) > 4:
                del ls[at:at + rng.randrange(1, 3)]
            else:
                ls[at:at + 1] = lines(rng.randrange(1, 3), tag)
        return ls

    env = dict(os.environ, GIT_AUTHOR_NAME="t", GIT_AUTHOR_EMAIL="t@e", GIT_COMMITTER_NAME="t", GIT_COMMITTER_EMAIL="t@e")
    git(repo, "init", "-q", "-b", "main")
    files = {"tests/test_a.py": lines(30, b"a"), "tests/test_b.py": lines(20, b"b"), "tests/test_c.py": lines(25, b"c")}
    history = []
    steps = ["edit", "edit", "delete_b", "edit", "readd_b", "move_a", "edit", "edit", "edit"]
    for k, step in enumerate(["init"] + steps):
        renames = {}
        if step == "edit":
            for p in list(files):
                if rng.random() < 0.8:
                    files[p] = edit(files[p], b"e%d" % k)
        elif step == "delete_b":
            b_old = files.pop("tests/test_b.py")
        elif step == "readd_b":
            files["tests/test_b.py"] = b_old[:10] + lines(5, b"r")
        elif step == "move_a":
            files["tests/unit/test_a.py"] = edit(files.pop("tests/test_a.py"), b"m")
            renames["tests/unit/test_a.py"] = "tests/test_a.py"
        for p in list(git(repo, "ls-files").decode().split()):
            if p not in files:
                git(repo, "rm", "-q", p)
        for p, ls in files.items():
            os.makedirs(os.path.join(repo, os.path.dirname(p)), exist_ok=True)
            with open(os.path.join(repo, p), "wb") as f:
                f.write(b"".join(ls))
            git(repo, "add", p)
        e = dict(env, GIT_AUTHOR_DATE="%d +0000" % (1_600_000_000 + k), GIT_COMMITTER_DATE="%d +0000" % (1_600_000_000 + k))
        git(repo, "commit", "-q", "-m", step, env=e)
        sha = git(repo, "rev-parse", "HEAD").decode().strip()
        history.append((sha, {p: b"".join(ls) for p, ls in files.items()}, renames))
    return history


needs_git = pytest.mark.skipif(shutil.which("git") is None, reason="needs git")


@needs_git
def test_py_blame_matches_git(tmp_path):
    repo = str(tmp_path / "r")
    os.makedirs(repo)
    hist = build_history(repo)
    assert any(r for _, _, r in hist)
    for end in (len(hist), len(hist) - 3):                 # HEAD and an older revision
        state = py_blame(hist[:end])
        rev = hist[end - 1][0]
        for path in hist[end - 1][1]:
            assert git_blame(repo, rev, path, True) == state[path], (end, path)


@needs_git
@pytest.mark.parametrize("n", [1, 3, 6])
def test_py_blame_window_matches_git(tmp_path, n):
    """A window of the last n commits: lines older than it belong to the boundary R~n, as in `git blame R~n..R`."""
    repo = str(tmp_path / "r")
    os.makedirs(repo)
    hist = build_history(repo)
    state = py_blame(hist, window=len(hist) - n)
    for path in hist[-1][1]:
        got = git_blame(repo, "%s~%d..%s" % (hist[-1][0], n, hist[-1][0]), path, False)
        assert got == state[path], (n, path)
        assert any(b for *_, b in got) == any(b for *_, b in state[path])


def block_middle(old_blocks, new_blocks, n_prefix, n_suffix):
    """(pre, suf) of a corpus_util.block_pair in closed form: leading empty block pairs put their common line in the prefix,
    the common line behind the last non-empty block pair and those of the empty pairs after it belong to the suffix."""
    nz = [i for i, (x, y) in enumerate(zip(old_blocks, new_blocks)) if x or y]
    return n_prefix + nz[0], n_suffix + len(old_blocks) - nz[-1]


def hashes(f):
    return np.array([r[0] for r in sr.py_line_records(f, 1)], np.uint64)


def test_untraced_marks_closed_form():
    """orc_marks.device_marks: on traced block pairs the serial marks, whose distance is the closed form's and whose first and
    last changed lines bound the closed-form middle; on untraced ones (D > 23 168, no serial search) the whole closed-form
    middle, common lines inside it included."""
    rng = random.Random(12)
    shapes = [(tuple(rng.randrange(0, 30) for _ in range(k)), tuple(rng.randrange(0, 30) for _ in range(k)))
              for k in (1, 2, 3, 5) for _ in range(8)]
    shapes += [((0, 7, 0), (0, 0, 0)), ((0, 0, 4), (3, 0, 0)), ((5,), (0,)), ((0,), (6,)), ((0, 2, 0, 0), (0, 0, 9, 0))]
    n = 0
    for i, (ob, nb) in enumerate(shapes):
        if not any(ob) and not any(nb):
            continue
        pre, suf = rng.randrange(0, 4), rng.randrange(0, 4)
        o, nw, w = cu.block_pair(b"m%d" % i, ob, nb, n_prefix=pre, n_suffix=suf)
        a, b = hashes(o), hashes(nw)
        p, s = orc_marks.middle(a, b)
        assert (p, s) == block_middle(ob, nb, pre, suf)
        d, dl, ins = orc_marks.diff_marks(a, b)
        assert d == len(w[3]) + len(w[4])
        assert np.flatnonzero(dl).tolist() == w[3] and np.flatnonzero(ins).tolist() == w[4]
        marks = ((np.flatnonzero(dl), len(a)), (np.flatnonzero(ins), len(b)))
        assert all(x.size == 0 or (x[0] >= p and x[-1] < k - s) for x, k in marks)
        assert any(x.size and x[0] == p for x, _ in marks) and any(x.size and x[-1] == k - s - 1 for x, k in marks)
        got = orc_marks.device_marks(a, b, d)
        assert np.array_equal(got[0], dl) and np.array_equal(got[1], ins)
        n += 1
    assert n > 30
    for i, (ob, nb) in enumerate((((11584,), (11585,)), ((6000, 5585), (6000, 5585)), ((23169,), (0,)), ((0, 9, 23161), (1, 0, 0)))):
        o, nw, w = cu.block_pair(b"u%d" % i, ob, nb, n_prefix=40 + i, n_suffix=30 + i)
        d = len(w[3]) + len(w[4])
        assert d > orc_marks.TRACE_MAX_D
        a, b = hashes(o), hashes(nw)
        p, s = block_middle(ob, nb, 40 + i, 30 + i)
        dl, ins = orc_marks.device_marks(a, b, d)
        assert np.flatnonzero(dl).tolist() == list(range(p, len(a) - s))
        assert np.flatnonzero(ins).tolist() == list(range(p, len(b) - s))
        assert set(w[3]) <= set(range(p, len(a) - s)) and set(w[4]) <= set(range(p, len(b) - s))


def test_marks_reference_matches_spec_ref():
    olds, news, exts = cu.tie_heavy_pairs(7)
    rng = random.Random(4)
    for i in range(12):
        o, n, _ = cu.block_pair(b"k%d" % i, tuple(rng.randrange(0, 40) for _ in range(3)), tuple(rng.randrange(0, 40) for _ in range(3)))
        olds.append(o); news.append(n); exts.append(1)
    olds += [b"", b"a\n", b"a\nb"]; news += [b"a\n", b"", b"a\nb\n"]; exts += [1, 1, 1]
    for o, n, x in zip(olds, news, exts):
        ha = [r[0] for r in sr.py_line_records(o, x)]
        hb = [r[0] for r in sr.py_line_records(n, x)]
        r = sr.py_diff_script(ha, hb, [0] * len(ha), [0] * len(hb))
        d, dl, ins = orc_marks.diff_marks(np.array(ha, np.uint64), np.array(hb, np.uint64))
        assert d == r[0] + r[1]
        assert np.nonzero(dl)[0].tolist() == r[7] and np.nonzero(ins)[0].tolist() == r[8]
