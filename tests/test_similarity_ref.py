"""The references of the rename similarity (docs/SPEC.md section 13), without a GPU: the plain-Python `py_similarity` equals
the C reference `orc_similarity` on generated files, and on a git repository whose lines are all shorter than 64 bytes
(where git's span hashing and whole-line hashing coincide) floor(100 * common / max size) is git's `R` score."""
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import orc_similarity as osim
import tosemscan as ts
from test_history import CLI, git


def gen_file(rng, n_lines, vocab, crlf=0.0, unterminated=False):
    out = []
    for _ in range(n_lines):
        line = rng.choice(vocab)
        out.append(line + (b"\r\n" if rng.random() < crlf else b"\n"))
    data = b"".join(out)
    if unterminated and data:
        data = data[:-1] if data.endswith(b"\n") else data
        if rng.random() < 0.5:
            data = data.rstrip(b"\n") + b"\r"                # a last line ending in a bare CR
    return data


def file_sets():
    rng = random.Random(0x5111)
    vocab = [b"x = %d" % i for i in range(40)] + [b"", b"    assert a == b", b"}", b"\r", b"  \t", b"a" * 90]
    files = [b"", b"\n", b"\r\n", b"a", b"a\r", b"a\n", b"a\r\n", b"\n\n\n", b"a\nb", b"a\r\nb\r\n", b"a\n" * 50, b"a\r\n" * 7 + b"a\n"]
    for k in range(120):
        files.append(gen_file(rng, rng.randrange(0, 80), vocab[:rng.randrange(2, len(vocab))], crlf=rng.choice([0, 0.3, 1]),
                              unterminated=rng.random() < 0.3))
    return files


def test_py_similarity_equals_orc_similarity():
    files = file_sets()
    corpus = ts.pack(files, [1] * len(files))
    rng = np.random.default_rng(3)
    n = len(files)
    co = np.concatenate([np.repeat(np.arange(n), 8), rng.integers(0, n, 2000)]).astype(np.int32)
    cn = np.concatenate([np.tile(np.arange(8), n) * 13 % n, rng.integers(0, n, 2000)]).astype(np.int32)
    got = osim.similarity(corpus, corpus, co, cn)
    want = [osim.py_similarity(files[a], files[b]) for a, b in zip(co, cn)]
    assert got.tolist() == want
    assert sum(1 for a, b in zip(co, cn) if a == b) > 0
    for i, f in enumerate(files):                          # a file against itself: every byte except the CR of a CRLF
        assert osim.py_similarity(f, f) == len(f) - f.count(b"\r\n")
    assert osim.py_similarity(b"assert 1\n", b"assert 1\nassert 2\n") * 100 // 18 == 50    # git: R050
    assert osim.py_similarity(b"", b"a\n") == 0


def test_orc_similarity_rejects_bad_indices():
    corpus = ts.pack([b"a\n", b"b\n"], [1, 1])
    with pytest.raises(ValueError):
        osim.similarity(corpus, corpus, [0, 2], [0, 0])
    with pytest.raises(ValueError):
        osim.similarity(corpus, corpus, [0], [-1])


def short_lines(tag, n):
    return [b"%s_%03d = %d\n" % (tag, i, i * 7) for i in range(n)]


def edited(lines, frac, tag, seed):
    rng = random.Random(seed)
    out = list(lines)
    for i in rng.sample(range(len(out)), int(round(frac * len(out)))):
        out[i] = b"%s_new_%03d = 0\n" % (tag, i)
    return out


@pytest.mark.skipif(shutil.which("git") is None, reason="needs the git command line")
def test_scores_equal_git_rename_scores(tmp_path):
    repo = tmp_path / "repo"
    os.makedirs(repo / "tests")
    git(repo, "init", "-q", ".")
    files = {}
    for k, frac in enumerate([0.0, 0.1, 0.2, 0.3, 0.35, 0.45]):
        files["tests/test_m%d.py" % k] = short_lines(b"m%d" % k, 20 + 7 * k)
    files["tests/test_crlf.py"] = [ln.replace(b"\n", b"\r\n") for ln in short_lines(b"cr", 30)]
    files["tests/test_dup.py"] = short_lines(b"dp", 5) * 6
    files["tests/test_grow.py"] = [b"assert 1\n"]
    for nm, lines in files.items():
        (repo / nm).write_bytes(b"".join(lines))
    git(repo, "add", "-A")
    git(repo, "commit", "-q", "-m", "one")
    os.makedirs(repo / "tests" / "moved")
    new = {}
    for k, frac in enumerate([0.0, 0.1, 0.2, 0.3, 0.35, 0.45]):
        new["tests/moved/test_m%d.py" % k] = edited(files["tests/test_m%d.py" % k], frac, b"m%d" % k, k)
    new["tests/moved/test_crlf.py"] = edited(files["tests/test_crlf.py"], 0.2, b"cr", 9)
    new["tests/moved/test_dup.py"] = files["tests/test_dup.py"][:20] + short_lines(b"dq", 4)
    new["tests/moved/test_grow.py"] = [b"assert 1\n", b"assert 2\n"]
    for nm in files:
        os.remove(repo / nm)
    for nm, lines in new.items():
        (repo / nm).write_bytes(b"".join(lines))
    git(repo, "add", "-A")
    git(repo, "commit", "-q", "-m", "move")
    out = git(repo, "diff", "-M", "--name-status", "-z", "HEAD~1", "HEAD").split("\0")
    seen = 0
    i = 0
    while i < len(out) and out[i]:
        st = out[i]
        if st.startswith("R"):
            old, nw = out[i + 1], out[i + 2]
            a = git(repo, "show", "HEAD~1:" + old, text=False)
            b = git(repo, "show", "HEAD:" + nw, text=False)
            common = osim.py_similarity(a, b)
            assert 100 * common // max(len(a), len(b)) == int(st[1:]), (old, nw, st)
            assert osim.similarity_percent(common, len(a), len(b)) == int(st[1:])
            seen += 1
            i += 3
        else:
            i += 2
    assert seen >= 7, out


def test_dry_run_with_find_renames_is_refused(tmp_path):
    r = subprocess.run([CLI, "history", str(tmp_path), "--dry-run", "--find-renames", "50"], capture_output=True, text=True)
    assert r.returncode == 2 and "--find-renames" in r.stderr
    for bad in ("101", "-1", "x", "5x"):
        r = subprocess.run([CLI, "history", str(tmp_path), "--find-renames", bad], capture_output=True, text=True)
        assert r.returncode == 2 and "--find-renames" in r.stderr
