"""The planted history of the moved-code tests (docs/SPEC.md section 20): one commit per scenario on top of a base commit, every
edit unambiguous (git's `--minimal` script and the canonical script of section 8 change the same lines), and a parser of git's
`--color-moved=blocks` output.  Flat layout: the pairs of a commit are its changed selected files in path order."""
import os
import re

from test_history import git

OLD_MOVED, NEW_MOVED, FRAG = "blue", "yellow", "white"   # ANSI 34, 33, 37: none of them git's default colours of -, + or @@
SGR = {"blue": "34", "yellow": "33"}


def tests(names, fmt=b"def test_%s(self):\n    self.assertEqual(compute_value_%s(x), expected_%s)\n"):
    return b"".join(fmt % (n, n, n) for n in names)


A1, A2 = b"    self.assertTrue(alpha_beta_gamma)\n", b"    self.assertTrue(delta_epsilon_zeta)\n"
B20, B19 = b"abcdefghij0123456789\n", b"abcdefghij012345678\n"
L12 = [b"value_alpha_%d\n" % i for i in range(3)]       # 12 alphanumerics each: two of them make a block, one does not
BLK = b"    self.assertIn(first_member, collection)\n    self.assertIn(second_member, collection)\n"
S1 = b"def test_s1(self):\n    check_first_thing(a)\n    check_first_other(b)\n"
S2 = b"def test_s2(self):\n    check_second_thing(c)\n"
REN = b"".join(b"    renamed_line_%d = prepare_%d()\n" % (i, i) for i in range(10))
BLK2 = b"    self.assertIsNone(leftover_handle)\n"

BASE = {
    "test_a.py": tests(b"%d" % i for i in range(1, 7)) + b"x = 1\n",
    "test_b.py": b"import os\n\ndef helper():\n    return 42\n",
    "test_r1.py": b"keep1\nab\ncd\n" + A1 + A2 + b"keep2\n",
    "test_r2.py": b"k3\nk4\nk5\n",
    "test_whole_old.py": tests([b"w1", b"w2", b"w3"]),
    "test_p.py": b"p1\n" + B20 + b"p2\n" + B19 + b"p3\n",
    "test_q.py": b"q1\nq2\n",
    "test_cut_a.py": b"ca\n" + b"".join(L12) + b"cb\n",
    "test_cut_b.py": b"cc\ncd\nce\n",
    "test_copy_x.py": b"x0\n" + BLK + b"x1\n",
    "test_copy_y.py": b"y0\ny1\n",
    "test_copy_z.py": b"z0\nz1\n",
    "test_blank_a.py": b"ba0\ndef test_blank(self):\n\n    self.assertEqual(first_value, second_value)\nba1\n",
    "test_blank_b.py": b"bb0\nbb1\n",
    "test_adj_x.py": b"ax0\n" + tests([b"adj1", b"adj2"]) + b"ax1\n",
    "test_adj_y.py": b"ay0\nay1\n",
    "test_adj_z.py": b"az0\naz1\n",
    "test_swap.py": b"sw0\n" + S1 + S2 + b"sw1\n",
    "test_ren_old.py": REN + BLK2,
    "test_ren_dst.py": b"rd0\nrd1\n",
}


def scenarios():
    """[(name, {path: bytes or None})]: the files each commit changes (None deletes)."""
    a = BASE["test_a.py"].splitlines(keepends=True)
    t = lambda i: a[2 * i - 2:2 * i]                           # noqa: E731 (the two lines of test_i)
    return [
        ("two files", {"test_a.py": b"".join(t(1) + [b"x = 1\n"] + t(3) + t(5) + t(4) + t(6)),
                       "test_b.py": BASE["test_b.py"] + b"".join(t(2))}),
        ("rewind", {"test_r1.py": b"keep1\nkeep2\n", "test_r2.py": b"k3\nab\ncd\nk4\ncd\n" + A1 + A2 + b"k5\n"}),
        ("whole file", {"test_whole_old.py": None, "test_whole_new.py": BASE["test_whole_old.py"]}),
        ("20 and 19", {"test_p.py": b"p1\np2\np3\n", "test_q.py": b"q1\n" + B20 + b"q2\n" + B19}),
        ("partner run ends", {"test_cut_a.py": b"ca\ncb\n", "test_cut_b.py": b"cc\n" + L12[0] + L12[1] + b"cd\n" + L12[2] + b"ce\n"}),
        ("two destinations", {"test_copy_x.py": b"x0\nx1\n", "test_copy_y.py": b"y0\n" + BLK + b"y1\n",
                              "test_copy_z.py": b"z0\n" + BLK + b"z1\n"}),
        ("blank lines", {"test_blank_a.py": b"ba0\nba1\n",
                         "test_blank_b.py": b"bb0\ndef test_blank(self):\n\n    self.assertEqual(first_value, second_value)\nbb1\n"}),
        ("adjacent blocks", {"test_adj_x.py": b"ax0\nax1\n", "test_adj_y.py": b"ay0\n" + tests([b"adj1"]) + b"ay1\n",
                             "test_adj_z.py": b"az0\n" + tests([b"adj2"]) + b"az1\n"}),
        ("swap", {"test_swap.py": b"sw0\n" + S2 + S1 + b"sw1\n"}),
        ("edited rename", {"test_ren_old.py": None, "test_ren_new.py": REN, "test_ren_dst.py": b"rd0\n" + BLK2 + b"rd1\n"}),
    ]


def build(repo):
    """The repository: the base commit, then one commit per scenario.  Returns [(name, commit)] of the scenarios."""
    os.makedirs(repo)
    git(repo, "init", "-q", ".")
    files = dict(BASE)

    def commit(msg):
        for fn in os.listdir(repo):
            if fn != ".git" and fn not in files:
                os.remove(os.path.join(repo, fn))
        for nm, data in files.items():
            with open(os.path.join(repo, nm), "wb") as f:
                f.write(data)
        git(repo, "add", "-A")
        git(repo, "commit", "-q", "-m", msg)
        return git(repo, "rev-parse", "HEAD").strip()

    commit("base")
    out = []
    for name, change in scenarios():
        for p, v in change.items():
            if v is None:
                files.pop(p)
            else:
                files[p] = v
        out.append((name, commit(name)))
    return out


def changed_paths(repo, parent, commit):
    return sorted(p for p in git(repo, "diff", "--no-renames", "--name-only", parent, commit).split("\n") if p)


def blob(repo, rev, path):
    try:
        return git(repo, "show", "%s:%s" % (rev, path), text=False)
    except Exception:
        return b""


def git_moved(repo, parent, commit, paths):
    """{path: (moved old lines, moved new lines, deleted lines, inserted lines)} as 0-based line sets, from git's
    `--color-moved=blocks` output of the commit against its parent."""
    out = git(repo, "-c", "color.diff.oldMoved=" + OLD_MOVED, "-c", "color.diff.newMoved=" + NEW_MOVED, "-c", "color.diff.frag=" + FRAG,
              "diff", "--minimal", "--no-renames", "-U0", "--color=always", "--color-moved=blocks", parent, commit, "--", *paths, text=False)
    res, cur, lo, ln = {}, None, 0, 0
    for raw in out.split(b"\n"):
        m = re.match(rb"^(?:\x1b\[[0-9;]*m)*", raw)
        sgr = re.findall(rb"\x1b\[([0-9;]*)m", m.group(0))
        line = re.sub(rb"\x1b\[[0-9;]*m", b"", raw)
        if line.startswith(b"diff --git "):
            cur = line.split(b" b/", 1)[1].decode()
            res[cur] = (set(), set(), set(), set())
        elif line.startswith(b"@@ "):
            h = re.match(rb"@@ -(\d+)(?:,(\d+))? \+(\d+)(?:,(\d+))? @@", line)
            lo, ln = int(h.group(1)) - 1, int(h.group(3)) - 1
        elif line.startswith(b"---") or line.startswith(b"+++") or cur is None:
            continue
        elif line.startswith(b"-"):
            res[cur][2].add(lo)
            if SGR["blue"].encode() in sgr:
                res[cur][0].add(lo)
            lo += 1
        elif line.startswith(b"+"):
            res[cur][3].add(ln)
            if SGR["yellow"].encode() in sgr:
                res[cur][1].add(ln)
            ln += 1
    return res
