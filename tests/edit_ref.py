"""Plain-Python restatement of the assertion edits of docs/SPEC.md section 17 (test infrastructure): hunks from the edit script
of spec_ref.py_diff_script, similarity from an O(nm) LCS table, the greedy pairing as written.  Written from the SPEC text; no
shared code with the kernels or tests/orc_assert_edits.py."""
from spec_ref import W, py_diff_script, py_line_records, py_lines

TRACE_MAX_D = 23168                                      # SPEC section 8: larger distances are not traced
SCORE_MIN = 30000                                        # 50 % on git's 60000 scale


def py_lcs(a: bytes, b: bytes) -> int:
    """Length of the longest common subsequence of two byte strings (dynamic programming, one row at a time)."""
    prev = [0] * (len(b) + 1)
    for x in a:
        cur = [0]
        for j, y in enumerate(b):
            cur.append(prev[j] + 1 if x == y else max(prev[j + 1], cur[j]))
        prev = cur
    return prev[-1]


def py_score(old_line: bytes, new_line: bytes) -> int:
    """SPEC section 17 point 3: floor(120000 * lcs / (|a| + |b|)) of the stripped lines."""
    a, b = old_line.strip(W), new_line.strip(W)
    return 120000 * py_lcs(a, b) // (len(a) + len(b))


def py_bitparallel_lcs(a: bytes, b: bytes) -> int:
    """The bit-parallel LCS of Allison-Dix / Hyyro the device runs: V starts all ones over |a| bits, each byte c of b does
    U = V & Peq[c]; V = (V + U) | (V - U); lcs = the zero bits of V."""
    m = len(a)
    full = (1 << m) - 1
    peq = {}
    for i, c in enumerate(a):
        peq[c] = peq.get(c, 0) | (1 << i)
    v = full
    for c in b:
        u = v & peq.get(c, 0)
        v = ((v + u) | (v - u)) & full
    return m - bin(v).count("1")


def py_assert_edits(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """SPEC section 17 as written for one revision pair: the edits as (old line, new line, score) with 0-based lines, in new
    line order."""
    ra, rb = py_line_records(old, ext_old), py_line_records(new, ext_new)
    la, lb = py_lines(old), py_lines(new)
    fa, fb = [r[2] for r in ra], [r[2] for r in rb]
    s = py_diff_script([r[0] for r in ra], [r[0] for r in rb], fa, fb)
    if s[0] + s[1] > TRACE_MAX_D:                        # not traced: no candidates
        return []
    # hunk of a changed line = the number of kept lines before it (its line minus the changed lines before it)
    olds = [(i, i - k) for k, i in enumerate(s[7]) if fa[i]]
    news = [(j, j - k) for k, j in enumerate(s[8]) if fb[j]]
    cands = []
    for i, hi in olds:
        for j, hj in news:
            if hi == hj:
                sc = py_score(la[i], lb[j])
                if sc >= SCORE_MIN:
                    cands.append((-sc, i, j))
    cands.sort()
    used_old, used_new, out = set(), set(), []
    for sc, i, j in cands:
        if i not in used_old and j not in used_new:
            used_old.add(i)
            used_new.add(j)
            out.append((i, j, -sc))
    return sorted(out, key=lambda e: e[1])


def py_hunks(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """The hunks of section 17 point 1 with assertion lines on both sides: [(deleted assertion lines, inserted ones)], 0-based."""
    ra, rb = py_line_records(old, ext_old), py_line_records(new, ext_new)
    fa, fb = [r[2] for r in ra], [r[2] for r in rb]
    s = py_diff_script([r[0] for r in ra], [r[0] for r in rb], fa, fb)
    ho, hn = {}, {}
    for k, i in enumerate(s[7]):
        if fa[i]:
            ho.setdefault(i - k, []).append(i)
    for k, j in enumerate(s[8]):
        if fb[j]:
            hn.setdefault(j - k, []).append(j)
    return [(ho[h], hn[h]) for h in sorted(set(ho) & set(hn))]


def py_changed_asserts(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """The changed assertion lines of a pair that can take part in an edit (0-based lines of each side): those of section 8 of
    a traced pair, in line order - the order of the pair's events in tsm_diff_pairs_asserts."""
    ra, rb = py_line_records(old, ext_old), py_line_records(new, ext_new)
    fa, fb = [r[2] for r in ra], [r[2] for r in rb]
    s = py_diff_script([r[0] for r in ra], [r[0] for r in rb], fa, fb)
    if s[0] + s[1] > TRACE_MAX_D:
        return [], []
    return [i for i in s[7] if fa[i]], [j for j in s[8] if fb[j]]


def py_batch_edits(olds, news, exts_old, exts_new):
    """The edits of a batch of pairs as tsm_diff_pairs_assert_edits reports them: (rev, aev, score) with rev / aev indices into
    the batch's deleted / inserted assertion events (pairs in order, lines in order), in aev order."""
    out, ko, kn = [], 0, 0
    for o, n, xo, xn in zip(olds, news, exts_old, exts_new):
        lo, ln = py_changed_asserts(o, n, xo, xn)
        at_o, at_n = {l: ko + k for k, l in enumerate(lo)}, {l: kn + k for k, l in enumerate(ln)}
        out += [(at_o[i], at_n[j], sc) for i, j, sc in py_assert_edits(o, n, xo, xn)]
        ko, kn = ko + len(lo), kn + len(ln)
    return out
