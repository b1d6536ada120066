"""numpy reference of the test-case records of tsm_diff_pairs_cases (docs/SPEC.md section 16), for inputs too large for the
plain-Python restatement (case_ref.py_case_churn).  TEST INFRASTRUCTURE ONLY.

The marks come from the serial tests/orc_diff_marks.c (orc_marks), the header and assertion lines from the oracle's events
(orc.scan); the cases, their counts and the step-1 match are array arithmetic over them.  case_rows applies step 2 (names)
and the row rule of section 16 to the records, as the CLI does."""
import collections

import numpy as np

import orc
import orc_marks
import case_ref as cr
import spec_ref as sr
import tosemscan as ts


def side_lines(side):
    """(line_base, header lines, assertion flag per line) of a packed side (arena, off, len, ext), global line indices."""
    arena, off, length, ext = side
    arena = np.asarray(arena, np.uint8)
    off = np.asarray(off, np.int64)
    res = orc.scan(arena, off, length, ext, np.zeros(len(length), np.uint16), 1, events=True, line_hashes=True)
    base = res["line_base"]
    nl = np.flatnonzero(arena[:int(off[-1])] == 10)

    def line_of(ev):                                     # lines before the event's line_off = LFs of its file in front of it
        f = ev["file"].astype(np.int64)
        return base[f] + np.searchsorted(nl, off[f] + ev["line_off"]) - np.searchsorted(nl, off[f])

    flag = np.zeros(int(base[-1]), np.uint8)
    flag[line_of(res["assert_events"])] = 1
    return base, np.unique(line_of(res["header_events"])), flag


def side_cases(base, heads, flag, mark):
    """CASE records (match -1) of one side: cases from each header line to the next one of its file or the file's end."""
    total = int(base[-1])
    out = np.zeros(len(heads), ts.CASE)
    f = np.searchsorted(base, heads, side="right") - 1
    end = np.minimum(np.append(heads[1:], total), base[f + 1])

    def pre(x):
        return np.concatenate([[0], np.cumsum(x, dtype=np.int64)])

    cf, cm, cfm = pre(flag), pre(mark), pre(flag & mark)
    out["pair"], out["line"], out["n_lines"] = f, heads - base[f], end - heads
    out["n_assert"], out["n_changed"], out["n_changed_assert"] = cf[end] - cf[heads], cm[end] - cm[heads], cfm[end] - cfm[heads]
    out["match"] = -1
    return out


def diff_cases(old, new, dist=None):
    """(old_cases, new_cases) of the packed sides old / new as tsm_diff_pairs_cases gives them.  dist as
    orc_marks.diff_pairs_marks: {pair: D} of the pairs whose distance is known in closed form (above the trace limit their
    whole middle is marked)."""
    ba, bb, dl, ins = orc_marks.diff_pairs_marks(old, new, dist)
    ba2, ha, fa = side_lines(old)
    bb2, hb, fb = side_lines(new)
    assert np.array_equal(ba, ba2) and np.array_equal(bb, bb2)
    oc, nc = side_cases(ba, ha, fa, dl), side_cases(bb, hb, fb, ins)
    kept_old = np.flatnonzero(dl == 0)                   # old line of every kept rank
    kept_new = (ins == 0).astype(np.int64)
    rank_new = np.cumsum(kept_new) - kept_new
    assert len(kept_old) == int(kept_new.sum())
    case_at = np.full(len(dl), -1, np.int64)
    case_at[ha] = np.arange(len(ha))
    sel = ins[hb] == 0
    m = np.full(len(hb), -1, np.int64)
    m[sel] = case_at[kept_old[rank_new[hb[sel]]]]
    nc["match"] = m
    return oc, nc


def case_rows(oc, nc, olds, news, exts_old, exts_new):
    """The rows of case_ref.py_case_churn for every pair, from the records: {pair: rows}.  olds / news: the files' bytes."""
    by_old, by_new = collections.defaultdict(list), collections.defaultdict(list)
    for k, c in enumerate(oc):
        by_old[int(c["pair"])].append(k)
    for j, c in enumerate(nc):
        by_new[int(c["pair"])].append(j)
    out = {}
    for i in sorted(set(by_old) | set(by_new)):
        la, lb = sr.py_lines(olds[i]), sr.py_lines(news[i])
        ko, kn = by_old[i], by_new[i]
        na = {k: cr.py_case_name(la[oc[k]["line"]], exts_old[i]) for k in ko}
        nb = {j: cr.py_case_name(lb[nc[j]["line"]], exts_new[i]) for j in kn}
        match = {j: int(nc[j]["match"]) for j in kn if nc[j]["match"] >= 0}
        used = set(match.values())
        cnt_new = collections.Counter(nb[j] for j in kn if j not in match)
        cnt_old = collections.Counter(na[k] for k in ko if k not in used)
        old_of = {na[k]: k for k in ko if k not in used}
        for j in kn:
            if j not in match and cnt_new[nb[j]] == 1 and cnt_old[nb[j]] == 1:
                match[j] = old_of[nb[j]]
        used = set(match.values())
        rows = []
        for k in ko:
            c = oc[k]
            if k not in used:
                rows.append((na[k], "D", None, int(c["line"]) + 1, None, int(c["n_lines"]), None, int(c["n_assert"]), None,
                             int(c["n_changed"]), None, int(c["n_changed_assert"])))
        for j in kn:
            c = nc[j]
            n, a, ch, cha = int(c["n_lines"]), int(c["n_assert"]), int(c["n_changed"]), int(c["n_changed_assert"])
            if j not in match:
                rows.append((nb[j], "A", int(c["line"]) + 1, None, n, None, a, None, ch, None, cha, None))
                continue
            o = oc[match[j]]
            if ch or o["n_changed"] or n != o["n_lines"]:
                rows.append((nb[j], "M", int(c["line"]) + 1, int(o["line"]) + 1, n, int(o["n_lines"]), a, int(o["n_assert"]), ch,
                             int(o["n_changed"]), cha, int(o["n_changed_assert"])))
        if rows:
            out[i] = rows
    return out
