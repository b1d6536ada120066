"""numpy reference of the test-smell churn of tsm_diff_pairs_smells (docs/SPEC.md section 19), for inputs too large for the
plain-Python restatement (smell_churn_ref.py_smell_churn).  TEST INFRASTRUCTURE ONLY.

The marks come from the serial tests/orc_diff_marks.c (orc_marks), the tests and line smells from the serial tests/orc_smells.c
(orc_smells), the header lines from the oracle's events (orc_cases.side_lines); the churn records are array arithmetic over
them.  churn_rows applies the matching and the event rule of section 19 to the records, as the CLI does."""
import collections
import types

import numpy as np

import case_ref as cr
import orc_cases
import orc_marks
import orc_smells
import spec_ref as sr
import tosemscan as ts


def _corpus(side):
    arena, off, length, ext = side
    return types.SimpleNamespace(arena=arena, off=off, len=length, ext=ext)


def side_churn(base, tests, smell, other_smell, mark, other_kept, heads):
    """TEST_CHURN records of one side: other_kept[rank] = the other side's kept line of that rank."""
    kept = mark == 0
    rank = np.cumsum(kept) - kept
    cp = np.zeros(len(smell), np.uint16)
    cp[kept] = other_smell[other_kept[rank[kept]]]
    churn = smell & ~cp
    out = np.zeros(len(tests), ts.TEST_CHURN)
    b = base[tests["file"]] + tests["line"]
    e = b + tests["body_lines"]
    out["case_idx"] = np.searchsorted(heads, b)
    for k in range(9):
        pi = np.concatenate([[0], np.cumsum((smell >> k) & 1, dtype=np.int64)])
        pc = np.concatenate([[0], np.cumsum((churn >> k) & 1, dtype=np.int64)])
        out["instances"][:, k] = pi[e] - pi[b]
        out["churned"][:, k] = pc[e] - pc[b]
    return out


def diff_smells(old, new, dist=None):
    """The dict of Scanner.diff_smells for the packed sides old / new (arena, off, len, ext), without added / removed / detail.
    dist as orc_marks.diff_pairs_marks."""
    ba, bb, dl, ins = orc_marks.diff_pairs_marks(old, new, dist)
    _, ha, fa = orc_cases.side_lines(old)
    _, hb, fb = orc_cases.side_lines(new)
    oc, nc = orc_cases.side_cases(ba, ha, fa, dl), orc_cases.side_cases(bb, hb, fb, ins)
    kept_old, kept_new = np.flatnonzero(dl == 0), np.flatnonzero(ins == 0)
    assert len(kept_old) == len(kept_new)
    case_at = np.full(len(dl), -1, np.int64)
    case_at[ha] = np.arange(len(ha))
    rank_new = np.cumsum(ins == 0) - (ins == 0)
    sel = ins[hb] == 0
    nc["match"][sel] = case_at[kept_old[rank_new[hb[sel]]]]
    so, sn = orc_smells.smells(_corpus(old)), orc_smells.smells(_corpus(new))
    assert np.array_equal(so["line_base"], ba) and np.array_equal(sn["line_base"], bb)
    return {"old_cases": oc, "new_cases": nc, "old_tests": so["tests"], "new_tests": sn["tests"],
            "old_churn": side_churn(ba, so["tests"], so["line_smell"], sn["line_smell"], dl, kept_new, ha),
            "new_churn": side_churn(bb, sn["tests"], sn["line_smell"], so["line_smell"], ins, kept_old, hb)}


def match_cases(ko, kn, na, nb):
    """Section 16 matching of the cases of one pair: {new case: old case}.  ko: the old case indices; kn: {new case index: its
    step-1 match or -1}; na / nb: the names of the cases."""
    match = {j: int(m) for j, m in kn.items() if m >= 0}
    used = set(match.values())
    cnt_new = collections.Counter(nb[j] for j in kn if j not in match)
    cnt_old = collections.Counter(na[k] for k in ko if k not in used)
    old_of = {na[k]: k for k in ko if k not in used}
    for j in kn:
        if j not in match and cnt_new[nb[j]] == 1 and cnt_old[nb[j]] == 1:
            match[j] = old_of[nb[j]]
    return match


def churn_rows(r, olds, news, exts_old, exts_new):
    """The rows of smell_churn_ref.py_smell_churn for every pair, from the records of diff_smells (device or reference):
    {pair: rows}.  olds / news: the files' bytes."""
    oc, nc, ot, nt, och, nch = (r[k] for k in ("old_cases", "new_cases", "old_tests", "new_tests", "old_churn", "new_churn"))
    by = [collections.defaultdict(list) for _ in range(4)]
    for k, c in enumerate(oc):
        by[0][int(c["pair"])].append(k)
    for j, c in enumerate(nc):
        by[1][int(c["pair"])].append(j)
    for t, x in enumerate(ot):
        by[2][int(x["file"])].append(t)
    for t, x in enumerate(nt):
        by[3][int(x["file"])].append(t)
    out = {}
    for i in sorted(set(by[2]) | set(by[3])):
        la, lb = sr.py_lines(olds[i]), sr.py_lines(news[i])
        na = {k: cr.py_case_name(la[oc[k]["line"]], exts_old[i]) for k in by[0][i]}
        nb = {j: cr.py_case_name(lb[nc[j]["line"]], exts_new[i]) for j in by[1][i]}
        match = match_cases(by[0][i], {j: nc[j]["match"] for j in by[1][i]}, na, nb)
        old_test = {int(och[t]["case_idx"]): t for t in by[2][i]}
        pairs = {}
        for t in by[3][i]:
            m = match.get(int(nch[t]["case_idx"]))
            if m is not None and m in old_test:
                pairs[t] = old_test[m]
        rows = []
        for t in by[2][i]:
            if t in pairs.values():
                continue
            x, c = ot[t], och[t]
            for k in range(9):
                if x["smells"] >> k & 1:
                    rows.append((na[int(c["case_idx"])], "D", None, int(x["line"]) + 1, ts.SMELLS[k], "removed", None,
                                 int(c["instances"][k]), None, int(c["churned"][k])))
        for t in by[3][i]:
            x, c = nt[t], nch[t]
            name = nb[int(c["case_idx"])]
            if t not in pairs:
                for k in range(9):
                    if x["smells"] >> k & 1:
                        rows.append((name, "A", int(x["line"]) + 1, None, ts.SMELLS[k], "introduced", int(c["instances"][k]), None,
                                     int(c["churned"][k]), None))
                continue
            y, d = ot[pairs[t]], och[pairs[t]]
            for k in range(9):
                hn, ho = x["smells"] >> k & 1, y["smells"] >> k & 1
                ev = ("introduced" if hn and not ho else "removed" if ho and not hn else
                      "changed" if hn and ho and (c["churned"][k] or d["churned"][k]) else None)
                if ev:
                    rows.append((name, "M", int(x["line"]) + 1, int(y["line"]) + 1, ts.SMELLS[k], ev, int(c["instances"][k]),
                                 int(d["instances"][k]), int(c["churned"][k]), int(d["churned"][k])))
        if rows:
            out[i] = rows
    return out
