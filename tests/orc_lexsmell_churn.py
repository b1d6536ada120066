"""numpy reference of the lexical test-smell churn of tsm_diff_pairs_smells_lexical (docs/SPEC.md section 26), for inputs too large
for the plain-Python restatement (lexsmell_churn_ref.py_lexsmell_churn).  TEST INFRASTRUCTURE ONLY.

Built on tests/orc_smell_churn.py as that is built on orc_smells: the marks of the serial tests/orc_diff_marks.c (orc_marks), the
cases of orc_cases, and the line_lsmell and lex records of each side from the serial tests/orc_lexsmells.c (orc_lexsmells); the
lexical churn records are array arithmetic over them.  churn_rows applies the matching and the event rule of section 19 to the
fourteen smells, as the CLI does."""
import collections

import numpy as np

import case_ref as cr
import orc_lexsmells
import orc_marks
import orc_smell_churn as osc
import spec_ref as sr
import tosemscan as ts

SMELLS = list(ts.SMELLS) + list(ts.LSMELLS)


def side_lex_churn(base, tests, lsmell, other_lsmell, mark, other_kept):
    """LEX_CHURN records of one side: other_kept[rank] = the other side's kept line of that rank."""
    kept = mark == 0
    rank = np.cumsum(kept) - kept
    cp = np.zeros(len(lsmell), np.uint8)
    cp[kept] = other_lsmell[other_kept[rank[kept]]]
    churn = lsmell & ~cp
    out = np.zeros(len(tests), ts.LEX_CHURN)
    b = base[tests["file"]] + tests["line"]
    e = b + tests["body_lines"]
    for k in range(len(ts.LSMELLS)):
        pi = np.concatenate([[0], np.cumsum((lsmell >> k) & 1, dtype=np.int64)])
        pc = np.concatenate([[0], np.cumsum((churn >> k) & 1, dtype=np.int64)])
        out["instances"][:, k] = pi[e] - pi[b]
        out["churned"][:, k] = pc[e] - pc[b]
    return out


def diff_smells_lexical(old, new, dist=None):
    """The dict of Scanner.diff_smells_lexical for the packed sides old / new (arena, off, len, ext), without added / removed /
    detail.  dist as orc_marks.diff_pairs_marks."""
    r = osc.diff_smells(old, new, dist)
    ba, bb, dl, ins = orc_marks.diff_pairs_marks(old, new, dist)
    lo, ln = orc_lexsmells.lexsmells(osc._corpus(old)), orc_lexsmells.lexsmells(osc._corpus(new))
    assert np.array_equal(lo["line_base"], ba) and np.array_equal(ln["line_base"], bb)
    assert len(lo["lex"]) == len(r["old_tests"]) and len(ln["lex"]) == len(r["new_tests"])
    kept_old, kept_new = np.flatnonzero(dl == 0), np.flatnonzero(ins == 0)
    r.update({"old_lex": lo["lex"].view(ts.LEX_TEST), "new_lex": ln["lex"].view(ts.LEX_TEST),
              "old_lex_churn": side_lex_churn(ba, r["old_tests"], lo["line_lsmell"], ln["line_lsmell"], dl, kept_new),
              "new_lex_churn": side_lex_churn(bb, r["new_tests"], ln["line_lsmell"], lo["line_lsmell"], ins, kept_old)})
    return r


def churn_rows(r, olds, news, exts_old, exts_new):
    """The rows of lexsmell_churn_ref.py_lexsmell_churn for every pair, from the records of diff_smells_lexical (device or
    reference): {pair: rows}.  olds / news: the files' bytes."""
    oc, nc, ot, nt, och, nch = (r[k] for k in ("old_cases", "new_cases", "old_tests", "new_tests", "old_churn", "new_churn"))
    n9 = len(ts.SMELLS)

    def fourteen(tests, churn, lex, lchurn):                 # per test: smells, instances[14], churned[14]
        sm = tests["smells"].astype(np.int64) | lex["smells"].astype(np.int64) << n9
        return (sm, np.concatenate([churn["instances"], lchurn["instances"]], 1),
                np.concatenate([churn["churned"], lchurn["churned"]], 1))

    osm, oin, ocu = fourteen(ot, och, r["old_lex"], r["old_lex_churn"])
    nsm, nin, ncu = fourteen(nt, nch, r["new_lex"], r["new_lex_churn"])
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
        match = osc.match_cases(by[0][i], {j: nc[j]["match"] for j in by[1][i]}, na, nb)
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
            rows += [(na[int(och[t]["case_idx"])], "D", None, int(ot[t]["line"]) + 1, s, "removed", None, int(oin[t, k]), None,
                      int(ocu[t, k])) for k, s in enumerate(SMELLS) if osm[t] >> k & 1]
        for t in by[3][i]:
            name = nb[int(nch[t]["case_idx"])]
            if t not in pairs:
                rows += [(name, "A", int(nt[t]["line"]) + 1, None, s, "introduced", int(nin[t, k]), None, int(ncu[t, k]), None)
                         for k, s in enumerate(SMELLS) if nsm[t] >> k & 1]
                continue
            u = pairs[t]
            for k, s in enumerate(SMELLS):
                hn, ho = nsm[t] >> k & 1, osm[u] >> k & 1
                ev = ("introduced" if hn and not ho else "removed" if ho and not hn else
                      "changed" if hn and ho and (ncu[t, k] or ocu[u, k]) else None)
                if ev:
                    rows.append((name, "M", int(nt[t]["line"]) + 1, int(ot[u]["line"]) + 1, s, ev, int(nin[t, k]), int(oin[u, k]),
                                 int(ncu[t, k]), int(ocu[u, k])))
        if rows:
            out[i] = rows
    return out
