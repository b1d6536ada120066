"""Reference of the similar-test churn of docs/SPEC.md section 24.  TEST INFRASTRUCTURE ONLY.

A revision is (files, exts); pair k is (pair_old[k], pair_new[k]), file indices of each revision or -1; the k-th unpaired file
of one revision is the k-th unpaired file of the other.
* `churn(old, new, pair_old, pair_new, min_lines, P)`: every pair of both revisions by brute force (simtest_ref.py_similar), the
  marks and kept-line correspondence of smell_churn_ref.py_script_lines and the section-16 matching of
  smell_churn_ref.py_case_match, then the changes and events written out from the SPEC text.  It has no notion of dirty
  tests, so it checks the device's restricted enumeration against the full answer.  Returns the dict of
  `tosemscan.Scanner.similar_churn`, with events as tuples (status, old_a, old_b, a, b, old_lcs, old_score, lcs, score).
"""
import simtest_ref as sr
import smell_churn_ref as scr
import spec_ref

STATUSES = ["changed", "removed", "dropped", "diverged", "created", "copied", "converged"]
NONE = 0xFFFFFFFF


def _unpaired(n, used):
    return [f for f in range(n) if f not in used]


def identity(old, new, pair_old, pair_new, to, tn):
    """(match_old, match_new, body marks): the section-24 test identity.  body marks: per side the set of (file, line) marked."""
    mo, mn = [-1] * len(to), [-1] * len(tn)
    at_o = {(f, b): t for t, (f, b, _) in enumerate(to)}
    at_n = {(f, b): t for t, (f, b, _) in enumerate(tn)}
    marked = (set(), set())
    uo = _unpaired(len(old[0]), set(pair_old))
    un = _unpaired(len(new[0]), set(pair_new))
    assert len(uo) == len(un)
    for fo, fn in zip(uo, un):
        ko = [t for t, x in enumerate(to) if x[0] == fo]
        kn = [t for t, x in enumerate(tn) if x[0] == fn]
        assert len(ko) == len(kn)
        for a, b in zip(ko, kn):
            mo[a], mn[b] = b, a
    for fo, fn in zip(pair_old, pair_new):
        if fo < 0 or fn < 0:
            for f, side, files in ((fo, 0, old[0]), (fn, 1, new[0])):
                if f >= 0:
                    marked[side].update((f, l) for l in range(len(spec_ref.py_lines(files[f]))))
            continue
        a, b, ea, eb = old[0][fo], new[0][fn], int(old[1][fo]), int(new[1][fn])
        deleted, inserted, corr = scr.py_script_lines(a, b, ea, eb)
        marked[0].update((fo, l) for l in deleted)
        marked[1].update((fn, l) for l in inserted)
        ca, cb, match = scr.py_case_match(spec_ref.py_lines(a), spec_ref.py_lines(b), ea, eb, corr)
        for j, k in match.items():
            x, y = at_o.get((fo, ca[k][0])), at_n.get((fn, cb[j][0]))
            if x is not None and y is not None:
                mo[x], mn[y] = y, x
    return mo, mn, marked


def churn(old, new, pair_old, pair_new, min_lines=5, P=70):
    pair_old, pair_new = [int(x) for x in pair_old], [int(x) for x in pair_new]
    to, so = sr.py_sequences(old[0], old[1])
    tn, sn = sr.py_sequences(new[0], new[1])
    mo, mn, marked = identity(old, new, pair_old, pair_new, to, tn)
    co, cn = [b"D"] * len(to), [b"A"] * len(tn)
    for a, b in enumerate(mo):
        if b < 0:
            continue
        (fa, ha, na), (fb, hb, nb) = to[a], tn[b]
        same = (na == nb and so[a] == sn[b] and not any((fa, l) in marked[0] for l in range(ha, ha + na))
                and not any((fb, l) in marked[1] for l in range(hb, hb + nb)))
        co[a] = cn[b] = b"=" if same else b"M"
    po = {(a, b): (l, s) for a, b, l, s in sr.py_similar(so, min_lines, P)}
    pn = {(a, b): (l, s) for a, b, l, s in sr.py_similar(sn, min_lines, P)}

    def scored(seqs, a, b):
        l = sr.lcs(seqs[a], seqs[b])
        return l, sr.score(l, len(seqs[a]), len(seqs[b]))
    ev_old, ev_new, images = [], [], set()
    for (a, b), (l, s) in sorted(po.items()):
        if co[a] == b"=" and co[b] == b"=":
            continue
        x, y = mo[a], mo[b]
        if x >= 0 and y >= 0 and (min(x, y), max(x, y)) in pn:
            images.add((min(x, y), max(x, y)))
            continue
        if x >= 0 and y >= 0:
            ev_old.append((3, a, b, x, y, l, s) + scored(sn, x, y))
        else:
            ev_old.append((1 if x < 0 and y < 0 else 2, a, b, x, y, l, s, NONE, NONE))
    for (a, b), (l, s) in sorted(pn.items()):
        if cn[a] == b"=" and cn[b] == b"=":
            continue
        x, y = mn[a], mn[b]
        if (a, b) in images:
            ev_new.append((0, x, y, a, b) + po[(min(x, y), max(x, y))] + (l, s))
        elif x >= 0 and y >= 0:
            ev_new.append((6, x, y, a, b) + scored(so, min(x, y), max(x, y)) + (l, s))
        else:
            ev_new.append((4 if x < 0 and y < 0 else 5, x, y, a, b, NONE, NONE, l, s))

    def side(tests, seqs, match, change):
        return {"tests": tests, "test_kept": [len(s) for s in seqs], "match": match, "change": b"".join(change)}
    return {"old": side(to, so, mo, co), "new": side(tn, sn, mn, cn), "events": ev_old + ev_new}


def rows(res):
    """The events as (status name, old_a, old_b, a, b, old similarity, similarity) with similarities in whole per cent."""
    pct = lambda s: None if s == NONE else s // 600
    return [(STATUSES[e[0]], e[1], e[2], e[3], e[4], pct(e[6]), pct(e[8])) for e in res["events"]]


def assert_equal(got, want):
    """got: the dict of Scanner.similar_churn; want: churn()."""
    for name in ("old", "new"):
        g, w = got[name], want[name]
        assert [(int(t["file"]), int(t["line"]), int(t["body_lines"])) for t in g["tests"]] == [tuple(t) for t in w["tests"]], name
        assert g["test_kept"].tolist() == w["test_kept"], name
        assert g["match"].tolist() == w["match"], name
        assert bytes(g["change"]) == w["change"], name
    assert [tuple(int(x) for x in e) for e in got["events"]] == [tuple(e) for e in want["events"]]
