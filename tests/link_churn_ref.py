"""Plain-Python restatement of the test-to-code link churn of docs/SPEC.md section 28 (test infrastructure): the links of each
revision alone (link_ref.py_links), the marks and kept-line correspondence of the section-8 script (smell_churn_ref.py_script_lines
over spec_ref's diff), the section-16 case matching (smell_churn_ref.py_case_match over case_ref), then the test changes, the
events and their order written out from the SPEC text.  No shared code with the kernels.

A revision is (files, exts, role, stem) and is one repository; pair k is (pair_old[k], pair_new[k]), file indices of each revision
or -1; the k-th unpaired file of one revision is the k-th unpaired file of the other.
* `churn(old, new, pair_old, pair_new)`: the dict of `tosemscan.Scanner.link_churn`, with events as tuples
  (event, cause, old_test, test, old_link, link, old_calls, calls, old_defs, defs).
* `rows(old, new, res)`: the events as readable rows (test name, change, event, callee, cause, ...).
"""
import numpy as np

import blind_ref as br
import lexsmell_ref as lxr
import link_ref as lr
import smell_churn_ref as scr
from spec_ref import py_bytes_hash, py_lines

EVENTS = ["added", "removed", "retargeted", "redefined", "eager_introduced", "eager_removed", "lazy_introduced", "lazy_removed"]
CAUSES = ["test", "call", "definition"]
ADDED, REMOVED, RETARGETED, REDEFINED = 0, 1, 2, 3
EAGER_IN, EAGER_OUT, LAZY_IN, LAZY_OUT = 4, 5, 6, 7


def _tests(files, exts, role):
    """Per link test (file, header line, body lines, {name hash: call tokens}), in the order of link_ref.py_links."""
    out = []
    for f, (data, ext) in enumerate(zip(files, exts)):
        fam = br.family(int(ext))
        if fam == br.NONE or not role[f]:
            continue
        lines = py_lines(data)
        toks = lr.file_tokens(lines, ext)
        for b, bend, _, code in lxr.bodies(lines, int(ext)):
            calls = {}
            for l in code:
                for nm, _ in lr.calls(toks[l], fam):
                    calls[py_bytes_hash(nm)] = calls.get(py_bytes_hash(nm), 0) + 1
            out.append((f, b, bend - b, calls))
    return out


def _side(rev):
    files, exts, role, stem = rev
    res = lr.py_links(files, exts, role, stem)
    tests = _tests(files, exts, role)
    assert [(int(t["file"]), int(t["line"])) for t in res["tests"]] == [(f, b) for f, b, _, _ in tests]
    keys = []                                                # the name hash of every definition
    for d in res["defs"]:
        o = int(d["name_off"])
        keys.append(py_bytes_hash(files[int(d["file"])][o:o + int(d["name_len"])]))
    n_defs = {}
    for k in keys:
        n_defs[k] = n_defs.get(k, 0) + 1
    return res, tests, keys, n_defs


def _unpaired(n, used):
    return [f for f in range(n) if f not in used]


def churn(old, new, pair_old, pair_new):
    pair_old, pair_new = [int(x) for x in pair_old], [int(x) for x in pair_new]
    (lo, to, ko, ndo), (ln, tn, kn, ndn) = _side(old), _side(new)
    at_o = {(f, b): t for t, (f, b, _, _) in enumerate(to)}
    at_n = {(f, b): t for t, (f, b, _, _) in enumerate(tn)}
    mo, mn = [-1] * len(to), [-1] * len(tn)
    marked = (set(), set())
    uo, un = _unpaired(len(old[0]), set(pair_old)), _unpaired(len(new[0]), set(pair_new))
    assert len(uo) == len(un)
    cfile, dmap = {}, {}                                     # old file -> new file; (old file, line) -> corresponding new line
    for fo, fn in zip(uo, un):
        cfile[fo] = fn
        for l in range(len(py_lines(old[0][fo]))):
            dmap[(fo, l)] = l
        a = [t for t, x in enumerate(to) if x[0] == fo]
        b = [t for t, x in enumerate(tn) if x[0] == fn]
        assert len(a) == len(b)
        for x, y in zip(a, b):
            mo[x], mn[y] = y, x
    for fo, fn in zip(pair_old, pair_new):
        if fo < 0 or fn < 0:
            for f, s, rev in ((fo, 0, old), (fn, 1, new)):
                if f >= 0:
                    marked[s].update((f, l) for l in range(len(py_lines(rev[0][f]))))
            if fo >= 0:
                cfile[fo] = -1
            continue
        cfile[fo] = fn
        a, b, ea, eb = old[0][fo], new[0][fn], int(old[1][fo]), int(new[1][fn])
        deleted, inserted, corr = scr.py_script_lines(a, b, ea, eb)
        marked[0].update((fo, l) for l in deleted)
        marked[1].update((fn, l) for l in inserted)
        for nl, ol in corr.items():
            dmap[(fo, ol)] = nl
        ca, cb, match = scr.py_case_match(py_lines(a), py_lines(b), ea, eb, corr)
        for j, k in match.items():
            x, y = at_o.get((fo, ca[k][0])), at_n.get((fn, cb[j][0]))
            if x is not None and y is not None:
                mo[x], mn[y] = y, x
    co, cn = [b"D"] * len(to), [b"A"] * len(tn)
    for x, y in enumerate(mo):
        if y < 0:
            continue
        (fa, ha, na, _), (fb, hb, nb, _) = to[x], tn[y]
        same = na == nb and not any((fa, l) in marked[0] for l in range(ha, ha + na)) and \
            not any((fb, l) in marked[1] for l in range(hb, hb + nb))
        co[x] = cn[y] = b"=" if same else b"M"

    def links_of(res, keys, t):
        return [(j, keys[int(l["name_def"])]) for j, l in enumerate(res["links"]) if int(l["test"]) == t]

    def corresponds(a, b):                                   # old target a, new target b (definition indices)
        da, db = lo["defs"][a], ln["defs"][b]
        if cfile.get(int(da["file"]), -1) != int(db["file"]):
            return RETARGETED
        return None if dmap.get((int(da["file"]), int(da["line"]))) == int(db["line"]) else REDEFINED

    events = []
    outs = [(a, -1) for a in range(len(to)) if mo[a] < 0] + [(mn[b], b) for b in range(len(tn))]
    for a, b in outs:
        fo = int(lo["tests"][a]["flags"]) if a >= 0 else 0
        fn = int(ln["tests"][b]["flags"]) if b >= 0 else 0
        for bit, ev_in, ev_out in ((lr.EAGER, EAGER_IN, EAGER_OUT), (lr.LAZY, LAZY_IN, LAZY_OUT)):
            if fn & bit and not fo & bit:
                events.append((ev_in, -1, a, b, -1, -1, -1, -1, -1, -1))
            if fo & bit and not fn & bit:
                events.append((ev_out, -1, a, b, -1, -1, -1, -1, -1, -1))
        old_links = links_of(lo, ko, a) if a >= 0 else []
        new_links = links_of(ln, kn, b) if b >= 0 else []
        old_by = {k: j for j, k in old_links}
        new_by = {k: j for j, k in new_links}
        oc = to[a][3] if a >= 0 else None
        nc = tn[b][3] if b >= 0 else None

        def row(ev, key, jo, jn):
            cause = -1
            if ev in (ADDED, REMOVED):
                absent = oc if ev == ADDED else nc
                cause = 0 if absent is None else 1 if absent.get(key, 0) == 0 else 2
            return (ev, cause, a, b, jo, jn, -1 if oc is None else oc.get(key, 0), -1 if nc is None else nc.get(key, 0),
                    ndo.get(key, 0), ndn.get(key, 0))
        for j, key in old_links:
            if key not in new_by:
                events.append(row(REMOVED, key, j, -1))
        for j, key in new_links:
            if key not in old_by:
                events.append(row(ADDED, key, -1, j))
                continue
            jo = old_by[key]
            ta, tb = int(lo["links"][jo]["target"]), int(ln["links"][j]["target"])
            if ta < 0 and tb < 0:
                continue
            ev = RETARGETED if (ta < 0) != (tb < 0) else corresponds(ta, tb)
            if ev is not None:
                events.append(row(ev, key, jo, j))

    def side(res, match, change):
        return {"tests": res["tests"], "links": res["links"], "defs": res["defs"], "match": match, "change": b"".join(change)}
    return {"old": side(lo, mo, co), "new": side(ln, mn, cn), "events": events}


def rows(old, new, res):
    """(test name, change, event, callee, cause, calls, old_calls, defs, old_defs, def line, old def line) per event: names as
    bytes, lines 1-based, None where a cell is empty."""
    from case_ref import py_case_name
    out = []
    for e in res["events"]:
        ev, cause, a, b, jo, jn, ocl, ncl, od, nd = (int(x) for x in e)
        s, rev, t = ("new", new, b) if b >= 0 else ("old", old, a)
        tr = res[s]["tests"][t]
        f = int(tr["file"])
        name = py_case_name(py_lines(rev[0][f])[int(tr["line"])], int(rev[1][f]))
        change = bytes([res[s]["change"][t]])
        if ev >= EAGER_IN:
            out.append((name, change, EVENTS[ev]) + (None,) * 8)
            continue

        def target(side, rv, j):
            if j < 0:
                return None, None
            lk = res[side]["links"][j]
            d = res[side]["defs"][int(lk["name_def"])]
            o = int(d["name_off"])
            callee = rv[0][int(d["file"])][o:o + int(d["name_len"])]
            tg = int(lk["target"])
            return callee, None if tg < 0 else int(res[side]["defs"][tg]["line"]) + 1
        cn, ln_ = target("new", new, jn)
        co, lo_ = target("old", old, jo)
        out.append((name, change, EVENTS[ev], cn or co, None if cause < 0 else CAUSES[cause], None if ncl < 0 else ncl,
                    None if ocl < 0 else ocl, nd, od, ln_, lo_))
    return out


def assert_equal(got, want):
    """got: the dict of Scanner.link_churn; want: churn()."""
    for name in ("old", "new"):
        g, w = got[name], want[name]
        for k in ("tests", "links", "defs"):
            assert np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(w[k]).view(np.uint8)), (name, k)
        assert g["match"].tolist() == w["match"], name
        assert bytes(g["change"]) == w["change"], name
    assert [tuple(int(x) for x in e) for e in got["events"]] == [tuple(e) for e in want["events"]]
