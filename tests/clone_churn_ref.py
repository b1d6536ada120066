"""References of the clone churn of docs/SPEC.md section 22.  TEST INFRASTRUCTURE ONLY.

A revision is (files, exts); pair k is (pair_old[k], pair_new[k]), file indices of each revision or -1.
* `churn(old, new, pair_old, pair_new, n, blind=False)`: from the existing references - the classes of tests/orc_clones.py
  (section 15) or tests/orc_blind.py (section 21), the marks of tests/orc_marks.py (section 14) - with the fragment counts,
  states and statuses in plain Python.  Returns {"old": ..., "new": ...}, each the dict of `tosemscan.Scanner.clone_churn`.
* `py_churn(old, new, pair_old, pair_new, n)`: a second restatement over line contents: orc_clones.py_clones for the classes,
  spec_ref.py_diff_files for the marks, and the status rules written out per class.  Exact classes only.
"""
import numpy as np

import orc
import orc_blind as ob
import orc_clones as oc
import orc_marks as om
import spec_ref

STATES = ["kept", "edited", "whole"]
STATUSES = ["untouched", "changed", "removed", "diverged", "dropped", "created", "copied", "joined"]
KEYS = ("changed", "changed_assert", "state", "class_counts", "status")


class _Packed:
    """The packed form orc and orc_clones read (arena, off, len, ext), without the library."""
    def __init__(self, files, exts):
        self.len = np.array([len(f) for f in files], np.int32)
        self.off = np.zeros(len(files) + 1, np.int32)
        pos = 0
        for i, f in enumerate(files):
            self.off[i] = pos
            pos += (len(f) + 127) // 128 * 128
        self.off[len(files)] = pos
        self.arena = np.zeros(max(pos, 1), np.uint8)
        for i, f in enumerate(files):
            self.arena[self.off[i]:self.off[i] + len(f)] = np.frombuffer(f, np.uint8)
        self.ext = np.ascontiguousarray(exts, np.uint8)


def _empty(nf, blind):
    d = {"line_base": np.zeros(nf + 1, np.int64), "file_dup": np.zeros(nf, np.uint32), "file_dup_assert": np.zeros(nf, np.uint32),
         "class_base": np.zeros(1, np.int64), "class_len": np.zeros(0, np.uint32), "member": np.zeros(0, np.int64)}
    if blind:
        d.update(kept_base=np.zeros(nf + 1, np.int64), kept_line=np.zeros(0, np.int64), blind_hash=np.zeros(0, np.uint64),
                 file_kept_assert=np.zeros(nf, np.uint32))
    return d


def status_of(kept, edited, whole, new_side):
    """Section 22's status of a class with these fragment counts (the first rule that holds)."""
    if edited + whole == 0:
        return 0
    if new_side:
        return 5 if kept + edited == 0 else 6 if kept and whole else 7 if kept else 1
    return 2 if kept + edited == 0 else 3 if kept and edited else 4 if kept else 1


def fragment_churn(cl, unit_mark, unit_flag, new_side):
    """The churn outputs of one side's classes `cl` (class_base, class_len, member over units) under per-unit marks."""
    cb, cln, mem = cl["class_base"], cl["class_len"].astype(np.int64), cl["member"]
    P = np.concatenate([[0], np.cumsum(unit_mark, dtype=np.int64)])
    PA = np.concatenate([[0], np.cumsum(unit_mark & unit_flag, dtype=np.int64)])
    L = np.repeat(cln, np.diff(cb))
    changed = (P[mem + L] - P[mem]).astype(np.uint32)
    state = np.where(changed == 0, 0, np.where(changed == L, 2, 1)).astype(np.uint8)
    counts = np.zeros((len(cln), 3), np.uint32)
    status = np.zeros(len(cln), np.uint8)
    for c in range(len(cln)):
        s = state[cb[c]:cb[c + 1]]
        counts[c] = [(s == 0).sum(), (s == 1).sum(), (s == 2).sum()]
        status[c] = status_of(*(int(x) for x in counts[c]), new_side)
    return {"changed": changed, "changed_assert": (PA[mem + L] - PA[mem]).astype(np.uint32), "state": state,
            "class_counts": counts, "status": status}


def revision_marks(old, new, pair_old, pair_new):
    """(del, ins): section 14's marks of the pairs on the lines of each revision (orc_marks.device_marks per pair)."""
    recs = []
    for files, exts in (old, new):
        if len(files):
            recs.append(om.line_hashes(_side(files, exts)))
        else:
            recs.append((np.zeros(1, np.int64), np.zeros(0, np.uint64)))
    marks = [np.zeros(int(b[-1]), np.uint8) for b, _ in recs]
    for fo, fn in zip(pair_old, pair_new):
        seq = []
        for f, (b, h) in zip((fo, fn), recs):
            seq.append(h[b[f]:b[f + 1]] if f >= 0 else np.zeros(0, np.uint64))
        if len(seq[0]) and len(seq[1]):
            dl, ins = om.device_marks(seq[0], seq[1])
        else:                                                 # a pure hunk: every line of the one side
            dl, ins = np.ones(len(seq[0]), np.uint8), np.ones(len(seq[1]), np.uint8)
        if fo >= 0:
            marks[0][recs[0][0][fo]:recs[0][0][fo + 1]] |= dl
        if fn >= 0:
            marks[1][recs[1][0][fn]:recs[1][0][fn + 1]] |= ins
    return marks


def _side(files, exts):
    p = _Packed(files, exts)
    return p.arena, p.off, p.len, p.ext


def churn(old, new, pair_old, pair_new, n, blind=False):
    marks = revision_marks(old, new, pair_old, pair_new)
    out = {}
    for name, (files, exts), mark, new_side in (("old", old, marks[0], False), ("new", new, marks[1], True)):
        if not len(files):
            cl = _empty(0, blind)
        else:
            p = _Packed(files, exts)
            if blind:
                cl = ob.clones_blind(p, n)
                _, _, _, flag = ob.blind_lines(p)
                unit_mark, unit_flag = mark[cl["kept_line"]], flag[cl["kept_line"]]
            else:
                cl = oc.clones(p, n)
                unit_mark, unit_flag = mark, orc.line_records(p.arena, p.off, p.len, p.ext)[3]
            if len(cl["class_len"]):
                cl.update(fragment_churn(cl, unit_mark, unit_flag.astype(np.uint8), new_side))
        for k, dt in zip(KEYS, (np.uint32, np.uint32, np.uint8, np.uint32, np.uint8)):
            cl.setdefault(k, np.zeros((0, 3) if k == "class_counts" else 0, dt))
        out[name] = cl
    return out


def py_churn(old, new, pair_old, pair_new, n):
    """Section 22 over line contents (exact classes)."""
    lines = []
    for files, exts in (old, new):
        recs = [spec_ref.py_line_records(f, int(e)) for f, e in zip(files, exts)]
        base = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
        lines.append((recs, base, [set() for _ in files]))
    for fo, fn in zip(pair_old, pair_new):
        a = old[0][fo] if fo >= 0 else b""
        b = new[0][fn] if fn >= 0 else b""
        ea = int(old[1][fo]) if fo >= 0 else 0
        eb = int(new[1][fn]) if fn >= 0 else 0
        res = spec_ref.py_diff_files(a, b, ea, eb)
        if fo >= 0:
            lines[0][2][fo].update(res[7])
        if fn >= 0:
            lines[1][2][fn].update(res[8])
    out = {}
    for name, (files, exts), (recs, base, marked), new_side in (("old", old) + (lines[0], False), ("new", new) + (lines[1], True)):
        cl = oc.py_clones(files, exts, n)
        fid = np.searchsorted(base, np.arange(int(base[-1])), side="right") - 1
        changed, changed_a, state, counts, status = [], [], [], [], []
        for c in range(len(cl["class_len"])):
            L = int(cl["class_len"][c])
            st = []
            for m in cl["member"][cl["class_base"][c]:cl["class_base"][c + 1]]:
                f = int(fid[m])
                rows = [int(m) - int(base[f]) + k for k in range(L)]
                hit = [r for r in rows if r in marked[f]]
                changed.append(len(hit))
                changed_a.append(sum(recs[f][r][2] for r in hit))
                st.append("kept" if not hit else "whole" if len(hit) == L else "edited")
            state += [STATES.index(s) for s in st]
            k, e, w = st.count("kept"), st.count("edited"), st.count("whole")
            counts.append([k, e, w])
            if not e and not w:
                s = "untouched"
            elif new_side:
                s = "created" if not k and not e else "copied" if k and w else "joined" if k else "changed"
            else:
                s = "removed" if not k and not e else "diverged" if k and e else "dropped" if k else "changed"
            status.append(STATUSES.index(s))
        cl.update(changed=np.array(changed, np.uint32), changed_assert=np.array(changed_a, np.uint32), state=np.array(state, np.uint8),
                  class_counts=np.array(counts, np.uint32).reshape(-1, 3), status=np.array(status, np.uint8))
        out[name] = cl
    return out


def assert_equal(got, want, blind=False):
    """Every array of both sides (the clones keys, the blind keys with blind, the churn keys)."""
    keys = oc.KEYS + KEYS + (("kept_base", "kept_line", "blind_hash", "file_kept_assert") if blind else ())
    for side in ("old", "new"):
        for k in keys:
            g, w = np.asarray(got[side][k]), np.asarray(want[side][k])
            assert g.shape == w.shape and np.array_equal(g.astype(np.int64), w.astype(np.int64)), (side, k)
