"""Plain-Python restatement of the test-smell churn of docs/SPEC.md section 19 (test infrastructure): the edit script of
spec_ref.py_diff_script, the cases and matching of section 16 (case_ref.py) and the tests and line smells of section 18
(smell_ref.py_file_smells).  Written from the SPEC text; no shared code with the kernels or tests/orc_smell_churn.py."""
import case_ref as cr
import smell_ref as smr
import spec_ref as sr

SMELLS = smr.SMELLS


def py_script_lines(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """(deleted, inserted, corr) of one pair: the deleted old and inserted new lines of the canonical script (the whole middle
    of an untraced pair), and corr[new kept line] = the corresponding old kept line (section 14)."""
    ra, rb = sr.py_line_records(old, ext_old), sr.py_line_records(new, ext_new)
    ha, hb = [r[0] for r in ra], [r[0] for r in rb]
    s = sr.py_diff_script(ha, hb, [r[2] for r in ra], [r[2] for r in rb])
    deleted, inserted = set(s[7]), set(s[8])
    if s[0] + s[1] > cr.TRACE_MAX_D:
        pre = 0
        while pre < len(ha) and pre < len(hb) and ha[pre] == hb[pre]:
            pre += 1
        suf = 0
        while suf < len(ha) - pre and suf < len(hb) - pre and ha[-1 - suf] == hb[-1 - suf]:
            suf += 1
        deleted, inserted = set(range(pre, len(ha) - suf)), set(range(pre, len(hb) - suf))
    corr = dict(zip([j for j in range(len(hb)) if j not in inserted], [i for i in range(len(ha)) if i not in deleted]))
    return deleted, inserted, corr


def py_case_match(la, lb, ext_old, ext_new, corr):
    """Section 16 matching: {new case index: old case index} after step 1 (kept header) and step 2 (unique name)."""
    ca, cb = cr.py_cases(la, ext_old), cr.py_cases(lb, ext_new)
    na = [cr.py_case_name(la[h], ext_old) for h, _ in ca]
    nb = [cr.py_case_name(lb[h], ext_new) for h, _ in cb]
    old_at = {h: k for k, (h, _) in enumerate(ca)}
    match = {j: old_at[corr[h]] for j, (h, _) in enumerate(cb) if h in corr and corr[h] in old_at}
    used = set(match.values())
    free_new = [j for j in range(len(cb)) if j not in match]
    free_old = [k for k in range(len(ca)) if k not in used]
    for j in free_new:
        same_old = [k for k in free_old if na[k] == nb[j]]
        if sum(nb[x] == nb[j] for x in free_new) == 1 and len(same_old) == 1:
            match[j] = same_old[0]
    return ca, cb, match


def py_test_churn(tests, line_smell, other_smell, changed, corr):
    """Per test of one side: (header line, smells, instances[9], churned[9]).  changed: the side's deleted / inserted lines;
    corr: this side's kept line -> the other side's corresponding line."""
    out = []
    for b, n, _, smells, _, _ in tests:
        inst, churn = [0] * 9, [0] * 9
        for l in range(b, b + n):
            bits = line_smell[l]
            c = bits if l in changed else bits & ~other_smell[corr[l]]
            for k in range(9):
                inst[k] += (bits >> k) & 1
                churn[k] += (c >> k) & 1
        out.append((b, smells, inst, churn))
    return out


def py_smell_churn(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """Section 19 as written: the rows of one revision pair, D tests in old line order, then A and M tests in new line order,
    each test's rows in smell order.  A row is (test, change, line, oldLine, smell, event, instances, oldInstances,
    addedInstances, removedInstances) with 1-based lines and None for a side the test does not have."""
    la, lb = sr.py_lines(old), sr.py_lines(new)
    deleted, inserted, corr = py_script_lines(old, new, ext_old, ext_new)
    back = {i: j for j, i in corr.items()}
    ta, lsa = smr.py_file_smells(old, ext_old)
    tb, lsb = smr.py_file_smells(new, ext_new)
    ca_, cb_ = py_test_churn(ta, lsa, lsb, deleted, back), py_test_churn(tb, lsb, lsa, inserted, corr)
    ca, cb, match = py_case_match(la, lb, ext_old, ext_new, corr)
    old_test = {t[0]: t for t in ca_}
    pairs = {}                                           # new test header -> old test header
    for j, k in match.items():
        if cb[j][0] in {t[0] for t in cb_} and ca[k][0] in old_test:
            pairs[cb[j][0]] = ca[k][0]
    rows = []
    for b, smells, inst, churn in ca_:
        if b in pairs.values():
            continue
        name = cr.py_case_name(la[b], ext_old)
        for k in range(9):
            if smells >> k & 1:
                rows.append((name, "D", None, b + 1, SMELLS[k], "removed", None, inst[k], None, churn[k]))
    for b, smells, inst, churn in cb_:
        name = cr.py_case_name(lb[b], ext_new)
        if b not in pairs:
            for k in range(9):
                if smells >> k & 1:
                    rows.append((name, "A", b + 1, None, SMELLS[k], "introduced", inst[k], None, churn[k], None))
            continue
        ob = pairs[b]
        _, osm, oinst, ochurn = old_test[ob]
        for k in range(9):
            hn, ho = smells >> k & 1, osm >> k & 1
            ev = ("introduced" if hn and not ho else "removed" if ho and not hn else
                  "changed" if hn and ho and (churn[k] or ochurn[k]) else None)
            if ev:
                rows.append((name, "M", b + 1, ob + 1, SMELLS[k], ev, inst[k], oinst[k], churn[k], ochurn[k]))
    return rows
