"""Plain-Python restatement of the lexical test-smell churn of docs/SPEC.md section 26 (test infrastructure): the edit script and
case matching of smell_churn_ref.py (sections 14 and 16), the tests and line smells of sections 18 and 25 of each side
(smell_ref.py_file_smells, lexsmell_ref.file_lexsmells) and the churn rule of section 19 over the fourteen smell bits.  Written
from the SPEC text; no shared code with the kernels or tests/orc_lexsmell_churn.py."""
import case_ref as cr
import lexsmell_ref as lr
import smell_churn_ref as scr
import smell_ref as smr
import spec_ref as sr

SMELLS = tuple(smr.SMELLS) + tuple(lr.LSMELLS)          # the nine, then the five: bit k of the fourteen is SMELLS[k]
N9 = len(smr.SMELLS)


def side_tests(data: bytes, ext: int):
    """(tests, bits) of one side: tests as (header line, body_lines, smells) over the fourteen bits, bits[line] the fourteen
    bits of every line."""
    t9, ls9 = smr.py_file_smells(data, ext)
    t5, ls5 = lr.file_lexsmells(data, ext)
    assert [(t[0], t[1]) for t in t9] == [(t[0], t[1]) for t in t5]
    tests = [(a[0], a[1], a[3] | b[6] << N9) for a, b in zip(t9, t5)]
    return tests, [x | y << N9 for x, y in zip(ls9, ls5)]


def test_churn(tests, bits, other_bits, changed, corr):
    """Per test of one side: (header line, smells, instances[14], churned[14]).  changed: the side's deleted / inserted lines;
    corr: this side's kept line -> the other side's corresponding line."""
    out = []
    for b, n, smells in tests:
        inst, churn = [0] * len(SMELLS), [0] * len(SMELLS)
        for l in range(b, b + n):
            x = bits[l]
            c = x if l in changed else x & ~other_bits[corr[l]]
            for k in range(len(SMELLS)):
                inst[k] += (x >> k) & 1
                churn[k] += (c >> k) & 1
        out.append((b, smells, inst, churn))
    return out


def py_lexsmell_churn(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """Section 26 as written: the --smells --lexical rows of one revision pair, D tests in old line order, then A and M tests in
    new line order, each test's rows in smell order (the nine, then the five).  A row is (test, change, line, oldLine, smell,
    event, instances, oldInstances, addedInstances, removedInstances) with 1-based lines and None for a side the test lacks."""
    la, lb = sr.py_lines(old), sr.py_lines(new)
    deleted, inserted, corr = scr.py_script_lines(old, new, ext_old, ext_new)
    back = {i: j for j, i in corr.items()}
    ta, ba = side_tests(old, ext_old)
    tb, bb = side_tests(new, ext_new)
    ca_, cb_ = test_churn(ta, ba, bb, deleted, back), test_churn(tb, bb, ba, inserted, corr)
    ca, cb, match = scr.py_case_match(la, lb, ext_old, ext_new, corr)
    old_test = {t[0]: t for t in ca_}
    new_heads = {t[0] for t in cb_}
    pairs = {cb[j][0]: ca[k][0] for j, k in match.items() if cb[j][0] in new_heads and ca[k][0] in old_test}
    rows = []
    for b, smells, inst, churn in ca_:
        if b in pairs.values():
            continue
        name = cr.py_case_name(la[b], ext_old)
        rows += [(name, "D", None, b + 1, s, "removed", None, inst[k], None, churn[k])
                 for k, s in enumerate(SMELLS) if smells >> k & 1]
    for b, smells, inst, churn in cb_:
        name = cr.py_case_name(lb[b], ext_new)
        if b not in pairs:
            rows += [(name, "A", b + 1, None, s, "introduced", inst[k], None, churn[k], None)
                     for k, s in enumerate(SMELLS) if smells >> k & 1]
            continue
        ob = pairs[b]
        _, osm, oinst, ochurn = old_test[ob]
        for k, s in enumerate(SMELLS):
            hn, ho = smells >> k & 1, osm >> k & 1
            ev = ("introduced" if hn and not ho else "removed" if ho and not hn else
                  "changed" if hn and ho and (churn[k] or ochurn[k]) else None)
            if ev:
                rows.append((name, "M", b + 1, ob + 1, s, ev, inst[k], oinst[k], churn[k], ochurn[k]))
    return rows
