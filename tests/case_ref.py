"""Plain-Python restatement of the test-case churn of docs/SPEC.md section 16 (test infrastructure): the header rule of section
5, the case names of section 10 and the cases, changed lines and matching of section 16, over the edit script of
spec_ref.py_diff_script.  Written from the SPEC text; no shared code with the oracle, the kernels or tests/orc_cases.py."""
from spec_ref import W, _ident, py_diff_script, py_line_records, py_lines


def py_is_header(line: bytes, ext: int) -> bool:
    """SPEC section 5: is the line (without its LF) a test-case header of a file with tag ext?"""
    if ext == 0:
        return False
    if ext == 1:
        s = line.strip(W)
        return b"def" in line or (s.startswith(b"class") and s[5:6] in (b" ", b"\t"))
    return b"test" in line.lower() and (b"{" in line or b"class" in line or b"void" in line)


def py_method_string(line: bytes, ext: int) -> bytes:
    """SPEC section 5: the method string of a header line."""
    s = line.strip(W)
    if ext == 1:
        if s.startswith(b"class"):
            s = s[5:]
        s = bytes(c for c in s.replace(b"def", b"") if c not in W)
        return s[:-1] if s.endswith(b":") else s
    if ext == 4:
        out, i = bytearray(), 0
        while i < len(s):
            w = next((w for w in (b"public", b"private", b"protected", b"static", b"void", b"class") if s.startswith(w, i)), None)
            if w:
                i += len(w)
                continue
            if s[i] not in W:
                out.append(s[i])
            i += 1
        return bytes(out)
    return s.split(b")", 1)[0].replace(b"{", b"").strip(W)


def py_case_name(line: bytes, ext: int) -> bytes:
    """SPEC section 10: the case name of a header line."""
    s = line.strip(W)
    if ext == 1:
        d = s.find(b"def")
        if d >= 0:
            i = d + 3
            while i < len(s) and s[i] in W:
                i += 1
            j = i
            while j < len(s) and _ident(s[j]):
                j += 1
            if j > i:
                return s[i:j]
        return py_method_string(line, ext)
    r = s.find(b")")
    if s.startswith((b"TEST(", b"TEST_F(", b"TEST_P(")):
        c = s.find(b",")
        if c >= 0 and (r < 0 or c < r):
            return s[c + 1:r if r >= 0 else len(s)].strip(W)
    if s.startswith(b"BOOST_AUTO_TEST_CASE("):
        return b"TEST_CASE(" + s[21:r if r >= 0 else len(s)].strip(W) + b")"
    return py_method_string(line, ext)


TRACE_MAX_D = 23168                                      # SPEC section 8: larger distances are not traced


def py_cases(lines, ext: int):
    """SPEC section 16: the cases of one file as (header line, end line) ranges; lines above the first header are in none."""
    heads = [i for i, ln in enumerate(lines) if py_is_header(ln, ext)]
    return [(h, heads[k + 1] if k + 1 < len(heads) else len(lines)) for k, h in enumerate(heads)]


def py_case_churn(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """SPEC section 16 as written: the case rows of one revision pair, the D rows in old line order, then the A and M rows
    in new line order.  A row is (case, change, line, oldLine, lines, oldLines, asserts, oldAsserts, insertedLines,
    deletedLines, insertedAsserts, deletedAsserts) with 1-based lines and None for a side that does not exist."""
    la, lb = py_lines(old), py_lines(new)
    ra, rb = py_line_records(old, ext_old), py_line_records(new, ext_new)
    ha, hb = [r[0] for r in ra], [r[0] for r in rb]
    fa, fb = [r[2] for r in ra], [r[2] for r in rb]
    s = py_diff_script(ha, hb, fa, fb)
    deleted, inserted = set(s[7]), set(s[8])
    if s[0] + s[1] > TRACE_MAX_D:                        # untraced: the whole middle between the common prefix and suffix
        pre = 0
        while pre < len(ha) and pre < len(hb) and ha[pre] == hb[pre]:
            pre += 1
        suf = 0
        while suf < len(ha) - pre and suf < len(hb) - pre and ha[-1 - suf] == hb[-1 - suf]:
            suf += 1
        deleted, inserted = set(range(pre, len(ha) - suf)), set(range(pre, len(hb) - suf))
    corr = dict(zip([j for j in range(len(lb)) if j not in inserted], [i for i in range(len(la)) if i not in deleted]))
    ca, cb = py_cases(la, ext_old), py_cases(lb, ext_new)

    def stats(rng, flags, changed):
        h, e = rng
        return (e - h, sum(flags[h:e]), sum(1 for i in range(h, e) if i in changed),
                sum(1 for i in range(h, e) if i in changed and flags[i]))

    sa = [stats(c, fa, deleted) for c in ca]
    sb = [stats(c, fb, inserted) for c in cb]
    na = [py_case_name(la[h], ext_old) for h, _ in ca]
    nb = [py_case_name(lb[h], ext_new) for h, _ in cb]
    old_at = {h: k for k, (h, _) in enumerate(ca)}
    match = {}                                           # step 1: the header line is kept and corresponds to an old header
    for j, (h, _) in enumerate(cb):
        if h in corr and corr[h] in old_at:
            match[j] = old_at[corr[h]]
    used = set(match.values())                           # step 2: a name that occurs once among the unmatched of each side
    free_new = [j for j in range(len(cb)) if j not in match]
    free_old = [k for k in range(len(ca)) if k not in used]
    for j in free_new:
        same_new = [x for x in free_new if nb[x] == nb[j]]
        same_old = [k for k in free_old if na[k] == nb[j]]
        if len(same_new) == 1 and len(same_old) == 1:
            match[j] = same_old[0]
    used = set(match.values())
    rows = []
    for k, (h, _) in enumerate(ca):
        if k not in used:
            n, a, c, ca_ = sa[k]
            rows.append((na[k], "D", None, h + 1, None, n, None, a, None, c, None, ca_))
    for j, (h, _) in enumerate(cb):
        n, a, c, ca_ = sb[j]
        if j not in match:
            rows.append((nb[j], "A", h + 1, None, n, None, a, None, c, None, ca_, None))
            continue
        k = match[j]
        no, ao, co, cao = sa[k]
        if c or co or n != no:
            rows.append((nb[j], "M", h + 1, ca[k][0] + 1, n, no, a, ao, c, co, ca_, cao))
    return rows
