"""Plain-Python restatement of the moved code of docs/SPEC.md section 20 (test infrastructure): the edit script of
spec_ref.py_diff_script, then runs, matches, reaches and the greedy block walk exactly as the section words them, with dicts and
direct walks.  Written from the SPEC text; no shared code with the kernels or tests/orc_moves.py."""
import spec_ref as sr

TRACE_MAX_D = 23168                          # the largest distance the device traces (include/tosemscan.h)
MIN_ALNUM = 20                               # git's COLOR_MOVED_MIN_ALNUM_COUNT


def alnum(line: bytes) -> int:
    """The [A-Za-z0-9] bytes of a section-2 line (no LF; a CR is not one of them)."""
    return sum(1 for c in line if 48 <= c <= 57 or 65 <= c <= 90 or 97 <= c <= 122)


def py_changed(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """(deleted, inserted) line index sets of one pair: the canonical script's, or the whole middle of an untraced pair."""
    ra, rb = sr.py_line_records(old, ext_old), sr.py_line_records(new, ext_new)
    ha, hb = [r[0] for r in ra], [r[0] for r in rb]
    s = sr.py_diff_script(ha, hb, [r[2] for r in ra], [r[2] for r in rb])
    if s[0] + s[1] <= TRACE_MAX_D or not s[7] or not s[8]:   # (a pure hunk is its whole middle at any distance)
        return set(s[7]), set(s[8])
    pre = 0
    while pre < len(ha) and pre < len(hb) and ha[pre] == hb[pre]:
        pre += 1
    suf = 0
    while suf < len(ha) - pre and suf < len(hb) - pre and ha[-1 - suf] == hb[-1 - suf]:
        suf += 1
    return set(range(pre, len(ha) - suf)), set(range(pre, len(hb) - suf))


def py_moves(pairs, steps=None):
    """pairs: [(old bytes, new bytes, ext_old, ext_new)], steps: the step of every pair (default: all in step 0).  Returns a dict
    with, per side ('old', 'new'), 'blocks': [(line, partner, n_lines, n_assert)] in line order (global lines of each side:
    pairs in order, then lines), 'moved': the set of moved global lines, 'changed': the set of changed global lines, and
    'base': the first global line of every pair (plus the total)."""
    steps = list(steps) if steps is not None else [0] * len(pairs)
    side = {s: {"hash": [], "text": [], "flag": [], "step": [], "run": [], "changed": set(), "base": [0]} for s in ("old", "new")}
    for (old, new, eo, en), st in zip(pairs, steps):
        dl, ins = py_changed(old, new, eo, en)
        for name, data, ext, chg in (("old", old, eo, dl), ("new", new, en, ins)):
            S = side[name]
            b = S["base"][-1]
            lines = sr.py_lines(data)
            run = None
            for i, (ln, rec) in enumerate(zip(lines, sr.py_line_records(data, ext))):
                g = b + i
                S["hash"].append(rec[0]); S["text"].append(ln); S["flag"].append(rec[2]); S["step"].append(st)
                if i in chg:
                    S["changed"].add(g)
                    run = run if run is not None and (i - 1) in chg else g   # a run: its first line
                else:
                    run = None
                S["run"].append(run)
            S["base"].append(b + len(lines))
    O, N = side["old"], side["new"]

    def in_run(S, x, r):
        return x < len(S["run"]) and S["run"][x] == r

    def length(X, Y, x, c):                  # len(x, c) of step 3
        rx, rc, L = X["run"][x], Y["run"][c], 0
        while in_run(X, x + L, rx) and in_run(Y, c + L, rc) and X["hash"][x + L] == Y["hash"][c + L]:
            L += 1
        return L

    out = {}
    for name, X, Y in (("old", O, N), ("new", N, O)):
        by_key = {}
        for c in sorted(Y["changed"]):
            by_key.setdefault((Y["step"][c], Y["hash"][c]), []).append(c)
        reach = {}                           # x -> (L(x), partner(x)) for x with a match
        for x in X["changed"]:
            best = (0, None)
            for c in by_key.get((X["step"][x], X["hash"][x]), []):
                L = length(X, Y, x, c)
                if L > best[0]:              # candidates ascend: the first of the longest is the smallest
                    best = (L, c)
            if best[0]:
                reach[x] = best
        blocks, moved = [], set()
        for x0 in sorted(X["changed"]):
            if X["run"][x0] != x0:
                continue                     # each run from its first line
            x = x0
            while in_run(X, x, x0):
                L, p = reach.get(x, (0, None))
                if L and sum(alnum(X["text"][x + k]) for k in range(L)) >= MIN_ALNUM:
                    blocks.append((x, p, L, sum(X["flag"][x:x + L])))
                    moved.update(range(x, x + L))
                    x += L
                else:
                    x += 1
        out[name] = {"blocks": blocks, "moved": moved, "changed": X["changed"], "base": X["base"]}
    return out


def file_moved(res, name, pair):
    """The moved lines of one pair's file on one side, 0-based in the file."""
    base = res[name]["base"]
    return sorted(g - base[pair] for g in res[name]["moved"] if base[pair] <= g < base[pair + 1])
