"""Plain-Python reference of the blind clones of docs/SPEC.md section 21.  TEST INFRASTRUCTURE ONLY.

* `lex_line(line, fam, state)`: the tokens that begin on one line (no LF) and the cross-line state after it;
* `blind_lines(data, ext)`: the blind form of every line of a file (section 2 lines);
* `py_blind_clones(files, exts, n)`: section 15 over the kept lines, windows equal when their blind forms are equal (content
  equality, independent of the hash).  Returns the dict of `tosemscan.Scanner.clones(..., blind=True)`.
"""
import numpy as np

import spec_ref

PY_KEYWORDS = frozenset(b"""and as assert async await break class continue def del elif else except finally for from global if
import in is lambda nonlocal not or pass raise return try while with yield""".split())
CJ_KEYWORDS = frozenset(b"""_ _Alignas _Alignof _Atomic _Bool _Complex _Generic _Imaginary _Noreturn _Static_assert _Thread_local
abstract alignas alignof and and_eq asm assert auto bitand bitor bool boolean break byte case catch char char16_t char32_t char8_t
class co_await co_return co_yield compl concept const const_cast consteval constexpr constinit continue decltype default delete do
double dynamic_cast else enum explicit export extends extern final finally float for friend goto if implements import inline
instanceof int interface long mutable namespace native new noexcept not not_eq operator or or_eq package private protected public
register reinterpret_cast requires restrict return short signed sizeof static static_assert static_cast strictfp struct super switch
synchronized template this thread_local throw throws transient try typedef typeid typename union unsigned using virtual void
volatile wchar_t while xor xor_eq""".split())
PY_LITERALS = frozenset([b"True", b"False", b"None"])
CJ_LITERALS = frozenset([b"true", b"false", b"null", b"nullptr"])
CJ_PREFIXES = frozenset([b"L", b"u", b"U", b"u8", b"R", b"LR", b"uR", b"UR", b"u8R"])

NONE, PY, CJ = 0, 1, 2
CODE = 0                                                 # PY 1 / 2: inside a triple-quoted " / ' literal; CJ 1: inside /* */
W = spec_ref.W
ALNUM_ = frozenset(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_")
DIGITS = frozenset(b"0123456789")


def family(ext):
    return PY if ext == 1 else CJ if 2 <= ext <= 6 else NONE


def _ident_byte(c):
    return c in ALNUM_ or c == 0x24 or c >= 0x80


def _close(line, i, fam, state):
    """Index behind the delimiter that closes `state`, searched from i; None when the line holds none."""
    if fam == CJ:
        k = line.find(b"*/", i)
        return None if k < 0 else k + 2
    triple = (b'"' if state == 1 else b"'") * 3
    n = len(line)
    while i < n:
        if line[i] == 0x5C:
            i += 2
        elif line[i:i + 3] == triple:
            return i + 3
        else:
            i += 1
    return None


def _string(line, i, fam):
    """The literal whose quote is at i: (index behind it, state after it)."""
    q, n = line[i], len(line)
    if fam == PY and line[i:i + 3] == bytes([q]) * 3:
        st = 1 if q == 0x22 else 2
        j = _close(line, i + 3, fam, st)
        return (n, st) if j is None else (j, CODE)
    j = i + 1
    while j < n:
        if line[j] == 0x5C:
            j += 2
        elif line[j] == q:
            return j + 1, CODE
        else:
            j += 1
    return n, CODE


def _number(line, i, fam):
    n, j = len(line), i + 1
    while j < n:
        c = line[j]
        if c in ALNUM_ or c == 0x2E or (c in b"+-" and line[j - 1] in b"eEpP"):
            j += 1
        elif fam == CJ and c == 0x27 and j + 1 < n and line[j + 1] in ALNUM_:
            j += 1
        else:
            break
    return j


def _is_prefix(word, fam):
    if fam == PY:
        return 1 <= len(word) <= 2 and all(c in b"rRbBuUfF" for c in word)
    return word in CJ_PREFIXES


def lex_line(line, fam, state):
    """(tokens that begin on the line, state at its end) for a line of family fam (PY or CJ) that starts in `state`."""
    toks, i, n = [], 0, len(line)
    if state != CODE:
        i = _close(line, 0, fam, state)
        if i is None:
            return toks, state
    kw, lit = (PY_KEYWORDS, PY_LITERALS) if fam == PY else (CJ_KEYWORDS, CJ_LITERALS)
    while i < n:
        c = line[i]
        nx = line[i + 1] if i + 1 < n else -1
        if c in W:
            i += 1
        elif fam == PY and c == 0x23:
            break
        elif fam == CJ and c == 0x2F and nx == 0x2F:
            break
        elif fam == CJ and c == 0x2F and nx == 0x2A:
            i = _close(line, i + 2, fam, 1)
            if i is None:
                return toks, 1
        elif c in DIGITS or (c == 0x2E and nx in DIGITS):
            i = _number(line, i, fam)
            toks.append(b"N")
        elif _ident_byte(c):
            j = i
            while j < n and _ident_byte(line[j]):
                j += 1
            word = line[i:j]
            if j < n and line[j] in b"\"'" and _is_prefix(word, fam):
                i, st = _string(line, j, fam)
                toks.append(b"S")
                if st != CODE:
                    return toks, st
                continue
            toks.append(word if word in kw else b"N" if word in lit else b"I")
            i = j
        elif c in b"\"'":
            i, st = _string(line, i, fam)
            toks.append(b"S")
            if st != CODE:
                return toks, st
        else:
            toks.append(bytes([c]))
            i += 1
    return toks, CODE


def blind_lines(data, ext):
    """The blind form of every line of a file, in order."""
    fam, state, out = family(int(ext)), CODE, []
    for line in spec_ref.py_lines(data):
        if fam == NONE:
            out.append(bytes(c for c in line if c not in W))
            continue
        toks, state = lex_line(line, fam, state)
        out.append(b" ".join(toks))
    return out


def blind_hash(form):
    return spec_ref.py_bytes_hash(form)


def clone_walk(key, flag, base, n):
    """Section 15 over a line sequence: key[p] (any hashable, equal keys = equal lines), flag[p] (assertion line) and the
    per-file bases; every line is non-empty.  Returns file_dup, file_dup_assert, class_base, class_len and member."""
    T, nf = len(key), len(base) - 1
    fid = np.searchsorted(np.asarray(base, np.int64), np.arange(T), side="right") - 1
    groups, wkey = {}, [None] * T
    for p in range(T):
        if p + n <= base[fid[p] + 1]:
            wkey[p] = tuple(key[p:p + n])
            groups.setdefault(wkey[p], []).append(p)

    def ext_of(g):
        preds = set()
        for q in g:
            if q == base[fid[q]] or wkey[q - 1] is None:
                return False
            preds.add(wkey[q - 1])
        return len(preds) == 1 and len(groups[preds.pop()]) == len(g)

    extendable = {k: len(g) >= 2 and ext_of(g) for k, g in groups.items()}
    covered = [False] * T
    class_base, class_len, member = [0], [], []
    for p in range(T):
        k = wkey[p]
        if k is None or len(groups[k]) < 2:
            continue
        for x in range(p, p + n):
            covered[x] = True
        if extendable[k] or groups[k][0] != p:
            continue
        r = 0
        while p + r + 1 < T and fid[p + r + 1] == fid[p] and wkey[p + r + 1] is not None and len(groups[wkey[p + r + 1]]) >= 2 \
                and extendable[wkey[p + r + 1]]:
            r += 1
        class_len.append(n + r)
        member += groups[k]
        class_base.append(len(member))
    dup = [sum(covered[base[f]:base[f + 1]]) for f in range(nf)]
    dup_a = [sum(1 for x in range(base[f], base[f + 1]) if covered[x] and flag[x]) for f in range(nf)]
    return {"file_dup": np.array(dup, np.uint32), "file_dup_assert": np.array(dup_a, np.uint32),
            "class_base": np.array(class_base, np.int64), "class_len": np.array(class_len, np.uint32),
            "member": np.array(member, np.int64)}


def py_blind_clones(files, exts, n):
    """Section 21: section 15 over the kept lines of the files, windows compared by blind form."""
    forms, flag, kept_line, line_base, kept_base, kept_assert = [], [], [], [0], [0], []
    for data, e in zip(files, exts):
        lines = spec_ref.py_lines(data)
        a = 0
        for k, (line, form) in enumerate(zip(lines, blind_lines(data, e))):
            if form:
                f = spec_ref.py_is_assert_line(line, int(e))
                forms.append(form)
                flag.append(f)
                kept_line.append(line_base[-1] + k)
                a += f
        line_base.append(line_base[-1] + len(lines))
        kept_base.append(len(forms))
        kept_assert.append(a)
    out = clone_walk(forms, flag, kept_base, n)
    out.update(line_base=np.array(line_base, np.int64), kept_base=np.array(kept_base, np.int64),
               kept_line=np.array(kept_line, np.int64), blind_hash=np.array([blind_hash(f) for f in forms], np.uint64),
               file_kept_assert=np.array(kept_assert, np.uint32))
    return out


KEYS = ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len", "member", "kept_base", "kept_line", "blind_hash",
        "file_kept_assert")


def assert_equal(got, want):
    for k in KEYS:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k
