"""Plain-Python restatements of docs/SPEC.md (test infrastructure): big integers and dicts, no shared code with the
oracle or the kernels, so that a rule both of them get wrong the same way still shows up."""
import os

M61 = (1 << 61) - 1
MASK = (1 << 64) - 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = b" \t\r\x0b\x0c"


def mix(h61: int, n: int) -> int:
    """The finaliser of SPEC section 3 (xor-shift-multiply of h61 and a length)."""
    x = h61 ^ ((n * 0x9E3779B97F4A7C15) & MASK)
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & MASK
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & MASK
    x ^= x >> 31
    return x


def py_bytes_hash(b: bytes) -> int:
    """SPEC section 3 with Python big integers."""
    return mix(int.from_bytes(b, "little") % M61, len(b))


def py_lines(data: bytes):
    """SPEC section 2."""
    if not data:
        return []
    parts = data.split(b"\n")
    if parts[-1] == b"":
        parts.pop()
    return parts


def py_is_assert_line(line: bytes, ext: int) -> bool:
    """SPEC section 4 (Rev A trigger)."""
    return ext != 0 and (b"assert" in line.lower() or b"EXPECT_" in line)


def py_line_records(data: bytes, ext: int = 1):
    """SPEC sections 2-3: (line_hash, line_end, line_flag) of every line of one file.  line_end is the position of the
    line's LF, or the file size for an unterminated last line; one trailing CR is not part of the hashed content."""
    out, pos = [], 0
    for line in py_lines(data):
        end = pos + len(line)
        content = line[:-1] if line.endswith(b"\r") else line
        out.append((py_bytes_hash(content), end, int(py_is_assert_line(line, ext))))
        pos = end + 1
    return out


def py_ngrams(hashes, n: int):
    """SPEC section 3 n-gram hashes of one file's line hashes (windows shorten at the end of the file)."""
    hs = [int(h) % M61 for h in hashes]
    out = []
    for i in range(len(hs)):
        m = min(n, len(hs) - i)
        acc = sum(hs[i + k] << (13 * k) for k in range(m)) % M61
        out.append(mix(acc, m))
    return out


def py_statement(line: bytes) -> bytes:
    """SPEC section 4: T = the stripped line cut before its first '(', right-stripped."""
    return line.strip(W).split(b"(", 1)[0].rstrip(W)


def _table():
    names = [ln.strip() for ln in open(os.path.join(ROOT, "spec", "categories.txt"))]
    names = [n for n in names if n and not n.startswith("#")]
    return {n.encode(): i for i, n in enumerate(names, start=1)}


CATEGORY_IDS = _table()
CATEGORY_NAMES = {i: n.decode() for n, i in CATEGORY_IDS.items()}
OTHER = 127
STEMS = {b"EQ": "assertEqual", b"NE": "assertNotEqual", b"TRUE": "assertTrue", b"FALSE": "assertFalse",
         b"GT": "assertGreater", b"GE": "assertGreaterEqual", b"LT": "assertLess", b"LE": "assertLessEqual",
         b"NEAR": "assertAlmostEqual", b"FLOAT_EQ": "assertFloatEqual", b"DOUBLE_EQ": "assertDoubleEqual",
         b"THROW": "assertRaises"}


def _ident(c: int) -> bool:
    return 48 <= c <= 57 or 65 <= c <= 90 or 97 <= c <= 122 or c == 95


def py_ident(t: bytes):
    """L of SPEC section 6: (offset, length) of the longest [A-Za-z0-9_] suffix of T."""
    s = len(t)
    while s and _ident(t[s - 1]):
        s -= 1
    return s, len(t) - s


def py_category(t: bytes) -> int:
    """SPEC section 6 (Rev A): the category id of a statement T."""
    s, n = py_ident(t)
    L = t[s:]
    name = CATEGORY_IDS.get
    if L.startswith(b"EXPECT_") or L.startswith(b"ASSERT_"):
        stem = STEMS.get(L[7:])
        return name(stem.encode()) if stem else 0
    if t == b"assert" or t.startswith(b"assert "):
        e = t[7:]
        if e.startswith(b"not "):
            r = "assertNotEqual"
        elif (b" not " in e and b" in " in e) or b" is not " in e:
            r = "assertFalse"
        else:
            r = next((c for op, c in ((b"True", "assertTrue"), (b"==", "assertEqual"), (b"!=", "assertNotEqual"),
                                      (b"<=", "assertLessEqual"), (b">=", "assertGreaterEqual"), (b"<", "assertLess"),
                                      (b">", "assertGreater")) if op in e), "assertTrue")
        return name(r.encode())
    if L == b"assert_":
        return name(b"assertTrue")
    if L.startswith(b"assert"):
        return name(L, OTHER)
    return 0


def py_category_string(t: bytes) -> str:
    """The category cell the lost tool printed: the table name, or the verbatim identifier for OTHER."""
    c = py_category(t)
    if c == OTHER:
        s, n = py_ident(t)
        return t[s:s + n].decode("latin-1")
    return CATEGORY_NAMES.get(c, "")


def py_diff_script(a, b, fa, fb):
    """SPEC section 8 as written, for line-hash lists a (old) and b (new) with assertion flags fa, fb.  Returns (added,
    removed, hunks_add, hunks_del, hunks_mod, added_assert, removed_assert, deleted_idx, inserted_idx): the deleted lines
    of a and the inserted lines of b as indices into the whole lists, in line order."""
    n0, m0 = len(a), len(b)
    pre = 0                                              # step 1: common prefix, then common suffix of the rest
    while pre < n0 and pre < m0 and a[pre] == b[pre]:
        pre += 1
    suf = 0
    while suf < n0 - pre and suf < m0 - pre and a[n0 - 1 - suf] == b[m0 - 1 - suf]:
        suf += 1
    A, B = a[pre:n0 - suf], b[pre:m0 - suf]
    n, m = len(A), len(B)
    if n == 0 or m == 0:                                 # the remainder is one pure hunk (or nothing)
        deleted, inserted = list(range(n)), list(range(m))
        hunks = [("del" if n else "add")] if n + m else []
        D = n + m
    else:
        V, rows, D = {1: 0}, [], None                    # step 2: rows[d][k] = furthest x on diagonal k after d edits
        for d in range(n + m + 1):
            row = {}
            for k in range(-d, d + 1, 2):
                if k == -d or (k != d and V[k - 1] < V[k + 1]):
                    x = V[k + 1]
                else:
                    x = V[k - 1] + 1
                y = x - k
                while x < n and y < m and A[x] == B[y]:
                    x += 1
                    y += 1
                row[k] = x
            V.update(row)
            rows.append(row)
            if row.get(n - m, -1) >= n:
                D = d
                break
        edits, x, y = [], n, m                           # step 3: (kind, x, y) where each edit starts, last to first
        for d in range(D, 0, -1):
            k, P = x - y, rows[d - 1]
            down = k == -d or (k != d and P[k - 1] < P[k + 1])
            pk = k + 1 if down else k - 1
            px = P[pk]
            py = px - pk
            edits.append(("ins" if down else "del", px, py))
            x, y = px, py
        edits.reverse()
        deleted = [ex for kind, ex, ey in edits if kind == "del"]
        inserted = [ey for kind, ex, ey in edits if kind == "ins"]
        hunks, cur, at = [], set(), None                 # a hunk: edits with no match between them
        for kind, ex, ey in edits:
            if at is not None and (ex, ey) != at:
                hunks.append(cur)
                cur = set()
            cur.add(kind)
            at = (ex + 1, ey) if kind == "del" else (ex, ey + 1)
        hunks.append(cur)
        hunks = ["mod" if len(h) == 2 else ("add" if "ins" in h else "del") for h in hunks]
    lcs = pre + suf + (n + m - D) // 2
    deleted = [pre + i for i in deleted]
    inserted = [pre + j for j in inserted]
    return (m0 - lcs, n0 - lcs, hunks.count("add"), hunks.count("del"), hunks.count("mod"),
            sum(1 for j in inserted if fb[j]), sum(1 for i in deleted if fa[i]), deleted, inserted)


def py_diff_files(old: bytes, new: bytes, ext_old: int, ext_new: int):
    """py_diff_script of two files, from their line records (SPEC sections 2-4)."""
    ra, rb = py_line_records(old, ext_old), py_line_records(new, ext_new)
    return py_diff_script([r[0] for r in ra], [r[0] for r in rb], [r[2] for r in ra], [r[2] for r in rb])


def py_line_starts(data: bytes):
    """File-relative start of every line (the line_off of its events)."""
    out, pos = [], 0
    for line in py_lines(data):
        out.append(pos)
        pos += len(line) + 1
    return out
