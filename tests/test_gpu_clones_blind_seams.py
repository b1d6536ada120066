"""`tsm_clones_blind` / `Scanner.clones(..., blind=True)` (docs/SPEC.md section 21) where tests/test_gpu_clones_blind.py never
reaches: every lexer construct at every line start and construct start modulo 8 (k_blind_lines reads through one cached 8-byte
word and reloads it when a lookahead crosses into the next), the SWAR identity filter of k_blind_state with the only quote or
'*' of a line at its bytes 0, 7, 8 and last and with a neighbour line's quote in a shared word, every keyword-table lookup
kind (every name in both families, each one byte longer and shorter, 16- and 17-byte identifiers, probes that walk the table's
chains and one that wraps from slot 511 to slot 0), the line-state scan across 32-line rounds with transfer functions that do
not commute, and the kept-assertion reduction of k_blind_files.  Every output array is compared with the C reference
(tests/orc_blind.c), and the blind hash of every kept line with bytes_hash of blind_ref's blind form, so that a failure names
the line.  The builders are in tests/front_seams.py, checked on the CPU by tests/test_clones_blind_ref.py; each test asserts
that its corpus reaches its seams."""
import numpy as np
import pytest

import blind_ref as br
import front_seams as fs
import orc_blind as ob
import spec_ref
import tosemscan as ts

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scanner():
    s = ts.Scanner(device=0, max_arena_bytes=1 << 24, max_files=1 << 12, max_groups=4)
    yield s
    s.close()


def check(s, files, exts, n=2):
    c = ts.pack(files, np.asarray(exts, np.uint8))
    got = s.clones(c, n, blind=True)
    lines = [ln for d in files for ln in spec_ref.py_lines(d)]
    forms = [f for d, e in zip(files, exts) for f in br.blind_lines(d, e)]
    kept = np.zeros(len(forms), bool)
    kept[got["kept_line"]] = True
    bad = np.nonzero(kept != np.array([bool(f) for f in forms], bool))[0]
    assert len(bad) == 0, "line %d %r: blind form %r, kept %s" % (bad[0], lines[bad[0]], forms[bad[0]], kept[bad[0]])
    for i, h in zip(got["kept_line"].tolist(), got["blind_hash"].tolist()):
        assert h == spec_ref.py_bytes_hash(forms[i]), "line %d %r: blind form %r" % (i, lines[i], forms[i])
    br.assert_equal(got, ob.clones_blind(c, n))
    return got


def test_constructs_on_the_load_grid(scanner):
    files, exts, reach = fs.blind_grid_corpus()
    assert all(fs.on_the_grid(reach).values()) and len(reach) == len(fs.PY_CONSTRUCTS) + len(fs.CJ_CONSTRUCTS)
    check(scanner, files, exts)


def test_identity_filter(scanner):
    files, exts, reach = fs.filter_corpus()
    for fam in ("py", "cj"):
        assert all(reach[(fam, k)] == set(range(8)) for k in ("byte0", "byte7", "byte8", "last"))
        assert reach[(fam, "neighbour_before")] and reach[(fam, "neighbour_after")]
    check(scanner, files, exts)


def test_keyword_table(scanner):
    files, exts, reach = fs.keyword_corpus()
    assert reach["searched_walk"] and reach["wraps"] and len(reach["displaced_found"]) == 12
    got = check(scanner, files, exts, 1)
    assert len(got["kept_line"]) == 2 * len(files[0].split(b"\n")[:-1])


def test_line_state_scan_across_rounds(scanner):
    files, exts, reach = fs.scan_corpus()
    for ext, n, lanes in reach["lanes"][:10]:
        assert {(l, r) for l in (0, 1, 30, 31) for r in range(n // 32 + 1) if 32 * r + l < n} <= set(lanes), (ext, n)
    assert reach["permutation"] and reach["noncommuting_neighbours"] >= 20
    got = check(scanner, files, exts, 1)
    kb = got["kept_base"]
    assert kb[11] - kb[10] == 1 and kb[12] == kb[11] and kb[14] - kb[13] == 1


def test_kept_assertions_per_file(scanner):
    files, exts, reach = fs.files_corpus()
    got = check(scanner, files, exts, 1)
    assert got["file_kept_assert"].tolist() == reach["asserts"]
    assert got["kept_base"][-4:].tolist() == [got["kept_base"][-1]] * 4
