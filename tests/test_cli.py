"""The C++ host driver `tosem-scan`: CSV schemas of the reference's shipped tables, rows built by the
product (GPU events + host method strings) against rows built from the oracle's line functions."""
import collections
import csv
import io
import os
import subprocess

import numpy as np
import pytest

import corpus_util as cu
import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "tosem-2021-replication_b200", "tosemscan", "tosem-scan")
EXT = {"py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}


def test_cli_builds_and_prints_usage():
    assert os.path.exists(CLI), "run __graft_entry__.build()"
    out = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert out.returncode == 0 and "tosem-scan scan" in out.stderr


def make_tree(root):
    files = {
        "tests/test_agent.py": cu.PY_SAMPLE,
        "modules/perception/fusion/common/dst_evidence_test.cc": cu.CC_SAMPLE,
        "integration/java/MapDecodeTest.java": cu.JAVA_SAMPLE,
        "external/lib/test_api.py": b"def test_fastCopyAndTranspose():\n    assert_equal(b, a.T)\n    assert_equal(b, a.T)\n",
        "third_party/protobuf-3.5/smoke/unit_test.cpp": b"TEST_F(Fix, A) {\n  EXPECT_EQ(1, 2);\n  EXPECT_EQ(1,\n 2);\n}\nvoid g() { ASSERT_TRUE(x); }\n",
        "regression/weird,name\"test.c": b"int testmain(void) {\n  assert(x == \"a,b\");\n  assert(x == \"a,b\");\n}\n",
        "src/main.py": b"assert False\n",                      # no `test` in the path: not selected
        "tests/data.json": b'{"assert": 1}\n',                  # no scannable extension: no rows
        "tests/empty_test.py": b"",
    }
    for rel, data in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        open(p, "wb").write(data)
    return files


def tag(rel, fixture):
    if rel.startswith("external/"):
        t = "external"
    elif "integration" in rel:
        t = "integration"
    elif "regression" in rel:
        t = "regression"
    elif "swarming" in rel:
        t = "swarming"
    else:
        t = "unit_test"
    comps = rel.split("/")[:-1]
    if any(c.startswith("protobuf-") for c in comps):
        t += ", Protocol Buffers"
    if "smoke" in comps:
        t += ", smoke"
    return t + (", Fixture" if fixture else "")


def expected(files):
    """Rows and per-file summaries from the oracle's line-level functions (docs/SPEC.md sections 2-7)."""
    rows, summ = [], []
    sel = sorted((r for r in files if "test" in r.lower() and r.rsplit(".", 1)[-1] in EXT), key=lambda r: r.split("/"))
    for i, rel in enumerate(sel, start=1):
        data, ext = files[rel], EXT[rel.rsplit(".", 1)[-1]]
        cur = (-1, False, b"xxxx")
        keyed = collections.OrderedDict()
        hist = collections.OrderedDict()
        pos = 0
        while pos < len(data):
            e = data.find(b"\n", pos)
            e = len(data) if e < 0 else e
            line = data[pos:e]
            hk = orc.header_kind(ext, line)
            if hk:
                cur = (pos, bool(hk & 2), orc.method_string(ext, line))
            if orc.is_assert_line(line):
                st = orc.statement(line)
                cat = orc.category_string(st)
                k = (cur[0], st)
                if k not in keyed:
                    keyed[k] = [cur, st, cat, 0]
                keyed[k][3] += 1
                hist[cat] = hist.get(cat, 0) + 1
            pos = e + 1
        for cur_, st, cat, n in keyed.values():
            rows.append([rel, rel.rsplit(".", 1)[-1], tag(rel, cur_[1]), cur_[2].decode("latin-1"), st.decode("latin-1"), str(n), cat])
        order = sorted(hist, key=lambda c: -hist[c])
        summ.append([str(i), rel, str(sum(hist.values())), ", ".join("%d:%s" % (hist[c], c) for c in order)])
    return rows, summ


def read_csv(path):
    raw = open(path, "rb").read()
    assert b"\n" not in raw.replace(b"\r\n", b""), "CRLF line ends only"
    return list(csv.reader(io.StringIO(raw.decode("latin-1"), newline="")))


@pytest.mark.gpu
def test_scan_rows_and_summary(tmp_path):
    files = make_tree(str(tmp_path / "proj"))
    rows_p, sum_p = str(tmp_path / "rows.csv"), str(tmp_path / "summary.csv")
    out = subprocess.run([CLI, "scan", str(tmp_path / "proj"), "--rows", rows_p, "--summary", sum_p], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    want_rows, want_sum = expected(files)
    got = read_csv(rows_p)
    assert got[0] == ["fileName", "extension", "test_name", "method", "statement", "counts", "category"]
    assert got[1:] == want_rows
    gs = read_csv(sum_p)
    assert gs[0] == ["Id", "FileName", "total assert", "assertion"] and gs[1:] == want_sum
    # spot checks against the reference's own example cells (ML-Testing-v1.xlsx!apollo_tests:R8-R10, !prefect_tests:R2)
    flat = {(r[0], r[3], r[4]): r for r in got[1:]}
    r = flat[("modules/perception/fusion/common/dst_evidence_test.cc", ': sensor1_dst_("test"', "EXPECT_NEAR")]
    assert r[2] == "unit_test" and r[5] == "1" and r[6] == "assertAlmostEqual"
    r = flat[("tests/test_agent.py", "test_docker_agent_init(monkeypatch,runner_token)", "assert agent.labels == []")]
    assert r[6] == "assertEqual"
    assert flat[("third_party/protobuf-3.5/smoke/unit_test.cpp", "TEST_F(Fix, A", "EXPECT_EQ")][2] == "unit_test, Protocol Buffers, smoke, Fixture"
    assert flat[("external/lib/test_api.py", "test_fastCopyAndTranspose()", "assert_equal")][5] == "2"
    # the aggregate table on stdout sums to the number of assertion lines
    agg = [l.split(",") for l in out.stdout.replace("\r\n", "\n").strip().split("\n")[1:]]
    assert sum(int(a[-1]) for a in agg) == sum(int(s[2]) for s in want_sum)


@pytest.mark.gpu
def test_reduce_tables(tmp_path):
    rng = np.random.default_rng(5)
    repos = ["autokeras", "auto_sklearn", "tpot", "Ray", "DeepSpeech2", "google_automl", "nni", "Apollo", "Nupic"]
    cols = ["Index", "Labels", "Cases", "Repo", "Data", "Model", "status_test", "Error_Type", "negative_test", "logical_statement",
            "logical_expression", "null_pointer", "value_range", "Approximation_Type", "checks_type", "regression",
            "Integration", "mock_test", "API"]
    lines, recs = [cols], []
    for i in range(600):
        repo = repos[int(rng.integers(0, 9))]
        rec = {"Index": str(i), "Labels": 'a "quoted", label\nwith a newline' if i % 50 == 0 else "x", "Cases": str(int(rng.integers(0, 120))) + repo[:2],
               "Repo": repo, "Data": ["", "Distribution", "Validity", "Data Error", "Time behaviour"][int(rng.integers(0, 5))],
               "Model": ["", "", "Resource Usage", "Compatibility"][int(rng.integers(0, 4))], "status_test": str(int(rng.random() < 0.3)), "Error_Type": ["", "ValueError", "RuntimeError", "Exception", "nullptr", "SyntaxError", "SchemaError", "FileError",
                              "AssertionError", "Timeout", "DataError"][int(rng.integers(0, 11))],
               "negative_test": str(int(rng.random() < 0.2)), "logical_statement": "0", "logical_expression": str(int(rng.random() < 0.1)),
               "null_pointer": "0", "value_range": str(int(rng.random() < 0.4)), "Approximation_Type": ["", "rounding_tolence"][int(rng.integers(0, 2))],
               "checks_type": ["", "instance_check"][int(rng.integers(0, 2))], "regression": "0", "Integration": str(int(rng.random() < 0.05)),
               "mock_test": str(int(rng.random() < 0.1)), "API": ""}
        recs.append(rec)
        lines.append([rec[c] for c in cols])
    tax = tmp_path / "taxonomy.csv"
    with open(tax, "w", newline="", encoding="utf-8") as f:
        csv.writer(f, lineterminator="\r\n").writerows(lines)
    sp, mp, pp = str(tmp_path / "s.csv"), str(tmp_path / "m.csv"), str(tmp_path / "p.csv")
    out = subprocess.run([CLI, "reduce", str(tax), "--strategy", sp, "--methods", mp, "--properties", pp], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    s = read_csv(sp)
    assert s[0][:10] == ["Tests"] + repos
    cases = {r: {x["Cases"] for x in recs if x["Repo"] == r} for r in repos}
    row = {x[0]: x for x in s[1:]}
    for name, pred in [("status_analysis", lambda x: x["status_test"] == "1"), ("value_error", lambda x: x["Error_Type"] == "ValueError"),
                       ("runtime_error", lambda x: x["Error_Type"] in ("RuntimeError", "Exception", "nullptr", "Timeout")),   # merged rows (SPEC section 9)
                       ("AssertionError", lambda x: x["Error_Type"] in ("AssertionError", "SyntaxError")),
                       ("FileError", lambda x: x["Error_Type"] in ("FileError", "SchemaError")),
                       ("logical_condition", lambda x: x["logical_statement"] == "1" or x["logical_expression"] == "1"),
                       ("rounding_tolence", lambda x: x["Approximation_Type"] == "rounding_tolence")]:
        for k, r in enumerate(repos):
            d = len({x["Cases"] for x in recs if x["Repo"] == r and pred(x)})
            v = round(round(100.0 * d / len(cases[r]), 4) / 1.1, 4)
            assert row[name][1 + k] == (("%.4f" % v).rstrip("0").rstrip(".") or "0"), (name, r)
    # property table: rows = repositories, cells = 100 * distinct / (Apollo's case count)
    pt = read_csv(pp)
    assert pt[0][0] == "Repos" and len(pt[0]) == 22 and [x[0] for x in pt[1:]][:2] == ["auto_sklearn", "google_automl"]
    prow = {x[0]: x for x in pt[1:]}
    for name, labels in [("Data Distribution", {"Distribution"}), ("Data Validity", {"Validity", "Data Error"}),
                         ("Efficiency", {"Time behaviour", "Resource Usage"}), ("Compatibility and Portability", {"Compatibility"})]:
        j = pt[0].index(name)
        for r in repos:
            dd = len({x["Cases"] for x in recs if x["Repo"] == r and (x["Data"] in labels or x["Model"] in labels)})
            assert prow[r][j] == (("%.4f" % round(100.0 * dd / len(cases["Apollo"]), 4)).rstrip("0").rstrip(".") or "0"), (name, r)
    m = {x[0]: x for x in read_csv(mp)[1:]}
    tot = sum(len(c) for c in cases.values())
    d = len({(x["Repo"], x["Cases"]) for x in recs if x["mock_test"] not in ("", "0")})
    assert m["mock_test"][1] == str(d) and m["mock_test"][2] == (("%.4f" % round(100.0 * d / tot, 4)).rstrip("0").rstrip(".") or "0")


@pytest.mark.gpu
def test_reduce_reproduces_the_shipped_tables(tmp_path):
    """The CLI on the package's own taxonomy (the columns it reads, tests/golden/taxonomy_min.csv.gz): every cell the
    ledger marks reproducible must come out bit-identical to RQs/RQ3/tests_strategy_rq32.csv, tests_prop_rq3.csv and
    RQs/RQ4/tests_methods_v2.csv (shipped cells kept in tests/golden/g3_reduce.npz)."""
    import gzip
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    tax = tmp_path / "taxonomy.csv"
    tax.write_bytes(gzip.open(os.path.join(gold, "taxonomy_min.csv.gz"), "rb").read())
    sp, mp, pp, cp = str(tmp_path / "s.csv"), str(tmp_path / "m.csv"), str(tmp_path / "p.csv"), str(tmp_path / "c.csv")
    ctex, ccnt, cmer = str(tmp_path / "ctex.csv"), str(tmp_path / "ccnt.csv"), str(tmp_path / "cmer.csv")
    out = subprocess.run([CLI, "reduce", str(tax), "--strategy", sp, "--methods", mp, "--properties", pp, "--correlate", cp,
                          "--correlate-tex", ctex, "--correlate-counts", ccnt, "--correlate-merged", cmer], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    d = np.load(os.path.join(gold, "g3_reduce.npz"))
    repos = [str(x) for x in d["repo_names"]]
    names = [str(x) for x in d["flag_names"]]
    s = read_csv(sp)
    assert s[0][1:10] == repos
    srow = {x[0]: x for x in s[1:]}
    ok, want = d["strategy_cell_reproduces"], d["want_strategy_cells"]
    n_ok = 0
    for j in range(ok.shape[0]):
        for k in range(ok.shape[1]):
            if ok[j, k]:
                assert srow[names[j]][1 + k] == str(want[j][k]), (names[j], repos[k])
                n_ok += 1
    assert n_ok == 171
    m = {x[0]: x for x in read_csv(mp)[1:]}
    mnames = [n[2:] for n in names if n.startswith("m:")]
    for j, name in enumerate(mnames):
        if d["method_reproduces"][j]:
            assert int(m[name][1]) == int(d["want_method_total_cases"][j]), name
    pt = read_csv(pp)
    prow = {x[0]: x for x in pt[1:]}
    pnames = [n[2:] for n in names if n.startswith("p:")]
    assert pt[0][1:] == pnames
    pok, pwant = d["property_cell_reproduces"], d["want_property_cells"]
    n_ok = 0
    for j in range(pok.shape[0]):
        for k in range(pok.shape[1]):
            if pok[j, k]:
                assert prow[repos[k]][1 + j] == str(pwant[j][k]), (pnames[j], repos[k])
                n_ok += 1
    assert n_ok == 172
    # RQs/RQ3/tests_correlate_rq3.csv: same header and row names, 394 of the 420 cells bit-identical; the other 26 are
    # checked against the oracle's distinct counts (the taxonomy revision shipped differs from the one the table was made from)
    ct = read_csv(cp)
    assert ct[0] == ["Tests"] + [str(x) for x in d["correlate_col_names"]]
    assert [x[0] for x in ct[1:]] == [str(x) for x in d["correlate_row_names"]]
    cok, cwant, cdist = d["correlate_cell_reproduces"], d["want_correlate_cells"], d["oracle_correlate_distinct"]
    order = [str(x) for x in d["correlate_repo_order"]]
    cpr = dict(zip(repos, (int(x) for x in d["oracle_cases_per_repo"])))
    n_ok = 0
    for j in range(cok.shape[0]):
        for q in range(cok.shape[1]):
            dd = [int(cdist[j * cok.shape[1] + q, repos.index(n)]) for n in order]
            mine = "0" if not any(dd) else "".join("%s:(%s%%), " % (n, repr(round(100.0 * v / cpr[n], 2))) for n, v in zip(order, dd))
            assert ct[1 + j][1 + q] == mine, (j, q)
            if cok[j, q]:
                assert ct[1 + j][1 + q] == str(cwant[j][q])
                n_ok += 1
    assert n_ok == 394
    # the same counts in the LaTeX layout (tests_correlate_rq4.csv) and as totals over the repositories (tests_combined_correlate_rq3.csv)
    tt, tn = read_csv(ctex), read_csv(ccnt)
    assert tt[0] == ct[0] and tn[0] == ct[0]
    tok, twant, nok, nwant = d["correlate_tex_cell_reproduces"], d["want_correlate_tex_cells"], d["correlate_count_cell_reproduces"], d["want_correlate_count_cells"]
    n_tex = n_cnt = 0
    for j in range(cok.shape[0]):
        for q in range(cok.shape[1]):
            dd = [int(cdist[j * cok.shape[1] + q, repos.index(n)]) for n in order]
            assert tn[1 + j][1 + q] == str(sum(dd))
            assert (tt[1 + j][1 + q] == "0") == (sum(dd) == 0)
            if tok[j, q]:
                assert tt[1 + j][1 + q] == str(twant[j][q]), (j, q)
                n_tex += 1
            if nok[j, q]:
                assert tn[1 + j][1 + q] == str(nwant[j][q]), (j, q)
                n_cnt += 1
    assert (n_tex, n_cnt) == (394, 382)
    # the four one-row tables of the merged strategy rows (tests_correlate_{FileError,RuntimeError,assertion,logical}.csv)
    tm = read_csv(cmer)
    assert tm[0] == ct[0] and [x[0] for x in tm[1:]] == [str(x) for x in d["merged_row_names"]]
    mok, mwant, mdist = d["merged_cell_reproduces"], d["want_merged_cells"], d["oracle_merged_distinct"]
    for j in range(mok.shape[0]):
        for q in range(mok.shape[1]):
            dd = [int(mdist[j * mok.shape[1] + q, repos.index(n)]) for n in order]
            mine = "0" if not any(dd) else "".join("%s:(%s%%), " % (n, repr(round(100.0 * v / cpr[n], 2))) for n, v in zip(order, dd))
            assert tm[1 + j][1 + q] == mine, (j, q)
            assert (mine == str(mwant[j][q])) == bool(mok[j, q])
    assert [int(x) for x in mok.sum(axis=1)] == [21, 16, 21, 20]


@pytest.mark.gpu
def test_diff_trees(tmp_path):
    old, new = tmp_path / "old", tmp_path / "new"
    os.makedirs(old / "a")
    os.makedirs(new / "a")
    (old / "a" / "x.py").write_bytes(b"1\n2\n3\n4\n")
    (new / "a" / "x.py").write_bytes(b"1\n3\n4\nassert 5\n6\n")
    (old / "gone.c").write_bytes(b"a\nb\n")
    (new / "fresh.c").write_bytes(b"c\n")
    (old / "same.h").write_bytes(b"s\n")
    (new / "same.h").write_bytes(b"s\n")
    (old / "blob.py").write_bytes(b"x = 1\n\x00\x01\n")            # binary on one side: skipped, like git's numstat
    (old / "a" / "tail.py").write_bytes(b"p\nq")                # only the final LF differs: no line changes (SPEC section 2)
    (new / "a" / "tail.py").write_bytes(b"p\nq\n")
    outp = str(tmp_path / "churn.csv")
    out = subprocess.run([CLI, "diff", str(old), str(new), "--out", outp], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "tosem-scan: 1 binary file(s) skipped" in out.stderr.splitlines()
    assert out.stdout.replace("\r\n", "\n").strip().split("\n") == ["cloc,added,removed", "6,3,3"]
    got = {r[0]: r[1:] for r in read_csv(outp)[1:]}
    # cloc, added, removed, hunks_add, hunks_del, hunks_mod, added_assert, removed_assert
    assert got == {"a/x.py": ["3", "2", "1", "1", "1", "0", "1", "0"], "gone.c": ["2", "0", "2", "0", "1", "0", "0", "0"],
                   "fresh.c": ["1", "1", "0", "1", "0", "0", "0", "0"]}


@pytest.mark.gpu
def test_scan_two_gpus_matches_one(tmp_path):
    """`--gpus 2`: batches dealt to two host threads / contexts, one ncclAllReduce of the count table."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import tosemscan as ts
    root = tmp_path / "big"
    c = ts.gen_corpus(21, 600, 1, n_groups=1, pinned=False)      # Zipf sizes; forces several batches? (no: one) -> two roots
    for r in ("a_tests", "b_tests"):
        os.makedirs(root / r)
    for i in range(c.n_files):
        ext = {1: "py", 2: "cc", 4: "java"}[int(c.ext[i])]
        (root / ("a_tests" if i % 2 else "b_tests") / ("f%04d_test.%s" % (i, ext))).write_bytes(c.file_bytes(i))
    outs = []
    for g in (1, 2):
        rows_p = str(tmp_path / ("rows%d.csv" % g))
        out = subprocess.run([CLI, "scan", str(root / "a_tests"), str(root / "b_tests"), "--rows", rows_p, "--gpus", str(g)],
                             capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        outs.append((out.stdout, open(rows_p, "rb").read(), out.stderr.strip().split("\n")[-1]))
    assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1]
    totals = [o[2].split(" on ")[0] for o in outs]           # "lines=.. assertion_lines=.. headers=.. fixture_headers=.."
    assert totals[0] == totals[1] and "on 2 GPU(s)" in outs[1][2]
    lo, hi = (int(x) for x in outs[1][2].split("shares ")[1].split(" bytes")[0].split(".."))
    assert hi - lo <= (1 << 20) + 128                        # LPT: the shares differ by less than the largest file


@pytest.mark.gpu
def test_scan_many_batches_match_one(tmp_path):
    """`--batch-bytes` small: dozens of batches per GPU, each loaded by the background task while the previous
    one is scanned; rows, summary and the aggregate table must not depend on the batching."""
    import tosemscan as ts
    root = tmp_path / "proj_tests"
    os.makedirs(root)
    c = ts.gen_corpus(33, 300, 1, n_groups=1, pinned=False)
    for i in range(c.n_files):
        ext = {1: "py", 2: "cc", 4: "java"}[int(c.ext[i])]
        (root / ("f%04d_test.%s" % (i, ext))).write_bytes(c.file_bytes(i))
    outs = []
    for extra in ([], ["--batch-bytes", "65536"]):
        tag = "b" if extra else "a"
        rows_p, sum_p = str(tmp_path / ("rows_%s.csv" % tag)), str(tmp_path / ("sum_%s.csv" % tag))
        out = subprocess.run([CLI, "scan", str(root), "--rows", rows_p, "--summary", sum_p] + extra, capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        outs.append((out.stdout, open(rows_p, "rb").read(), open(sum_p, "rb").read()))
    assert outs[0] == outs[1]


def py_case_name(ext, line):
    s = line.strip(b" \t\r\x0b\x0c").decode("latin-1")
    if ext == 1:
        import re
        m = re.search(r"def\s*([A-Za-z0-9_]+)", s)
        if m:
            return m.group(1)
    else:
        if s.startswith(("TEST(", "TEST_F(", "TEST_P(")):
            c, r = s.find(","), s.find(")")
            if c >= 0 and (r < 0 or c < r):
                return s[c + 1:(len(s) if r < 0 else r)].strip(" \t\r\x0b\x0c")
        if s.startswith("BOOST_AUTO_TEST_CASE("):
            r = s.find(")")
            return "TEST_CASE(" + s[21:(len(s) if r < 0 else r)].strip(" \t\r\x0b\x0c") + ")"
    return orc.method_string(ext, line).decode("latin-1")


def expected_body(files):
    """SPEC section 10 rows from the oracle's statement kinds and header rule."""
    rows, index, cases = [], 0, 0
    sel = sorted((r for r in files if "test" in r.lower() and r.rsplit(".", 1)[-1] in EXT), key=lambda r: r.split("/"))
    for file_id, rel in enumerate(sel, start=1):
        data, ext = files[rel], EXT[rel.rsplit(".", 1)[-1]]
        arena, off, length = orc.pack([data])
        _, end, kind = orc.statements(arena, off, length)
        in_case, cur, listed, pos = False, None, False, 0

        def flush():
            nonlocal index, cur
            if cur is not None and listed and cur.strip(b"{}(); \t\r\x0b\x0c"):
                index += 1
                rows.append([str(index), cur.decode("latin-1"), "", str(cases), str(file_id), ""])
            cur = None
        for e, k in zip(end.tolist(), kind.tolist()):
            line = data[pos:e]
            is_hdr = bool(orc.header_kind(ext, line))
            if k == 1:
                flush()
                listed = in_case and not is_hdr
                cur = b""
            if is_hdr:
                in_case = True
                cases += 1
                index += 1
                rows.append([str(index), py_case_name(ext, line), "", str(cases), str(file_id), ""])
            if k != 0 and cur is not None:
                st = line.strip(b" \t\r\x0b\x0c")
                cur = st if not cur else cur + b" " + st
            pos = e + 1
        flush()
    return rows


@pytest.mark.gpu
def test_body_statements(tmp_path):
    files = make_tree(str(tmp_path / "proj"))
    extra = {"tests/math/aabox2d_test.cc": b"TEST(AABox2dTest, GetAllCorners) {\n  AABox2d box1({0, 0}, 4, 2);\n  EXPECT_EQ(\n      box1.DebugString(),\n"
                                           b"      \"aabox2d ( center = vec2d ( x = 0 ) )\");\n}\n\nBOOST_AUTO_TEST_CASE(Query) {\n  BOOST_CHECK_EQUAL(1, 2);\n}\n"}
    for rel, data in extra.items():
        p = os.path.join(str(tmp_path / "proj"), rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        open(p, "wb").write(data)
    files.update(extra)
    outp = str(tmp_path / "body.csv")
    out = subprocess.run([CLI, "body", str(tmp_path / "proj"), "--out", outp], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = read_csv(outp)
    assert got[0] == ["Index", "text", "Category", "cases", "File_ID", "Component"]
    want = expected_body(files)
    assert got[1:] == want
    texts = [r[1] for r in got[1:]]
    # the reference's own example: ML-Analysis-v4.xlsx!Apollo:R2-R3 and the joined multi-line row :R14
    assert "GetAllCorners" in texts and "AABox2d box1({0, 0}, 4, 2);" in texts
    assert 'EXPECT_EQ( box1.DebugString(), "aabox2d ( center = vec2d ( x = 0 ) )");' in texts
    assert "TEST_CASE(Query)" in texts and "}" not in texts


@pytest.mark.gpu
def test_release_presence_matrix(tmp_path):
    """S7 (SPEC section 11): identities across snapshots by path, by content (pure move), by unique base name."""
    a = b"def test_a(self):\n    self.assertEqual(1, 2)\n    self.assertEqual(3, 4)\n    assert x\n"
    b = b"TEST(S, T) {\n  EXPECT_EQ(1, 2);\n}\n"
    snaps = {
        "v1": {"tests/test_image_supervised.py": a, "tests/test_search.py": b"def test_s():\n    assert y\n", "unit_test/x_test.cc": b},
        "v2": {"tests/image/test_image_supervised.py": a, "tests/test_search.py": b"def test_s():\n    assert y\n    assert z\n", "unit_test/x_test.cc": b},
        "v3": {"tests/image/test_image_supervised.py": a + b"    assert more\n", "lib/tests/x_test.cc": b + b"// moved and edited\n",
               "tests/test_new.py": b"assert True\n"},
    }
    args = []
    for tag, files in snaps.items():
        for rel, data in files.items():
            p = tmp_path / tag / rel
            os.makedirs(p.parent, exist_ok=True)
            p.write_bytes(data)
        args.append("%s=%s" % (tmp_path / tag, tag))
    outp = str(tmp_path / "release_meta.csv")
    out = subprocess.run([CLI, "releases"] + args + ["--out", outp], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = read_csv(outp)
    assert got[0] == ["Id", "FileName", "v1", "v2", "v3", "total assert", "assertion"]
    assert got[1:] == [
        ["1", "tests/test_image_supervised.py", "tests/test_image_supervised.py", "tests/image/test_image_supervised.py",
         "tests/image/test_image_supervised.py", "4", "2:assertEqual, 2:assertTrue"],
        ["2", "tests/test_search.py", "tests/test_search.py", "tests/test_search.py", "", "2", "2:assertTrue"],
        ["3", "unit_test/x_test.cc", "unit_test/x_test.cc", "unit_test/x_test.cc", "lib/tests/x_test.cc", "1", "1:assertEqual"],
        ["4", "tests/test_new.py", "", "", "tests/test_new.py", "1", "1:assertTrue"],
    ]
