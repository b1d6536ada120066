"""Cost of the assertion edits (docs/SPEC.md section 17) over tsm_diff_pairs_asserts, on two corpora: the 50 000 pairs of
BASELINE config C5, and a hunk-heavy corpus in which every edit replaces a run of assertion lines by a run of similar ones (so
that the score kernel has real work).  Per corpus, alternating on the same batch: diff_pairs(asserts=True) and
diff_assert_edits, with the whole call on the host clock (both synchronise) and the phases of tsm_assert_edits_last_ms; medians
over the repetitions.  The kernels are timed in a separate torch.profiler run of one call each.  Candidates (deleted x inserted
assertion lines of one hunk) are counted on the host from the reference entries (tests/orc_assert_edits.py).

    python tools/bench_assert_edits.py [--pairs 50000] [--reps 10] [--out F]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tosemscan as ts  # noqa: E402


def kernel_ms(call):
    """{kernel name: device ms} of one call under torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {}
    for k in prof.key_averages():
        name = k.key.split("(")[0].replace("void ", "").split("<")[0]
        out[name] = out.get(name, 0.0) + getattr(k, "device_time_total", 0.0) / 1e3
    return out


def hunk_heavy(n_pairs, hunks=16, run=12, seed=9):
    """Pairs of `hunks` runs of `run` assertion lines each, every run replaced by `run` similar lines, kept lines between."""
    rng = np.random.default_rng(seed)
    olds, news = [], []
    for p in range(n_pairs):
        o, n = [], []
        for h in range(hunks):
            o.append(b"    x_%d_%d = f(%d)\n" % (p, h, h))
            n.append(b"    x_%d_%d = f(%d)\n" % (p, h, h))
            for k in range(run):
                v = int(rng.integers(1000))
                o.append(b"    self.assertEqual(result_%d[%d], expected_%d)\n" % (h, k, v))
                n.append(b"    self.assertAlmostEqual(result_%d[%d], expected_%d, 6)\n" % (h, k, v + 1))
        olds.append(b"".join(o)); news.append(b"".join(n))
    return ts.pack(olds, [1] * n_pairs), ts.pack(news, [1] * n_pairs)


def candidates(A, B):
    import orc_assert_edits as oae
    import orc_cases
    import orc_marks
    sa, sb = (A.arena, A.off, A.len, A.ext), (B.arena, B.off, B.len, B.ext)
    ba, bb, dl, ins = orc_marks.diff_pairs_marks(sa, sb)
    cd, ci = np.concatenate([[0], np.cumsum(dl, dtype=np.int64)]), np.concatenate([[0], np.cumsum(ins, dtype=np.int64)])
    traced = cd[ba[1:]] - cd[ba[:-1]] + ci[bb[1:]] - ci[bb[:-1]] <= orc_marks.TRACE_MAX_D
    ko, _ = oae.entries(sa, ba, orc_cases.side_lines(sa)[2], dl, traced)
    kn, _ = oae.entries(sb, bb, orc_cases.side_lines(sb)[2], ins, traced)
    uo, co = np.unique(ko, return_counts=True)
    un, cn = np.unique(kn, return_counts=True)
    common, io, jn = np.intersect1d(uo, un, return_indices=True)
    return int((co[io].astype(np.int64) * cn[jn]).sum())


def measure(sc, name, A, B, reps):
    first = sc.diff_assert_edits(A, B)
    cap = max(len(first[5]), len(first[6]), 1)
    plain, edits, wall = [], [], [[], []]
    for r in range(reps + 2):                              # two warm-up rounds
        t0 = time.perf_counter()
        d = sc.diff_pairs(A, B, asserts=True)
        t1 = time.perf_counter()
        plain.append(sc.diff_last_ms())
        g = sc.diff_assert_edits(A, B, cap=cap)
        t2 = time.perf_counter()
        edits.append(sc.assert_edits_last_ms())
        if r < 2:
            plain.pop(); edits.pop()
            continue
        wall[0].append(t1 - t0); wall[1].append(t2 - t1)
    assert all(np.array_equal(x, y) for x, y in zip(d, g[:7]))
    kp = kernel_ms(lambda: sc.diff_pairs(A, B, asserts=True))
    ke = kernel_ms(lambda: sc.diff_assert_edits(A, B, cap=cap))
    n_cand = candidates(A, B)
    med = lambda v: float(np.median(v))                    # noqa: E731
    score_ms = ke.get("tsm::k_edit_score", 0.0) + ke.get("tsm::k_edit_score_long", 0.0)
    lines = [
        "## %s: %d pairs, %d deleted / %d inserted assertion lines, %d candidates, %d edits; medians of %d alternating repetitions" % (
            name, A.n_files, len(g[6]), len(g[5]), n_cand, len(g[7]), reps),
        "phase                             tsm_diff_pairs_asserts (ms)   tsm_diff_pairs_assert_edits (ms)",
        "k_scan (both sides)               %10.3f                    %10.3f" % (med([p[0] for p in plain]), med([e[0] for e in edits])),
        "diff kernels                      %10.3f                    %10.3f  (EMIT / MARKS)" % (
            med([p[1] + p[2] for p in plain]), med([e[1] for e in edits])),
        "compact to pairing, host clock           -                    %10.3f" % med([e[2] for e in edits]),
        "whole call, host clock            %10.3f                    %10.3f" % (1e3 * med(wall[0]), 1e3 * med(wall[1])),
        "# one call each under torch.profiler, device ms per kernel:",
    ]
    for k in sorted(set(kp) | set(ke)):
        if any(s in k for s in ("k_edit", "k_case_kept", "k_classify", "k_diff_small", "k_myers", "xscan", "k_scan")):
            lines.append("%-33s %10.3f                    %10.3f" % (k.replace("tsm::", ""), kp.get(k, 0.0), ke.get(k, 0.0)))
    if score_ms > 0:
        lines.append("candidates scored per second (score kernels only): %.3g" % (n_cand / (score_ms / 1e3)))
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=50_000)
    ap.add_argument("--heavy-pairs", type=int, default=4_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().split("\n")[0]
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    lines = ["# tools/bench_assert_edits.py", "# card, power limit, max SM clock: %s" % card]
    A, B = ts.gen_pairs(0x7053454D0005, a.pairs)
    lines += measure(sc, "C5", A, B, a.reps)
    A, B = hunk_heavy(a.heavy_pairs)
    lines += measure(sc, "hunk-heavy", A, B, a.reps)
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)
    sc.close()


if __name__ == "__main__":
    main()
