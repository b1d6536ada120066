"""Device time of the test-case churn (docs/SPEC.md section 16) on the 50 000 pairs of BASELINE config C5.  Alternating on the
same batch: tsm_diff_pairs_detail (plain kernels) and tsm_diff_pairs_cases (k_scan with header events, DIFF_MARKS kernels,
the case kernels), each with its device phases from CUDA events inside the library (tsm_diff_last_ms) and the whole call on
the host clock (both calls synchronise); medians over the repetitions.  The case kernels and the exclusive scans they launch
are timed in a separate torch.profiler run of one call each (the profiler slows the host, so it is not part of the above).

    python tools/bench_cases.py [--pairs 50000] [--reps 10] [--out F]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().split("\n")[0]
    A, B = ts.gen_pairs(0x7053454D0005, a.pairs)
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    first = sc.diff_cases(A, B)
    cap = max(len(first[3]), len(first[4]))                 # arrays of the right size: one library call per timed call
    plain, cases, wall = [], [], [[], []]
    for r in range(a.reps + 2):                            # two warm-up rounds
        t0 = time.perf_counter()
        d = sc.diff_pairs(A, B, detail=True)
        t1 = time.perf_counter()
        plain.append(sc.diff_last_ms())
        g = sc.diff_cases(A, B, cap=cap)
        t2 = time.perf_counter()
        cases.append(sc.diff_last_ms())
        if r < 2:
            plain.pop(); cases.pop()
            continue
        wall[0].append(t1 - t0); wall[1].append(t2 - t1)
    assert all(np.array_equal(x, y) for x, y in zip(d, g[:3]))
    kp = kernel_ms(lambda: sc.diff_pairs(A, B, detail=True))
    kc = kernel_ms(lambda: sc.diff_cases(A, B, cap=cap))
    med = lambda v: float(np.median(v))                    # noqa: E731
    lines = [
        "# tools/bench_cases.py: %d C5 pairs, %d old cases, %d new cases; medians of %d alternating repetitions" % (
            a.pairs, len(g[3]), len(g[4]), a.reps),
        "# card: %s" % card,
        "phase                           tsm_diff_pairs_detail (ms)   tsm_diff_pairs_cases (ms)",
        "k_scan (both sides)             %10.3f                  %10.3f  (+ header events)" % (med([p[0] for p in plain]), med([c[0] for c in cases])),
        "k_diff_small (four sizes)       %10.3f                  %10.3f  (marks)" % (med([p[1] for p in plain]), med([c[1] for c in cases])),
        "k_myers + k_myers_trace         %10.3f                  %10.3f" % (med([p[2] for p in plain]), med([c[2] for c in cases])),
        "whole call, host clock          %10.3f                  %10.3f" % (1e3 * med(wall[0]), 1e3 * med(wall[1])),
        "# one call each under torch.profiler, device ms per kernel:",
    ]
    for name in sorted(set(kp) | set(kc)):
        if "k_case" in name or "xscan" in name or name.startswith(("tsm::k_scan", "k_scan")):
            lines.append("%-31s %10.3f                  %10.3f" % (name.replace("tsm::", ""), kp.get(name, 0.0), kc.get(name, 0.0)))
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)
    sc.close()


if __name__ == "__main__":
    main()
