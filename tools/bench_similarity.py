#!/usr/bin/env python3
"""Cost of the rename similarity (docs/SPEC.md section 13) on a synthetic reorganisation commit, one GPU:

    python tools/bench_similarity.py [--files 4000] [--steps 10] [--warmup 3] [--sample 100000]

The commit deletes D = --files files and adds as many: the old files follow BASELINE config C5's size law (seeded), 3/4 of
the added files are gen_edit(lambda = 6) of a deleted file and the rest are new.  Every D x A candidate that passes git's
size filter at --find-renames 50 (100 * min size >= 50 * max size) is scored by one tsm_similarity call.  Reported: the
median call time and the median device time of its three phases (tsm_similarity_last_ms) over --steps calls after
--warmup, candidates per second, a check digest (sum of `common` over a seeded sample of --sample candidates) equal to the
CPU reference's on the same sample, the CPU reference's rate there, and the card's name and power limit.  Each call
synchronises before it returns, so a host clock around it is its whole time.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tosem-2021-replication_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import tosemscan as ts  # noqa: E402
from bench_diff_asserts import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=4000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=100000)
    args = ap.parse_args()
    d = args.files
    edited = d * 3 // 4
    olds, edits = ts.gen_pairs(0x7053454D0013, d, lam=6.0, pinned=False)      # C5's size law; news = gen_edit(lambda = 6)
    fresh, _ = ts.gen_pairs(0x7053454D0014, d - edited, lam=0.0, pinned=False)
    news = ts.pack([edits.file_bytes(i) for i in range(edited)] + [fresh.file_bytes(i) for i in range(d - edited)], [1] * d)
    so, sn = olds.len.astype(np.int64), news.len.astype(np.int64)
    lo, hi = np.minimum.outer(so, sn), np.maximum.outer(so, sn)
    keep = (100 * lo >= 50 * hi) & (hi > 0)
    co, cn = (x.astype(np.int32) for x in np.nonzero(keep))
    sc = ts.Scanner(0, 1 << 20, 16, 1)
    for _ in range(args.warmup):
        sc.similarity(olds, news, co, cn)
    t, ms = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        common = sc.similarity(olds, news, co, cn)
        t.append(1e3 * (time.perf_counter() - t0))
        ms.append(sc.similarity_last_ms())
    rng = np.random.default_rng(0x5A)
    pick = np.sort(rng.choice(co.size, min(args.sample, co.size), replace=False))
    import orc_similarity as osim
    t0 = time.perf_counter()
    ref = osim.similarity(olds, news, co[pick], cn[pick])
    cpu_s = time.perf_counter() - t0
    gpu_digest, cpu_digest = int(common[pick].sum()), int(ref.sum())
    assert gpu_digest == cpu_digest and np.array_equal(common[pick], ref), "the GPU differs from the CPU reference"
    med = float(np.median(t))
    print(json.dumps({"metric": "tsm_similarity over a reorganisation commit", "unit": "ms", "deleted": d, "added": d,
                      "added_edited": edited, "candidates": int(co.size), "bytes": olds.source_bytes + news.source_bytes,
                      "steps": args.steps, "warmup": args.warmup, "ms_median": med, "ms_min": float(min(t)),
                      "device_ms_median": dict(zip(("k_scan both sides", "sort_merge", "k_similarity"),
                                                   (float(x) for x in np.median(np.array(ms), axis=0)))),
                      "candidates_per_s": co.size / (med / 1e3),
                      "check": {"sample": int(pick.size), "sum_common_gpu": gpu_digest, "sum_common_cpu": cpu_digest},
                      "cpu_reference_candidates_per_s": pick.size / cpu_s, "gpu": card()}))
    sc.close()


if __name__ == "__main__":
    main()
