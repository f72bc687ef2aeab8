"""Index peeks (mzgpu_peek / mzgpu_peek_many) against a ~10 M-row R32 index of 10 batches (--rows, keys uniform over
--rows / 4 values, so about four rows per key).

1. Point lookups: --lookups (default 1,000) single-key peeks with the identity plan, three ways, each ending in a
   device synchronise: peek_many calls of MZGPU_PEEK_MANY_MAX requests each, one peek call per key, and the host
   path a Rust worker takes today (per batch mzgpu_batch_seek_keys for all keys, then mzgpu_batch_rows per found
   run, and the times accumulated on the host).
2. A full scan with ORDER BY val DESC LIMIT 10: time per call, and the scanned R32 bytes per second as a share of
   the H100 SXM's 3.35 TB/s (the index read once; a lower bound on the bytes the peek moves).
Each way runs --reps times after one warm-up; the median is reported.  Prints one JSON line with the card's name and
power limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import materialize_b200 as mz  # noqa: E402


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception:  # noqa: BLE001
        return "unknown"


def timed(ctx, fn, reps):
    fn()
    ctx.sync()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ctx.sync()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--lookups", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    ctx = mz.Context(0)
    sp = mz.Spine(ctx, 32)
    per = a.rows // a.batches
    keys_n = max(1, a.rows // 4)
    batches = []
    for i in range(a.batches):
        r = np.zeros(per, dtype=mz.R32)
        r["key"] = rng.integers(0, keys_n, per, dtype=np.uint64)
        r["val"] = rng.integers(0, 1 << 40, per, dtype=np.uint64)
        r["time"] = i
        r["diff"] = 1
        b = mz.Batch.build(ctx, r, i, i + 1)
        batches.append(b)
        sp.insert(b)
    as_of = a.batches - 1
    ident = [[(0, 0, 64, 0)], [(1, 0, 64, 0)]]
    plan = mz.PeekPlan(ctx, ident)
    keys = rng.integers(0, keys_n, a.lookups, dtype=np.uint64)
    K = mz.PEEK_MANY_MAX

    def many():
        for s in range(0, len(keys), K):
            mz.peek_many(ctx, sp, [{"plan": plan, "as_of": as_of, "literals": [k]} for k in keys[s:s + K]])

    def single():
        for k in keys:
            mz.peek(ctx, plan, sp, as_of, literals=[k])

    def host_path():
        acc = {}
        for b in batches:
            runs = b.seek_keys(keys)
            for k, run in zip(keys, runs):
                if run["len"] and run["key"] == k:
                    rows = b.rows_range(int(run["first"]), int(run["len"]))
                    for row in rows:
                        if row["time"] <= as_of:
                            p = (int(row["key"]), int(row["val"]))
                            acc[p] = acc.get(p, 0) + int(row["diff"])
        return acc

    topk = mz.PeekPlan(ctx, ident, order=[mz.order_lane(src=1, descending=True)], limit=10)

    def scan():
        mz.peek(ctx, topk, sp, as_of)

    # the three lookup ways must agree
    got = {}
    for s in range(0, len(keys), K):
        for st, rows in mz.peek_many(ctx, sp, [{"plan": plan, "as_of": as_of, "literals": [k]} for k in keys[s:s + K]]):
            assert st == "rows"
            for row in rows:
                got[(int(row["key"]), int(row["val"]))] = got.get((int(row["key"]), int(row["val"])), 0) + int(row["diff"])
    assert got == {p: c for p, c in host_path().items() if c}, "peek_many and the host path disagree"

    t_many = timed(ctx, many, a.reps)
    t_single = timed(ctx, single, a.reps)
    t_host = timed(ctx, host_path, max(1, a.reps // 2))
    t_scan = timed(ctx, scan, a.reps)
    scanned = a.rows * 32
    print(json.dumps({
        "gpu": gpu_name(), "rows": a.rows, "batches": a.batches, "lookups": a.lookups,
        "peek_many_us_per_lookup": t_many / a.lookups * 1e6,
        "peek_us_per_lookup": t_single / a.lookups * 1e6,
        "host_path_us_per_lookup": t_host / a.lookups * 1e6,
        "scan_order_by_limit10_ms": t_scan * 1e3,
        "scan_bytes_per_s": scanned / t_scan,
        "scan_share_of_3_35_TBps": scanned / t_scan / 3.35e12,
    }))


if __name__ == "__main__":
    main()
