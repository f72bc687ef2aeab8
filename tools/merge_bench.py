#!/usr/bin/env python
"""Batch merges at update-batch-to-spine sizes: device time of mzgpu_batch_merge for two sorted,
consolidated R32 batches of n/2 rows each (the merges a spine schedules while the Q3 workload steps).
Run on a GPU box."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import materialize_b200 as mz  # noqa: E402

ctx = mz.Context(0)
rng = np.random.default_rng(1)
for n in (40_000, 160_000, 320_000, 640_000, 1_000_000, 1_280_000, 2_560_000):
    halves = []
    for h in range(2):
        a = np.zeros(n // 2, dtype=mz.R32)
        a["key"] = rng.integers(0, 60_000_000, size=n // 2, dtype=np.uint64)
        a["val"] = rng.integers(0, 1 << 36, size=n // 2, dtype=np.uint64)
        a["time"] = h
        a["diff"] = 1
        halves.append(mz.Batch.build(ctx, a, h, h + 1))
    best = None
    for rep in range(4):
        ctx.sync()
        ctx.profile(True)
        ctx.profile_report()
        m = halves[0].merge(halves[1], 0)
        ln = len(m)
        rep_ms = sum(v["ms"] for v in ctx.profile_report().values())
        ctx.profile(False)
        best = rep_ms if best is None else min(best, rep_ms)
        del m
    print(f"merge of 2 x {n // 2:>8} rows -> {ln:>8}: {1e3 * best:8.1f} us device ({n * 64 / best / 1e6:7.1f} GB/s algorithmic)")
