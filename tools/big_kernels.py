#!/usr/bin/env python
"""Bulk-regime kernel timings (BASELINE configs 1 and 2 sizes) for tuning: live CUDA-event
time and algorithmic GB/s per kernel."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import materialize_b200 as mz  # noqa: E402
from materialize_b200 import harness  # noqa: E402

ctx = mz.Context(0)
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 6650.0
which = sys.argv[1] if len(sys.argv) > 1 else "both"
out = {}


def table():
    rep = ctx.profile_report()
    return {k: {"launches": v["launches"], "ms": round(v["ms"], 4),
                "GBps": round(v["bytes"] / (v["ms"] / 1e3) / 1e9, 1) if v["bytes"] and v["ms"] else None,
                "frac": round(v["bytes"] / (v["ms"] / 1e3) / 1e9 / peak, 4) if v["bytes"] and v["ms"] else None}
            for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])[:8]}


if which in ("both", "sort"):
    n = 100_000_000
    for rep in range(2):
        d = harness.gen_cfg1(ctx, 1, n, 64)
        d.consolidate()
        len(d)
    d = harness.gen_cfg1(ctx, 1, n, 64)
    ctx.profile(True)
    ctx.profile_report()
    d.consolidate()
    len(d)
    out["cfg1_100M_64bit"] = table()
    ctx.profile(False)
    del d
if which in ("both", "join"):
    n2 = 10_000_000
    for rep in range(2):
        a, b = harness.gen_cfg2(ctx, 1, n2, n2), harness.gen_cfg2(ctx, 2, n2, n2)
        ba, bb = mz.Batcher(ctx, 32), mz.Batcher(ctx, 32)
        ba.push_device(a)
        bb.push_device(b)
        xa, xb = ba.seal(1), bb.seal(1)
        sa, sb = mz.Spine(ctx, 32), mz.Spine(ctx, 32)
        j = mz.JoinCore(ctx, sa, sb)
        sa.insert(xa)
        j.push(0, xa, 0)
        sb.insert(xb)
        j.push(1, xb, 0)
        if rep == 1:
            ctx.profile(True)
            ctx.profile_report()
        j.work()
        if rep == 1:
            out["cfg2_join_10Mx10M"] = table()
            ctx.profile(False)
print(json.dumps(out))
