#!/usr/bin/env python
"""bench_kernels.py — per-kernel roofline numbers at BASELINE sizes (configs 1, 2, 4).

Not the driver's contract bench (that is bench.py, config 3/5): this script
reports, for the bulk regimes, update-rows/s per operator and achieved GB/s per
kernel = algorithmic bytes (DESIGN.md §4) / live CUDA-event duration, against
MEASURED_PEAKS.json (the H100 SXM data sheet's 3350 GB/s when that file is
absent).  Output: one JSON document.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def kernel_table(ctx, peak):
    rep = ctx.profile_report()
    rows = []
    tot = sum(v["ms"] for v in rep.values()) or 1.0
    for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"]):
        gbps = v["bytes"] / (v["ms"] / 1000.0) / 1e9 if v["ms"] > 0 and v["bytes"] else None
        rows.append(
            {
                "kernel": k,
                "launches": v["launches"],
                "ms": round(v["ms"], 4),
                "share": round(v["ms"] / tot, 4),
                "algorithmic_GBps": None if gbps is None else round(gbps, 1),
                "frac_of_measured_hbm": None if gbps is None else round(gbps / peak, 4),
            }
        )
    return rows


def timed(ctx, fn, reps=3):
    best = None
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        fn()
        ctx.sync()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, help="run only the cases whose name contains this string")
    args = ap.parse_args()
    import materialize_b200 as mz
    from materialize_b200 import harness

    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")
    ) else 3350.0
    ctx = mz.Context(0)
    scale = 10 if args.quick else 1
    res = {"peak_hbm_gbs": peak, "cases": []}

    def case(name, n_rows, build, run, reps=3):
        if args.only and args.only not in name:
            return
        state = build()
        run(state)  # warm-up (also warms the memory pool)
        secs = None
        for _ in range(reps):
            state = build()
            ctx.sync()
            t0 = time.perf_counter()
            run(state)
            ctx.sync()
            dt = time.perf_counter() - t0
            secs = dt if secs is None else min(secs, dt)
        state = build()
        ctx.profile(True)
        ctx.profile_report()
        run(state)
        table = kernel_table(ctx, peak)
        ctx.profile(False)
        entry = {"case": name, "rows": n_rows, "seconds": secs, "rows_per_sec": n_rows / secs, "kernels": table[:10]}
        # the two-pass probe as one unit: its algorithmic bytes over count + write time
        pr = [t for t in table if "k_probe<" in t["kernel"]]
        if pr:
            ms = sum(t["ms"] for t in pr)
            gb = sum((t["algorithmic_GBps"] or 0.0) * t["ms"] for t in pr) / ms
            entry["probe_both_passes"] = {
                "ms": round(ms, 4),
                "algorithmic_GBps": round(gb, 1),
                "frac_of_measured_hbm": round(gb / peak, 4),
            }
        res["cases"].append(entry)
        print(name, f"{n_rows / secs / 1e6:.1f} M rows/s", file=sys.stderr, flush=True)

    # ---- config 1: consolidate() on (u64 key, i64 diff)
    for n, bits in ((1_000_000, 20), (1_000_000, 64), (100_000_000 // scale, 64), (100_000_000 // scale, 26)):
        case(
            f"cfg1 consolidate R16 n={n} key_bits={bits}",
            n,
            lambda n=n, bits=bits: harness.gen_cfg1(ctx, 1, n, bits),
            lambda d: d.consolidate(),
        )
    # ---- config 2: arrange + join_core, 2 x 10M rows, uniform keys
    n2 = 10_000_000 // scale

    def build2():
        return harness.gen_cfg2(ctx, 1, n2, n2), harness.gen_cfg2(ctx, 2, n2, n2)

    def run2(st):
        a, b = st
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
        j.work()
        run2.out = len(j.out)

    case(f"cfg2 arrange+join_core 2x{n2} R32", 2 * n2, build2, run2, reps=2)
    if res["cases"] and "cfg2" in res["cases"][-1]["case"]:
        res["cases"][-1]["join_output_rows"] = run2.out
    # ---- config 4: reduce COUNT/SUM, Zipf(0.9) over 1M keys
    n4 = 100_000_000 // scale
    nk = 1_000_000 // scale
    # zipf inverse CDF built on the host with numpy (same formula as the oracle's mzo_zipf_cdf)
    w = 1.0 / np.power(np.arange(1, nk + 1, dtype=np.float64), 0.9)
    cdf = np.cumsum(w / w.sum())
    cdf[-1] = 1.0

    def run4(d):
        r = mz.ReduceAccumulable(ctx, mz.AGG_COUNT_SUM_I64)
        out = mz.DeviceRows(ctx, 64)
        from materialize_b200 import _ffi as F

        ctx.check(F.lib.mzgpu_reduce_accumulable(r.h, d.device_ptr(), len(d), F.MEM_DEVICE, 1, out.h))
        run4.out = len(out)

    case(f"cfg4 reduce COUNT/SUM n={n4} zipf0.9 keys={nk}", n4, lambda: harness.gen_cfg4(ctx, 3, n4, cdf), run4, reps=2)
    if res["cases"] and "cfg4" in res["cases"][-1]["case"]:
        res["cases"][-1]["groups_out"] = run4.out
    txt = json.dumps(res, indent=1)
    if args.out:
        open(args.out, "w").write(txt)
    print(txt)


if __name__ == "__main__":
    main()
