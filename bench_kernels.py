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

    # ---- config 4 with several aggregate columns per key (mzgpu_reduce_lanes_*): an int64 column
    # (val1) and a float64 column (val2) generated from the same seed, R40 rows.  Each variant runs on
    # a context of its own, so device_bytes_peak is that variant's.
    def lanes_of(k):
        cols = [mz.accum_lane(mz.AGG_COUNT_SUM_I64, 1), mz.accum_lane(mz.AGG_COUNT_SUM_F64, 2)]
        return (cols * 4)[:k]

    # COUNT(DISTINCT) / SUM(DISTINCT) next to the plain columns: the two plain lanes of lanes_of(2), a
    # distinct lane over val1 (nearly every value new) and one over its low 12 bits, sign-extended (values
    # repeat within a key)
    def distinct_lanes():
        d = mz.AGG_COUNT_SUM_I64 | mz.ACCUM_DISTINCT
        return lanes_of(2) + [mz.accum_lane(d, 1), mz.accum_lane(d, 1, 0, 12, True)]

    def r40_cfg4(c, seed, n, first=0, t=0, diff=1):
        a = harness.gen_cfg4(c, seed, n, cdf, first=first, t=t, diff=diff).download()
        f = harness.gen_cfg4(c, seed, n, cdf, as_f64=True, first=first, t=t, diff=diff).download()
        r = np.zeros(n, dtype=mz.R40)
        r["key"], r["val1"], r["val2"], r["time"], r["diff"] = a["key"], a["val"], f["val"], a["time"], a["diff"]
        return r

    def lanes_case(name, n_rows, build, run):
        if args.only and args.only not in name:
            return
        c = mz.Context(0)
        run(c, build(c))  # warm-up
        state = build(c)
        c.sync()
        syncs0 = c.stats()["host_syncs"]
        t0 = time.perf_counter()
        run(c, state)
        c.sync()
        secs = time.perf_counter() - t0
        syncs = c.stats()["host_syncs"] - syncs0  # host waits of the timed run, its closing sync included
        state = build(c)
        c.profile(True)
        c.profile_report()
        run(c, state)
        table = kernel_table(c, peak)
        c.profile(False)
        res["cases"].append(
            {"case": name, "rows": n_rows, "seconds": secs, "rows_per_sec": n_rows / secs, "kernels": table[:10],
             "device_bytes_peak": c.stats()["device_bytes_peak"], "host_syncs": syncs}
        )
        del state
        c.close()  # its cached blocks go back before the next variant measures its peak
        print(name, f"{n_rows / secs / 1e6:.1f} M rows/s", file=sys.stderr, flush=True)

    # the bulk seal holds the exploded rows, their sorted copy, the consolidated batch and the segment
    # sums at once (about 5 x the row width per input row): next to this script's other buffers, 2 lanes
    # (128-byte rows) run at 50 M rows and 4 lanes (224 bytes) at 25 M
    for k, n in ((2, n4 // 2), (4, n4 // 4)):
        name = f"cfg4 bulk reduce lanes={k} n={n} zipf0.9 keys={nk} R40"
        host = r40_cfg4(ctx, 3, n) if not args.only or args.only in name else None
        lanes_case(
            name,
            n,
            lambda c, host=host: mz.DeviceRows(c, 40).upload(host),
            lambda c, d, k=k: mz.ReduceLanes(c, lanes_of(k), 40).step_dev(d, 1),
        )
        del host
    name = f"cfg4 bulk reduce lanes=4 (2 plain + 2 distinct) n={n4 // 4} zipf0.9 keys={nk} R40"
    host = r40_cfg4(ctx, 3, n4 // 4) if not args.only or args.only in name else None
    lanes_case(
        name,
        n4 // 4,
        lambda c, host=host: mz.DeviceRows(c, 40).upload(host),
        lambda c, d: mz.ReduceLanes(c, distinct_lanes(), 40).step_dev(d, 1),
    )
    del host

    # incremental regime: 1M-row batches, half of each batch retracting rows of the batch before; one
    # 4-lane operator against four one-lane operators on the same batches
    nb, per = 20 // (2 if args.quick else 1), 1_000_000 // scale
    batches = {}

    def inc_batches(c):
        if not batches:
            prev = None
            for b in range(nb):
                fresh = r40_cfg4(c, 5, per // 2, first=b * (per // 2), t=b, diff=1)
                if prev is not None:
                    back = prev.copy()
                    back["time"], back["diff"] = b, -1
                    fresh = np.concatenate([fresh, back])
                batches[b] = fresh
                prev = fresh[: per // 2]
        return [mz.DeviceRows(c, 40).upload(batches[b]) for b in range(nb)]

    def run_inc(c, bufs, ops_lanes):
        ops = [mz.ReduceLanes(c, ls, 40) for ls in ops_lanes]
        outs = [mz.DeviceRows(c, op.out_row_bytes) for op in ops]
        for b, d in enumerate(bufs):
            for op, o in zip(ops, outs):
                op.step_dev(d, b + 1, o)

    lanes_case(
        f"cfg4 incremental lanes=4, one operator, {nb}x{per} R40",
        nb * per,
        inc_batches,
        lambda c, bufs: run_inc(c, bufs, [lanes_of(4)]),
    )
    lanes_case(
        f"cfg4 incremental lanes=4 (2 plain + 2 distinct), one operator, {nb}x{per} R40",
        nb * per,
        inc_batches,
        lambda c, bufs: run_inc(c, bufs, [distinct_lanes()]),
    )
    lanes_case(
        f"cfg4 incremental lanes=4, four one-lane operators, {nb}x{per} R40",
        nb * per,
        inc_batches,
        lambda c, bufs: run_inc(c, bufs, [[l] for l in lanes_of(4)]),
    )
    # HAVING inside the operator: the same 4-lane incremental run without and with a two-predicate filter
    # (COUNT(val1) >= 2 AND SUM(val1) > 0), alternating on one context; the best of three rounds each
    name = f"cfg4 incremental lanes=4, without / with a two-predicate HAVING, {nb}x{per} R40"
    if not args.only or args.only in name:
        hv = mz.having([mz.h_count(0), mz.h_int(2), mz.h_cmp("ge")], [mz.h_sum(2), mz.h_num(0), mz.h_cmp("gt")])
        c = mz.Context(0)

        def run_having(bufs, having):
            op = mz.ReduceLanes(c, lanes_of(4), 40, having=having)
            out = mz.DeviceRows(c, op.out_row_bytes)
            for b, d in enumerate(bufs):
                op.step_dev(d, b + 1, out)
            return len(out)

        best, rows_out = {"without": None, "with": None}, {}
        for rnd in range(4):  # round 0 warms up
            for label, having in (("without", None), ("with", hv)):
                bufs = inc_batches(c)
                c.sync()
                t0 = time.perf_counter()
                rows_out[label] = run_having(bufs, having)
                c.sync()
                dt = time.perf_counter() - t0
                if rnd > 0:
                    best[label] = dt if best[label] is None else min(best[label], dt)
        res["cases"].append(
            {"case": name, "rows": nb * per, "seconds_without": best["without"], "seconds_with": best["with"],
             "output_rows_without": rows_out["without"], "output_rows_with": rows_out["with"]}
        )
        c.close()
        print(name, f"{best['without']:.4f} s / {best['with']:.4f} s", file=sys.stderr, flush=True)

    # Monotonic MIN / MAX: cfg 4's incremental regime made insert-only, 4 unsigned lanes (MIN / MAX of val1
    # and of val2's bits).  One monotonic operator against four MIN / MAX operators, which take R32
    # (key, value) projections made before the timed region; alternating on one context, best of two rounds
    # after a warm-up.  The four operators walk every live value of a hot key once per batch, so the
    # comparison runs over the first `nb_cmp` batches; the monotonic operator alone then runs all nb.
    name = f"cfg4 incremental insert-only MIN/MAX lanes=4, monotonic vs four MIN/MAX operators, {nb}x{per} R40"
    if not args.only or args.only in name:
        nb_cmp = min(nb, 5)
        c = mz.Context(0)
        ins = [r40_cfg4(c, 7, per, first=b * per, t=b, diff=1) for b in range(nb)]
        mono_lanes = [mz.accum_lane(mz.AGG_MIN, 1), mz.accum_lane(mz.AGG_MAX, 1), mz.accum_lane(mz.AGG_MIN, 2),
                      mz.accum_lane(mz.AGG_MAX, 2)]
        kinds = [(mz.AGG_MIN, "val1"), (mz.AGG_MAX, "val1"), (mz.AGG_MIN, "val2"), (mz.AGG_MAX, "val2")]

        def proj(r, col):
            p = np.zeros(len(r), dtype=mz.R32)
            p["key"], p["val"], p["time"], p["diff"] = r["key"], r[col], r["time"], r["diff"]
            return p

        def collect(coll, rows, vals):
            for k, v, d in zip(rows["key"].tolist(), vals, rows["diff"].tolist()):
                coll[(k, v)] = coll.get((k, v), 0) + d

        def run_mono(k):
            cm = mz.Context(0)  # one context per leg: its own device_bytes_peak
            bufs = [mz.DeviceRows(cm, 40).upload(ins[b]) for b in range(k)]
            op = mz.ReduceMonotonic(cm, mono_lanes, 40)
            out, errs = mz.DeviceRows(cm, op.out_row_bytes), mz.DeviceRows(cm, 16)
            cm.sync()
            t0 = time.perf_counter()
            for b, d in enumerate(bufs):
                op.step_dev(d, b + 1, out, errs)
            cm.sync()
            dt = time.perf_counter() - t0
            r = (dt, out.download(), len(errs), len(op.input_trace().export()), cm.stats()["device_bytes_peak"])
            del op, out, errs, bufs
            cm.close()
            return r

        def run_four(k):
            from materialize_b200 import _ffi as F

            cf = mz.Context(0)
            bufs = [[mz.DeviceRows(cf, 32).upload(proj(ins[b], col)) for b in range(k)] for _, col in kinds]
            ops = [mz.ReduceAccumulable(cf, kind) for kind, _ in kinds]
            outs = [mz.DeviceRows(cf, 64) for _ in kinds]
            cf.sync()
            t0 = time.perf_counter()
            for b in range(k):
                for j in range(4):
                    ops[j].step_dev(bufs[j][b], b + 1, outs[j])
            cf.sync()
            dt = time.perf_counter() - t0
            r = (dt, [o.download() for o in outs], sum(len(mz.Spine(cf, 32, _borrowed=F.lib.mzgpu_reduce_input_trace(op.h)).export()) for op in ops),
                 cf.stats()["device_bytes_peak"])
            del ops, outs, bufs
            cf.close()
            return r

        best = {"mono": None, "four": None}
        for rnd in range(3):  # round 0 warms up
            dm, mout, n_err, marr, peak_m = run_mono(nb_cmp)
            df, fouts, farr, peak_f = run_four(nb_cmp)
            if rnd > 0:
                best["mono"] = dm if best["mono"] is None else min(best["mono"], dm)
                best["four"] = df if best["four"] is None else min(best["four"], df)
        agree = n_err == 0
        for j in range(4):
            cm_, cf_ = {}, {}
            collect(cm_, mout, mout["vals"][:, j].tolist())
            collect(cf_, fouts[j], fouts[j]["sum_lo"].tolist())
            agree = agree and {k: d for k, d in cm_.items() if d} == {k: d for k, d in cf_.items() if d}
        dm_all, _, _, marr_all, peak_all = run_mono(nb)
        res["cases"].append(
            {"case": name, "rows": nb_cmp * per, "batches_compared": nb_cmp,
             "seconds_monotonic": best["mono"], "seconds_four_minmax": best["four"], "outputs_agree": agree,
             "arrangement_rows_monotonic": marr, "arrangement_bytes_monotonic": 48 * marr,
             "arrangement_rows_four_minmax": farr, "arrangement_bytes_four_minmax": 32 * farr,
             "device_bytes_peak_monotonic": peak_m, "device_bytes_peak_four_minmax": peak_f,
             "monotonic_all_batches": {"batches": nb, "seconds": dm_all, "arrangement_rows": marr_all,
                                       "device_bytes_peak": peak_all}}
        )
        print(name, f"{best['mono']:.4f} s / {best['four']:.4f} s, agree={agree}, all {nb}: {dm_all:.4f} s",
              file=sys.stderr, flush=True)
        del ins
        c.close()

    name = f"bulk monotonic MIN/MAX lanes=4 n={n4} zipf0.9 keys={nk} R40"
    host = r40_cfg4(ctx, 3, n4) if not args.only or args.only in name else None
    lanes_case(
        name,
        n4,
        lambda c, host=host: mz.DeviceRows(c, 40).upload(host),
        lambda c, d: mz.ReduceMonotonic(c, [mz.accum_lane(mz.AGG_MIN, 1), mz.accum_lane(mz.AGG_MAX, 1),
                                            mz.accum_lane(mz.AGG_MIN, 2), mz.accum_lane(mz.AGG_MAX, 2)],
                                        40).step_dev(d, 1),
    )
    del host

    # Monotonic TopK: the same insert-only regime, Top1 (ORDER BY val1 DESC: the latest row per key) and
    # limit 3, against the TopK operator on the R32 (key, val1) projection over the first `nb_cmp` batches
    # (that operator refuses a group of more than 32 distinct values late, and reports it).
    for limit in (1, 3):
        name = f"cfg4 incremental insert-only monotonic TopK limit={limit} val1 desc vs TopK operator, {nb}x{per} R40"
        if args.only and args.only not in name:
            continue
        nb_cmp = min(nb, 3)
        c = mz.Context(0)
        ins = [r40_cfg4(c, 11, per, first=b * per, t=b, diff=1) for b in range(nb)]

        def run_topk_mono(k, limit=limit, ins=ins):
            cm = mz.Context(0)
            bufs = [mz.DeviceRows(cm, 40).upload(ins[b]) for b in range(k)]
            op = mz.TopKMonotonic(cm, [mz.order_lane(1, descending=True)], limit, 40)
            out, errs = mz.DeviceRows(cm, 40), mz.DeviceRows(cm, 16)
            cm.sync()
            t0 = time.perf_counter()
            for b, d in enumerate(bufs):
                op.step_dev(d, b + 1, out, errs)
                op.input_trace().set_logical_compaction(b + 1)
            cm.sync()
            dt = time.perf_counter() - t0
            r = (dt, out.download(), len(errs), len(op.input_trace().export()), cm.stats()["device_bytes_peak"])
            del op, out, errs, bufs
            cm.close()
            return r

        def run_topk_old(k, limit=limit, ins=ins):
            from materialize_b200 import _ffi as F

            cf = mz.Context(0)
            bufs = []
            for b in range(k):
                p = np.zeros(per, dtype=mz.R32)
                p["key"], p["val"], p["time"], p["diff"] = ins[b]["key"], ins[b]["val1"], ins[b]["time"], 1
                bufs.append(mz.DeviceRows(cf, 32).upload(p))
            op = mz.TopK(cf, limit, 0, True)
            out = mz.DeviceRows(cf, 64)
            cf.sync()
            t0 = time.perf_counter()
            status = "ok"
            try:
                for b in range(k):
                    op.step_dev(bufs[b], b + 1, out)
                cf.sync()
            except mz.MzGpuError as e:
                status = f"error {e.status}"
            dt = time.perf_counter() - t0
            arr = len(mz.Spine(cf, 32, _borrowed=F.lib.mzgpu_reduce_input_trace(op.h)).export()) if status == "ok" else None
            r = (dt, out.download() if status == "ok" else None, arr, cf.stats()["device_bytes_peak"], status)
            del op, out, bufs
            cf.close()
            return r

        dm = df = None
        for rnd in range(3):  # round 0 warms up
            t_m, mout, n_err, marr, peak_m = run_topk_mono(nb_cmp)
            t_f, fout, farr, peak_f, fstatus = run_topk_old(nb_cmp)
            if rnd > 0:
                dm = t_m if dm is None else min(dm, t_m)
                df = t_f if df is None else min(df, t_f)
        agree = None
        if fout is not None:
            cm_, cf_ = {}, {}
            for k_, v_, d_ in zip(mout["key"].tolist(), mout["val1"].tolist(), mout["diff"].tolist()):
                cm_[(k_, v_)] = cm_.get((k_, v_), 0) + d_
            for k_, v_, d_ in zip(fout["key"].tolist(), fout["sum_lo"].tolist(), fout["diff"].tolist()):
                cf_[(k_, v_)] = cf_.get((k_, v_), 0) + d_
            agree = n_err == 0 and {k: d for k, d in cm_.items() if d} == {k: d for k, d in cf_.items() if d}
        dm_all, _, _, marr_all, peak_all = run_topk_mono(nb)
        res["cases"].append(
            {"case": name, "rows": nb_cmp * per, "batches_compared": nb_cmp,
             "seconds_monotonic_topk": dm, "seconds_topk_operator": df, "topk_operator_status": fstatus,
             "outputs_agree": agree, "arrangement_rows_monotonic_topk": marr,
             "arrangement_bytes_monotonic_topk": 72 * marr, "arrangement_rows_topk_operator": farr,
             "arrangement_bytes_topk_operator": None if farr is None else 32 * farr,
             "device_bytes_peak_monotonic_topk": peak_m, "device_bytes_peak_topk_operator": peak_f,
             "monotonic_topk_all_batches": {"batches": nb, "seconds": dm_all, "arrangement_rows": marr_all,
                                            "device_bytes_peak": peak_all}}
        )
        print(name, f"{dm:.4f} s / {df:.4f} s ({fstatus}), agree={agree}, all {nb}: {dm_all:.4f} s",
              file=sys.stderr, flush=True)
        del ins
        c.close()

    for limit in (1, 3):
        name = f"bulk monotonic TopK limit={limit} val1 desc n={n4} zipf0.9 keys={nk} R40"
        host = r40_cfg4(ctx, 5, n4) if not args.only or args.only in name else None
        lanes_case(
            name,
            n4,
            lambda c, host=host: mz.DeviceRows(c, 40).upload(host),
            lambda c, d, limit=limit: mz.TopKMonotonic(c, [mz.order_lane(1, descending=True)], limit, 40).step_dev(d, 1),
        )
        del host
    txt = json.dumps(res, indent=1)
    if args.out:
        open(args.out, "w").write(txt)
    print(txt)


if __name__ == "__main__":
    main()
