"""FlatMap on the device (mzgpu_flat_map_new) against what a caller does without it: expand on the host, upload,
and run mzgpu_mfp_step on the expanded rows.  The two are timed alternately in one process.

- bulk: N R32 rows, each generate_series(1, k) with k uniform in 0..16 (k in val), plus one predicate
  (value % 4 <> 3, written NOT(value % 4 = 3)); one activation per step, paged by --fuel.  Reports the step time
  (all pages, host clock ending in a device synchronise), function rows/s, the expansion kernel's time from
  torch.profiler in a separate pass and device_bytes_peak.
- hop: --hop-rows new rows per step, each fanned out to the 4 windows (of 20, hopping by 5) that contain its event
  time, with mz_now() >= window and mz_now() < window + 20 on the series column; median and p90 step time over
  --hop-steps steps.
The baseline's host expansion is numpy (np.repeat), and its time is included.  Prints one JSON line per
measurement with the card's name and power limit.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import materialize_b200 as mz  # noqa: E402
from materialize_b200 import _ffi as F  # noqa: E402
from materialize_b200 import api as A  # noqa: E402

K = lambda i: A.hop(F.HOP_INT, konst=i)  # noqa: E731
FN = A.col(F.SRC_FN0, 0, 64)


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception:  # noqa: BLE001
        return "unknown"


# value % 4 <> 3 over a column `v`
def pred(v):
    return [v, K(0), A.hop(F.HOP_MOD, 64), K(1), A.hop(F.HOP_CMP, 0), A.hop(F.HOP_NOT)]


PRED_CONSTS = [(4, 0), (3, 0)]


def bulk_ops(ctx):
    fm = A.FlatMap(ctx, F.TF_GENERATE_SERIES_INT64, [[K(0)], [A.col(1, 0, 64)], [K(0)]],
                   [[(0, 0, 64, 0)], [A.field_fn(0)], []], arg_consts=[(1, 0)], predicates=[pred(FN)],
                   consts=PRED_CONSTS)
    mfp = A.Mfp(ctx, [[(0, 0, 64, 0)], [(1, 0, 64, 0)], []], predicates=[pred(A.col(1, 0, 64))], consts=PRED_CONSTS)
    return fm, mfp


def host_expand_series(rows, first, last, step):
    """generate_series(first[i], last[i], step) per row, on the host: (key, value, time, diff) rows."""
    cnt = np.maximum((last - first) // step + 1, 0)
    idx = np.repeat(np.arange(len(rows)), cnt)
    j = np.arange(len(idx)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    out = np.zeros(len(idx), dtype=mz.R32)
    out["key"] = rows["key"][idx]
    out["val"] = (first[idx] + j * step).astype(np.uint64)
    out["time"] = rows["time"][idx]
    out["diff"] = rows["diff"][idx]
    return out


def run_fm(ctx, fm, dev, upper, fuel, out, errs):
    out_, errs_, done = fm.step_dev(dev, upper, fuel, out, errs)
    while not done:
        _, _, done = fm.work(fuel, out, errs)


def bulk(args, gpu):
    ctx = mz.Context(0)
    rng = np.random.default_rng(0)
    n = args.rows
    rows = np.zeros(n, dtype=mz.R32)
    rows["key"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    rows["val"] = rng.integers(0, 17, n, dtype=np.uint64)
    rows["diff"] = 1
    fm, mfp = bulk_ops(ctx)
    dev = A.DeviceRows(ctx, 32).upload(rows)
    out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    t_fm, t_base = [], []
    fn_rows = int(rows["val"].astype(np.int64).sum())
    for i in range(args.warmup + args.reps):
        for which in ("fm", "base"):
            F.lib.mzgpu_buf_clear(out.h)
            F.lib.mzgpu_buf_clear(errs.h)
            ctx.sync()
            t0 = time.perf_counter()
            if which == "fm":
                run_fm(ctx, fm, dev, 16 + i, args.fuel, out, errs)
            else:
                ex = host_expand_series(rows, np.ones(n, dtype=np.int64), rows["val"].astype(np.int64), 1)
                d2 = A.DeviceRows(ctx, 32).upload(ex)
                mfp.step_dev(d2, 16 + i, out, errs)
            ctx.sync()
            if i >= args.warmup:
                (t_fm if which == "fm" else t_base).append(time.perf_counter() - t0)
    kernel_ms = None
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.reps):
                F.lib.mzgpu_buf_clear(out.h)
                run_fm(ctx, fm, dev, 100 + i, args.fuel, out, errs)
            ctx.sync()
        ev = [e for e in prof.events() if "k_fm_expand" in e.name]
        if ev:
            kernel_ms = sum(e.time_range.elapsed_us() for e in ev) / args.reps / 1e3
    fm_ms, base_ms = float(np.median(t_fm)) * 1e3, float(np.median(t_base)) * 1e3
    print(json.dumps({"bench": "bulk", "rows": n, "function_rows": fn_rows, "fuel": args.fuel,
                      "pages": -(-fn_rows // args.fuel), "flat_map_step_ms_median": round(fm_ms, 3),
                      "function_rows_per_s": round(fn_rows / (fm_ms / 1e3)),
                      "k_fm_expand_ms_per_activation": kernel_ms,
                      "host_expand_upload_mfp_ms_median": round(base_ms, 3),
                      "device_bytes_peak": ctx.stats().get("device_bytes_peak"), "gpu": gpu}), flush=True)


def hop(args, gpu):
    ctx = mz.Context(0)
    rng = np.random.default_rng(1)
    t_ = A.col(1, 0, 32, signed=True)
    start = [t_, t_, K(0), A.hop(F.HOP_MOD, 64), A.hop(F.HOP_SUB, 64), K(1), A.hop(F.HOP_SUB, 64)]
    stop = [t_, t_, K(0), A.hop(F.HOP_MOD, 64), A.hop(F.HOP_SUB, 64)]
    temporal = [(5, [FN, A.hop(F.HOP_INT_TO_MZTS)]), (2, [FN, K(0), A.hop(F.HOP_ADD, 64), A.hop(F.HOP_INT_TO_MZTS)])]
    fm = A.FlatMap(ctx, F.TF_GENERATE_SERIES_INT64, [start, stop, [K(0)]], [[(0, 0, 64, 0)], [A.field_fn(0)], []],
                   arg_consts=[(5, 0), (15, 0)], temporal=temporal, consts=[(20, 0)])
    tb = A.col(1, 0, 64)
    base = A.Mfp(ctx, [[(0, 0, 64, 0)], [(1, 0, 64, 0)], []],
                 temporal=[(5, [tb, A.hop(F.HOP_INT_TO_MZTS)]), (2, [tb, K(0), A.hop(F.HOP_ADD, 64),
                                                                    A.hop(F.HOP_INT_TO_MZTS)])], consts=[(20, 0)])
    out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    res = {"fm": [], "base": []}
    for s in range(args.hop_steps):
        r = np.zeros(args.hop_rows, dtype=mz.R32)
        r["key"] = rng.integers(0, 1 << 40, args.hop_rows, dtype=np.uint64)
        ev = (s * 5 + 20 + rng.integers(0, 5, args.hop_rows)).astype(np.int64)
        r["val"] = ev.astype(np.uint64)
        r["time"] = s * 5
        r["diff"] = 1
        for which in ("fm", "base"):
            F.lib.mzgpu_buf_clear(out.h)
            F.lib.mzgpu_buf_clear(errs.h)
            ctx.sync()
            t0 = time.perf_counter()
            if which == "fm":
                d = A.DeviceRows(ctx, 32).upload(r)
                run_fm(ctx, fm, d, s * 5 + 5, args.fuel, out, errs)
            else:
                w0 = ev - ev % 5 - 15
                ex = host_expand_series(r, w0, ev - ev % 5, 5)
                base.step_dev(A.DeviceRows(ctx, 32).upload(ex), s * 5 + 5, out, errs)
            ctx.sync()
            if s >= args.warmup:
                res[which].append((time.perf_counter() - t0) * 1e3)
    f, b = np.array(res["fm"]), np.array(res["base"])
    print(json.dumps({"bench": "hop", "rows_per_step": args.hop_rows, "steps": len(f),
                      "flat_map_step_ms_median": round(float(np.median(f)), 3),
                      "flat_map_step_ms_p90": round(float(np.percentile(f, 90)), 3),
                      "host_expand_upload_mfp_ms_median": round(float(np.median(b)), 3),
                      "host_expand_upload_mfp_ms_p90": round(float(np.percentile(b, 90)), 3), "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1000000)
    ap.add_argument("--fuel", type=int, default=1000000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", type=int, default=1)
    ap.add_argument("--hop-rows", type=int, default=100000)
    ap.add_argument("--hop-steps", type=int, default=200)
    ap.add_argument("--which", default="bulk,hop")
    args = ap.parse_args()
    gpu = gpu_name()
    if "bulk" in args.which:
        bulk(args, gpu)
    if "hop" in args.which:
        hop(args, gpu)


if __name__ == "__main__":
    main()
