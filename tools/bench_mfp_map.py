"""Map expressions in the device MfpPlan (mzgpu_mfp_new_map): mzgpu_mfp_step_buf rows/s and k_mfp_eval kernel time.

Plans, over R32 rows (key, val) at time 0 stepped to upper 16:
- identity: no expressions, (key, val) projected as they are (the mzgpu_mfp_new path);
- maps4: val * 3, IF(val > 100, 1, 0), key % 16 and ABS(val - 500), projected as
  (key % 16, val * 3 | flag << 40 | ABS(val - 500) << 48);
- maps4_temporal: the same with mz_now() >= (val % 16)::mz_timestamp read from a fifth expression: every bound is
  below the upper, so nothing is held and each step's work stays its new rows.
Step time is a host clock around one step that ends in a device synchronise (it includes the consolidation of the
output); kernel time is k_mfp_eval's device time from torch.profiler in a separate pass.  Prints one JSON line per
(plan, rows) with the card's name and power limit.  Needs a GPU.
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

HOP_INT = lambda k: A.hop(F.HOP_INT, konst=k)  # noqa: E731
VAL32 = A.col(1, 0, 32, signed=True)
KEY = A.col(0, 0, 64)
MAPS4 = [[VAL32, HOP_INT(0), A.hop(F.HOP_MUL, 64)],
         [VAL32, HOP_INT(1), A.hop(F.HOP_CMP, 4), HOP_INT(2), HOP_INT(3), A.hop(F.HOP_IF)],
         [KEY, HOP_INT(4), A.hop(F.HOP_MOD, 64)],
         [VAL32, HOP_INT(5), A.hop(F.HOP_SUB, 32), A.hop(F.HOP_ABS, 32)]]
MAP_CONSTS = [(3, 0), (100, 0), (1, 0), (0, 0), (16, 0), (500, 0)]
MZTS = [VAL32, HOP_INT(4), A.hop(F.HOP_MOD, 32), A.hop(F.HOP_INT_TO_MZTS)]


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception:  # noqa: BLE001
        return "unknown"


def make(ctx, plan):
    if plan == "identity":
        return A.Mfp(ctx, [[(0, 0, 64, 0)], [(1, 0, 64, 0)], []])
    fields = [[A.field_map(2)], [A.field_map(0, 0, 40, 0), A.field_map(1, 0, 1, 40), A.field_map(3, 0, 16, 48)], []]
    if plan == "maps4":
        return A.Mfp(ctx, fields, maps=MAPS4, map_consts=MAP_CONSTS)
    return A.Mfp(ctx, fields, temporal=[(5, [A.map_ref(4)])], maps=MAPS4 + [MZTS], map_consts=MAP_CONSTS)


def rows_of(rng, n):
    r = np.zeros(n, dtype=mz.R32)
    r["key"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    r["val"] = rng.integers(0, 1000, n, dtype=np.uint64)
    r["diff"] = 1
    return r


def measure(args, plan, n):
    ctx = mz.Context(0)
    op = make(ctx, plan)
    dev = A.DeviceRows(ctx, 32).upload(rows_of(np.random.default_rng(0), n))
    out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    times = []
    for i in range(args.warmup + args.reps):
        F.lib.mzgpu_buf_clear(out.h)
        F.lib.mzgpu_buf_clear(errs.h)
        ctx.sync()
        t0 = time.perf_counter()
        op.step_dev(dev, 16, out, errs)
        ctx.sync()
        if i >= args.warmup:
            times.append(time.perf_counter() - t0)
    kernel_ms = None
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                F.lib.mzgpu_buf_clear(out.h)
                op.step_dev(dev, 16, out, errs)
            ctx.sync()
        ev = [e for e in prof.events() if "k_mfp_eval" in e.name]
        if ev:
            kernel_ms = sum(e.time_range.elapsed_us() for e in ev) / len(ev) / 1e3
    w = np.array(times) * 1e3
    return {"plan": plan, "rows": n, "step_ms_median": round(float(np.median(w)), 3),
            "rows_per_s": round(n / (float(np.median(w)) / 1e3)), "k_mfp_eval_ms": kernel_ms,
            "out_rows": len(out)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1000000,10000000")
    ap.add_argument("--plans", default="identity,maps4,maps4_temporal")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", type=int, default=1)
    args = ap.parse_args()
    gpu = gpu_name()
    for n in (int(x) for x in args.rows.split(",")):
        for plan in args.plans.split(","):
            r = measure(args, plan, n)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
