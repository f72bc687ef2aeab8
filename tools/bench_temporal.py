"""Sliding-window temporal filter: the Mfp operator against pushing the same future updates into a batcher.

Each step inserts `--tick` rows at time t with `mz_now() < t + W` (W = --window steps), so every row's
retraction is held W steps ahead and the held set grows to tick * W rows.  The operator releases only due
updates; the baseline pushes (+1 at t, -1 at t + W) into a batcher and seals at t + 1, which re-sorts every
held retraction at each seal.  Prints one JSON line per path: median / p90 step time (host clock around work
that ends in a device synchronise) over the last --measure steps, and device_bytes_peak.  Needs a GPU.
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


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception:  # noqa: BLE001
        return "unknown"


def rows_at(rng, n, t):
    r = np.zeros(n, dtype=mz.R32)
    r["key"] = rng.integers(0, 1 << 20, n, dtype=np.uint64)
    r["val"] = t
    r["time"] = t
    r["diff"] = 1
    return r


def run_mfp(args, rng):
    ctx = mz.Context(0)
    op = A.Mfp(ctx, [[(0, 0, 64, 0)], [(1, 0, 64, 0)], []], [],
               [(5, [A.col(1, 0, 64, code=F.HOP_COL_MZTS)]),  # mz_now() >= val
                (2, [A.col(1, 0, 40), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_ADD, 64), A.hop(F.HOP_INT_TO_MZTS)])],
               [(args.window, 0)])
    dev, out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    times = []
    for t in range(args.steps):
        dev.upload(rows_at(rng, args.tick, t))
        ctx.sync()
        t0 = time.perf_counter()
        F.lib.mzgpu_buf_clear(out.h)
        op.step_dev(dev, t + 1, out, errs)
        ctx.sync()
        times.append(time.perf_counter() - t0)
    return times, ctx.stats(), op.stats()


def run_batcher(args, rng):
    ctx = mz.Context(0)
    b = mz.Batcher(ctx, 32)
    dev = A.DeviceRows(ctx, 32)
    times = []
    for t in range(args.steps):
        r = rows_at(rng, args.tick, t)
        neg = r.copy()
        neg["time"] = t + args.window
        neg["diff"] = -1
        dev.upload(np.concatenate([r, neg]))
        ctx.sync()
        t0 = time.perf_counter()
        F.lib.mzgpu_batcher_push_buf(b.h, dev.h)
        b.seal(t + 1)
        ctx.sync()
        times.append(time.perf_counter() - t0)
    return times, ctx.stats(), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tick", type=int, default=100_000)
    ap.add_argument("--window", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=1100)
    ap.add_argument("--measure", type=int, default=50)
    ap.add_argument("--paths", default="mfp,batcher")
    args = ap.parse_args()
    gpu = gpu_name()
    for path in args.paths.split(","):
        rng = np.random.default_rng(0)
        times, st, ops = (run_mfp if path == "mfp" else run_batcher)(args, rng)
        w = np.array(times[-args.measure:]) * 1e3
        print(json.dumps({"path": path, "gpu": gpu, "tick": args.tick, "window": args.window, "steps": args.steps,
                          "step_ms_median": round(float(np.median(w)), 3),
                          "step_ms_p90": round(float(np.percentile(w, 90)), 3),
                          "device_bytes_peak": st["device_bytes_peak"],
                          "held_rows": ops[0] if ops else None, "buckets": ops[1] if ops else None}), flush=True)


if __name__ == "__main__":
    main()
