"""Join closures in the probe: a Q3-sized half join (mzgpu_half_join_buf / mzgpu_half_join_mfp_buf) three ways.

The stream (--stream rows, default 100,000, at time 1) probes one arrangement of --trace rows (default 64 Mi rows,
2 GiB of R32 rows plus the hash index, about four rows per key) at time 0.  Values are 40-bit: bits 0-23 and 24-31
of the lookup value are Q3's extendedprice and discount.  The closures:
- bit:       the bit-field closure key = v1 bits 0-19, val = a * (100 - b) (MZGPU_EXPR_MUL_CONST_MINUS);
- mfp_q3:    the same closure as an MfpPlan: one map expression a * (100 - b), projected as the value;
- mfp_cross: an MfpPlan with two cross-side predicates (v1 bits 0-15 < v2 bits 0-15, and key % 3 <> v1 % 3) and two
             map expressions (v1 * 3 - v2 and (v1 + v2) % 1000), both projected.
The three run alternately in one process, --reps calls each after --warmup: each call is timed by a host clock
around the call and a device synchronise (the unconsolidated output stays on the device).  A separate pass under
torch.profiler gives the probe kernels' device time per call.  Prints one JSON line per closure with the card's
name and power limit, read in the same run.  Needs a GPU.
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

SRC_MAP0 = F.SRC_MAP0
KONST = lambda k: A.hop(F.HOP_INT, konst=k)  # noqa: E731


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception:  # noqa: BLE001
        return "unknown"


def closures(ctx):
    bit = A.make_closure(key_fields=[(1, 0, 20, 0)], expr=((2, 0, 24), (2, 24, 8), 100))
    q3 = A.JoinClosure(ctx, [[(1, 0, 20, 0)], [(SRC_MAP0, 0, 64, 0)]],
                       maps=[[A.col(2, 0, 24), KONST(0), A.col(2, 24, 8), A.hop(F.HOP_SUB, 64),
                              A.hop(F.HOP_MUL, 64)]], map_consts=[(100, 0)])
    cross = A.JoinClosure(
        ctx, [[(0, 0, 64, 0)], [A.field_map(0, 0, 32, 0), A.field_map(1, 0, 16, 32)]],
        predicates=[[A.col(1, 0, 16), A.col(2, 0, 16), A.hop(F.HOP_CMP, 2)],
                    [A.col(0, 0, 32), KONST(0), A.hop(F.HOP_MOD, 64), A.col(1, 0, 32), KONST(0), A.hop(F.HOP_MOD, 64),
                     A.hop(F.HOP_CMP, 1)]],
        consts=[(3, 0)],
        maps=[[A.col(1, 0, 32), KONST(0), A.hop(F.HOP_MUL, 64), A.col(2, 0, 32), A.hop(F.HOP_SUB, 64)],
              [A.col(1, 0, 32), A.col(2, 0, 32), A.hop(F.HOP_ADD, 64), KONST(1), A.hop(F.HOP_MOD, 64)]],
        map_consts=[(3, 0), (1000, 0)])
    return {"bit": bit, "mfp_q3": q3, "mfp_cross": cross}


def rows(rng, n, keys, t):
    r = np.zeros(n, dtype=mz.R32)
    r["key"] = rng.integers(0, keys, n, dtype=np.uint64)
    r["val"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    r["time"] = t
    r["diff"] = 1
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stream", type=int, default=100_000)
    ap.add_argument("--trace", type=int, default=64 << 20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--profile", type=int, default=1)
    args = ap.parse_args()
    gpu = gpu_name()
    rng = np.random.default_rng(0)
    ctx = mz.Context(0)
    keys = max(1, args.trace // 4)
    sp = mz.Spine(ctx, 32)
    sp.insert(mz.Batch.build(ctx, rows(rng, args.trace, keys, 0), 0, 1))
    stream = A.DeviceRows(ctx, 32).upload(rows(rng, args.stream, keys, 1))
    cls = closures(ctx)
    outs = {k: (A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)) for k in cls}

    def call(name):
        out, errs = outs[name]
        F.lib.mzgpu_buf_clear(out.h)
        F.lib.mzgpu_buf_clear(errs.h)
        if name == "bit":
            A.half_join_dev(ctx, stream, sp, F.HALFJOIN_LE, cls[name], False, out)
        else:
            A.half_join_mfp_dev(ctx, stream, sp, F.HALFJOIN_LE, cls[name], False, out, errs)

    times = {k: [] for k in cls}
    for i in range(args.warmup + args.reps):
        for name in cls:  # alternating: the three share the machine's state within each round
            ctx.sync()
            t0 = time.perf_counter()
            call(name)
            ctx.sync()
            if i >= args.warmup:
                times[name].append((time.perf_counter() - t0) * 1e3)
    same_as_bit = outs["mfp_q3"][0].download().tobytes() == outs["bit"][0].download().tobytes()
    kernel_ms = {k: None for k in cls}
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        for name in cls:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    call(name)
                ctx.sync()
            ev = [e for e in prof.events() if "k_probe" in e.name]
            if ev:
                kernel_ms[name] = round(sum(e.time_range.elapsed_us() for e in ev) / args.reps / 1e3, 4)
    for name in cls:
        w = np.array(times[name])
        print(json.dumps({"closure": name, "stream_rows": args.stream, "trace_rows": args.trace,
                          "out_rows": len(outs[name][0]), "err_rows": len(outs[name][1]),
                          "call_ms_median": round(float(np.median(w)), 4),
                          "call_ms_p90": round(float(np.percentile(w, 90)), 4),
                          "probe_kernel_ms": kernel_ms[name], "mfp_q3_output_equals_bit": same_as_bit,
                          "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
