"""Activation times and arrangement bytes of the basic TopK (mzgpu_topk_basic_new).

1. Against the TopK operator (mzgpu_topk_new): 1 M-row R32 batches over Zipf(0.9) keys, ~10 % of each batch
   retracting earlier rows (never below zero, which the TopK operator refuses late), limit 3, one descending
   lane on val1.  Both operators see the same batches; the seconds are per activation, host input included.
2. One activation's time for a key of 10^3, 10^5 and 10^7 live rows: the key's group is loaded and compacted,
   then each timed activation inserts 50 rows and retracts 50 live rows of that key.  With the work bounded by
   the window, the time stays near flat as the group grows.

Prints one JSON object (and writes it to --out), with the card's name and power limit.
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001  (the numbers are still worth reporting)
        return {"gpu": None, "power_limit": None, "error": str(e)}


def zipf(rng, n, nk, s=0.9):
    p = 1.0 / np.arange(1, nk + 1) ** s
    return rng.choice(nk, size=n, p=p / p.sum()).astype(np.uint64)


def versus_topk_operator(mz, ctx, n, n_batches, limit):
    rng = np.random.default_rng(1)
    batches, live_k, live_v = [], np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    for b in range(n_batches):
        rows = np.zeros(n, dtype=mz.R32)
        rows["key"] = zipf(rng, n, 1_000_000)
        rows["val"] = rng.integers(0, 1 << 40, size=n, dtype=np.uint64)
        rows["time"] = 2 * b
        rows["diff"] = 1
        if len(live_k):  # retract ~10 % of the batch from distinct live rows
            m = min(n // 10, len(live_k))
            pick = rng.choice(len(live_k), size=m, replace=False)
            rows["key"][:m], rows["val"][:m], rows["diff"][:m] = live_k[pick], live_v[pick], -1
            keep = np.ones(len(live_k), bool)
            keep[pick] = False
            live_k, live_v = live_k[keep], live_v[keep]
        ins = rows["diff"] > 0
        live_k, live_v = np.concatenate([live_k, rows["key"][ins]]), np.concatenate([live_v, rows["val"][ins]])
        batches.append(rows)

    def run(make, step):
        op = make()
        secs, outs = [], []
        for b, rows in enumerate(batches):
            ctx.sync()
            t0 = time.perf_counter()
            out = step(op, rows, 2 * b + 2)
            ctx.sync()
            secs.append(time.perf_counter() - t0)
            outs.append(out)
        return op, secs, outs

    lane = [mz.order_lane(1, 0, 64, False, True)]
    g, s_new, o_new = run(lambda: mz.TopKBasic(ctx, lane, limit), lambda op, r, up: op.step(r, up)[0])
    old, s_old, o_old = run(lambda: mz.TopK(ctx, limit, 0, True), lambda op, r, up: op.step(r, up))
    agree = True
    for a, b in zip(o_new, o_old):
        ga = sorted(zip(a["key"].tolist(), a["val"].tolist(), a["diff"].tolist()))
        gb = sorted(zip(b["key"].tolist(), b["sum_lo"].tolist(), b["diff"].tolist()))
        agree &= ga == gb
    return {
        "rows_per_batch": n, "batches": n_batches, "limit": limit,
        "seconds_per_activation_topk_basic": s_new, "seconds_per_activation_topk_operator": s_old,
        "outputs_agree": agree,
        "arrangement_bytes_topk_basic": g.input_trace().size()["size_bytes"],
        "negatives_arrangement_bytes_topk_basic": g.negatives_trace().size()["size_bytes"],
        "arrangement_bytes_topk_operator": old.input_trace().size()["size_bytes"],
    }


def one_hot_key(mz, ctx, group, limit, reps=5):
    rng = np.random.default_rng(group)
    g = mz.TopKBasic(ctx, [mz.order_lane(1, 0, 64, False, True)], limit, 2)
    vals = rng.permutation(np.arange(1, group + 1, dtype=np.uint64) * 7)
    t0 = time.perf_counter()
    rows = np.zeros(group, dtype=mz.R32)  # the group in one activation (one thread walks a key's new rows)
    rows["key"], rows["val"], rows["time"], rows["diff"] = 5, vals, 0, 1
    g.step(rows, 1)
    t = 1
    tr = g.input_trace()
    tr.set_logical_compaction(t)
    for _ in range(8):  # idle activations fuel the spine's merges
        g.step(np.zeros(0, dtype=mz.R32), t + 1)
        t += 1
        tr.set_logical_compaction(t)
        tr.exert(1 << 40)
    load = time.perf_counter() - t0
    secs = []
    for r in range(reps):
        rows = np.zeros(100, dtype=mz.R32)
        rows["key"], rows["time"] = 5, t
        rows["val"][:50] = rng.integers(1, 1 << 40, size=50, dtype=np.uint64) * 7 + 3  # new values
        rows["diff"][:50] = 1
        rows["val"][50:] = vals[r * 50:(r + 1) * 50]  # live values retracted
        rows["diff"][50:] = -1
        dev = mz.DeviceRows(ctx, 32).upload(rows)
        ctx.sync()
        t1 = time.perf_counter()
        out, errs = g.step_dev(dev, t + 1)
        ctx.sync()
        secs.append(time.perf_counter() - t1)
        assert len(errs) == 0
        t += 1
    return {"live_rows": group, "limit": limit, "offset": 2, "load_seconds": load,
            "activation_seconds": secs, "activation_seconds_median": float(np.median(secs)),
            "arrangement_bytes": g.input_trace().size()["size_bytes"],
            "arrangement_batches": g.input_trace().size()["batches"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--batches", type=int, default=3)
    ap.add_argument("--groups", default="1000,100000,10000000")
    args = ap.parse_args()
    import materialize_b200 as mz

    ctx = mz.Context(0)
    res = dict(card())
    # warm-up: every kernel of both operators once
    versus_topk_operator(mz, ctx, 10_000, 2, 3)
    res["versus_topk_operator"] = versus_topk_operator(mz, ctx, args.rows, args.batches, 3)
    res["hot_key"] = [one_hot_key(mz, ctx, int(gs), 3) for gs in args.groups.split(",")]
    ctx.sync()
    text = json.dumps(res)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
