"""The temporal filter (mzgpu_mfp_new) on the GPU, step for step against tests/mfp_oracle.py."""
import json
import os

import numpy as np
import pytest

import mfp_oracle as O

pytestmark = pytest.mark.gpu

mz = pytest.importorskip("materialize_b200")
from materialize_b200 import api as A  # noqa: E402
from materialize_b200 import _ffi as F  # noqa: E402

IDENT32 = [[(0, 0, 64, 0)], [(1, 0, 64, 0)], []]
IDENT40 = [[(0, 0, 64, 0)], [(1, 0, 64, 0)], [(2, 0, 64, 0)]]


@pytest.fixture(scope="module")
def ctx():
    return mz.Context(0)


def rows_of(rb, key, val, time, diff, val2=None):
    r = np.zeros(len(key), dtype=mz.R32 if rb == 32 else mz.R40)
    r["key"] = key
    if rb == 32:
        r["val"] = val
    else:
        r["val1"] = val
        r["val2"] = val2 if val2 is not None else val
    r["time"] = time
    r["diff"] = diff
    return r


def as_tuples(arr, rb):
    nw = rb // 8
    v = arr.view(np.uint64).reshape(-1, nw)
    return [(tuple(int(x) for x in r[: nw - 2]), int(r[nw - 2]), O.s64(int(r[nw - 1]))) for r in v]


def err_tuples(arr):
    v = arr.view(np.uint64).reshape(-1, 4)
    return [((int(r[0]), int(r[1])), int(r[2]), O.s64(int(r[3]))) for r in v]


def plan_of(fields, predicates=(), temporal=(), consts=()):
    return {"fields": [f for f in fields if f or fields.index(f) < 2], "predicates": list(predicates),
            "temporal": list(temporal), "consts": list(consts)}


def run_history(ctx, fields, predicates, temporal, consts, steps, in_rb=32, out_rb=32, until=O.EMPTY,
                check_frontier=True):
    op = A.Mfp(ctx, fields, predicates, temporal, consts, in_row_bytes=in_rb, out_row_bytes=out_rb, until=until)
    ref = O.Operator({"fields": fields[: out_rb // 8 - 2], "predicates": predicates, "temporal": temporal,
                      "consts": consts}, until, in_rb // 8)
    for rows, upper in steps:
        out, errs = op.step(rows, upper)
        want_out, want_err = ref.step(rows, upper)
        ref_out = [(tuple(w[: out_rb // 8 - 2]), t, d) for w, t, d in want_out]
        assert as_tuples(out, out_rb) == ref_out, upper
        assert err_tuples(errs) == want_err, upper
        if check_frontier:
            assert op.frontier() == ref.frontier()
            assert op.stats()[0] == ref.held()
    return op, ref


# mz_now() CMP (val + offset)::mz_timestamp, or val itself as an mz_timestamp column
def window_expr(kind, shift=0):
    if kind == "col":
        return [A.col(1, 0, 64, code=F.HOP_COL_MZTS)]
    if kind == "int":
        return [A.col(1, 0, 32), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_ADD, 64), A.hop(F.HOP_INT_TO_MZTS)]
    if kind == "ts":  # (val::timestamp + interval '1 second')::mz_timestamp
        return [A.col(1, 0, 64, signed=True, code=F.HOP_COL_TS), A.hop(F.HOP_TS_ADD_IV, konst=1),
                A.hop(F.HOP_TS_TO_MZTS)]
    if kind == "date":
        return [A.col(1, 0, 16, code=F.HOP_COL_DATE), A.hop(F.HOP_DATE_TO_MZTS)]
    raise ValueError(kind)


CONSTS = [(50, 0), A.interval_const(micros=1_000_000)]


def zipf_steps(rng, n_steps, rb, per_step=300, tmax=400, val_hi=300):
    steps, live = [], []
    for s in range(n_steps):
        n = per_step
        key = rng.zipf(1.3, n).astype(np.uint64) % 1000
        val = rng.integers(0, val_hi, n, dtype=np.uint64)
        time = np.full(n, s * 5, dtype=np.uint64)
        diff = rng.choice([1, 1, 2, -1], n).astype(np.int64)
        r = rows_of(rb, key, val, time, diff, val2=rng.integers(0, 4, n, dtype=np.uint64))
        if live and s % 3 == 2:  # retract some earlier rows
            old = live[rng.integers(0, len(live))].copy()[:50]
            old["time"] = s * 5
            old["diff"] = -old["diff"]
            r = np.concatenate([r, old])
        live.append(r)
        steps.append((r, s * 5 + 5))
    return steps


@pytest.mark.parametrize("rb", [32, 40])
@pytest.mark.parametrize("cmp", [O.EQ, O.LT, O.LE, O.GT, O.GE])
@pytest.mark.parametrize("kind", ["col", "int"])
def test_history_each_cmp(ctx, rb, cmp, kind):
    rng = np.random.default_rng(cmp * 7 + rb + len(kind))
    fields = IDENT32 if rb == 32 else IDENT40
    run_history(ctx, fields, [], [(cmp, window_expr(kind))], CONSTS, zipf_steps(rng, 40, rb), in_rb=rb, out_rb=rb)


@pytest.mark.parametrize("until", [O.EMPTY, 120, 0])
def test_sliding_window_with_predicate_and_projection(ctx, until):
    # WHERE key % 3 <> 1 AND mz_now() >= val AND mz_now() < val + 50; projected to (val, key) as R40 -> R32
    rng = np.random.default_rng(until % 97)
    pred = [A.col(0, 0, 32), A.hop(F.HOP_INT, konst=2), A.hop(F.HOP_DIV, 64), A.hop(F.HOP_INT, konst=2),
            A.hop(F.HOP_MUL, 64), A.col(0, 0, 32), A.hop(F.HOP_SUB, 64), A.hop(F.HOP_INT, konst=3),
            A.hop(F.HOP_CMP, O.NE)]
    consts = CONSTS + [(3, 0), (2**64 - 1, 2**64 - 1)]
    temporal = [(O.GE, window_expr("col")), (O.LT, window_expr("int"))]
    fields = [[(1, 0, 64, 0)], [(0, 0, 32, 0), (2, 0, 8, 32)], []]
    run_history(ctx, fields, [pred], temporal, consts, zipf_steps(rng, 40, 40), in_rb=40, out_rb=32, until=until)


def test_four_temporal_predicates_and_casts(ctx):
    rng = np.random.default_rng(5)
    temporal = [(O.GE, window_expr("col")), (O.LE, window_expr("int")), (O.LT, window_expr("ts")),
                (O.GT, window_expr("date"))]
    run_history(ctx, IDENT32, [], temporal, CONSTS, zipf_steps(rng, 30, 32, val_hi=2000))


def test_errors_and_suppressed_errors(ctx):
    # predicate val / (key - 5) > 0: division by zero at key 5;  bounds: val::mz_timestamp (negative values fail)
    pred = [A.col(1, 0, 64, signed=True), A.col(0, 0, 64), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_SUB, 64),
            A.hop(F.HOP_DIV, 64), A.hop(F.HOP_INT, konst=1), A.hop(F.HOP_CMP, O.GE)]
    neg_cast = [A.col(1, 0, 64, signed=True), A.hop(F.HOP_INT_TO_MZTS)]
    step_max = [A.col(0, 0, 64, code=F.HOP_COL_MZTS)]  # mz_now() <= key: step(u64::MAX) overflows
    ts_range = [A.col(1, 0, 64, signed=True, code=F.HOP_COL_TS), A.hop(F.HOP_TS_ADD_IV, konst=2),
                A.hop(F.HOP_TS_TO_MZTS)]
    consts = [(5, 0), (0, 0), A.interval_const(days=10**8)]
    cases = [
        ([pred], [(O.GE, neg_cast)]),
        ([], [(O.LE, step_max)]),
        ([], [(O.LT, ts_range)]),
        # lower not valid (until): a later upper-bound error is never raised
        ([], [(O.GE, [A.col(0, 0, 64, code=F.HOP_COL_MZTS)]), (O.LE, step_max)]),
        # upper == lower stops evaluation: the second upper bound's error is suppressed
        ([], [(O.LT, [A.hop(F.HOP_INT, konst=1), A.hop(F.HOP_INT_TO_MZTS)]), (O.LT, neg_cast)]),
        # the first lower-bound error wins
        ([], [(O.GE, neg_cast), (O.GT, step_max)]),
    ]
    key = np.array([5, 5, 1, 2, 2**64 - 1, 7, 9], dtype=np.uint64)
    val = np.array([3, 2**64 - 5, 2**64 - 1, 10, 4, 2**63 + 1, 0], dtype=np.uint64)
    for until in (O.EMPTY, 2**64 - 2):
        for preds, temporal in cases:
            rows = rows_of(32, key, val, np.arange(7, dtype=np.uint64), np.array([1, 2, 3, -1, 1, 1, 4]))
            run_history(ctx, IDENT32, preds, temporal, consts, [(rows, 3), (rows[:0], 20), (rows[:0], O.EMPTY)],
                        until=until)


def test_bucket_chain_edges(ctx):
    # rows held millions of ticks ahead, released a few at a time; a straddling split at each step; an upper
    # jumping past many buckets; upper = FRONTIER_EMPTY; empty steps
    rng = np.random.default_rng(11)
    n = 5000
    key = rng.integers(0, 100, n, dtype=np.uint64)
    val = (rng.integers(0, 3_000_000, n) + 1_000_000).astype(np.uint64)
    rows = rows_of(32, key, val, np.zeros(n, dtype=np.uint64), np.ones(n, dtype=np.int64))
    temporal = [(O.GE, window_expr("col"))]
    steps = [(rows, 1)]
    up = 1_000_000
    for _ in range(10):
        up += int(rng.integers(1, 50))
        steps.append((rows[:0], up))
    steps += [(rows[:0], 2_500_000), (rows[:0], 2_500_000), (rows[:0], 3_999_000)]
    for _ in range(5):
        up = steps[-1][1] + 7
        steps.append((rows[:0], up))
    steps.append((rows[:0], O.EMPTY))
    steps.append((rows[:0], O.EMPTY))
    run_history(ctx, IDENT32, [], temporal, CONSTS, steps)
    # time u64::MAX is released only by the empty frontier
    far = rows_of(32, [1], [2**64 - 1], [0], [1])
    run_history(ctx, IDENT32, [], temporal, CONSTS, [(far, 10), (far[:0], 2**64 - 2), (far[:0], O.EMPTY)])


def test_device_input_with_device_length(ctx):
    rng = np.random.default_rng(3)
    temporal = [(O.GE, window_expr("col")), (O.LT, window_expr("int"))]
    op = A.Mfp(ctx, IDENT32, [], temporal, CONSTS)
    ref = O.Operator({"fields": IDENT32[:2], "predicates": [], "temporal": temporal, "consts": CONSTS})
    out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    want = []
    for rows, upper in zipf_steps(rng, 12, 32):
        dev = A.DeviceRows(ctx, 32).upload(np.concatenate([rows, rows[:10]]))
        F.lib.mzgpu_buf_consolidate(dev.h)  # the length now lives on the device
        cons = O.consolidate([((int(r["key"]), int(r["val"])), int(r["time"]), int(r["diff"]))
                              for r in np.concatenate([rows, rows[:10]])])
        crow = rows_of(32, [w[0] for w, _, _ in cons], [w[1] for w, _, _ in cons], [t for _, t, _ in cons],
                       [d for _, _, d in cons]) if cons else rows[:0]
        op.step_dev(dev, upper, out, errs)
        want.extend(ref.step(crow, upper)[0])
    assert as_tuples(out.download(), 32) == [(w, t, d) for w, t, d in want]


def test_work_bound(ctx):
    n = 1_000_000
    rows = rows_of(32, np.arange(n, dtype=np.uint64), np.full(n, 10**12, dtype=np.uint64),
                   np.zeros(n, dtype=np.uint64), np.ones(n, dtype=np.int64))
    op = A.Mfp(ctx, IDENT32, [], [(O.GE, window_expr("col"))], CONSTS)
    op.step(rows, 1)
    for _ in range(3):  # restore the chain
        op.step(rows[:0], 2)
    touched = []
    for u in range(3, 200):
        op.step(rows[:0], u * 1000)
        touched.append(op.stats()[2])
    assert max(touched) == 0, touched
    assert op.stats()[0] == n


def test_sliding_window_work_is_amortised(ctx):
    # each step inserts R rows whose retraction is W ticks ahead; rows touched stay within
    # (new + released) * (2 + 2 * (log2(W) + 2)) over the run
    rng = np.random.default_rng(9)
    W, R, steps = 512, 2000, 300
    temporal = [(O.LT, window_expr("int"))]
    consts = [(W, 0)]
    op = A.Mfp(ctx, IDENT32, [], temporal, consts)
    total = 0
    for s in range(steps):
        rows = rows_of(32, rng.integers(0, 100, R, dtype=np.uint64), np.full(R, s, dtype=np.uint64),
                       np.full(R, s, dtype=np.uint64), np.ones(R, dtype=np.int64))
        op.step(rows, s + 1)
        total += op.stats()[2]
    moved = steps * R * 2
    assert total <= moved * (2 + 2 * (np.log2(W) + 2)), (total, moved)


def test_end_to_end_sliding_count(ctx):
    # SELECT key, COUNT(*) ... WHERE mz_now() >= val AND mz_now() < val + 20 GROUP BY key, built as
    # Mfp -> batcher -> spine -> mzgpu_reduce_lanes_new (one COUNT lane); the reduce's accumulated output equals a
    # direct count over the rows valid at every step, and the batcher holds nothing after each seal
    rng = np.random.default_rng(21)
    temporal = [(O.GE, window_expr("col")), (O.LT, window_expr("int"))]
    op = A.Mfp(ctx, IDENT32, [], temporal, [(20, 0)])
    batcher, spine = mz.Batcher(ctx, 32), mz.Spine(ctx, 32)
    red = mz.ReduceLanes(ctx, [mz.accum_lane(F.AGG_COUNT_SUM_I64, 1, 0, 64)], 32)
    history, counts = [], {}
    for s in range(40):
        n = 200
        rows = rows_of(32, rng.integers(0, 30, n, dtype=np.uint64), s + rng.integers(0, 4, n, dtype=np.uint64),
                       np.full(n, s, dtype=np.uint64), rng.choice([1, 1, 1, 2], n).astype(np.int64))
        if history and s % 4 == 3:  # retract rows inserted earlier
            old = history[-2][:40].copy()
            old["time"] = s
            old["diff"] = -old["diff"]
            rows = np.concatenate([rows, old])
        history.append(rows)
        out, errs = op.step(rows, s + 1)
        assert len(errs) == 0
        batcher.push_container(out)
        batch = batcher.seal(s + 1)
        assert F.lib.mzgpu_batcher_len(batcher.h) == 0  # only due rows were released
        batch_rows = batch.rows()
        spine.insert(batch)
        for r in red.step(batch_rows, s + 1):
            k = int(r["key"])
            counts[k] = counts.get(k, 0) + int(r["diff"]) * int(r["lanes"][0]["count"])
        want = {}
        for r in np.concatenate(history):
            if int(r["val"]) <= s < int(r["val"]) + 20:
                want[int(r["key"])] = want.get(int(r["key"]), 0) + int(r["diff"])
        assert {k: v for k, v in counts.items() if v} == {k: v for k, v in want.items() if v}, s


GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "temporal_filters.json")))


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[c["view"] for c in GOLDEN["cases"]])
def test_golden_answers(ctx, case):
    """Materialize's expected answers (temporal.slt, temporal.td) from the operator on the device."""
    plan = O.golden_plan(case)
    op = A.Mfp(ctx, IDENT32, [], plan["temporal"], plan["consts"])

    def step(rows, upper):
        arr = rows_of(32, [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], [r[3] for r in rows])
        out, errs = op.step(arr, upper)
        return as_tuples(out, 32), err_tuples(errs)

    assert O.golden_check(case, step) == []


def test_projection_r32_to_r40(ctx):
    # R32 input projected to R40 output: (key, val >> 8, val & 0xff | key << 8) under a sliding window
    rng = np.random.default_rng(17)
    fields = [[(0, 0, 64, 0)], [(1, 8, 56, 0)], [(1, 0, 8, 0), (0, 0, 16, 8)]]
    temporal = [(O.GE, [A.col(1, 0, 8, code=F.HOP_COL_MZTS)]), (O.LT, [A.col(1, 0, 8), A.hop(F.HOP_INT, konst=0),
                                                                       A.hop(F.HOP_ADD, 64), A.hop(F.HOP_INT_TO_MZTS)])]
    steps = zipf_steps(rng, 30, 32, val_hi=1 << 16)
    run_history(ctx, fields, [], temporal, CONSTS, steps, in_rb=32, out_rb=40)


def test_creation_refusals_leave_the_context_usable(ctx):
    ok = [(O.GE, window_expr("col"))]
    good = dict(fields=IDENT32, predicates=[], temporal=ok, consts=CONSTS)

    def refused(code, **kw):
        args = dict(good)
        args.update(kw)
        rb_in = args.pop("in_row_bytes", 32)
        rb_out = args.pop("out_row_bytes", 32)
        with pytest.raises(A.MzGpuError) as e:
            A.Mfp(ctx, args["fields"], args["predicates"], args["temporal"], args["consts"], in_row_bytes=rb_in,
                  out_row_bytes=rb_out)
        assert e.value.status == code, e.value
        A.Mfp(ctx, IDENT32, [], ok, CONSTS).step(rows_of(32, [1], [2], [0], [1]), 1)

    INV, UNS = F.E_INVALID, F.E_UNSUPPORTED
    refused(INV, in_row_bytes=24)
    refused(INV, out_row_bytes=48)
    refused(INV, fields=[[(0, 0, 64, 0)], [(2, 0, 64, 0)], []])  # VAL2 of an R32 input
    refused(INV, fields=[[(0, 0, 64, 0)], [(1, 0, 64, 0)], [(1, 0, 8, 0)]])  # val2 of an R32 output
    refused(INV, fields=[[(0, 0, 0, 0)], [], []])
    refused(INV, predicates=[[A.hop(F.HOP_COUNT)]])
    refused(INV, predicates=[[A.hop(F.HOP_SUM)]])
    refused(INV, predicates=[[A.hop(F.HOP_NUM)]])
    refused(INV, predicates=[[A.hop(F.HOP_FLOAT)]])
    refused(INV, predicates=[[A.col(0), A.col(0)]])  # leaves two values
    refused(INV, predicates=[[A.hop(F.HOP_ADD, 64)]])  # underflow
    refused(INV, predicates=[[A.col(0)] * 9])  # overflow
    refused(INV, predicates=[[A.hop(99)]])
    refused(INV, predicates=[[A.col(0), A.hop(F.HOP_INT, konst=7), A.hop(F.HOP_CMP, 0)]])  # constant index
    refused(INV, predicates=[[]])
    refused(INV, predicates=[[A.col(0)]] * 5)
    refused(INV, temporal=[(O.GE, [A.col(1)])])  # leaves an INT
    refused(INV, temporal=[(9, window_expr("col"))])
    refused(INV, temporal=[(O.GE, [A.col(1), A.hop(F.HOP_TS_TO_MZTS)])])  # INT is not a timestamp
    refused(INV, temporal=ok * 5)
    refused(UNS, temporal=[(O.NE, window_expr("col"))])
    refused(UNS, temporal=[(O.LT, window_expr("ts"))], consts=[(0, 0), A.interval_const(months=1)])
    refused(UNS, predicates=[[A.col(1, code=F.HOP_COL_MZTS), A.col(1, code=F.HOP_COL_MZTS), A.hop(F.HOP_CMP, 0)]])
    refused(UNS, predicates=[[A.col(1, code=F.HOP_COL_F64), A.col(1, code=F.HOP_COL_F64), A.hop(F.HOP_CMP, 0)]])
    refused(INV, temporal=[(O.GE, [A.col(1, 0, 32, signed=True, code=F.HOP_COL_MZTS)])])  # mz_timestamp is unsigned
