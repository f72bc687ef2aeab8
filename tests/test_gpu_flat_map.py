"""FlatMap (mzgpu_flat_map_new) on the GPU, byte for byte against tests/flat_map_oracle.py."""
import json
import os
import random

import numpy as np
import pytest

import flat_map_oracle as FM
import mfp_map_oracle as M
import mfp_oracle as O

pytestmark = pytest.mark.gpu

mz = pytest.importorskip("materialize_b200")
from materialize_b200 import api as A  # noqa: E402
from materialize_b200 import _ffi as F  # noqa: E402

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "table_func.json")))
U64 = 2**64


@pytest.fixture(scope="module")
def ctx():
    return mz.Context(0)


def rows_of(rb, words, time, diff):
    """rows from lists of words (key, val1[, val2])"""
    r = np.zeros(len(words), dtype=mz.R32 if rb == 32 else mz.R40)
    if len(words):
        w = np.array([[x % U64 for x in ws] + [0] * (3 - len(ws)) for ws in words], dtype=np.uint64)
        r["key"] = w[:, 0]
        if rb == 32:
            r["val"] = w[:, 1]
        else:
            r["val1"], r["val2"] = w[:, 1], w[:, 2]
    r["time"] = np.asarray(time, dtype=np.uint64) if np.ndim(time) else time
    r["diff"] = np.asarray([d % U64 for d in diff], dtype=np.uint64) if np.ndim(diff) else diff % U64
    return r


def as_tuples(arr, rb):
    nw = rb // 8
    v = arr.view(np.uint64).reshape(-1, nw)
    return [(tuple(int(x) for x in r[: nw - 2]), int(r[nw - 2]), O.s64(int(r[nw - 1]))) for r in v]


def err_tuples(arr):
    v = arr.view(np.uint64).reshape(-1, 4)
    return [((int(r[0]), int(r[1])), int(r[2]), O.s64(int(r[3]))) for r in v]


def make(ctx, tf, plan, in_rb, out_rb, until=O.EMPTY):
    fields = [list(f) for f in plan["fields"]] + [[]] * (3 - len(plan["fields"]))
    return A.FlatMap(ctx, tf["kind"], tf["args"], fields, with_ordinality=tf.get("with_ordinality", False),
                     arg_consts=tf.get("consts", []), step_iv=(tf.get("step_us", 0), 0),
                     predicates=plan["predicates"], temporal=plan["temporal"], consts=plan["consts"],
                     in_row_bytes=in_rb, out_row_bytes=out_rb, until=until, maps=plan.get("maps", []),
                     map_consts=plan.get("map_consts", []))


def run_both(ctx, tf, plan, steps, in_rb=32, out_rb=32, until=O.EMPTY, fuel=10**6):
    """steps of (rows, upper) through the device and the restatement, page by page, compared byte for byte."""
    op, ref = make(ctx, tf, plan, in_rb, out_rb, until), FM.Operator(tf, plan, until, in_rb // 8)
    acc_out, acc_err = [], []
    for rows, upper in steps:
        out, errs, done = op.step(rows, upper, fuel)
        r_out, r_err, r_done = ref.step(rows, upper, fuel)
        while True:
            assert as_tuples(out, out_rb) == r_out
            assert err_tuples(errs) == r_err
            assert done == r_done
            acc_out += r_out
            acc_err += r_err
            if done:
                break
            out, errs, done = op.work(fuel)
            r_out, r_err, r_done = ref.work(fuel)
    return O.consolidate(acc_out), O.consolidate(acc_err)


def _consts(vals):
    return [(v % U64, U64 - 1 if v < 0 else 0) for v in vals]


def tf_of(kind, args, consts=(), ordinality=False, step_us=0):
    return {"kind": kind, "args": args, "consts": _consts(consts), "with_ordinality": ordinality, "step_us": step_us}


def k(i):
    return (O.HOP_INT, 0, 0, 0, 0, i)


def c32(word, shift=0):
    return (O.HOP_COL, word, shift, 32, 1, 0)


def c64(word):
    return (O.HOP_COL, word, 0, 64, 0, 0)


def plan_of(out_rb, fn_cols, predicates=(), temporal=(), consts=()):
    """output: key = input key, val1 = the first extension column (or the input val1), val2 = the second"""
    f1 = [(F.SRC_FN0, 0, 64, 0)] if fn_cols >= 1 else [(1, 0, 64, 0)]
    fields = [[(0, 0, 64, 0)], f1]
    if out_rb == 40:
        fields.append([(F.SRC_FN0 + 1, 0, 64, 0)] if fn_cols >= 2 else [(1, 0, 64, 0)])
    return {"fields": fields, "predicates": list(predicates), "temporal": list(temporal), "consts": _consts(consts),
            "maps": [], "map_consts": []}


def random_rows(rng, rb, n, diffs=(1, 2, -1, -3)):
    words = [[rng.randrange(U64), rng.randrange(U64), rng.randrange(U64)] for _ in range(n)]
    return rows_of(rb, words, [rng.randrange(4) for _ in range(n)], [rng.choice(diffs) for _ in range(n)])


# ------------------------------------------------------------------ every function, R32 / R40
FUNCS = [
    # generate_series(int32): start = key's low byte (signed), stop = val1's low byte (signed), step = +-1 / +-3
    ("series32", lambda o: tf_of(F.TF_GENERATE_SERIES_INT32, [[(O.HOP_COL, 0, 0, 8, 1, 0)], [(O.HOP_COL, 1, 0, 8, 1, 0)],
                                                              [k(0)]], [o]), 1),
    ("series64", lambda o: tf_of(F.TF_GENERATE_SERIES_INT64, [[(O.HOP_COL, 0, 0, 8, 1, 0)], [(O.HOP_COL, 1, 0, 8, 1, 0)],
                                                              [k(0)]], [o]), 1),
    ("series_ts", lambda o: tf_of(F.TF_GENERATE_SERIES_TIMESTAMP, [[(O.HOP_COL_TS, 0, 0, 8, 1, 0)],
                                                                   [(O.HOP_COL_TS, 1, 0, 8, 1, 0)]], step_us=o), 1),
    ("repeat_row", lambda o: tf_of(F.TF_REPEAT_ROW, [[(O.HOP_COL, 0, 0, 3, 1, 0)]]), 0),
    ("repeat_row_non_negative", lambda o: tf_of(F.TF_REPEAT_ROW_NON_NEGATIVE, [[(O.HOP_COL, 0, 0, 4, 1, 0)]]), 0),
    ("guard_subquery_size", lambda o: tf_of(F.TF_GUARD_SUBQUERY_SIZE, [[(O.HOP_COL, 0, 0, 3, 1, 0)]]), 0),
]


# repeat_row WITH ORDINALITY is refused (test_host_refusals)
CASES = [(f, o) for f in FUNCS for o in (False, True) if not (f[0] == "repeat_row" and o)]


@pytest.mark.parametrize("name,mk,ncol,ordinality", [f + (o,) for f, o in CASES],
                         ids=[f[0] + ("_ordinality" if o else "") for f, o in CASES])
@pytest.mark.parametrize("in_rb,out_rb", [(32, 32), (32, 40), (40, 32), (40, 40)])
def test_every_function(ctx, name, mk, ncol, ordinality, in_rb, out_rb):
    rng = random.Random(hash((name, ordinality, in_rb, out_rb)) & 0xFFFF)
    for step in (1, -1, 3, -3):
        tf = mk(step)
        tf["with_ordinality"] = ordinality
        plan = plan_of(out_rb, ncol + ordinality)
        steps = [(random_rows(rng, in_rb, 300), 2), (random_rows(rng, in_rb, 200), O.EMPTY)]
        run_both(ctx, tf, plan, steps, in_rb, out_rb, fuel=rng.choice([1000, 10**6]))


def test_golden_answers(ctx):
    for case in GOLDEN["cases"]:
        n_in = max(len(r) for r in case["input"])
        rows = rows_of(40, [FM.encode_columns(r) for r in case["input"]], 0, 1)
        refused = False
        for st in case["stages"]:
            tf, plan, n_out = FM.golden_stage(st, n_in)
            if "refused" in case and st is case["stages"][-1]:
                with pytest.raises(mz.MzGpuError):
                    make(ctx, tf, plan, 40, 40)
                refused = True
                break
            out, errs = run_both(ctx, tf, plan, [(rows, O.EMPTY)], 40, 40)
            assert errs == []
            rows = rows_of(40, [list(w) for w, t, d in out], [t for w, t, d in out], [d for w, t, d in out])
            n_in = n_out
        if not refused:
            got = [((w, t, d), n_in) for w, t, d in as_tuples(rows, 40)]
            assert FM.golden_rows(case, got) == sorted(case["expect"])


def test_diffs_errors_and_wrapping(ctx):
    rng = random.Random(3)
    # repeat_row with huge n: the diff product wraps
    tf = tf_of(F.TF_REPEAT_ROW, [[c64(1)]])
    words = [[rng.randrange(16), rng.choice([2**62, 2**63 - 1, U64 - 1, 3, 2**63]), 0] for _ in range(200)]
    rows = rows_of(32, words, 0, [rng.choice([-3, 2, 2**62, -(2**63)]) for _ in range(200)])
    run_both(ctx, tf, plan_of(32, 0), [(rows, O.EMPTY)])
    # argument errors (1 / val1), function errors (a zero step), MfpPlan errors (value + i64::MAX overflows)
    tf = tf_of(F.TF_GENERATE_SERIES_INT64, [[k(0)], [k(0), c32(1), (O.HOP_DIV, 64, 0, 0, 0, 0)], [c32(1, 32)]], [1])
    plan = plan_of(32, 1, predicates=[[(O.HOP_COL, F.SRC_FN0, 0, 64, 0, 0), k(0), (O.HOP_ADD, 64, 0, 0, 0, 0), k(0),
                                       (O.HOP_CMP, O.GE, 0, 0, 0, 0)]], consts=[2**63 - 1])
    words = [[rng.randrange(8), rng.choice([0, 1, 2, -1]) % 2**32 | (rng.choice([0, 1, -1, 2]) % 2**32) << 32, 0]
             for _ in range(300)]
    rows = rows_of(32, words, [rng.randrange(3) for _ in range(300)], [rng.choice([1, -2]) for _ in range(300)])
    out, errs = run_both(ctx, tf, plan, [(rows, O.EMPTY)], fuel=7)
    codes = {c for (c, _p), _t, _d in errs}
    assert {O.E_DIV0, FM.E_INVALID_PARAMETER_VALUE, O.E_OVF} <= codes


def test_hopping_windows(ctx):
    """Each event fanned out to the 4 windows (of 10, hopping by 5) that contain it: mz_now() >= window start and
    mz_now() < window start + 20 on the series column, stepped over many uppers."""
    rng = random.Random(9)
    # window starts: generate_series(t - t % 5 - 15, t - t % 5, 5) over the event time in val1
    t_ = (O.HOP_COL, 1, 0, 32, 1, 0)
    start = [t_, t_, k(0), (M.HOP_MOD, 64, 0, 0, 0, 0), (O.HOP_SUB, 64, 0, 0, 0, 0), k(1), (O.HOP_SUB, 64, 0, 0, 0, 0)]
    stop = [t_, t_, k(0), (M.HOP_MOD, 64, 0, 0, 0, 0), (O.HOP_SUB, 64, 0, 0, 0, 0)]
    tf = tf_of(F.TF_GENERATE_SERIES_INT64, [start, stop, [k(0)]], [5, 15])
    ws = (O.HOP_COL, F.SRC_FN0, 0, 64, 0, 0)
    plan = plan_of(32, 1, temporal=[(O.GE, [ws, (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)]),
                                    (O.LT, [ws, k(0), (O.HOP_ADD, 64, 0, 0, 0, 0), (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)])],
                   consts=[20])
    steps = []
    for s in range(40):
        n = rng.randrange(0, 60)
        words = [[rng.randrange(100), 20 + s * 3 + rng.randrange(10), 0] for _ in range(n)]
        steps.append((rows_of(32, words, s * 3, [rng.choice([1, -1]) for _ in range(n)]), s * 3 + 3))
    steps.append((rows_of(32, [], 0, []), O.EMPTY))
    run_both(ctx, tf, plan, steps, fuel=50)
    # until drops the windows at or past it
    run_both(ctx, tf, plan, steps, until=70, fuel=10**6)


def test_device_input_chained_and_empty(ctx):
    rng = random.Random(11)
    tf1 = tf_of(F.TF_GENERATE_SERIES_INT64, [[k(0)], [(O.HOP_COL, 0, 0, 3, 0, 0)], [k(0)]], [1])
    plan1 = {"fields": [[(0, 0, 64, 0)], [(F.SRC_FN0, 0, 64, 0)]], "predicates": [], "temporal": [], "consts": [],
             "maps": [], "map_consts": []}
    tf2 = tf_of(F.TF_REPEAT_ROW_NON_NEGATIVE, [[c64(1)]], ordinality=True)
    plan2 = plan_of(40, 1)
    rows = random_rows(rng, 32, 500, diffs=(1, 2, -1))
    a, b = make(ctx, tf1, plan1, 32, 32), make(ctx, tf2, plan2, 32, 40)
    src = A.DeviceRows(ctx, 32)
    src.upload(rows)
    mid, _e1, done = a.step_dev(src, O.EMPTY, fuel=100)
    while not done:
        mid, _e1, done = a.work(100, out=mid, errs=_e1)
    out, _e2, done = b.step_dev(mid, O.EMPTY, fuel=333)
    while not done:
        out, _e2, done = b.work(333, out=out, errs=_e2)
    got = O.consolidate(as_tuples(out.download(), 40))
    r1 = FM.Operator(tf1, plan1, O.EMPTY, 4)
    o1, _, _ = r1.step(rows, O.EMPTY)
    mid_rows = rows_of(32, [list(w) for w, t, d in o1], [t for w, t, d in o1], [d for w, t, d in o1])
    r2 = FM.Operator(tf2, plan2, O.EMPTY, 4)
    o2, _, _ = r2.step(mid_rows, O.EMPTY)
    assert got == o2
    # an empty input
    out, errs, done = a.step(rows_of(32, [], 0, []), O.EMPTY, fuel=1)
    assert done and len(out) == 0 and len(errs) == 0


def test_fuel_does_not_change_the_output(ctx):
    rng = random.Random(13)
    tf = tf_of(F.TF_GENERATE_SERIES_INT32, [[(O.HOP_COL, 0, 0, 4, 1, 0)], [(O.HOP_COL, 1, 0, 5, 0, 0)], [k(0)]], [2],
               ordinality=True)
    plan = plan_of(40, 2, temporal=[(O.GE, [(O.HOP_COL, F.SRC_FN0 + 1, 0, 64, 0, 0),
                                            (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)])])
    steps = [(random_rows(rng, 32, 200), 3), (random_rows(rng, 32, 200), 9), (random_rows(rng, 32, 10), O.EMPTY)]
    res = [run_both(ctx, tf, plan, steps, 32, 40, fuel=f) for f in (1, 7, 10**6)]
    assert res[0] == res[1] == res[2]


def test_pending_activation(ctx):
    """A step is refused while an activation is unfinished; frontier covers the unexpanded rows; stats count them;
    a step or work waits for the device at most once."""
    tf = tf_of(F.TF_GENERATE_SERIES_INT64, [[c64(0)], [c64(1)], [k(0)]], [1])
    plan = plan_of(32, 1)
    op = make(ctx, tf, plan, 32, 32)
    # one row of 2^64 function rows, then a row of 3
    rows = rows_of(32, [[2**63, 2**63 - 1], [0, 2]], [4, 2], [1, 1])
    src, out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    src.upload(rows)
    ctx.sync()
    s0 = ctx.stats()["host_syncs"]
    out, errs, done = op.step_dev(src, O.EMPTY, fuel=5, out=out, errs=errs)
    assert ctx.stats()["host_syncs"] - s0 <= 1
    assert not done
    assert [w[1] for w, t, d in as_tuples(out.download(), 32)] == sorted((2**63 + j) % U64 for j in range(5))
    assert op.stats()[3] == U64 - 2  # 2^64 + 3 - 5
    assert op.frontier() == 2  # the row of 3 at time 2 is not expanded yet
    with pytest.raises(mz.MzGpuError) as ei:
        op.step(rows, O.EMPTY, fuel=5)
    assert ei.value.status == F.E_FRONTIER
    s0 = ctx.stats()["host_syncs"]
    out2, errs2, done = op.work(7, out=A.DeviceRows(ctx, 32), errs=A.DeviceRows(ctx, 32))
    assert ctx.stats()["host_syncs"] - s0 <= 1
    assert not done and len(out2.download()) == 7


def test_skewed_activation(ctx):
    """10^5 rows of 0-3 function rows and one row of 10^7, checked by closed forms."""
    rng = np.random.default_rng(17)
    n = 100000
    stop = rng.integers(0, 4, size=n, dtype=np.int64)
    words = np.zeros((n + 1, 2), dtype=np.uint64)
    words[:, 0] = np.arange(n + 1, dtype=np.uint64)
    words[:n, 1] = stop.astype(np.uint64)
    words[n // 2, 1] = 10**7
    r = np.zeros(n + 1, dtype=mz.R32)
    r["key"], r["val"], r["time"], r["diff"] = words[:, 0], words[:, 1], 0, 1
    tf = tf_of(F.TF_GENERATE_SERIES_INT64, [[k(0)], [c64(1)], [k(0)]], [1])
    # output: key = input key, val1 = the value; predicate: value is odd
    plan = plan_of(32, 1, predicates=[[c64(F.SRC_FN0), k(0), (M.HOP_MOD, 64, 0, 0, 0, 0), k(1),
                                       (O.HOP_CMP, O.EQ, 0, 0, 0, 0)]], consts=[2, 1])
    op = make(ctx, tf, plan, 32, 32)
    total_rows, total_val, pages = 0, 0, 0
    out, errs, done = op.step(r, O.EMPTY, fuel=3 * 10**6)
    while True:
        v = out.view(np.uint64).reshape(-1, 4)
        total_rows += len(v)
        total_val += int(v[:, 1].sum())
        pages += 1
        if done:
            break
        out, errs, done = op.work(3 * 10**6)
    stops = [int(x) for x in words[:, 1]]
    exp_rows = sum((s + 1) // 2 for s in stops)
    exp_val = sum(((s + 1) // 2) ** 2 for s in stops)  # 1 + 3 + ... + (2m - 1) = m^2
    assert (total_rows, total_val) == (exp_rows, exp_val)
    assert pages == -(-(sum(stops)) // (3 * 10**6))


def test_host_refusals(ctx):
    ok_args = [[k(0)], [k(0)], [k(0)]]
    plan = plan_of(32, 1)
    bad = [
        (tf_of(F.TF_GENERATE_SERIES_INT64, ok_args[:2], [1]), plan, F.E_INVALID),  # argument count
        (tf_of(F.TF_GENERATE_SERIES_INT32, [[k(0)], [k(0)], [c64(0)]], [1]), plan, F.E_INVALID),  # int64 arg
        (tf_of(F.TF_GENERATE_SERIES_INT64, [[k(0)], [(23, 0, 0, 0, 0, 0)], [k(0)]], [1]), plan, F.E_INVALID),  # MAP
        (tf_of(F.TF_REPEAT_ROW, [[k(0)]], [1]), plan_of(32, 1), F.E_INVALID),  # FN0 beyond 0 columns
        (tf_of(F.TF_REPEAT_ROW, [[k(0)]], [1], ordinality=True), plan_of(32, 0), F.E_INVALID),
        (tf_of(F.TF_GENERATE_SERIES_INT64, ok_args, [1]), plan_of(40, 2), F.E_INVALID),  # FN1 without ordinality
        (tf_of(F.TF_GENERATE_SERIES_TIMESTAMP, [[(O.HOP_COL_TS, 0, 0, 64, 1, 0)]] * 2), plan, F.E_UNSUPPORTED),
        (tf_of(7, [[k(0)]], [1]), plan_of(32, 0), F.E_UNSUPPORTED),  # another table function
    ]
    bad[6][0]["step_us"] = 0
    for tf, p, st in bad:
        if tf["kind"] == F.TF_GENERATE_SERIES_TIMESTAMP:
            fields = [list(f) for f in p["fields"]] + [[]]
            with pytest.raises(mz.MzGpuError) as ei:
                A.FlatMap(ctx, tf["kind"], tf["args"], fields, step_iv=A.interval_const(days=1, months=1))
        else:
            with pytest.raises(mz.MzGpuError) as ei:
                make(ctx, tf, p, 32, p["fields"].__len__() == 3 and 40 or 32)
        assert ei.value.status == st, (tf, ei.value)
    # the context stays usable
    run_both(ctx, tf_of(F.TF_REPEAT_ROW, [[c64(1)]]), plan_of(32, 0),
             [(rows_of(32, [[1, 2], [3, -1]], 0, [1, 1]), O.EMPTY)])
    op = make(ctx, tf_of(F.TF_REPEAT_ROW, [[c64(1)]]), plan_of(32, 0), 32, 32)
    with pytest.raises(mz.MzGpuError):
        op.step(rows_of(32, [[1, 2]], 0, [1]), O.EMPTY, fuel=0)
