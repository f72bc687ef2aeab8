"""The MfpPlan with map expressions (mzgpu_mfp_new_map) on the GPU, byte for byte against tests/mfp_map_oracle.py."""
import ctypes as C
import random

import numpy as np
import pytest

import mfp_map_oracle as M
import mfp_oracle as O

pytestmark = pytest.mark.gpu

mz = pytest.importorskip("materialize_b200")
from materialize_b200 import api as A  # noqa: E402
from materialize_b200 import _ffi as F  # noqa: E402

MIN32, MIN64 = 2**64 - 2**31, 2**63  # the minimum values as u64 words
EDGE = [0, 1, 5, 2**31 - 1, MIN32, 2**64 - 1, 2**63 - 1, MIN64, 2**31, 2**64 - 2**31 - 1, 2**32 - 1, 16, 2**64 - 16]


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


def make(ctx, plan, in_rb, out_rb, until=O.EMPTY):
    fields = [list(f) for f in plan["fields"]] + [[]] * (3 - len(plan["fields"]))
    return A.Mfp(ctx, fields, plan["predicates"], plan["temporal"], plan["consts"], in_row_bytes=in_rb,
                 out_row_bytes=out_rb, until=until, maps=plan["maps"], map_consts=plan["map_consts"])


def run_history(ctx, plan, steps, in_rb=32, out_rb=32, until=O.EMPTY):
    op = make(ctx, plan, in_rb, out_rb, until)
    ref = M.Operator(plan, until, in_rb // 8)
    for rows, upper in steps:
        out, errs = op.step(rows, upper)
        want_out, want_err = ref.step(rows, upper)
        assert as_tuples(out, out_rb) == want_out, upper
        assert err_tuples(errs) == want_err, upper
    assert op.frontier() == ref.frontier()
    return op


def edge_rows(rb, n=None):
    """Every pair of edge values in (key, val), val2 cycling, at times 0..3."""
    pairs = [(a, b) for a in EDGE for b in EDGE]
    key = np.array([a for a, _ in pairs], dtype=np.uint64)
    val = np.array([b for _, b in pairs], dtype=np.uint64)
    k = len(pairs)
    return rows_of(rb, key, val, np.arange(k, dtype=np.uint64) % 4, np.ones(k, dtype=np.int64),
                   val2=np.array([EDGE[i % len(EDGE)] for i in range(k)], dtype=np.uint64))


def plan_of(maps, fields, predicates=(), temporal=(), consts=(), map_consts=()):
    return {"fields": fields, "predicates": list(predicates), "temporal": list(temporal), "consts": list(consts),
            "maps": list(maps), "map_consts": list(map_consts)}


COL32 = A.col(0, 0, 32, signed=True)        # key as an int4
COL32B = A.col(1, 0, 32, signed=True)       # val as an int4
COL64 = A.col(0, 0, 64)                     # key as an int8
COL64B = A.col(1, 0, 64)                    # val as an int8


@pytest.mark.parametrize("rb", [(32, 32), (40, 40), (32, 40), (40, 32)])
@pytest.mark.parametrize("expr", ["neg", "abs", "mod", "cast", "div"])
@pytest.mark.parametrize("width", [32, 64])
def test_each_function_at_its_edges(ctx, rb, expr, width):
    in_rb, out_rb = rb
    a, b = (COL32, COL32B) if width == 32 else (COL64, COL64B)
    ops = {"neg": [a, A.hop(M.HOP_NEG, width)], "abs": [a, A.hop(M.HOP_ABS, width)],
           "mod": [a, b, A.hop(M.HOP_MOD, width)], "div": [a, b, A.hop(F.HOP_DIV, width)],
           "cast": [COL64, A.hop(M.HOP_INT64_TO_INT32)]}[expr]
    fields = [[A.field_map(0)], [A.field_map(0, 0, 32, 0), (0, 0, 16, 48)]]
    if out_rb == 40:
        fields.append([(2 if in_rb == 40 else 1, 0, 64, 0)])
    plan = plan_of([ops], fields)
    rows = edge_rows(in_rb)
    run_history(ctx, plan, [(rows, 2), (rows[:0], 5)], in_rb, out_rb)


def test_if_errors(ctx):
    # map 0 = IF(key < 5, 100 / val, -val); map 1 = IF(100 / val > 1, 1, 0): an error in the untaken branch never
    # surfaces, one in the condition always does
    consts = [(5, 0), (100, 0), (1, 0), (0, 0)]
    m0 = [A.col(0, 0, 64), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_CMP, O.LT), A.hop(F.HOP_INT, konst=1), COL64B,
          A.hop(F.HOP_DIV, 64), COL64B, A.hop(M.HOP_NEG, 64), A.hop(M.HOP_IF)]
    m1 = [A.hop(F.HOP_INT, konst=1), COL64B, A.hop(F.HOP_DIV, 64), A.hop(F.HOP_INT, konst=2), A.hop(F.HOP_CMP, O.GT),
          A.hop(F.HOP_INT, konst=2), A.hop(F.HOP_INT, konst=3), A.hop(M.HOP_IF)]
    for maps in ([m0], [m1], [m0, m1]):
        plan = plan_of(maps, [[A.field_map(len(maps) - 1)], [(0, 0, 64, 0)]], map_consts=consts)
        run_history(ctx, plan, [(edge_rows(32), 4)])


def test_unneeded_map_error_only_for_rows_that_pass(ctx):
    # WHERE key > 10; map 0 = 100 / val (never read, never projected): its error only for rows with key > 10
    consts = [(10, 0), (100, 0)]
    pred = [COL64, A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_CMP, O.GT)]
    m0 = [A.hop(F.HOP_INT, konst=1), COL64B, A.hop(F.HOP_DIV, 64)]
    plan = plan_of([m0], [[(0, 0, 64, 0)], [(1, 0, 64, 0)]], [pred], consts=consts, map_consts=consts)
    rng = np.random.default_rng(1)
    n = 4000
    rows = rows_of(32, rng.integers(0, 20, n, dtype=np.uint64), rng.integers(0, 3, n, dtype=np.uint64),
                   rng.integers(0, 3, n, dtype=np.uint64), rng.choice([1, -1, 2], n).astype(np.int64))
    run_history(ctx, plan, [(rows, 3)])
    errs = M.Operator(plan).step(rows, 3)[1]
    assert sum(d for _, _, d in errs) == int(rows["diff"][(rows["key"] > 10) & (rows["val"] == 0)].sum()) != 0


def test_support_forces_early_evaluation(ctx):
    # map 0 = 100 / val, map 1 = key % 7; predicate map 1 > 2 has support 2: map 0's error fires for every
    # row with val = 0, the predicate's drop notwithstanding.  Reversed (map 0 = key % 7), map 1's error must
    # not fire for the rows the predicate drops.
    consts = [(2, 0), (100, 0), (7, 0)]
    div = [A.hop(F.HOP_INT, konst=1), COL64B, A.hop(F.HOP_DIV, 64)]
    mod = [COL64, A.hop(F.HOP_INT, konst=2), A.hop(M.HOP_MOD, 64)]
    rng = np.random.default_rng(2)
    n = 3000
    rows = rows_of(32, rng.integers(0, 50, n, dtype=np.uint64), rng.integers(0, 3, n, dtype=np.uint64),
                   rng.integers(0, 2, n, dtype=np.uint64), np.ones(n, dtype=np.int64))
    for maps, j in (([div, mod], 1), ([mod, div], 0)):
        pred = [A.map_ref(j), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_CMP, O.GT)]
        plan = plan_of(maps, [[A.field_map(1 - j)], [A.field_map(j)]], [pred], consts=consts, map_consts=consts)
        run_history(ctx, plan, [(rows, 2)])
        n_err = sum(d for _, _, d in M.Operator(plan).step(rows, 2)[1])
        zero = rows["val"] == 0
        want = int(zero.sum()) if j == 1 else int((zero & (rows["key"] % 7 > 2)).sum())
        assert n_err == want and 0 < want


@pytest.mark.parametrize("in_rb", [32, 40])
def test_maps_read_by_temporal_bounds_and_chained(ctx, in_rb):
    # map 0 = val % 64 (int4); map 1 = (map 0 + 3)::mz_timestamp; map 2 = map 1's source * 2 - key % 5;
    # WHERE map 2 >= 0 AND mz_now() >= map 1 AND mz_now() < (map 0 + 20)::mz_timestamp; project (key, maps 2 | 0)
    mconsts = [(64, 0), (3, 0), (2, 0), (5, 0)]
    consts = [(0, 0), (20, 0)]
    m0 = [COL32B, A.hop(F.HOP_INT, konst=0), A.hop(M.HOP_MOD, 32)]
    m1 = [A.map_ref(0), A.hop(F.HOP_INT, konst=1), A.hop(F.HOP_ADD, 32), A.hop(F.HOP_INT_TO_MZTS)]
    m2 = [A.map_ref(0), A.hop(F.HOP_INT, konst=2), A.hop(F.HOP_MUL, 64), COL64, A.hop(F.HOP_INT, konst=3),
          A.hop(M.HOP_MOD, 64), A.hop(F.HOP_SUB, 64)]
    pred = [A.map_ref(2), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_CMP, O.GE)]
    temporal = [(O.GE, [A.map_ref(1)]),
                (O.LT, [A.map_ref(0), A.hop(F.HOP_INT, konst=1), A.hop(F.HOP_ADD, 64), A.hop(F.HOP_INT_TO_MZTS)])]
    fields = [[(0, 0, 64, 0)], [A.field_map(2, 0, 32, 0), A.field_map(0, 0, 8, 32), A.field_map(1, 0, 8, 40)]]
    plan = plan_of([m0, m1, m2], fields, [pred], temporal, consts, mconsts)
    rng = np.random.default_rng(in_rb)
    steps = []
    for s in range(30):
        n = 300
        key = rng.zipf(1.3, n).astype(np.uint64) % 500
        val = rng.integers(0, 2**32, n, dtype=np.uint64)
        steps.append((rows_of(in_rb, key, val, np.full(n, s * 3, dtype=np.uint64), rng.choice([1, 1, -1], n)), s * 3 + 3))
    steps.append((steps[0][0][:0], O.EMPTY))
    run_history(ctx, plan, steps, in_rb, 32)


def zipf_rows(rng, rb, n, t):
    key = rng.zipf(1.3, n).astype(np.uint64) % 1000
    edge = np.array(EDGE + [3, 7, 100], dtype=np.uint64)
    val = np.where(rng.random(n) < 0.1, edge[rng.integers(0, len(EDGE), n)], rng.integers(0, 300, n, dtype=np.uint64))
    val2 = edge[rng.integers(0, len(edge), n)]
    return rows_of(rb, key, val, np.full(n, t, dtype=np.uint64), rng.choice([1, 1, 2, -1], n).astype(np.int64), val2)


@pytest.mark.parametrize("seed", range(12))
def test_random_plans_over_zipf_histories(ctx, seed):
    rng, nrng = random.Random(seed), np.random.default_rng(seed)
    in_rb, out_rb = rng.choice([32, 40]), rng.choice([32, 40])
    plan = M.random_plan(rng, in_words=in_rb // 8, out_words=out_rb // 8)
    steps = [(zipf_rows(nrng, in_rb, 400, s * 10), s * 10 + 10) for s in range(15)]
    run_history(ctx, plan, steps, in_rb, out_rb, until=rng.choice([O.EMPTY, 120]))


def test_device_input(ctx):
    rng, nrng = random.Random(7), np.random.default_rng(7)
    plan = M.random_plan(rng, n_maps=4, n_preds=1)
    op = make(ctx, plan, 32, 32)
    ref = M.Operator(plan)
    out, errs = A.DeviceRows(ctx, 32), A.DeviceRows(ctx, 32)
    want_out, want_err = [], []
    for s in range(10):
        rows = zipf_rows(nrng, 32, 500, s)
        op.step_dev(A.DeviceRows(ctx, 32).upload(rows), s + 1, out, errs)
        o, e = ref.step(rows, s + 1)
        want_out.extend(o)
        want_err.extend(e)
    assert as_tuples(out.download(), 32) == want_out
    assert err_tuples(errs.download()) == want_err


def test_no_expressions_is_mfp_new(ctx):
    # mzgpu_mfp_new_map with n_exprs == 0 against mzgpu_mfp_new on the same histories, byte for byte
    rng, nrng = random.Random(3), np.random.default_rng(3)
    for _ in range(4):
        plan = M.random_plan(rng, n_maps=0, temporal=[(O.GE, [A.col(1, 0, 8, code=F.HOP_COL_MZTS)])], new_ops=False)
        fields = [list(f) for f in plan["fields"]] + [[]]
        a = A.Mfp(ctx, fields, plan["predicates"], plan["temporal"], plan["consts"])
        b = A.Mfp(ctx, fields, plan["predicates"], plan["temporal"], plan["consts"])
        # re-create b through mzgpu_mfp_new_map with an empty map
        m, h = F.Mfp(), C.c_void_p()
        F.lib.mzgpu_mfp_free(b.h)
        b.h = None
        m.in_row_bytes = m.out_row_bytes = 32
        for w, fl in enumerate(fields):
            m.n_fields[w] = len(fl)
            for i, f in enumerate(fl):
                m.fields[w][i] = F.Field(*f)
        m.n_predicates, m.n_temporal, m.n_consts = len(plan["predicates"]), len(plan["temporal"]), len(plan["consts"])
        for p, ops in enumerate(plan["predicates"]):
            m.n_ops[p] = len(ops)
            for i, o in enumerate(ops):
                d = m.ops[p][i]
                d.code, d.arg, d.shift, d.bits, d.sign_extend, d.konst = o
        for p, (cmp, ops) in enumerate(plan["temporal"]):
            m.temporal_cmp[p], m.n_temporal_ops[p] = cmp, len(ops)
            for i, o in enumerate(ops):
                d = m.temporal_ops[p][i]
                d.code, d.arg, d.shift, d.bits, d.sign_extend, d.konst = o
        for k, (lo, hi) in enumerate(plan["consts"]):
            m.consts[k].lo, m.consts[k].hi = lo, hi
        empty = F.MfpMap()
        empty.n_consts = 99  # ignored: no expressions is exactly mzgpu_mfp_new
        ctx.check(F.lib.mzgpu_mfp_new_map(ctx.h, C.byref(m), C.byref(empty), O.EMPTY, C.byref(h)))
        b.h = h
        for s in range(8):
            rows = zipf_rows(nrng, 32, 600, s * 20)
            (oa, ea), (ob, eb) = a.step(rows, s * 20 + 20), b.step(rows, s * 20 + 20)
            assert oa.tobytes() == ob.tobytes() and ea.tobytes() == eb.tobytes()
        assert a.frontier() == b.frontier()


def test_end_to_end_reduce_over_computed_columns(ctx):
    # SELECT k % 16, COUNT(*), SUM(a * b), SUM(CASE WHEN a > 10 THEN 1 ELSE 0 END) FROM t GROUP BY k % 16:
    # R40 (k, a, b) -> maps [a * b, IF(a > 10, 1, 0), k % 16] -> R40 (k % 16, a * b, flag) -> ReduceLanes, all on
    # the device, against numpy
    mconsts = [(10, 0), (1, 0), (0, 0), (16, 0)]
    maps = [[A.col(1, 0, 32, signed=True), A.col(2, 0, 32, signed=True), A.hop(F.HOP_MUL, 64)],
            [A.col(1, 0, 32, signed=True), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_CMP, O.GT),
             A.hop(F.HOP_INT, konst=1), A.hop(F.HOP_INT, konst=2), A.hop(M.HOP_IF)],
            [A.col(0, 0, 64), A.hop(F.HOP_INT, konst=3), A.hop(M.HOP_MOD, 64)]]
    fields = [[A.field_map(2)], [A.field_map(0)], [A.field_map(1)]]
    op = A.Mfp(ctx, fields, in_row_bytes=40, out_row_bytes=40, maps=maps, map_consts=mconsts)
    red = mz.ReduceLanes(ctx, [mz.accum_lane(F.AGG_COUNT_SUM_I64, A.SRC_VAL1, 0, 64),
                               mz.accum_lane(F.AGG_COUNT_SUM_I64, A.SRC_VAL2, 0, 64)], 40)
    rng = np.random.default_rng(31)
    acc = {}
    hist = []
    for s in range(12):
        n = 20000
        k = rng.integers(0, 10**6, n, dtype=np.uint64)
        a = rng.integers(-1000, 1000, n)
        b = rng.integers(-1000, 1000, n)
        d = rng.choice([1, 1, 2, -1], n).astype(np.int64)
        rows = rows_of(40, k, a.astype(np.uint64), np.full(n, s, dtype=np.uint64), d, b.astype(np.uint64))
        hist.append((k, a, b, d))
        out, errs = op.step_dev(A.DeviceRows(ctx, 40).upload(rows), s + 1)
        assert errs.download().size == 0
        for r in red.step_dev(out, s + 1).download().view(F.ROUT_LANES[2]):
            key = int(r["key"])
            c, s0, s1 = acc.get(key, (0, 0, 0))
            dd = int(r["diff"])
            acc[key] = (c + dd * int(r["lanes"][0]["count"]), s0 + dd * int(np.int64(r["lanes"][0]["sum_lo"])),
                        s1 + dd * int(np.int64(r["lanes"][1]["sum_lo"])))
        kk = np.concatenate([h[0] for h in hist]) % 16
        aa, bb, dd = (np.concatenate([h[i] for h in hist]) for i in (1, 2, 3))
        want = {}
        for g in range(16):
            m = kk == g
            want[g] = (int(dd[m].sum()), int((aa[m] * bb[m] * dd[m]).sum()), int(((aa[m] > 10) * dd[m]).sum()))
        assert {g: v for g, v in acc.items() if v != (0, 0, 0)} == {g: v for g, v in want.items() if v != (0, 0, 0)}, s


def test_creation_refusals_leave_the_context_usable(ctx):
    ok_map = [COL64, A.hop(M.HOP_NEG, 64)]
    good = dict(maps=[ok_map], fields=[[A.field_map(0)], [(1, 0, 64, 0)], []], predicates=[], temporal=[],
                consts=[(1, 0)], map_consts=[(1, 0)])

    def refused(code, **kw):
        args = dict(good)
        args.update(kw)
        with pytest.raises(A.MzGpuError) as e:
            A.Mfp(ctx, args["fields"], args["predicates"], args["temporal"], args["consts"], maps=args["maps"],
                  map_consts=args["map_consts"])
        assert e.value.status == code, e.value
        out, _ = A.Mfp(ctx, good["fields"], maps=[ok_map]).step(rows_of(32, [3], [2], [0], [1]), 1)
        assert as_tuples(out, 32) == [((2**64 - 3, 2), 0, 1)]

    INV, UNS = F.E_INVALID, F.E_UNSUPPORTED
    refused(INV, maps=[[A.map_ref(0)]])                                # reads itself
    refused(INV, maps=[ok_map, [A.map_ref(2)], ok_map])                # forward reference
    refused(INV, maps=[ok_map] * 9)                                    # too many expressions
    refused(INV, maps=[[COL64] * 9])                                   # stack overflow
    refused(INV, maps=[[COL64, A.hop(M.HOP_NEG, 64)] * 8 + [A.hop(F.HOP_ADD, 64)]])  # 17 ops
    refused(INV, maps=[[COL64, COL64]])                                # leaves two values
    refused(INV, maps=[[A.hop(M.HOP_NEG, 64)]])                        # underflow
    refused(INV, maps=[[COL64, A.hop(M.HOP_NEG, 32)]])                 # 32-bit op on an int8
    refused(INV, maps=[[COL64, A.hop(M.HOP_ABS, 16)]])                 # width
    refused(INV, maps=[[COL64, COL64, A.hop(M.HOP_MOD, 48)]])
    refused(INV, maps=[[COL64, COL64, COL64, A.hop(M.HOP_IF)]])        # non-BOOL condition
    refused(INV, maps=[[COL64, COL64, A.hop(F.HOP_CMP, O.EQ), COL64, COL64, A.hop(F.HOP_CMP, O.EQ),
                        A.hop(M.HOP_IF), A.hop(M.HOP_NEG, 64)]])       # NEG of a BOOL
    refused(INV, maps=[[COL64, COL64, A.hop(F.HOP_CMP, O.EQ), COL64, A.col(1, code=F.HOP_COL_MZTS),
                        A.hop(M.HOP_IF)]])                             # branches of different types
    refused(INV, maps=[[A.hop(F.HOP_INT, konst=3)]])                   # map constant index
    refused(INV, map_consts=[(1, 0)] * 9)                              # too many constants
    refused(INV, fields=[[A.field_map(1)], [], []])                    # projects a missing expression
    refused(INV, fields=[[A.field_map(0, 60, 8)], [], []])             # past the value's 64 bits
    refused(INV, predicates=[[A.map_ref(1), A.map_ref(0), A.hop(F.HOP_CMP, O.EQ)]])  # predicate reads map 1 of 1
    refused(INV, predicates=[[A.map_ref(0)]])                          # leaves an INT
    refused(INV, temporal=[(O.GE, [A.map_ref(0)])])                    # an INT is not an mz_timestamp
    mzts = [COL64, A.hop(F.HOP_INT_TO_MZTS)]
    refused(UNS, maps=[mzts], predicates=[[A.map_ref(0), A.map_ref(0), A.hop(F.HOP_CMP, O.EQ)]])
    cast_cmp = [COL64, A.hop(M.HOP_INT64_TO_INT32), A.hop(F.HOP_INT, konst=0), A.hop(F.HOP_CMP, O.EQ)]
    refused(UNS, maps=[cast_cmp + cast_cmp + [A.hop(F.HOP_AND)]])      # AND over a varying payload
    refused(UNS, predicates=[cast_cmp + [COL64, COL64, A.hop(F.HOP_CMP, O.EQ), A.hop(F.HOP_OR)]])
    refused(UNS, maps=[[A.col(1, code=F.HOP_COL_F64)]])
    refused(UNS, maps=[[A.col(0, code=F.HOP_COL_TS), A.hop(F.HOP_TS_ADD_IV, konst=0)]],
            map_consts=[A.interval_const(months=1)])
    # AND over a map read is allowed: the map's error stopped the row before the predicate
    A.Mfp(ctx, good["fields"], [[A.map_ref(1), A.map_ref(1), A.hop(F.HOP_AND)]], consts=[(0, 0)],
          maps=[ok_map, cast_cmp], map_consts=[(0, 0)])
    # the HAVING interpreter keeps refusing the new opcodes
    for code in (M.HOP_MAP, M.HOP_NEG, M.HOP_ABS, M.HOP_MOD, M.HOP_INT64_TO_INT32, M.HOP_IF):
        with pytest.raises(A.MzGpuError) as e:
            mz.ReduceLanes(ctx, [mz.accum_lane(F.AGG_COUNT_SUM_I64, 1, 0, 64)], 32,
                           having=A.having([A.h_key(), A.h_key(), (code, 64, 0, 0, 0, None), A.h_int(0),
                                            A.h_cmp("eq")]))
        assert e.value.status == INV
