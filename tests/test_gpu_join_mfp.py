"""The probe operators with an MfpPlan closure (mzgpu_join_closure) on the GPU, byte for byte against
`join_mfp_ref`: output rows in probe order, error rows consolidated.  Every probe path: the single-pass
k_probe_lb, the two-pass k_probe (inexact fan-out, bound past MZ_BOUND_MAX_ROWS), the chains of
half_join_many_mfp and the join_core work loop."""
import json
import os
import random

import numpy as np
import pytest

import join_mfp_ref as jref
import mfp_map_oracle as M
import probe_ref as ref
from test_gpu_probe_paths import Trace, dev, gen, pending_spine, rows_of, runs, same

pytestmark = pytest.mark.gpu

LE, LT, JOIN = ref.LE, ref.LT, ref.JOIN
M64 = ref.M64
COL, INT, ADD, SUB, MUL, DIV, CMP, AND, OR = (M.O.HOP_COL, M.O.HOP_INT, M.O.HOP_ADD, M.O.HOP_SUB, M.O.HOP_MUL,
                                             M.O.HOP_DIV, M.O.HOP_CMP, M.O.HOP_AND, M.O.HOP_OR)
HOP_MOD = M.HOP_MOD
EQ, NE, LT_, LE_, GT, GE = range(6)
SRC_MAP0 = M.SRC_MAP0
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


def col(src, bits=20, signed=False):
    return (COL, src, 0, bits, 1 if signed else 0, 0)


def konst(i):
    return (INT, 0, 0, 0, 0, i)


def op(code, arg=64):
    return (code, arg, 0, 0, 0, 0)


def plan_of(fields, predicates=(), consts=(), maps=(), map_consts=()):
    return {"fields": [list(f) for f in fields], "predicates": [list(p) for p in predicates], "temporal": [],
            "consts": list(consts), "maps": [list(m) for m in maps], "map_consts": list(map_consts)}


def closure(mz, ctx, plan):
    out_rb = 8 * (2 + len(plan["fields"]))
    return mz.JoinClosure(ctx, plan["fields"], plan["predicates"], plan["consts"], out_rb, plan["maps"],
                          plan["map_consts"])


# A cross-side plan: v1 < v2 OR key % 7 = 0; out = (key, (v1 * 3 - v2) | v2 << 32) and, for R40, v1 / (v2 % 5)
# (with `divide`, a division by zero for every fifth lookup value)
def cross_plan(out_words=4, divide=False):
    maps = [[col(1), konst(0), op(MUL), col(2), op(SUB)]]
    fields = [[(0, 0, 64, 0)], [(SRC_MAP0, 0, 32, 0), (2, 0, 20, 32)]]
    if divide:
        maps.append([col(1), col(2), konst(1), op(HOP_MOD), op(DIV)])
    if out_words == 5:
        fields.append([(SRC_MAP0 + len(maps) - 1, 0, 64, 0)])
    preds = [[col(1), col(2), (CMP, LT_, 0, 0, 0, 0),
              col(0, 32), konst(0), op(HOP_MOD), konst(1), (CMP, EQ, 0, 0, 0, 0), op(OR)]]
    return plan_of(fields, preds, [(7, 0), (0, 0)], maps, [(3, 0), (5, 0)])


def check_half(mz, ctx, stream, sp, refb, mode, plan, consolidate=False):
    jc = closure(mz, ctx, plan)
    out, errs = mz.half_join_mfp_dev(ctx, dev(mz, ctx, stream), sp, mode, jc, consolidate)
    want, want_e = jref.probe_mfp(stream, refb, mode, plan)
    if consolidate and len(want):
        want = ref.aref.consolidate(want)
    same(out.download(), want)
    same(errs.download(), want_e)
    return len(want), len(want_e)


def kernels(t, word):
    return {k for k in t.kernels if word in k}


@pytest.mark.parametrize("mode", [LE, LT], ids=["le", "lt"])
@pytest.mark.parametrize("ow", [4, 5], ids=["r32", "r40"])
def test_single_pass(mz, ctx, mode, ow):
    rng = np.random.default_rng(10 + mode * 2 + ow)
    sp, refb = pending_spine(mz, ctx, [gen(rng, 3000, 800, times=(i, i + 1)) for i in range(3)])
    stream = gen(rng, 4000, 800, times=(0, 5))
    plan = cross_plan(ow, divide=True)
    with Trace(ctx) as t:
        n, ne = check_half(mz, ctx, stream, sp, refb, mode, plan)
    assert n > 0 and ne > 0
    assert kernels(t, "MfpClosure") == {f"k_probe_lb<{ow},_MfpClosure>"}, t.kernels


def test_more_than_8_batches_and_128_candidates(mz, ctx):
    rng = np.random.default_rng(3)
    ws = [np.concatenate([runs(rng, [5], [40], i), gen(rng, 800, 2000, times=(i, i + 1))]) for i in range(20)]
    sp, refb = pending_spine(mz, ctx, ws)
    stream = gen(rng, 2000, 2000, times=(20, 21))
    stream[::3, 0] = 5
    plan = cross_plan(4, divide=True)
    plan["fields"][1].append((SRC_MAP0 + 1, 0, 8, 52))
    for mode in (LE, LT):
        check_half(mz, ctx, stream, sp, refb, mode, plan, consolidate=True)


def test_two_pass(mz, ctx):
    rng = np.random.default_rng(5)
    w0 = np.concatenate([runs(rng, [77], [1500], 0), gen(rng, 2000, 3000, key_base=100)])
    sp, refb = pending_spine(mz, ctx, [w0, gen(rng, 2000, 3100, key_base=100)])
    stream = gen(rng, 4000, 3100, times=(0, 5), key_base=100)
    stream[::50, 0] = 77
    for ow in (4, 5):
        with Trace(ctx) as t:
            check_half(mz, ctx, stream, sp, refb, LE, cross_plan(ow, divide=True))
        assert kernels(t, "MfpClosure") == {f"k_probe<{ow},_false,_MfpClosure>", f"k_probe<{ow},_true,_MfpClosure>"}
    # n_ub x fan-out past MZ_BOUND_MAX_ROWS
    w1 = np.concatenate([runs(rng, [9], [1000], 1), gen(rng, 500, 600, key_base=20)])
    sp1, refb1 = pending_spine(mz, ctx, [w1])
    big = gen(rng, 60_000, 1 << 30, times=(0, 3), key_base=1 << 20)
    big[::500, 0] = 9
    with Trace(ctx) as t:
        check_half(mz, ctx, big, sp1, refb1, LT, cross_plan(4, divide=True))
    assert "k_probe<4,_false,_MfpClosure>" in t.kernels


def test_every_match_errors(mz, ctx):
    """Every key of the trace has a run of exactly 6 rows at time 0 and every stream row meets one: the matches are
    n_ub x fan-out, the bound the single pass sizes its error space by, and every one errors."""
    rng = np.random.default_rng(8)
    keys = np.arange(500, dtype=np.uint64) * np.uint64(7)
    sp, refb = pending_spine(mz, ctx, [runs(rng, keys, [6] * len(keys))])
    stream = gen(rng, 3000, 500, times=(6, 7))
    stream[:, 0] = keys[rng.integers(0, len(keys), size=len(stream))]
    plan = plan_of([[(0, 0, 64, 0)], [(1, 0, 64, 0)]], [[col(1), konst(0), op(DIV), konst(0), (CMP, EQ, 0, 0, 0, 0)]],
                   [(0, 0)])
    jc = closure(mz, ctx, plan)
    with Trace(ctx) as t:
        out, errs = mz.half_join_mfp_dev(ctx, dev(mz, ctx, stream), sp, LE, jc, False)
    want, want_e = jref.probe_mfp(stream, refb, LE, plan)
    assert len(want) == 0 and len(want_e) > 0
    n_matches = len(stream) * 6
    assert len(jref.probe_mfp(stream, refb, LE, plan_of([[(0, 0, 64, 0)], [(1, 0, 64, 0)]]))[0]) == n_matches
    same(out.download(), want)
    same(errs.download(), want_e)
    assert kernels(t, "MfpClosure") == {"k_probe_lb<4,_MfpClosure>"}, t.kernels


def test_equivalences(mz, ctx):
    """JoinClosure(equivalences=...) lowers as the reference does, with classes of 2 and 3 expressions: an error in
    e0 (v1 / (v2 % 3)), an error in a later expression, and a mismatch before a failing one."""
    rng = np.random.default_rng(16)
    sp, refb = pending_spine(mz, ctx, [gen(rng, 2000, 200, vals=8)])
    stream = gen(rng, 2000, 200, vals=8, times=(1, 2))
    e_div = [col(1), col(2), konst(0), op(HOP_MOD), op(DIV)]
    cases = [
        [[[col(1)], [col(2)]]],
        [[e_div, [col(2)]]],
        [[[col(1)], [col(2)], e_div]],
        [[[col(1)], e_div], [[col(0, 1)], [konst(1)]]],
    ]
    fields = [[(0, 0, 64, 0)], [(1, 0, 8, 0), (2, 0, 8, 8)]]
    for classes in cases:
        jc = mz.JoinClosure(ctx, fields, consts=[(3, 0), (0, 0)], equivalences=classes)
        plan = plan_of(fields, jref.lower_equivalences(classes), [(3, 0), (0, 0)])
        assert [list(p) for p in mz.lower_equivalences(classes)] == plan["predicates"]
        out, errs = mz.half_join_mfp_dev(ctx, dev(mz, ctx, stream), sp, LE, jc, False)
        want, want_e = jref.probe_mfp(stream, refb, LE, plan)
        same(out.download(), want)
        same(errs.download(), want_e)
        for w in ([1, 1, 0], [1, 2, 0], [2, 2, 3], [1, 2, 3], [0, 0, 3]):
            err, ok = jref.join_closure_apply(classes, dict(plan, predicates=[]), w)
            upd, e2, _ = M.evaluate(plan, w, 0, 1, M64)
            assert ((e2[0][0], e2[0][1]) if e2 else None) == err and bool(upd) == ok


def test_empty_stream_and_trace(mz, ctx):
    rng = np.random.default_rng(9)
    sp, refb = pending_spine(mz, ctx, [gen(rng, 100, 50)])
    plan = cross_plan(4, divide=True)
    check_half(mz, ctx, np.zeros((0, 4), np.uint64), sp, refb, LE, plan)
    empty = mz.Spine(ctx, 32)
    check_half(mz, ctx, gen(rng, 100, 50), empty, [], LE, plan)
    # host rows
    jc = closure(mz, ctx, plan)
    stream = gen(rng, 500, 50, times=(0, 3))
    got, errs = mz.half_join_mfp(ctx, rows_of(mz, stream), sp, LE, jc)
    want, want_e = jref.probe_mfp(stream, refb, LE, plan)
    same(got, ref.aref.consolidate(want) if len(want) else want)
    same(errs, want_e)


def test_random_plans_zipf(mz, ctx):
    rng = np.random.default_rng(11)
    r = random.Random(11)
    keys = np.minimum(rng.zipf(1.3, size=6000), 400).astype(np.uint64)
    w = gen(rng, 6000, 400)
    w[:, 0] = keys
    sp, refb = pending_spine(mz, ctx, [w[:3000], w[3000:]])
    stream = gen(rng, 3000, 400, times=(0, 4))
    stream[:, 0] = np.minimum(rng.zipf(1.3, size=3000), 400).astype(np.uint64)
    ran = 0
    for i in range(12):
        plan = M.random_plan(r, in_words=5, out_words=4 + i % 2, temporal=[])
        try:
            jc = closure(mz, ctx, plan)
        except mz.MzGpuError as e:
            assert e.status == mz._ffi.E_UNSUPPORTED, e
            continue
        out, errs = mz.half_join_mfp_dev(ctx, dev(mz, ctx, stream), sp, LE, jc, False)
        want, want_e = jref.probe_mfp(stream, refb, LE, plan)
        same(out.download(), want)
        same(errs.download(), want_e)
        ran += 1
    assert ran >= 6


def test_chains(mz, ctx):
    """Four requests (split into 3 + 1), two naming one output, the last probing an earlier one's output."""
    rng = np.random.default_rng(12)
    tr = [pending_spine(mz, ctx, [gen(rng, 2000, 500, times=(i, i + 1)) for i in range(2)]) for _ in range(3)]
    plan = cross_plan(4, divide=True)
    jc = closure(mz, ctx, plan)
    s0, s1, s2 = (gen(rng, 1500, 500, times=(2, 4)) for _ in range(3))
    outs = [mz.DeviceRows(ctx, 32) for _ in range(3)]
    reqs = [(dev(mz, ctx, s0), tr[0][0], LE, jc, outs[0]), (dev(mz, ctx, s1), tr[1][0], LT, jc, outs[0]),
            (dev(mz, ctx, s2), tr[2][0], LE, jc, outs[1]), (outs[1], tr[0][0], LE, jc, outs[2])]
    with Trace(ctx) as t:
        errs = mz.half_join_many_mfp(ctx, reqs)
    assert "k_probe_chains<4,_MfpClosure>" in t.kernels, t.kernels
    o0a, e0a = jref.probe_mfp(s0, tr[0][1], LE, plan)
    o0b, e0b = jref.probe_mfp(s1, tr[1][1], LT, plan)
    o1, e1 = jref.probe_mfp(s2, tr[2][1], LE, plan)
    o2, e2 = jref.probe_mfp(o1, tr[0][1], LE, plan)
    same(outs[0].download(), np.concatenate([o0a, o0b]))
    same(outs[1].download(), o1)
    same(outs[2].download(), o2)
    same(errs.download(), ref.aref.consolidate(np.concatenate([e0a, e0b, e1, e2])))


def join_plan():
    """(key, v1 | v2 << 20) where v1 < v2 OR key % 7 = 0, and v1 / (v2 % 5) evaluated: an error for every fifth v2."""
    plan = cross_plan(4, divide=True)
    plan["fields"] = [[(0, 0, 64, 0)], [(1, 0, 20, 0), (2, 0, 20, 20)]]
    return plan


@pytest.mark.parametrize("long_run", [False, True], ids=["single_pass", "two_pass"])
def test_join_core_pushes_both_sides(mz, ctx, long_run):
    """The pre-loaded side-1 batch against three pending trace-1 batches (values swapped), a side-0 push with the
    capability above both times, a side-1 push with it in between; each push's output and errors against the
    reference.  A 1500-row run makes the fan-out inexact: the two-pass form and its counted error flush."""
    rng = np.random.default_rng(600 + long_run)
    w1 = [gen(rng, 600, 400, times=(i, i + 1)) for i in range(3)]
    w1[0] = np.concatenate([w1[0], runs(rng, [401], [1500 if long_run else 700], 0, val_base=1 << 17)])
    t1, r1 = pending_spine(mz, ctx, w1)
    w2 = gen(rng, 3000, 402, times=(0, 1))
    w2[3:40, 0] = 401
    t2, r2 = pending_spine(mz, ctx, [w2])
    plan = join_plan()
    jc = closure(mz, ctx, plan)
    j = mz.JoinCore(ctx, t1, t2, jc)
    seen = [0, 0]

    def step(want, two_pass):
        with Trace(ctx) as t:
            assert j.work_mfp(1 << 40)
        got, errs = ref._w(j.out.download()), ref._w(j.errs.download())
        same(got[seen[0]:], want[0])
        same(errs[seen[1]:], want[1])
        seen[0], seen[1] = len(got), len(errs)
        assert len(want[0]) > 0 and len(want[1]) > 0
        kind = {"k_probe<4,_false,_MfpClosure>"} if two_pass else {"k_probe_lb<4,_MfpClosure>"}
        assert kind <= kernels(t, "MfpClosure"), t.kernels

    step(jref.join_core_push(r2[0], r1, 1, 0, plan), long_run)
    cap = 1 << 40
    wb = gen(rng, 2000, 402, times=(3, 4))
    bb = mz.Batch.build(ctx, rows_of(mz, wb), 3, 4)
    t1.insert(bb)
    j.push(0, bb, cap)
    step(jref.join_core_push(ref.aref.consolidate(wb), r2, 0, cap, plan), False)
    wc = gen(rng, 2000, 402, times=(1, 2))
    bc = mz.Batch.build(ctx, rows_of(mz, wc), 1, 2)
    t2.insert(bc)
    j.push(1, bc, 2)
    step(jref.join_core_push(ref.aref.consolidate(wc), r1 + [ref.aref.consolidate(wb)], 1, 2, plan), long_run)
    with pytest.raises(mz.MzGpuError) as ei:
        j.ctx.check(mz._ffi.lib.mzgpu_join_core_work(j.h, 1, j.out.h, None))
    assert ei.value.status == mz._ffi.E_INVALID
    with pytest.raises(mz.MzGpuError) as ei:
        j.ctx.check(mz._ffi.lib.mzgpu_join_core_work_until(j.h, 1, 0, j.out.h, None))
    assert ei.value.status == mz._ffi.E_INVALID


def test_join_core_errors_count_as_fuel(mz, ctx):
    """Two work items whose every match errors: with fuel 1 the first item's errors use up the fuel, so the call
    stops with the second item still queued (were errors not fuel, it would run both)."""
    rng = np.random.default_rng(601)
    plan = plan_of([[(0, 0, 64, 0)], [(1, 0, 64, 0)]], [[col(1), konst(0), op(DIV), konst(0), (CMP, EQ, 0, 0, 0, 0)]],
                   [(0, 0)])
    w1 = gen(rng, 500, 100)
    t1, r1 = pending_spine(mz, ctx, [w1])
    w2a, w2b = gen(rng, 500, 100, times=(0, 1)), gen(rng, 500, 100, times=(1, 2))
    t2, r2 = pending_spine(mz, ctx, [w2a, w2b])
    j = mz.JoinCore(ctx, t1, t2, closure(mz, ctx, plan))
    ea = jref.join_core_push(r2[0], r1, 1, 0, plan)
    eb = jref.join_core_push(r2[1], r1, 1, 0, plan)
    assert len(ea[0]) == len(eb[0]) == 0 and len(ea[1]) > 0 and len(eb[1]) > 0
    assert not j.work_mfp(1)
    same(j.errs.download(), ea[1])
    assert j.work_mfp(1)
    same(j.errs.download(), np.concatenate([ea[1], eb[1]]))
    assert len(j.out.download()) == 0


def test_join_core_slices(mz, ctx):
    """A 1.5 M-row side-1 batch (more than one 1 M-row slice) with a deadline already past: one slice per call, each
    slice's output and errors consolidated and appended in order."""
    rng = np.random.default_rng(602)
    big = gen(rng, 1_500_000, 1 << 30, times=(0, 1))
    ws = gen(rng, 400, 1, times=(0, 1))
    ws[:, 0] = big[rng.integers(0, len(big), size=400), 0]
    t1, r1 = pending_spine(mz, ctx, [ws])
    t2 = mz.Spine(ctx, 32)
    plan = join_plan()
    j = mz.JoinCore(ctx, t1, t2, closure(mz, ctx, plan))
    bb = mz.Batch.build(ctx, rows_of(mz, big), 0, 1)
    t2.insert(bb)
    j.push(1, bb, 0)
    rows = ref.aref.consolidate(big)
    slices = [rows[: 1 << 20], rows[1 << 20:]]
    want = [jref.join_core_push(s, r1, 1, 0, plan) for s in slices]
    assert not j.work_mfp(1 << 40, 1)
    same(j.out.download(), want[0][0])
    same(j.errs.download(), want[0][1])
    assert j.work_mfp(1 << 40, 1)
    same(j.out.download(), np.concatenate([want[0][0], want[1][0]]))
    same(j.errs.download(), np.concatenate([want[0][1], want[1][1]]))
    assert all(len(w[0]) and len(w[1]) for w in want)


def test_q3_closure_matches_bit_field(mz, ctx):
    rng = np.random.default_rng(14)
    w = gen(rng, 20000, 5000, vals=1 << 40)
    sp, refb = pending_spine(mz, ctx, [w])
    stream = gen(rng, 10000, 5000, vals=1 << 40, times=(1, 3))
    bit = mz.make_closure(key_fields=[(1, 0, 20, 0)], expr=((2, 0, 24), (2, 24, 8), 100))
    plan = plan_of([[(1, 0, 20, 0)], [(SRC_MAP0, 0, 64, 0)]],
                   maps=[[col(2, 24), konst(0), (COL, 2, 24, 8, 0, 0), op(SUB), op(MUL)]], map_consts=[(100, 0)])
    want = mz.half_join_dev(ctx, dev(mz, ctx, stream), sp, LE, bit, False).download()
    got, errs = mz.half_join_mfp_dev(ctx, dev(mz, ctx, stream), sp, LE, closure(mz, ctx, plan), False)
    assert got.download().tobytes() == want.tobytes()
    assert len(errs.download()) == 0


def test_golden(mz, ctx):
    cases = json.load(open(os.path.join(HERE, "golden", "join_closures.json")))
    for case in cases:
        l = np.array(case["left"], dtype=np.int64).reshape(-1)
        r = np.array(case["right"], dtype=np.int64).reshape(-1)
        # a cross join: every row under key 0
        lw = np.zeros((len(l), 4), np.uint64)
        lw[:, 1], lw[:, 2], lw[:, 3] = l.view(np.uint64), 1, 1
        rw = np.zeros((len(r), 4), np.uint64)
        rw[:, 1], rw[:, 2], rw[:, 3] = r.view(np.uint64), 0, 1
        sp, refb = pending_spine(mz, ctx, [rw])
        plan = plan_of([[(1, 0, 64, 0)], [(SRC_MAP0, 0, 64, 0)]], [[tuple(o) for o in p] for p in case["predicates"]],
                       [tuple(c) for c in case["consts"]], [[tuple(o) for o in m] for m in case["maps"]],
                       [tuple(c) for c in case["map_consts"]])
        out, errs = mz.half_join_mfp_dev(ctx, dev(mz, ctx, lw), sp, LE, closure(mz, ctx, plan), True)
        want, want_e = jref.probe_mfp(lw, refb, LE, plan)
        same(out.download(), ref.aref.consolidate(want) if len(want) else want)
        same(errs.download(), want_e)
        got = sorted((int(np.uint64(x).view(np.int64)), int(np.uint64(y).view(np.int64)))
                     for x, y in ref._w(out.download())[:, :2])
        assert got == sorted(tuple(x) for x in case["expect_rows"])
        assert [int(e[0]) for e in ref._w(errs.download())] == case["expect_error_codes"]


def test_refusals(mz, ctx):
    plan = cross_plan(4)
    for kw, st in ((dict(temporal=[(GE, [col(1)])]), mz._ffi.E_INVALID), (dict(in_row_bytes=32), mz._ffi.E_INVALID)):
        with pytest.raises(mz.MzGpuError) as ei:
            mz.JoinClosure(ctx, plan["fields"], plan["predicates"], plan["consts"], 32, plan["maps"],
                           plan["map_consts"], **kw)
        assert ei.value.status == st
    # a well-formed closure still works afterwards
    rng = np.random.default_rng(15)
    sp, refb = pending_spine(mz, ctx, [gen(rng, 500, 100)])
    check_half(mz, ctx, gen(rng, 500, 100, times=(0, 7)), sp, refb, LE, plan)
