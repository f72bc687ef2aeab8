"""Index peeks (mzgpu_peek / mzgpu_peek_many) on the GPU, byte for byte against `peek_ref`: full scans and literal
lookups, both output widths, as_of around batch boundaries, compaction, a merge in flight, the frontier checks, the
error trace, failure precedence, the finishing and max_rows, and k requests in one call."""
import random

import numpy as np
import pytest

import arrangement_ref as aref
import mfp_map_oracle as M
import peek_ref as P
from test_gpu_probe_paths import pending_spine, rows_of

pytestmark = pytest.mark.gpu

COL, INT, SUB, DIV, CMP = M.O.HOP_COL, M.O.HOP_INT, M.O.HOP_SUB, M.O.HOP_DIV, M.O.HOP_CMP
EQ, NE, LT, LE, GT, GE = range(6)
M64 = P.M64


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


IDENT = plan_of([[(0, 0, 64, 0)], [(1, 0, 64, 0)]])
IDENT40 = plan_of([[(0, 0, 64, 0)], [(1, 0, 64, 0)], [(1, 0, 8, 0)]])


def gen(rng, n, keys, vals, t0, t1, neg=0.0):
    """n R32 rows with times in [t0, t1); diffs +1 / +2, or -1 with probability `neg`."""
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = rng.integers(0, keys, n)
    w[:, 1] = rng.integers(0, vals, n)
    w[:, 2] = rng.integers(t0, t1, n)
    d = np.where(rng.random(n) < neg, -1, rng.integers(1, 3, n))
    w[:, 3] = d.astype(np.int64).view(np.uint64)
    return w


def trace(mz, ctx, parts, step=10):
    """A spine of one batch per part, part i covering times [step * i, step * (i + 1))."""
    sp = mz.Spine(ctx, 32)
    for i, w in enumerate(parts):
        sp.insert(mz.Batch.build(ctx, rows_of(mz, w), step * i, step * (i + 1)))
    return sp


def pplan(mz, ctx, plan, out_rb=32, **fin):
    return mz.PeekPlan(ctx, plan["fields"], plan["predicates"], plan["consts"], out_rb, plan["maps"],
                       plan["map_consts"], **fin)


def want_of(parts, plan, as_of, out_rb=32, fin=None, **kw):
    fin = fin or {}
    allw = np.concatenate(parts) if parts else np.zeros((0, 4), np.uint64)
    return P.peek(rows32(allw), plan, as_of, out_words=out_rb // 8 - 2, **fin, **kw)


def rows32(w):
    import materialize_b200 as m

    return aref.as_rows(np.asarray(w, dtype=np.uint64).reshape(-1, 4), m.R32)


def same(got, want, out_rb):
    assert got[0] == want[0], (got, want)
    if got[0] == "rows":
        g = aref.words(got[1], out_rb)
        assert g.shape == want[1].shape and g.tobytes() == want[1].tobytes(), (g[:8].tolist(), want[1][:8].tolist())
    else:
        assert got[1] == want[1], (got, want)


def check(mz, ctx, sp, parts, plan, as_of, out_rb=32, fin=None, literals=None, max_rows=0):
    fin = fin or {}
    got = mz.peek(ctx, pplan(mz, ctx, plan, out_rb, **fin), sp, as_of, literals=literals, max_rows=max_rows)
    want = want_of(parts, plan, as_of, out_rb, fin, literals=literals, max_rows=max_rows)
    same(got, want, out_rb)
    return got


def rand_fin(r, out_words):
    order = []
    for _ in range(r.randrange(4)):
        shift = r.choice([0, 8])
        order.append((r.randrange(out_words), shift, r.choice([8, 16, 64 - shift]), r.random() < 0.5,
                      r.random() < 0.5, False))
    fin = {"order": order, "limit": r.choice([None, 0, 1, 5, 37]), "offset": r.choice([0, 0, 1, 3, 20])}
    if r.random() < 0.4:
        fin["project"] = [[(r.randrange(out_words), 0, 16, 0)] for _ in range(out_words)]
    return fin


@pytest.mark.parametrize("out_rb", [32, 40])
def test_random_plans_scan_and_literals(mz, ctx, out_rb):
    rng = np.random.default_rng(out_rb)
    parts = [gen(rng, 3000, 300, 16, 10 * i, 10 * (i + 1)) for i in range(5)]
    sp = trace(mz, ctx, parts)
    r = random.Random(out_rb)
    for i in range(24):
        plan = M.random_plan(r, in_words=4, out_words=out_rb // 8, temporal=[])
        fin = rand_fin(r, out_rb // 8 - 2)
        as_of = r.choice([0, 9, 10, 25, 30, 49])
        lits = None if i % 3 == 0 else [r.randrange(320) for _ in range(r.choice([0, 1, 5, 40]))] * r.choice([1, 2])
        check(mz, ctx, sp, parts, plan, as_of, out_rb, fin, lits)


def test_identity_orders_and_cuts(mz, ctx):
    rng = np.random.default_rng(1)
    parts = [gen(rng, 2000, 100, 1 << 20, 10 * i, 10 * (i + 1)) for i in range(3)]
    sp = trace(mz, ctx, parts)
    for order in ([], [(1, 0, 20, True, False, False)], [(1, 0, 64, False, True, False)],
                  [(0, 0, 8, False, False, False), (1, 4, 12, True, True, False)]):
        for limit, offset in ((None, 0), (0, 0), (1, 0), (3, 1), (10, 7), (None, 50), (5, 10**6)):
            check(mz, ctx, sp, parts, IDENT, 29, 32, {"order": order, "limit": limit, "offset": offset})
    # a cut inside one row's copies: key 5 carries 7 copies of one value
    w = np.array([[5, 1, 0, 7], [6, 2, 0, 3]], dtype=np.uint64)
    sp2 = trace(mz, ctx, [w])
    for limit, offset in ((2, 3), (4, 6), (1, 9), (0, 0)):
        got = check(mz, ctx, sp2, [w], IDENT, 5, 32, {"limit": limit, "offset": offset})
    assert got[0] == "rows"
    # a projection that drops the order column
    check(mz, ctx, sp, parts, IDENT40, 29, 40, {"order": [(1, 0, 20, False, True, False)], "limit": 9,
                                               "project": [[(0, 0, 64, 0)], [(2, 0, 8, 0)], []]})


def test_as_of_and_compaction(mz, ctx):
    rng = np.random.default_rng(2)
    parts = [gen(rng, 1500, 200, 8, 10 * i, 10 * (i + 1), neg=0.0) for i in range(6)]
    sp = trace(mz, ctx, parts)
    for as_of in (0, 9, 10, 11, 35, 59):
        check(mz, ctx, sp, parts, IDENT, as_of)
        check(mz, ctx, sp, parts, IDENT, as_of, literals=list(range(0, 200, 7)))
    # logical compaction to 30 and merges: the answers at as_of >= 30 are unchanged, earlier ones are SINCE
    sp.set_logical_compaction(30)
    sp.set_physical_compaction(60)
    for _ in range(8):
        sp.exert(10**6)
    check(mz, ctx, sp, parts, IDENT, 45)
    assert mz.peek(ctx, pplan(mz, ctx, IDENT), sp, 29) == ("error", (P.ERR_SINCE, (30, 29, 0, 0)))


def test_pending_merge_and_export_unchanged(mz, ctx):
    rng = np.random.default_rng(3)
    ws = [gen(rng, 4000, 500, 4, i, i + 1) for i in range(8)]
    sp, _ = pending_spine(mz, ctx, ws)
    before = sp.export()
    plan = pplan(mz, ctx, IDENT)
    for as_of in (3, 7):
        got = mz.peek(ctx, plan, sp, as_of)
        same(got, want_of(ws, IDENT, as_of), 32)
        got = mz.peek(ctx, plan, sp, as_of, literals=[1, 2, 3, 499, 10**9])
        same(got, want_of(ws, IDENT, as_of, literals=[1, 2, 3, 499, 10**9]), 32)
    assert sp.export().tobytes() == before.tobytes()
    sp.set_physical_compaction(8)
    sp.exert(10**6)
    same(mz.peek(ctx, plan, sp, 7), want_of(ws, IDENT, 7), 32)
    assert sp.export().tobytes() == before.tobytes()


def test_long_key_run_literal(mz, ctx):
    w = np.zeros((3000, 4), dtype=np.uint64)
    w[:, 0] = 42
    w[:, 1] = np.arange(3000)
    w[:, 3] = 1
    w2 = np.array([[41, 1, 0, 1], [43, 2, 0, 1]], dtype=np.uint64)
    parts = [np.concatenate([w, w2])]
    sp = trace(mz, ctx, parts)
    for lits in ([42], [42, 42, 41], [40], []):
        check(mz, ctx, sp, parts, IDENT, 5, 32, {"order": [(1, 0, 64, False, True, False)], "limit": 100},
              literals=lits)


def test_refusals_and_frontiers(mz, ctx):
    rng = np.random.default_rng(4)
    parts = [gen(rng, 20, 10, 4, i, i + 1) for i in range(65)]
    sp = trace(mz, ctx, parts, step=1)
    with pytest.raises(mz.MzGpuError) as e:
        mz.peek(ctx, pplan(mz, ctx, IDENT), sp, 64)
    assert e.value.status == -4
    sp.set_physical_compaction(65)
    sp.exert(10**6)
    check(mz, ctx, sp, parts, IDENT, 64)
    # NOT_READY on the ok trace, then on the error trace
    assert mz.peek(ctx, pplan(mz, ctx, IDENT), sp, 65) == ("not_ready", None)
    errs = trace(mz, ctx, [np.zeros((0, 4), np.uint64)], step=20)
    assert mz.peek(ctx, pplan(mz, ctx, IDENT), sp, 30, err_spine=errs) == ("not_ready", None)
    # refused plans
    bad = dict(IDENT, fields=[[(0, 0, 64, 0)], [(1, 0, 64, 0)]])
    with pytest.raises(mz.MzGpuError) as e:
        mz.PeekPlan(ctx, bad["fields"], in_row_bytes=40)
    assert e.value.status == -1
    with pytest.raises(mz.MzGpuError) as e:
        mz.PeekPlan(ctx, bad["fields"], limit=-1)
    assert e.value.status == -4
    with pytest.raises(mz.MzGpuError) as e:
        mz.PeekPlan(ctx, bad["fields"], order=[(1, 0, 64, False, False, True)])
    assert e.value.status == -4
    with pytest.raises(mz.MzGpuError) as e:
        mz.PeekPlan(ctx, bad["fields"], order=[(2, 0, 64, False, False, False)])
    assert e.value.status == -1


def test_error_trace(mz, ctx):
    ok = [np.array([[1, 1, 0, 1]], dtype=np.uint64)]
    sp = trace(mz, ctx, ok)
    plan = pplan(mz, ctx, IDENT)
    e_pos = [np.array([[7, 3, 2, 1], [9, 1, 1, 2], [5, 5, 8, 1]], dtype=np.uint64)]
    errs = trace(mz, ctx, e_pos)
    assert mz.peek(ctx, plan, sp, 5, err_spine=errs) == ("error", (P.ERR_ERRS_ROW, (7, 3, 0, 0)))
    assert mz.peek(ctx, plan, sp, 9, err_spine=errs) == ("error", (P.ERR_ERRS_ROW, (5, 5, 0, 0)))
    neg = [np.array([[4, 0, 1, np.uint64(M64)], [7, 3, 2, 1]], dtype=np.uint64)]
    errs2 = trace(mz, ctx, neg)
    assert mz.peek(ctx, plan, sp, 5, err_spine=errs2) == ("error", (P.ERR_ERRS_RETRACTION, (4, 0, M64, 0)))
    # the error trace's rows after as_of do not count
    assert mz.peek(ctx, plan, sp, 0, err_spine=errs2)[0] == "rows"


def test_failure_precedence(mz, ctx):
    # key / (val - 3) >= 0: val == 3 is DivisionByZero; val == 7 is filtered out (key 0 / 4 = 0 >= 0 is kept)
    div = [col(0), col(1), konst(0), op(SUB), op(DIV), konst(1), (CMP, GE, 0, 0, 0, 0)]
    ne7 = [col(1), konst(2), (CMP, NE, 0, 0, 0, 0)]
    plan = plan_of([[(0, 0, 64, 0)], [(1, 0, 64, 0)]], [ne7, div], [(3, 0), (0, 0), (7, 0)])
    m1 = np.uint64(M64)
    cases = [
        [[2, 3, 0, 1], [5, 4, 0, m1]],  # the MFP error (key 2) comes first
        [[2, 4, 0, m1], [5, 3, 0, 1]],  # the retraction (key 2) comes first
        [[2, 7, 0, m1], [3, 5, 0, 1]],  # a filtered-out pair's negative count is not reported
        [[2, 3, 1, 1], [3, 5, 0, 1]],  # the error is after as_of = 0
    ]
    for w in cases:
        parts = [np.array(w, dtype=np.uint64)]
        sp = trace(mz, ctx, parts)
        check(mz, ctx, sp, parts, plan, 0)
        check(mz, ctx, sp, parts, plan, 0, literals=[2, 3, 5])


def test_max_rows(mz, ctx):
    rng = np.random.default_rng(5)
    parts = [gen(rng, 500, 100, 4, 0, 10)]
    sp = trace(mz, ctx, parts)
    n = len(want_of(parts, IDENT, 9)[1])
    for m in (1, n - 1, n, n + 1):
        check(mz, ctx, sp, parts, IDENT, 9, max_rows=m)
    check(mz, ctx, sp, parts, IDENT, 9, fin={"limit": 3}, max_rows=3)


def test_peek_many_equals_single_peeks(mz, ctx):
    rng = np.random.default_rng(6)
    parts = [gen(rng, 3000, 400, 16, 10 * i, 10 * (i + 1)) for i in range(4)]
    sp = trace(mz, ctx, parts)
    e = [np.array([[3, 1, 35, 1]], dtype=np.uint64)]
    errs = trace(mz, ctx, e, step=40)
    r = random.Random(6)
    plans = []
    for i in range(6):
        out_rb = 32 if i % 2 else 40
        plan = M.random_plan(r, in_words=4, out_words=out_rb // 8, temporal=[])
        plans.append((pplan(mz, ctx, plan, out_rb, **rand_fin(r, out_rb // 8 - 2)), out_rb))
    for k in (1, 2, 7, 33, mz.PEEK_MANY_MAX):
        reqs = []
        for j in range(k):
            p, out_rb = plans[r.randrange(len(plans))]
            lits = None if r.random() < 0.5 else [r.randrange(450) for _ in range(r.randrange(30))]
            reqs.append({"plan": p, "as_of": r.choice([5, 10, 20, 34, 35, 39, 45]), "literals": lits,
                         "max_rows": r.choice([0, 0, 50])})
        got = mz.peek_many(ctx, sp, reqs, err_spine=errs)
        for j, q in enumerate(reqs):
            one = mz.peek(ctx, q["plan"], sp, q["as_of"], literals=q["literals"], err_spine=errs,
                          max_rows=q["max_rows"])
            assert got[j][0] == one[0]
            if one[0] == "rows":
                assert got[j][1].tobytes() == one[1].tobytes()
            else:
                assert got[j][1] == one[1]
    with pytest.raises(mz.MzGpuError):
        mz.peek_many(ctx, sp, [{"plan": plans[0][0], "as_of": 5}] * (mz.PEEK_MANY_MAX + 1))


def test_sqllogictest_answers(mz, ctx):
    """The golden cases of tests/golden/index_peeks.json on the device, each as one peek and all as one peek_many."""
    import test_ref_peek as G

    g = G.golden()
    reqs, cases, spines = [], [], {}
    for case in g["cases"]:
        w, plan, fin, lits, as_of, decode = G.golden_lowering(case, g["tables"])
        key = (case["table"], tuple(case.get("index_columns", [])), bool(case.get("after_delete")))
        if key not in spines:
            parts = [w[w[:, 2] == 0], w[w[:, 2] == 1]]
            spines[key] = trace(mz, ctx, parts, step=1)
        p = pplan(mz, ctx, plan, 32, **fin)
        got = mz.peek(ctx, p, spines[key], as_of, literals=lits)
        assert got[0] == "rows", case
        assert G.golden_answer(case, decode, aref.words(got[1], 32)) == case["expect"], (case["file"], case["line"])
        reqs.append(({"plan": p, "as_of": as_of, "literals": lits}, spines[key]))
        cases.append((case, decode))
    for key, sp in spines.items():
        mine = [(q, c) for (q, s), c in zip(reqs, cases) if s is sp]
        for (case, decode), (st, rows) in zip([c for _, c in mine], mz.peek_many(ctx, sp, [q for q, _ in mine])):
            assert st == "rows" and G.golden_answer(case, decode, aref.words(rows, 32)) == case["expect"]


def test_full_scans_share_one_gather(mz, ctx):
    """Full-scan requests at one as_of read one gathered slot; each still gets its own plan, finishing, failure and
    max_rows, against the reference."""
    rng = np.random.default_rng(8)
    parts = [gen(rng, 2000, 150, 16, 10 * i, 10 * (i + 1), neg=0.02) for i in range(3)]
    sp = trace(mz, ctx, parts)
    r = random.Random(8)
    reqs, wants = [], []
    for j in range(12):
        out_rb = 32 if j % 3 else 40
        plan = M.random_plan(r, in_words=4, out_words=out_rb // 8, temporal=[])
        fin = rand_fin(r, out_rb // 8 - 2)
        as_of = (15, 29)[j % 2]
        max_rows = r.choice([0, 0, 40])
        reqs.append({"plan": pplan(mz, ctx, plan, out_rb, **fin), "as_of": as_of, "max_rows": max_rows})
        wants.append((want_of(parts, plan, as_of, out_rb, fin, max_rows=max_rows), out_rb))
    for got, (want, out_rb) in zip(mz.peek_many(ctx, sp, reqs), wants):
        same(got, want, out_rb)
