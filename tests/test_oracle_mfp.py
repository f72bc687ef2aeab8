"""CPU checks of tests/mfp_oracle.py: the step restatement against the direct definition, the bucket chain
against a plain time filter, and MfpPlan::evaluate's quirks on hand-written rows."""
import json
import os
import random

import pytest

import mfp_oracle as O

COL = (O.HOP_COL_MZTS, 1, 0, 64, 0, 0)
PLUS_K = [(O.HOP_COL, 1, 0, 32, 0, 0), (O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_ADD, 64, 0, 0, 0, 0),
          (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)]
TS = [(O.HOP_COL_TS, 1, 0, 64, 1, 0), (O.HOP_TS_ADD_IV, 0, 0, 0, 0, 1), (O.HOP_TS_TO_MZTS, 0, 0, 0, 0, 0)]
DATE = [(O.HOP_COL_DATE, 1, 0, 16, 0, 0), (O.HOP_DATE_TO_MZTS, 0, 0, 0, 0, 0)]
CONSTS = [(7, 0), (3000, 0)]
EXPRS = {"col": [COL], "int": PLUS_K, "ts": TS, "date": DATE}


def plan(temporal, predicates=()):
    return {"fields": [[(0, 0, 64, 0)], [(1, 0, 64, 0)]], "predicates": list(predicates), "temporal": temporal,
            "consts": CONSTS}


def test_bounds_follow_create_from():
    t = [(O.EQ, []), (O.LT, []), (O.LE, []), (O.GT, []), (O.GE, [])]
    assert O.bounds(t) == ([(0, False), (3, True), (4, False)], [(0, True), (1, False), (2, True)])
    with pytest.raises(ValueError):
        O.bounds([(O.NE, [])])


@pytest.mark.parametrize("cmp", [O.EQ, O.LT, O.LE, O.GT, O.GE])
@pytest.mark.parametrize("kind", sorted(EXPRS))
@pytest.mark.parametrize("until", [O.EMPTY, 40, 0])
@pytest.mark.parametrize("nw", [4, 5])
def test_steps_against_the_definition(cmp, kind, until, nw):
    rng = random.Random(cmp * 100 + len(kind) + nw + until % 7)
    p = plan([(cmp, EXPRS[kind]), (O.LT, PLUS_K)] if kind != "int" else [(cmp, EXPRS[kind])])
    op = O.Operator(p, until, nw)
    history, acc = [], {}
    t = 0
    for s in range(25):
        rows = []
        for _ in range(20):
            r = [rng.randrange(5), rng.randrange(60), rng.randrange(3)][: nw - 2] + [t, rng.choice([1, 1, 2, -1])]
            rows.append(r)
        history.extend(rows)
        upper = t + rng.randrange(1, 6)
        out, _ = op.step(rows, upper)
        for w, ut, d in out:
            assert ut < upper
            acc[w] = acc.get(w, 0) + d
        # the accumulation up to upper - 1 equals the definition at that time (when valid)
        if O.valid(upper - 1, until):
            want = {w: d for w, _, d in O.direct(p, history, upper - 1, until, nw)}
            got = {w: d for w, d in acc.items() if d}
            assert got == want
        t = upper


def test_times_near_the_ends():
    p = plan([(O.LE, [COL])])  # mz_now() <= val: upper = val + 1
    for until in (O.EMPTY, O.MAX - 1):
        op = O.Operator(p, until)
        out, errs = op.step([[1, O.MAX, 0, 1], [2, O.MAX - 1, 0, 1], [3, 0, 0, 1]], 1)
        assert errs == [((O.E_STEP, 0), 0, 1)]
        assert out == [((2, O.MAX - 1), 0, 1), ((3, 0), 0, 1)]
        out, _ = op.step([], O.MAX - 1)
        assert out == [((3, 0), 1, -1)]
        out, _ = op.step([], O.EMPTY)
        # the retraction at u64::MAX is released only by the empty frontier (upper = FRONTIER_EMPTY), and is
        # not valid under until = u64::MAX - 1
        assert out == ([((2, O.MAX - 1), O.MAX, -1)] if until == O.EMPTY else [])


def test_quirks():
    neg = [(O.HOP_COL, 1, 0, 64, 1, 0), (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)]
    w = [0, O.U64 - 3, 0]
    # the first lower-bound error wins
    p = plan([(O.GE, neg), (O.GT, [(O.HOP_COL_MZTS, 0, 0, 64, 0, 0)])])
    assert O.evaluate(p, [O.MAX, O.U64 - 3, 0], 0, 1, O.EMPTY) == ([], [(O.E_MZTS_RANGE, O.U64 - 3, 0, 1)])
    # an invalid lower drops the row before an upper bound's error
    p = plan([(O.GE, [COL]), (O.LT, neg)])
    assert O.evaluate(p, [0, 50, 0], 0, 1, 10) == ([], [])
    # upper == lower stops evaluation
    p = plan([(O.LT, [(O.HOP_INT, 0, 0, 0, 0, 2), (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)]), (O.LT, neg)])
    p["consts"] = CONSTS + [(0, 0)]
    assert O.evaluate(p, w, 0, 1, O.EMPTY) == ([], [])
    # the upper bound is clamped to the lower bound
    p = plan([(O.GE, [COL]), (O.LT, PLUS_K)])
    assert O.evaluate(p, [0, 20, 0], 5, 1, O.EMPTY) == ([(20, 1), (27, -1)], [])
    assert O.evaluate(p, [0, 20, 0], 30, 1, O.EMPTY) == ([], [])
    # an invalid upper becomes none
    assert O.evaluate(p, [0, 20, 0], 5, 1, 25) == ([(20, 1)], [])
    # a predicate error is an error update at (time, diff)
    div = [(O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_COL, 0, 0, 8, 0, 0), (O.HOP_DIV, 64, 0, 0, 0, 0),
           (O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_CMP, O.GT, 0, 0, 0, 0)]
    assert O.evaluate(plan([], [div]), [0, 1, 0], 4, -2, O.EMPTY) == ([], [(O.E_DIV0, 0, 4, -2)])
    # timestamp casts round toward -inf; out of range errors
    assert O.run(TS, [(0, 0), (0, 0)], [0, 1999, 0])[2] == 1
    assert O.run(TS, [(0, 0), (0, 0)], [0, O.U64 - 1, 0])[:2] == (O.E_MZTS_RANGE, O.U64 - 1)
    assert O.run(TS, [(0, 0), (0, 10**8)], [0, 0, 0])[0] == O.E_TS_RANGE


@pytest.mark.parametrize("seed", range(6))
def test_chain_peel_is_a_time_filter(seed):
    rng = random.Random(seed)
    chain = O.BucketChain()
    held = []
    upper = 0
    for _ in range(40):
        rows = [(upper + rng.choice([rng.randrange(10), rng.randrange(10**6), rng.randrange(2**40)]), i)
                for i in range(rng.randrange(30))]
        chain.insert(rows)
        held.extend(rows)
        upper += rng.choice([0, 1, 5, 1000, 10**5, 2**30])
        got = sorted(chain.peel(upper))
        want = sorted(r for r in held if r[0] < upper)
        held = [r for r in held if r[0] >= upper]
        assert got == want
        chain.restore(rng.choice([1, 10, 10**6]))
        assert chain.held() == len(held)
        starts = sorted(chain.content)
        assert not starts or starts[0] == upper
    assert sorted(chain.peel(O.EMPTY)) == sorted(held)


GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "temporal_filters.json")))


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[c["view"] for c in GOLDEN["cases"]])
def test_golden_answers(case):
    """The restatement reproduces Materialize's own expected answers (temporal.slt, temporal.td)."""
    op = O.Operator(O.golden_plan(case))
    assert O.golden_check(case, op.step) == []
