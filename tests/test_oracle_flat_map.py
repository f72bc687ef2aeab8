"""tests/flat_map_oracle.py (CPU): Materialize's expected answers, series counts against a literal iteration of
range_step_inclusive, error codes and payloads, and the paging contract."""
import json
import os
import random

import pytest

import flat_map_oracle as FM
import mfp_oracle as O

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "table_func.json")))
I32, I64 = (-(2**31), 2**31 - 1), (-(2**63), 2**63 - 1)


def run_golden(case, fuel=10**6):
    """The case through the restatement, stage by stage: (rows with their column counts) or None if refused."""
    n_in = max(len(r) for r in case["input"])
    rows = [tuple(FM.encode_columns(r)) + (0, 1) for r in case["input"]]
    for st in case["stages"]:
        tf, plan, n_out = FM.golden_stage(st, n_in)
        if tf["kind"] == FM.TF_REPEAT_ROW and tf["with_ordinality"]:
            return None
        op = FM.Operator(tf, plan, O.EMPTY, 5)
        out, errs, done = op.step(rows, O.EMPTY, fuel)
        while not done:
            more, e2, done = op.work(fuel)
            out, errs = out + more, errs + e2
        assert errs == []
        rows = [tuple(w) + (t, d % 2**64) for w, t, d in O.consolidate(out)]
        n_in = n_out
    return [((r[:3], r[3], O.s64(r[4])), n_in) for r in rows]


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[c["slt"] for c in GOLDEN["cases"]])
def test_golden_answers(case):
    got = run_golden(case)
    if "refused" in case:
        assert got is None
        return
    assert FM.golden_rows(case, got) == sorted(case["expect"])


def test_golden_answers_do_not_depend_on_fuel():
    for case in GOLDEN["cases"]:
        if "refused" not in case:
            assert run_golden(case, 1) == run_golden(case)


def _edges(lo, hi):
    return [lo, lo + 1, lo + 2, -3, -1, 0, 1, 2, 7, hi - 2, hi - 1, hi]


@pytest.mark.parametrize("bits", [32, 64])
def test_series_count_matches_iteration(bits):
    lo, hi = I32 if bits == 32 else I64
    rng = random.Random(bits)
    cases = []
    for a in _edges(lo, hi):
        for b in _edges(lo, hi):
            for s in [1, 2, 3, -1, -2, -5, hi, lo, hi // 2, lo // 2 + 1]:
                if s and abs(b - a) // abs(s) < 5000:  # iterate only short series literally
                    cases.append((a, b, s))
    for _ in range(3000):
        a, s = rng.randint(lo, hi), rng.choice([1, -1]) * rng.randint(1, 50)
        cases.append((a, max(lo, min(hi, a + rng.randint(-500, 500))), s))
    for a, b, s in cases:
        assert FM.series_count(a, b, s) == sum(1 for _ in FM.range_step_inclusive(a, b, s, bits)), (a, b, s)


def test_series_count_at_the_extremes():
    # the overflow stop and the formula agree next to INT32_MAX / INT64_MAX
    for bits, (lo, hi) in ((32, I32), (64, I64)):
        assert list(FM.range_step_inclusive(hi - 2, hi, 1, bits)) == [hi - 2, hi - 1, hi]
        assert list(FM.range_step_inclusive(hi - 4, hi, 3, bits)) == [hi - 4, hi - 1]
        assert list(FM.range_step_inclusive(lo + 2, lo, -1, bits)) == [lo + 2, lo + 1, lo]
        assert FM.series_count(hi - 4, hi, 3) == 2
        assert FM.series_count(lo, hi, 1) == 2**bits
        assert FM.series_count(hi, lo, -1) == 2**bits
        assert FM.series_count(lo, hi, hi) == 3
        assert FM.series_count(1, 0, 1) == 0 and FM.series_count(0, 1, -1) == 0


def _tf(kind, args, ordinality=False, step_us=0):
    consts = [(a % 2**64, 2**64 - 1 if a < 0 else 0) for a in args]
    return {"kind": kind, "with_ordinality": ordinality, "consts": consts, "step_us": step_us,
            "args": [[(O.HOP_INT, 0, 0, 0, 0, k)] for k in range(len(args))]}


def test_function_errors_and_payloads():
    w = [0] * 10
    assert FM.evaluate_func(_tf(FM.TF_GENERATE_SERIES_INT64, [1, 5, 0]), w) == (FM.E_INVALID_PARAMETER_VALUE, 0)
    assert FM.evaluate_func(_tf(FM.TF_GENERATE_SERIES_TIMESTAMP, [1, 5], step_us=0), w) == (
        FM.E_INVALID_PARAMETER_VALUE, 0)
    assert FM.evaluate_func(_tf(FM.TF_REPEAT_ROW_NON_NEGATIVE, [-7]), w) == (FM.E_INVALID_PARAMETER_VALUE, 2**64 - 7)
    assert FM.evaluate_func(_tf(FM.TF_GUARD_SUBQUERY_SIZE, [2]), w) == (FM.E_MULTIPLE_ROWS, 0)
    assert FM.evaluate_func(_tf(FM.TF_GUARD_SUBQUERY_SIZE, [-1]), w) == (FM.E_NEGATIVE_ROWS, 0)
    assert FM.evaluate_func(_tf(FM.TF_GUARD_SUBQUERY_SIZE, [0]), w) == (FM.E_INTERNAL, 0)
    assert FM.evaluate_func(_tf(FM.TF_GUARD_SUBQUERY_SIZE, [1]), w)[0] == 0
    assert FM.function_rows(_tf(FM.TF_REPEAT_ROW, [-3]), w) == [([], -3)]
    assert FM.function_rows(_tf(FM.TF_REPEAT_ROW, [0]), w) == []
    assert FM.function_rows(_tf(FM.TF_REPEAT_ROW_NON_NEGATIVE, [3], True), w) == [([1], 1), ([2], 1), ([3], 1)]
    assert FM.function_rows(_tf(FM.TF_REPEAT_ROW_NON_NEGATIVE, [3]), w) == [([], 3)]
    # an argument error comes first: 1 / 0 in the step
    tf = _tf(FM.TF_GENERATE_SERIES_INT64, [1, 5, 0])
    tf["args"][2] = [(O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_INT, 0, 0, 0, 0, 2), (O.HOP_DIV, 64, 0, 0, 0, 0)]
    assert FM.evaluate_func(tf, w) == (O.E_DIV0, 0)


def test_operator_pages():
    """Errors ride on the first page, every page is consolidated, and the accumulation does not depend on fuel."""
    rng = random.Random(5)
    tf = {"kind": FM.TF_GENERATE_SERIES_INT64, "with_ordinality": True, "consts": [(1, 0)],
          "args": [[(O.HOP_INT, 0, 0, 0, 0, 0)], [(O.HOP_COL, 0, 0, 8, 1, 0)], [(O.HOP_COL, 1, 0, 8, 1, 0)]]}
    plan = {"fields": [[(FM.SRC_FN0, 0, 32, 0), (0, 0, 8, 32)], [(FM.SRC_FN0 + 1, 0, 64, 0)]], "predicates": [],
            "temporal": [], "consts": [], "maps": [], "map_consts": []}
    rows = [(rng.randrange(256), rng.choice([0, 1, 2, 255]), rng.randrange(3), rng.choice([1, 2, 2**64 - 1]))
            for _ in range(60)]
    totals = []
    for fuel in (1, 7, 10**6):
        op = FM.Operator(tf, plan, O.EMPTY, 4)
        out, errs, done = op.step(rows, 10, fuel)
        pages = 1
        while not done:
            more, e2, done = op.work(fuel)
            out, errs, pages = out + more, errs + e2, pages + 1
        if fuel == 1:
            assert pages > 1
        totals.append((O.consolidate(out), O.consolidate(errs)))
    assert totals[0] == totals[1] == totals[2]
    assert totals[0][1] and all(c == FM.E_INVALID_PARAMETER_VALUE for (c, _p), _t, _d in totals[0][1])
