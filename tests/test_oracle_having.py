"""HAVING filters of the multi-column accumulable reduce, restated on the CPU (tests/having_oracle.py),
pinned by their definition -- at every time the accumulated output is GROUP BY over the accumulated input,
filtered by the predicates evaluated on each group, error rows kept -- by evaluator answers written from
the reference's rules, and by reference-held sqllogictest answers."""
import json
import os

import numpy as np
import pytest
from having_oracle import (
    DIVISION_BY_ZERO,
    ERR_SHIFT,
    INT32_OUT_OF_RANGE,
    INT64_OUT_OF_RANGE,
    NUMERIC_FIELD_OVERFLOW,
    ReduceLanesHaving,
    add,
    and_,
    cmp,
    count,
    div,
    evaluate,
    filter_row,
    float_,
    int_,
    key,
    mul,
    not_,
    num,
    or_,
    sub,
    sum_,
)
from test_oracle_distinct_lanes import D, accumulated, distinct_activations, expected
from test_oracle_reduce_lanes import F64, I64, VAL1, VAL2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
NAN, INF = float("nan"), float("inf")

# (input row bytes, lanes, predicates): every lane class, R32 and R40, distinct lanes, every value type
SCENARIOS = {
    "c1_r32_count": (32, [(I64, VAL1, 0, 64, False)], [[count(0), int_(3), cmp("gt")]]),
    "c1_r32_f64_sum": (32, [(F64, VAL1, 0, 64, False)], [[sum_(0), float_(0.0), cmp("ge")]]),
    "c2_r40_num_past_i64": (
        40,
        [(I64, VAL1, 0, 64, False), (I64 | D, VAL2, 0, 64, False)],
        [[sum_(0), num(2**63), cmp("lt"), sum_(1), num(-(2**64)), cmp("gt"), or_()], [count(1), int_(1), cmp("ne")]],
    ),
    "c2_r32_count_distinct": (
        32,
        [(I64 | D, VAL1, 0, 64, False), (I64, VAL1, 0, 20, True)],
        [[count(0), int_(2), cmp("ge"), sum_(1), num(0), cmp("le"), or_()]],
    ),
    "c4_r32_bit_fields": (
        32,
        [(I64, VAL1, 0, 64, False), (I64 | D, VAL1, 8, 16, True), (F64, VAL1, 0, 64, False), (I64, VAL1, 32, 32, True)],
        [[count(1), key(0, 8), add(64), int_(3), cmp("gt")],
         [sum_(3), num(-(2**40)), cmp("ge"), sum_(2), float_(-INF), cmp("ne"), and_(), key(0, 4), int_(5), cmp("eq"), or_()]],
    ),
    "c8_r32_seven_lanes": (
        32,
        [(I64, VAL1, 0, 64, False), (I64 | D, VAL1, 0, 64, False), (F64, VAL1, 0, 64, False), (I64, VAL1, 0, 8, True),
         (I64 | D, VAL1, 60, 4, True), (I64, VAL1, 16, 16, False), (I64, VAL1, 40, 24, True)],
        [[count(4), int_(1), cmp("ne"), key(0, 32, True), int_(4), sub(32), int_(0), cmp("ne"), and_()],
         [count(0), key(0, 32, True), int_(4), sub(32), div(64), int_(0), cmp("ge")]],
    ),
    "c4_r40_division_by_key": (
        40,
        [(I64, VAL1, 0, 64, False), (I64 | D, VAL2, 0, 64, False), (I64, VAL1, 8, 16, True), (F64, VAL2, 0, 64, False)],
        # count(0) / (key - 3) >= 1: key 3 divides by zero; the first predicate keeps odd keys only
        [[key(0, 32, True), int_(2), div(32), int_(2), mul(32), key(0, 32, True), cmp("ne")],
         [count(0), key(0, 32, True), int_(3), sub(32), div(64), int_(1), cmp("ge"), sum_(3), sum_(3), cmp("eq"), not_(), or_()]],
    ),
    "c8_r40_eight_lanes": (
        40,
        [(I64, VAL1, 0, 64, False), (I64 | D, VAL1, 0, 64, False), (F64, VAL2, 0, 64, False), (I64 | D, VAL2, 0, 64, False),
         (I64, VAL1, 3, 17, True), (I64 | D, VAL1, 60, 4, True), (I64, VAL2, 32, 32, False), (I64 | D, VAL2, 0, 8, True)],
        [[count(0), count(4), mul(64), int_(4), cmp("ge"), sum_(2), float_(NAN), cmp("lt"), and_()],
         [sum_(6), num(0), cmp("ne"), count(7), int_(2**62), mul(64), int_(0), cmp("gt"), and_()]],
    ),
}


def run_scenario(make_op, name, steps=8, keys=12, seed=0):
    """Steps of distinct_activations through one operator; yields (rows so far, outputs so far, upper, op)."""
    in_rb, lanes, preds = SCENARIOS[name]
    op = make_op(in_rb, lanes, preds)
    rng = np.random.default_rng(seed + len(name))
    seen, outs = [], []
    for a, upper in distinct_activations(rng, in_rb // 8, steps=steps, keys=keys):
        seen.append(a)
        outs.append(op.step(a, upper))
        yield np.concatenate(seen), outs, upper, op


def filtered_expected(rows, lanes, preds, in_words, cls, tau):
    kinds = [l[0] & ~D for l in lanes] + [0] * (cls - len(lanes))
    out = set()
    for row, _ in expected(rows, lanes, in_words, cls, tau).values():
        r = filter_row(preds, kinds, row)
        if r is not None:
            out.add(r)
    return out


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_having_is_filtered_group_by_of_accumulated_input(oracle, name):
    in_rb, lanes, preds = SCENARIOS[name]
    errs = 0
    for rows, outs, upper, op in run_scenario(lambda i, l, p: ReduceLanesHaving(oracle, l, i, p), name):
        out = np.concatenate(outs)
        errs += int(((out["flags"].astype(np.uint64) >> np.uint64(ERR_SHIFT)) & np.uint64(7) != 0).sum())
        for tau in range(upper - 3, upper):
            assert accumulated(out, op.cls, tau) == filtered_expected(rows, lanes, preds, in_rb // 8, op.cls, tau), (name, tau)
    if name == "c4_r40_division_by_key":
        assert errs > 0  # the division by zero occurs, and its rows come and go


# Small scenarios, each one operator: (lanes, predicates, [(rows of one activation, upper)]).  The CPU tests
# pin their answers; the GPU module runs the same activations and compares byte for byte.
ONE_LANE = [(I64, VAL1, 0, 64, False)]
# SUM > 10: hidden changes emit nothing, crossing up is one insertion, crossing down one retraction
CROSSING = (ONE_LANE, [[sum_(0), num(10), cmp("gt")]], [([(1, v, t, 1)], t + 1) for t, v in enumerate([5, 3, 4, 1, -10, 2])])
# count / key: the key-0 group is an error row (kept whatever the filter says) until its rows leave
DIVISION_RETRACTED = (ONE_LANE, [[count(0), key(), div(64), int_(0), cmp("ge")]],
                      [([(2, 7, 0, 1), (0, 5, 0, 1)], 1), ([(0, 5, 1, -1)], 2)])
# a plain and a distinct lane over (k,1,+1), (k,3,+1), (k,2,-2): the total is 3 (one plain lane: sum of diffs 0,
# plus three present pairs) and the plain lane's accumulation is zero, so its SUM is NULL (flag bit 0)
NULL_SUM_LANES = [(I64, VAL1, 0, 64, False), (I64 | D, VAL1, 0, 64, False)]
NULL_SUM_ROWS = [(1, 1, 0, 1), (1, 3, 0, 1), (1, 2, 0, -2)]
NULL_SUM_PREDS = [  # (predicates, visible)
    ([[sum_(0), num(0), cmp("eq")]], False),
    ([[sum_(0), num(0), cmp("eq"), not_()]], False),
    ([[sum_(0), num(0), cmp("eq"), count(1), int_(3), cmp("eq"), or_()]], True),
]


def _r32(rows):
    a = np.zeros(len(rows), dtype=np.dtype([("key", "<u8"), ("val", "<u8"), ("time", "<u8"), ("diff", "<i8")]))
    for i, (k, v, t, d) in enumerate(rows):
        a[i] = (np.int64(k).view(np.uint64), np.int64(v).view(np.uint64), t, d)
    return a


def run_steps(op, steps):
    return [op.step(_r32(rows), upper) for rows, upper in steps]


def _rows_of(out):
    return [(int(o["key"]), int(o["lanes"][0]["sum_lo"]), int(o["flags"]), int(o["time"]), int(o["diff"])) for o in out]


def test_threshold_crossings_and_silence_while_filtered(oracle):
    lanes, preds, steps = CROSSING
    got = [_rows_of(o) for o in run_steps(ReduceLanesHaving(oracle, lanes, 32, preds), steps)]
    assert got == [[], [], [(1, 12, 0, 2, 1)], [(1, 12, 0, 3, -1), (1, 13, 0, 3, 1)], [(1, 13, 0, 4, -1)], []]


def test_division_by_zero_appears_and_is_retracted(oracle):
    lanes, preds, steps = DIVISION_RETRACTED
    got = [_rows_of(o) for o in run_steps(ReduceLanesHaving(oracle, lanes, 32, preds), steps)]
    assert got == [[(0, 5, DIVISION_BY_ZERO << ERR_SHIFT, 0, 1), (2, 7, 0, 0, 1)], [(0, 5, DIVISION_BY_ZERO << ERR_SHIFT, 1, -1)]]


def evaluator_cases():
    """(predicates, key word, whether lane 0's SUM is NULL, answer) from the reference's rules.  Only constants,
    key fields and lane 0's (NULL) SUM are read, so each case runs through a one-key operator as well: key =
    the key word, and the NULL_SUM rows when the SUM is NULL, else one row (key, 5, +1)."""
    T, Fl = "pass", "drop"
    cases = []

    def case(preds, want, key_word=0, null=False):
        cases.append((preds, key_word, null, want))

    # comparisons: INT, NUM past i64, INT widened against NUM, FLOAT as OrderedFloat
    for op, want in [("eq", Fl), ("ne", T), ("lt", T), ("le", T), ("gt", Fl), ("ge", Fl)]:
        case([[int_(-5), int_(3), cmp(op)]], want)
        case([[num(-(2**100)), num(2**70), cmp(op)]], want)
        case([[int_(2**63 - 1), num(2**63), cmp(op)]], want)
        case([[float_(-INF), float_(NAN), cmp(op)]], want)
        case([[int_(7), int_(7), cmp(op)]], {"eq": T, "ne": Fl, "lt": Fl, "le": T, "gt": Fl, "ge": T}[op])
    case([[float_(NAN), float_(NAN), cmp("eq")]], T)
    case([[float_(NAN), float_(INF), cmp("gt")]], T)
    case([[float_(-0.0), float_(0.0), cmp("eq")]], T)
    case([[float_(-0.0), float_(0.0), cmp("lt")]], Fl)
    case([[float_(INF), float_(1e308), cmp("gt")]], T)
    case([[float_(-INF), float_(-1e308), cmp("le")]], T)
    # checked arithmetic at both widths
    i32max, i64max = 2**31 - 1, 2**63 - 1
    case([[int_(i32max), int_(1), add(32), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([[int_(i32max), int_(1), add(64), int_(0), cmp("gt")]], T)
    case([[int_(-(2**31)), int_(1), sub(32), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([[int_(i64max), int_(1), add(64), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([[int_(-i64max), int_(2), sub(64), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([[int_(-i64max), int_(1), sub(64), int_(0), cmp("lt")]], T)
    case([[int_(2**32), int_(2**31), mul(64), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([[int_(-(2**32)), int_(2**31), mul(64), int_(-(2**63)), cmp("eq")]], T)
    case([[int_(65536), int_(32768), mul(32), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([[int_(-(2**31)), int_(-1), div(32), int_(0), cmp("gt")]], ("err", INT32_OUT_OF_RANGE))
    case([[int_(-(2**31)), int_(-1), div(64), int_(2**31), cmp("eq")]], T)
    case([[int_(-(2**63)), int_(-1), div(64), int_(0), cmp("gt")]], ("err", INT64_OUT_OF_RANGE))
    case([[int_(-7), int_(2), div(64), int_(-3), cmp("eq")]], T)  # truncation toward zero
    case([[int_(7), int_(-2), div(32), int_(-3), cmp("eq")]], T)
    case([[int_(1), int_(0), div(64), int_(0), cmp("gt")]], ("err", DIVISION_BY_ZERO))
    case([[int_(1), int_(0), div(32), int_(0), cmp("gt")]], ("err", DIVISION_BY_ZERO))
    # the first operand's error wins; an error wins over NULL; NULL propagates
    ovf = [int_(i32max), int_(1), add(32)]
    dz = [int_(1), int_(0), div(64)]
    case([ovf + dz + [add(64), int_(0), cmp("gt")]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([dz + ovf + [add(64), int_(0), cmp("gt")]], ("err", DIVISION_BY_ZERO))
    case([[sum_(0), num(1), cmp("eq")] + dz + [int_(0), cmp("gt"), and_()]], ("err", DIVISION_BY_ZERO), null=True)
    case([[sum_(0), num(1), cmp("eq")]], Fl, null=True)  # NULL drops the row
    case([[sum_(0), num(1), cmp("eq"), not_()]], Fl, null=True)
    case([[sum_(0), num(5), cmp("eq")]], T)  # the same SUM, not NULL
    # AND / OR: FALSE (TRUE) beats an error, two errors give the larger, NULL beats TRUE (FALSE)
    false, true = [int_(0), int_(1), cmp("eq")], [int_(1), int_(1), cmp("eq")]
    e_dz, e_ovf = dz + [int_(0), cmp("gt")], ovf + [int_(0), cmp("gt")]
    e_i64 = [int_(-(2**63)), int_(-1), div(64), int_(0), cmp("gt")]
    null = [sum_(0), num(0), cmp("eq")]
    case([false + e_dz + [and_()]], Fl)
    case([e_dz + false + [and_()]], Fl)
    case([e_dz + e_ovf + [and_()]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([e_ovf + e_dz + [and_()]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([e_i64 + e_ovf + [and_()]], ("err", INT64_OUT_OF_RANGE))
    case([e_ovf + e_dz + [or_()]], ("err", NUMERIC_FIELD_OVERFLOW))
    case([e_dz + e_i64 + [or_()]], ("err", INT64_OUT_OF_RANGE))
    case([true + e_dz + [or_()]], T)
    case([e_dz + true + [or_()]], T)
    case([true + e_dz + [and_()]], ("err", DIVISION_BY_ZERO))
    case([false + e_dz + [or_()]], ("err", DIVISION_BY_ZERO))
    case([true + true + [and_()]], T)
    case([false + false + [or_()]], Fl)
    case([null + true + [and_()]], Fl, null=True)
    case([null + false + [and_(), not_()]], T, null=True)  # FALSE
    case([null + true + [or_(), not_()]], Fl, null=True)
    case([null + false + [or_(), not_()]], Fl, null=True)  # NULL
    case([null + e_dz + [or_()]], ("err", DIVISION_BY_ZERO), null=True)
    case([null + e_dz + [and_()]], ("err", DIVISION_BY_ZERO), null=True)
    # an error in predicate 2 is masked by a FALSE predicate 1, not by a later one
    case([false, e_dz], Fl)
    case([true, e_dz], ("err", DIVISION_BY_ZERO))
    case([e_dz, false], ("err", DIVISION_BY_ZERO))
    case([true, true, true, false], Fl)
    case([true, true, true, true], T)
    # key fields: sign extension and shifts
    case([[key(0, 32, True), int_(-1), cmp("eq")]], T, key_word=0xFFFFFFFF)
    case([[key(0, 32, False), int_(2**32 - 1), cmp("eq")]], T, key_word=0xFFFFFFFF)
    case([[key(60, 4, True), int_(-8), cmp("eq")]], T, key_word=0x8 << 60)
    case([[key(8, 16, True), int_(-2), cmp("eq")]], T, key_word=0xFFFE00)
    case([[key(), int_(-1), cmp("eq")]], T, key_word=2**64 - 1)
    return cases


def test_evaluator_answers_from_the_reference_rules():
    for preds, key_word, null, want in evaluator_cases():
        got = evaluate(preds, key_word, [0, 0], [0, 0, 0] if null else [1, 5, 0], 1 if null else 0)
        assert got == want, (preds, key_word, null)


def evaluator_case_op_rows(key_word, null):
    """The one-key activation of an evaluator case (NULL_SUM_LANES)."""
    k = key_word - (1 << 64) if key_word >> 63 else key_word
    return [(k, v, t, d) for _, v, t, d in NULL_SUM_ROWS] if null else [(k, 5, 0, 1)]


def test_evaluator_cases_through_one_key_operators(oracle):
    """Each evaluator case through the restatement: the row is visible exactly when the answer says so, with
    the answer's error in flag bits 16-18."""
    for preds, key_word, null, want in evaluator_cases():
        (out,) = run_steps(ReduceLanesHaving(oracle, NULL_SUM_LANES, 32, preds), [(evaluator_case_op_rows(key_word, null), 1)])
        visible = want != "drop"
        assert len(out) == (1 if visible else 0), (preds, want)
        if visible:
            err = want[1] if isinstance(want, tuple) else 0
            assert int(out[0]["flags"]) == (err << ERR_SHIFT) | (1 if null else 0), (preds, want)


def test_null_sum_through_the_distinct_total_rule(oracle):
    """On the NULL SUM a predicate is NULL and drops the row, its negation too, and an OR with TRUE keeps it."""
    for preds, visible in NULL_SUM_PREDS:
        (out,) = run_steps(ReduceLanesHaving(oracle, NULL_SUM_LANES, 32, preds), [(NULL_SUM_ROWS, 1)])
        assert len(out) == (1 if visible else 0), preds
        if visible:
            assert int(out[0]["flags"]) == 1 and int(out[0]["lanes"][1]["count"]) == 3


# ---------------------------------------------------------------- reference-held answers
def load_fixture():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "sqllogictest_having.json")))


# the mapping of each case's plan to lanes and predicates, as a renderer would write it
# filter=(((#3 - integer_to_bigint(#0{a})) > 2) AND ((#3 / integer_to_bigint((1 + #0{a}))) >= 1)) with the map
# #3 = #2 + 1 (#2 = count(b)) inline: the plan's predicate list, one conjunct per predicate
_MFP_FILTER = [
    [count(1), int_(1), add(64), key(0, 32, True), sub(64), int_(2), cmp("gt")],
    [count(1), int_(1), add(64), int_(1), key(0, 32, True), add(32), div(64), int_(1), cmp("ge")],
]
FIXTURE_PLANS = {
    "reduce_mfp_fusable_accumulable": (32, [(I64, VAL1, 0, 32, True), (I64, VAL1, 0, 32, True)], _MFP_FILTER, 0),
    "reduce_mfp_complex_accumulable": (32, [(I64, VAL1, 0, 32, True), (I64, VAL1, 0, 32, True)], _MFP_FILTER, 1),
    "cockroach_having_count_star": (32, [(I64, VAL1, 0, 64, True)], [[count(0), int_(1), cmp("gt")]], None),
    "cockroach_having_count_distinct": (
        40, [(I64 | D, VAL1, 0, 64, True), (I64 | D, VAL2, 0, 64, True)], [[count(0), int_(1), cmp("gt")]], None),
}


def _case_rows(name, table_rows, time, diff, in_rb):
    dt = np.dtype([(f"w{i}", "<u8") for i in range(in_rb // 8)])
    a = np.zeros(len(table_rows), dtype=dt)
    for i, r in enumerate(table_rows):
        if name.startswith("reduce_mfp"):  # t(a, b): GROUP BY a, aggregates over b
            words = [r[0], r[1]]
        elif name == "cockroach_having_count_star":  # kv(k, v, w, s): GROUP BY s, count(*) over k
            words = [r[3], r[0]]
        else:  # GROUP BY length(s): DISTINCT s, DISTINCT length(s)
            words = [1, r[3], 1]
        words += [time, diff]
        for j, x in enumerate(words):
            a[i][f"w{j}"] = np.int64(x).view(np.uint64)
    return a


def run_fixture_case(make_op, case):
    """Every step of one case through one operator; returns per step the answer rows (or "error: <name>")."""
    in_rb, lanes, preds, sum_plus = FIXTURE_PLANS[case["name"]]
    op = make_op(in_rb, lanes, preds)
    cur, answers = {}, []
    for t, step in enumerate(case["steps"]):
        rows = step.get("insert") or step.get("delete")
        out = op.step(_case_rows(case["name"], rows, t, 1 if "insert" in step else -1, in_rb), t + 1)
        for o in out:
            cls = o["lanes"].shape[0]
            k = (int(o["key"]),) + tuple(int(x) & M64 for l in range(cls) for x in o["lanes"][l].tolist()) + (int(o["flags"]),)
            cur[k] = cur.get(k, 0) + int(o["diff"])
        vis = [k for k, d in cur.items() if d != 0]
        assert all(cur[k] == 1 for k in vis)
        errors = [k for k in vis if (k[-1] >> ERR_SHIFT) & 7]
        if errors:
            assert all((k[-1] >> ERR_SHIFT) & 7 == DIVISION_BY_ZERO for k in errors)
            answers.append("error: division by zero")
            continue
        ans = []
        for k in vis:
            kw = k[0] - (1 << 64) if k[0] >> 63 else k[0]
            lane_words = k[1:-1]
            if sum_plus is not None:  # a, SUM(b) (+ 1 downstream)
                s = lane_words[1] | (lane_words[2] << 64)
                ans.append([kw, s + sum_plus])
            else:
                ans.append([kw] + [lane_words[3 * l] for l in range(len(lanes))])
        answers.append(sorted(ans))
    return answers


def fixture_expect(case):
    return [("error: " + s["expect_error"]) if "expect_error" in s else sorted(s["expect"]) for s in case["steps"]]


def test_fixture_cases_through_one_operator(oracle):
    # every program here fits the descriptor (mzgpu_having: 4 predicates of at most 16 ops)
    for _, _, preds, _ in FIXTURE_PLANS.values():
        assert len(preds) <= 4 and all(len(p) <= 16 for p in preds)
    for _, _, preds in SCENARIOS.values():
        assert len(preds) <= 4 and all(len(p) <= 16 for p in preds)
    for case in load_fixture()["cases"]:
        got = run_fixture_case(lambda i, l, p: ReduceLanesHaving(oracle, l, i, p), case)
        assert got == fixture_expect(case), case["name"]


def having_sum_cases():
    """The having_sum* cases of sqllogictest_join_reduce.json with HAVING sum(b) = 3 inside the operator."""
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "sqllogictest_join_reduce.json")))
    t = [tuple(r) for r in fx["tables"]["t"]["rows"]]
    for case in fx["cases"]:
        if case["shape"] == "having_sum":
            yield case, t
        elif case["shape"] == "having_sum_expr_key":
            yield case, [(a + 1, b) for a, b in t]  # the key's map runs in front of the reduce


def run_having_sum(make_op, pairs):
    op = make_op(32, [(I64, VAL1, 0, 64, True)], [[sum_(0), num(3), cmp("eq")]])
    out = op.step(_r32([(k, v, 0, 1) for k, v in pairs]), 1)
    assert (out["diff"] == 1).all() and (out["flags"] == 0).all()
    return sorted([int(np.int64(k))] for k in out["key"])


def test_join_reduce_having_sum_cases_inside_the_operator(oracle):
    n = 0
    for case, pairs in having_sum_cases():
        assert run_having_sum(lambda i, l, p: ReduceLanesHaving(oracle, l, i, p), pairs) == sorted(case["expect"]), case["name"]
        n += 1
    assert n == 2


def test_no_predicates_is_the_unfiltered_restatement(oracle):
    from distinct_lanes_oracle import ReduceLanesDistinct

    in_rb, lanes, _ = SCENARIOS["c4_r40_division_by_key"]
    a, b = ReduceLanesHaving(oracle, lanes, in_rb, []), ReduceLanesDistinct(oracle, lanes, in_rb)
    for rows, upper in distinct_activations(np.random.default_rng(1), in_rb // 8, steps=5):
        assert a.step(rows, upper).tobytes() == b.step(rows, upper).tobytes()


def test_having_descriptor_limits_in_python():
    """having() builds the descriptor on the host (no device): past its limits it raises E_INVALID, not an
    IndexError from ctypes."""
    import materialize_b200 as mz

    p = [mz.h_count(0), mz.h_int(1), mz.h_cmp("gt")]
    hv = mz.having(*[p] * 4)
    assert hv.n_predicates == 4 and hv.n_consts == 1 and list(hv.n_ops) == [3] * 4
    def sums(ks):  # sum of the constants ks > 0: len(ks) + 1 ops
        return [mz.h_int(k) for k in ks] + [mz.h_add()] * (len(ks) - 1) + [mz.h_int(0), mz.h_cmp("gt")]

    for preds in ([p] * 5, [[mz.h_int(1)] * 17], [sums(range(1, 6)), sums(range(6, 10))]):  # 5 + 4 + 1 constants
        with pytest.raises(mz.MzGpuError) as e:
            mz.having(*preds)
        assert e.value.status == -1
    assert mz.having(sums(range(1, 5)), sums(range(5, 8))).n_consts == 8
