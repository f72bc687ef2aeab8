"""CPU checks of tests/mfp_map_oracle.py: the restatement of the MfpPlan with map expressions against an eager
per-row statement of evaluate_inner's order, against Materialize's expected answers for the new integer functions,
and against mfp_oracle for plans without expressions."""
import json
import os
import random

import pytest

import mfp_map_oracle as M
import mfp_oracle as O

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mfp_map_arithmetic.json")))
EDGE = [0, 1, 2**31 - 1, 2**31, 2**32 - 2**31, 2**63, 2**64 - 1, 2**64 - 2**31, 12345, 2**64 - 16]


def eager(plan, w, time, diff, until):
    """evaluate_inner's outcome from every expression and predicate evaluated up front: the first erroring
    expression E fires at the first predicate whose support passes E (or after the last predicate), unless an
    earlier predicate errors or is not TRUE.  The bounds are then mfp_oracle's, over the expression values."""
    maps, mv, first_err = plan["maps"], [], None
    for i, ops in enumerate(maps):
        e, p, v = M.run(ops, plan["map_consts"], w, mv + [0] * (len(maps) - len(mv)))
        if e and first_err is None:
            first_err = (i, e, p)
        mv.append(0 if e or first_err else v)
    for ops in plan["predicates"]:
        if first_err and M.support(ops) > first_err[0]:
            return [], [(first_err[1], first_err[2], time, diff)]
        e, p, v = M.run(ops, plan["consts"], w, mv)
        if e:
            return [], [(e, p, time, diff)]
        if v == 0:
            return [], []
    if first_err:
        return [], [(first_err[1], first_err[2], time, diff)]
    # the temporal part, with the expression values substituted for MAP reads
    temporal = [(c, [(O.HOP_INT, 0, 0, 0, 0, 100 + o[1]) if o[0] == M.HOP_MAP else o for o in ops])
                for c, ops in plan["temporal"]]
    consts = dict(enumerate(plan["consts"]))
    consts.update({100 + j: (v % M.U64, 0) for j, v in enumerate(mv)})
    p2 = {"fields": plan["fields"], "predicates": [], "temporal": temporal, "consts": consts}
    return O.evaluate(p2, w, time, diff, until)


@pytest.mark.parametrize("seed", range(40))
def test_restatement_against_eager_evaluation(seed):
    rng = random.Random(seed)
    for _ in range(8):
        plan = M.random_plan(rng, in_words=rng.choice([4, 5]))
        for _ in range(40):
            w = [rng.choice(EDGE + [rng.randrange(2**64), rng.randrange(200)]) for _ in range(3)]
            time, diff = rng.randrange(200), rng.choice([1, -1, 3])
            until = rng.choice([O.EMPTY, 100])
            upd, err, _ = M.evaluate(plan, w, time, diff, until)
            assert (upd, err) == eager(plan, w, time, diff, until), plan


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[str(c["line"]) for c in GOLDEN["cases"]])
def test_golden_arithmetic(case):
    """Materialize's expected answers (arithmetic.slt) from the restatement's interpreter."""
    ops, consts = M.golden_program(case)
    e, p, v = M.run(ops, consts, [0, 0, 0], [])
    want_e, want_p, want_v = M.golden_expect(case)
    assert e == want_e
    if want_p is not None:
        assert p == want_p
    if want_v is not None:
        assert v == want_v


def test_function_edges():
    ops = lambda *o: [tuple(list(x) + [0] * (6 - len(x))) for x in o]  # noqa: E731
    col32 = (O.HOP_COL, 0, 0, 32, 1)
    col64 = (O.HOP_COL, 0, 0, 64, 0)
    assert M.run(ops(col32, (M.HOP_NEG, 32)), [], [2**31], []) == (O.E_I32, 2**64 - 2**31, -(2**31))
    assert M.run(ops(col32, (M.HOP_NEG, 64)), [], [2**31], []) == (0, 0, 2**31)
    assert M.run(ops(col32, (M.HOP_ABS, 32)), [], [2**32 - 5], []) == (0, 0, 5)
    assert M.run(ops(col64, (M.HOP_ABS, 64)), [], [2**63], []) == (O.E_I64, 2**63, -(2**63))
    assert M.run(ops(col64, (M.HOP_INT64_TO_INT32,)), [], [2**31], []) == (O.E_I32, 2**31, 2**31)
    assert M.run(ops(col64, (M.HOP_INT64_TO_INT32,)), [], [2**64 - 2**31], [])[:2] == (0, 0)
    # -7 % 3 = -1 and 7 % -3 = 1 (the dividend's sign, as Rust's %)
    k = [(2**64 - 7, 2**64 - 1), (3, 0), (7, 0), (2**64 - 3, 2**64 - 1)]
    assert M.run(ops((O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_INT, 0, 0, 0, 0, 1), (M.HOP_MOD, 64)), k, [], [])[2] == -1
    assert M.run(ops((O.HOP_INT, 0, 0, 0, 0, 2), (O.HOP_INT, 0, 0, 0, 0, 3), (M.HOP_MOD, 64)), k, [], [])[2] == 1


def test_if_is_lazy_in_the_branch_not_taken():
    div0 = [(O.HOP_INT, 0, 0, 0, 0, 1), (O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_DIV, 64, 0, 0, 0, 0)]
    cond = [(O.HOP_COL, 0, 0, 8, 0, 0), (O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_CMP, O.EQ, 0, 0, 0, 0)]
    one = [(O.HOP_INT, 0, 0, 0, 0, 1)]
    k = [(0, 0), (1, 0)]
    iff = [(M.HOP_IF, 0, 0, 0, 0, 0)]
    assert M.run(cond + one + div0 + iff, k, [0], []) == (0, 0, 1)  # the erroring else is not taken
    assert M.run(cond + one + div0 + iff, k, [5], [])[0] == O.E_DIV0
    # an error in the condition is the result, whatever the branches
    cond_err = div0 + [(O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_CMP, O.EQ, 0, 0, 0, 0)]
    assert M.run(cond_err + one + one + iff, k, [0], [])[0] == O.E_DIV0


def test_evaluation_order():
    # maps: [0] = 10 / key (errors at key 0), [1] = val; predicate: #1 > 5 (support 2)
    k = [(10, 0), (5, 0), (0, 0)]
    div = [(O.HOP_INT, 0, 0, 0, 0, 0), (O.HOP_COL, 0, 0, 64, 0, 0), (O.HOP_DIV, 64, 0, 0, 0, 0)]
    val = [(O.HOP_COL, 1, 0, 64, 0, 0)]
    gt = [(M.HOP_MAP, 1, 0, 0, 0, 0), (O.HOP_INT, 0, 0, 0, 0, 1), (O.HOP_CMP, O.GT, 0, 0, 0, 0)]
    plan = {"fields": [[(0, 0, 64, 0)], [(M.SRC_MAP0 + 1, 0, 64, 0)]], "predicates": [gt], "temporal": [],
            "consts": k, "maps": [div, val], "map_consts": k}
    # support 2 forces map 0 before the predicate: its error fires even for a row the predicate would drop
    assert M.evaluate(plan, [0, 1, 0], 3, 1, O.EMPTY)[:2] == ([], [(O.E_DIV0, 0, 3, 1)])
    # with the maps swapped the predicate needs only map 0 (= val): map 1 fires only for rows that pass
    plan2 = dict(plan, maps=[val, div], predicates=[[(M.HOP_MAP, 0, 0, 0, 0, 0)] + gt[1:]])
    assert M.evaluate(plan2, [0, 1, 0], 3, 1, O.EMPTY)[:2] == ([], [])
    assert M.evaluate(plan2, [0, 9, 0], 3, 1, O.EMPTY)[:2] == ([], [(O.E_DIV0, 0, 3, 1)])
    assert M.evaluate(plan2, [2, 9, 0], 3, 1, O.EMPTY) == ([(3, 1)], [], [9, 5])
    assert M.project(plan2, [2, 9, 0], [9, 5]) == [2, 5]


@pytest.mark.parametrize("seed", range(10))
def test_without_expressions_is_mfp_oracle(seed):
    rng = random.Random(seed)
    for _ in range(10):
        plan = M.random_plan(rng, n_maps=0, temporal=[(O.GE, [(O.HOP_COL_MZTS, 1, 0, 8, 0, 0)])], new_ops=False)
        for _ in range(30):
            w = [rng.choice(EDGE + [rng.randrange(300)]) for _ in range(3)]
            upd, err, _ = M.evaluate(plan, w, 7, 1, O.EMPTY)
            assert (upd, err) == O.evaluate(plan, w, 7, 1, O.EMPTY)
            assert M.project(plan, w, []) == O.project(plan, w)
