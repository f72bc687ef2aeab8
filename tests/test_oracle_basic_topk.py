"""The basic TopK restatement (tests/basic_topk_oracle.py) against its direct definition, the C++ oracle's
TopK, the monotonic TopK's definition and the reference's sqllogictest answers.  CPU only."""
import json
import os
import random
from collections import Counter

import numpy as np
import pytest

from basic_topk_oracle import NO_LIMIT, BasicTopKDefinition, NegatedStage
from monotonic_topk_oracle import TopKDefinition as MonotonicDefinition

HERE = os.path.dirname(os.path.abspath(__file__))
VAL1, VAL2 = 1, 2
LANES = {
    0: [],
    1: [(VAL1, 0, 64, False, True)],
    3: [(VAL1, 0, 4, False, False), (VAL2, 0, 64, True, True), (VAL1, 4, 60, True, False)],
}


def history(rng, r40, n_acts=12, n_keys=6, n_vals=8, neg=True):
    """random activations of rows over a few keys and values: retractions, negative counts and their
    repairs, rows that cancel inside one activation"""
    acts = []
    for a in range(n_acts):
        rows = []
        for _ in range(rng.randint(0, 25)):
            k, v1 = rng.randrange(n_keys), rng.choice([rng.randrange(n_vals), rng.getrandbits(64)])
            v2 = rng.randrange(4) if r40 else 0
            d = rng.choice([1, 1, 2, 3, -1, -2] if neg else [1, 2, 3])
            rows.append((k, v1, v2, 2 * a + rng.randrange(2), d))
        if neg and rows and rng.random() < 0.3:  # a row and its retraction in one activation
            k, v1, v2, t, _ = rows[0]
            rows.append((k, v1, v2, t, -1))
            rows.append((k, v1, v2, t, 1))
        acts.append(rows)
    return acts


@pytest.mark.parametrize("limit", [0, 1, 3, 40, NO_LIMIT])
@pytest.mark.parametrize("offset", [0, 2, 50])
@pytest.mark.parametrize("r40", [False, True])
def test_restatement_matches_definition(limit, offset, r40):
    """Every activation's output and errors, the input arrangement and the negative counts agree."""
    rng = random.Random(limit % 997 * 100 + offset * 2 + r40)
    saw_error = saw_window = False
    for n_lanes in (0, 1, 3):
        lanes = LANES[n_lanes] if r40 else [(VAL1,) + l[1:] for l in LANES[n_lanes]]
        rb = 40 if r40 else 32
        s, d = NegatedStage(lanes, limit, offset, rb), BasicTopKDefinition(lanes, limit, offset, rb)
        for rows in history(rng, r40):
            got, want = s.step(rows), d.step(rows)
            assert got == want
            saw_error |= bool(want[1])
            saw_window |= bool(want[0])
            assert s.negatives() == d.negatives()
        assert s.input_rows(10) == d.input_rows(10)
    assert saw_error
    assert saw_window or limit == 0 or offset == 50


def test_enter_stay_and_leave_the_error_state():
    """A key with a negative count has no window until the count is repaired; its window comes back whole."""
    d = BasicTopKDefinition([], 2, 1)
    out, errs = d.step([(7, 1, 0, 0, 1), (7, 2, 0, 0, 1), (7, 3, 0, 0, 1)])
    assert out == [(7, 2, 0, 0, 1), (7, 3, 0, 0, 1)] and errs == []
    out, errs = d.step([(7, 9, 0, 1, -1)])
    assert out == [(7, 2, 0, 1, -1), (7, 3, 0, 1, -1)] and errs == [(7, 0, 1, 1)]
    out, errs = d.step([(7, 1, 0, 2, -5)])  # a second negative row: still in the state, nothing changes
    assert out == [] and errs == [] and d.negatives() == {7: 2}
    out, errs = d.step([(7, 9, 0, 3, 1), (7, 1, 0, 3, 5)])
    assert out == [(7, 2, 0, 3, 1), (7, 3, 0, 3, 1)] and errs == [(7, 0, 3, -1)]
    assert d.negatives() == {}


def test_limit_and_offset_cut_inside_a_row():
    d = BasicTopKDefinition([], 3, 2)
    out, _ = d.step([(1, 5, 0, 0, 4), (1, 6, 0, 0, 4)])
    assert out == [(1, 5, 0, 0, 2), (1, 6, 0, 0, 1)]
    out, _ = d.step([(1, 5, 0, 1, -3)])  # one unit of 5 left: the offset eats it and one of 6
    assert out == [(1, 5, 0, 1, -2), (1, 6, 0, 1, 2)]


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("limit,offset", [(1, 0), (3, 0), (3, 2), (NO_LIMIT, 1)])
def test_agrees_with_oracle_topk(descending, limit, offset):
    """One unsigned full-width lane over R32 with no negative counts: the C++ oracle's TopK (values in sum_lo)."""
    oracle = pytest.importorskip("oracle.binding")
    rng = random.Random(limit % 97 + offset + descending)
    lane = [(VAL1, 0, 64, False, descending)]
    d = BasicTopKDefinition(lane, limit, offset)
    o = oracle.TopK(-1 if limit == NO_LIMIT else limit, offset, descending)
    live = Counter()
    for a in range(10):
        rows = []
        for _ in range(rng.randint(0, 30)):
            k, v = rng.randrange(5), rng.randrange(12)
            dd = rng.choice([1, 2, -1])
            if live[(k, v)] + dd < 0:
                dd = 1
            live[(k, v)] += dd
            rows.append((k, v, 0, 2 * a, dd))
        want, errs = d.step(rows)
        assert errs == []
        arr = np.zeros(len(rows), dtype=oracle.R32)
        for i, (k, v, _, t, dd) in enumerate(rows):
            arr[i] = (k, v, t, dd)
        got = sorted((int(r["key"]), int(r["sum_lo"]), 0, int(r["time"]), int(r["diff"])) for r in o.step(arr, 2 * a + 2))
        assert got == want


@pytest.mark.parametrize("limit", [1, 3, NO_LIMIT])
@pytest.mark.parametrize("n_lanes", [0, 1, 3])
def test_agrees_with_monotonic_topk_on_insert_only_input(limit, n_lanes):
    rng = random.Random(limit % 89 + n_lanes)
    lanes = LANES[n_lanes]
    d, m = BasicTopKDefinition(lanes, limit, 0, 40), MonotonicDefinition(lanes, limit, 40)
    for rows in history(rng, True, neg=False):
        assert d.step(rows) == (m.step(rows)[0], [])


def golden():
    return json.load(open(os.path.join(HERE, "golden", "sqllogictest_topk.json")))


def city_rows(fx, case):
    """the cities as R40 rows (key = state, val1 = pop, val2 = city); NULL above every population (DESC NULLS
    FIRST) or below (DESC NULLS LAST), as tests/test_oracle_ops.py encodes it"""
    rows = fx["cities"]["rows"]
    states = sorted({r[1] for r in rows})
    names = [r[0] for r in rows]
    out = []
    for name, state, pop in rows:
        if pop is None:
            pop = (1 << 40) - 1 if case["nulls_first"] else 0
        out.append((states.index(state), pop, names.index(name), 0, 1))
    return out, states, names


def test_sqllogictest_per_group():
    fx = golden()
    for case in fx["per_group"]:
        rows, states, names = city_rows(fx, case)
        d = BasicTopKDefinition([(VAL1, 0, 64, False, case["descending"])], case["limit"], 0, 40)
        out, errs = d.step(rows)
        assert errs == [] and all(r[4] == 1 for r in out)
        assert sorted((states[r[0]], names[r[2]]) for r in out) == sorted(tuple(x) for x in case["answer"])


def test_sqllogictest_global_limit_then_limit_offset():
    """Two chained operators, fed all at once and then with deletions and re-inserts."""
    fx = golden()
    for case in fx["global"]:
        stages = [BasicTopKDefinition([(VAL1, 0, 64, False, False)], s["limit"], s["offset"]) for s in case["stages"]]
        final = Counter()

        def feed(rows):
            for st in stages:
                rows, errs = st.step(rows)
                assert errs == []
            for k, v1, _, _, d in rows:
                final[v1] += d

        feed([(0, x, 0, 0, 1) for x in case["t"]])
        assert sorted(v for v, c in final.items() if c) == case["answer"]
        feed([(0, x, 0, 1, -1) for x in case["t"][:3]])  # 1, 2, 3 leave: the window moves up by three
        assert sorted(v for v, c in final.items() if c) == [x + 3 for x in case["answer"]]
        feed([(0, x, 0, 2, 1) for x in case["t"][:3]])
        assert sorted(v for v, c in final.items() if c) == case["answer"]
        assert all(c in (0, 1) for c in final.values())
