"""The monotonic TopK restatement (tests/monotonic_topk_oracle.py) against its direct definition at every
time, on hand-written cases, and on the reference's testdrive answers."""
import itertools
import json
import os
import random
from collections import Counter

import pytest

from monotonic_topk_oracle import M64, NO_LIMIT, TopKDefinition, TopKRestatement, order_words

HERE = os.path.dirname(os.path.abspath(__file__))

LANE_SETS = {
    0: [],
    1: [(1, 0, 64, False, True)],
    2: [(1, 0, 8, True, False), (1, 8, 8, False, True)],
    3: [(1, 0, 4, False, False), (2, 0, 64, True, True), (1, 4, 60, True, False)],
}


def gen(rng, n, t, r40, keys=6, vals=12):
    rows = []
    for _ in range(n):
        v1 = rng.choice([rng.randrange(vals), rng.randrange(1 << 64), M64, 1 << 63])
        v2 = rng.randrange(vals) if r40 else 0
        rows.append((rng.randrange(keys), v1, v2, t + rng.randrange(2), rng.choice([1, 1, 2, 5, 0, -1])))
    return rows


@pytest.mark.parametrize("limit", [0, 1, 3, 40, NO_LIMIT])
@pytest.mark.parametrize("n_lanes", [0, 1, 2, 3])
@pytest.mark.parametrize("r40", [False, True])
@pytest.mark.parametrize("must", [False, True])
def test_restatement_equals_definition(limit, n_lanes, r40, must):
    lanes = LANE_SETS[n_lanes]
    if not r40:
        lanes = [(1,) + lane[1:] for lane in lanes]
    rng = random.Random(limit * 97 + n_lanes * 7 + 2 * r40 + must)
    d = TopKDefinition(lanes, limit, 40 if r40 else 32, must)
    r = TopKRestatement(lanes, limit, 40 if r40 else 32, must)
    for t in range(0, 40, 2):
        rows = gen(rng, rng.choice([0, 1, 5, 30]), t, r40)
        assert d.step(rows) == r.step(rows)


def accumulate(model, batches):
    acc, errs = Counter(), Counter()
    for b in batches:
        out, e = model.step(b)
        for k, v1, v2, _, dd in out:
            acc[(k, v1, v2)] += dd
        for t, c in e:
            errs[t] += c
    return {k: c for k, c in acc.items() if c}, dict(errs)


@pytest.mark.parametrize("model", [TopKDefinition, TopKRestatement])
def test_hand_cases(model):
    desc = [(1, 0, 64, False, True)]
    # multiplicity above the limit: the limit cuts inside one row's copies; Top1 yields diff 1
    assert accumulate(model(desc, 1), [[(1, 5, 0, 0, 7)]])[0] == {(1, 5, 0): 1}
    assert accumulate(model(desc, 3), [[(1, 5, 0, 0, 7), (1, 9, 0, 0, 1)]])[0] == {(1, 9, 0): 1, (1, 5, 0): 2}
    # ties on the lane are broken by the row (val1, then val2)
    lane = [(1, 0, 4, False, False)]
    got = accumulate(model(lane, 2, 40), [[(0, 0x31, 9, 0, 1), (0, 0x21, 8, 0, 1), (0, 0x21, 3, 0, 1)]])[0]
    assert got == {(0, 0x21, 3): 1, (0, 0x21, 8): 1}
    # one row displacing several: a new head of multiplicity 3 evicts the whole window of limit 3
    m = model(desc, 3)
    out1, _ = m.step([(2, 1, 0, 0, 1), (2, 2, 0, 0, 1), (2, 3, 0, 0, 1)])
    out2, _ = m.step([(2, 10, 0, 1, 3)])
    assert sorted(out2) == [(2, 1, 0, 1, -1), (2, 2, 0, 1, -1), (2, 3, 0, 1, -1), (2, 10, 0, 1, 3)]
    # several times per activation: each time's change at its own time
    m = model(desc, 1)
    out, _ = m.step([(3, 1, 0, 5, 1), (3, 2, 0, 6, 1), (3, 0, 0, 7, 1)])
    assert out == [(3, 1, 0, 5, 1), (3, 1, 0, 6, -1), (3, 2, 0, 6, 1)]


@pytest.mark.parametrize("model", [TopKDefinition, TopKRestatement])
def test_rejected_rows(model):
    desc = [(1, 0, 64, False, True)]
    rows = [(1, 5, 0, 3, 0), (1, 6, 0, 3, -1), (1, 7, 0, 4, 1), (1, 7, 0, 4, -1), (1, 8, 0, 4, 1)]
    out, errs = model(desc, 2).step(rows)
    assert errs == [(3, 2), (4, 1)]
    assert out == [(1, 7, 0, 4, 1), (1, 8, 0, 4, 1)]
    # consolidated first: the cancelling pair and the zero row vanish, the -1 stays an error
    out, errs = model(desc, 2, must_consolidate=True).step(rows)
    assert errs == [(3, 1)]
    assert out == [(1, 8, 0, 4, 1)]


def test_order_words():
    assert order_words(5, 0, []) == (0, 0, 0)
    assert order_words(0xFF, 0, [(1, 0, 8, True, False)]) == ((M64 ^ (1 << 63)), 0, 0)
    assert order_words(1, 0, [(1, 0, 64, False, True)]) == (M64 - 1, 0, 0)
    # signed order: -1 < 0 < 1 as words
    w = [order_words(v & M64, 0, [(1, 0, 64, True, False)])[0] for v in (-1, 0, 1)]
    assert w == sorted(w)


def fixture_cases():
    return json.load(open(os.path.join(HERE, "golden", "testdrive_monotonic_topk.json")))["cases"]


def encode(v, flip):
    v &= M64
    return v ^ (1 << 63) if flip else v


@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c: c["name"])
@pytest.mark.parametrize("model", [TopKDefinition, TopKRestatement])
def test_testdrive_answers(case, model):
    lanes = [(1, 0, 64, bool(sx), bool(desc)) for sx, desc in case["order"]]
    m = model(lanes, case["limit"])
    acc = Counter()
    for ingest, expect in zip(case["ingest"], case["expect"]):
        rows = [(k, encode(v, case["flip_sign"]), 0, t, 1) for k, v, t in ingest]
        out, errs = m.step(rows)
        assert errs == []
        for k, v1, _, _, d in out:
            acc[(k, v1)] += d
        got = sorted(itertools.chain.from_iterable([kv] * c for kv, c in acc.items() if c))
        want = sorted((k, encode(v, case["flip_sign"])) for k, v in expect)
        assert got == want
