"""COUNT(DISTINCT x) / SUM(DISTINCT x) lanes of the multi-column accumulable reduce, restated on the CPU
(tests/distinct_lanes_oracle.py), pinned by their definition -- a GROUP BY over the accumulated input, with
the reference's rule for the total word -- and by reference-held sqllogictest answers."""
import json
import os

import numpy as np
import pytest
from distinct_lanes_oracle import ACCUM_DISTINCT, ReduceLanesDistinct
from test_oracle_reduce_lanes import F64, I64, VAL1, VAL2, pick, s64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64, M128 = (1 << 64) - 1, (1 << 128) - 1
D = ACCUM_DISTINCT


def f64_fixed(x):
    y = x * 16777216.0
    if y >= 2.0**127:
        return (1 << 127) - 1
    if y <= -(2.0**127):
        return -(1 << 127)
    return int(y)


def expected(rows, lanes, in_words, cls, tau):
    """GROUP BY key of the input rows with time <= tau.  A plain lane accumulates every row; a distinct lane
    the values whose accumulated multiplicity is non-zero (negative included), each once.  The total is
    [some lane is plain] * (sum of diffs) + the number of present (value, lane) pairs."""
    plain = any(not (l[0] & D) for l in lanes)
    acc, mult = {}, {}
    for r in rows:
        w = [int(x) for x in r.tolist()]
        if w[in_words - 2] > tau:
            continue
        d = s64(w[in_words - 1])
        a = acc.setdefault(w[0], [0] + [[0, 0, 0, 0, 0] for _ in lanes])
        if plain:
            a[0] += d
        for l, lane in enumerate(lanes):
            kind = lane[0] & ~D
            v = pick(w, (kind, *lane[1:]))
            if lane[0] & D:
                mult[(l, w[0], v)] = s64(mult.get((l, w[0], v), 0) + d)
                continue
            x = a[1 + l]
            x[0] += d
            if kind == F64:
                f = float(np.uint64(v).view(np.float64))
                if np.isnan(f):
                    x[4] += d
                elif f == np.inf:
                    x[2] += d
                elif f == -np.inf:
                    x[3] += d
                else:
                    x[1] += f64_fixed(f) * d
            else:
                x[1] += s64(v) * d
    for (l, k, v), m in mult.items():
        if m != 0:
            a = acc[k]
            a[0] += 1
            a[1 + l][0] += 1
            a[1 + l][1] += s64(v)
    out = {}
    for k, a in acc.items():
        total = s64(a[0])
        lanes_w = [[s64(x[0]), x[1] & M128, s64(x[2]), s64(x[3]), s64(x[4])] for x in a[1:]]
        if total == 0 and all(not any(x) for x in lanes_w):
            continue
        vals, flags = [], 0
        for l, (lane, (nn, s, pinf, ninf, nan)) in enumerate(zip(lanes, lanes_w)):
            zero = nn == 0 and s == 0 and pinf == 0 and ninf == 0 and nan == 0
            lf = (1 if total > 0 and zero else 0) | (2 if total == 0 and not zero else 0)
            if lane[0] == F64:
                if nan > 0 or (pinf > 0 and ninf > 0):
                    lo = 0x7FF8000000000000
                elif pinf > 0:
                    lo = 0x7FF0000000000000
                elif ninf > 0:
                    lo = 0xFFF0000000000000
                else:
                    si = s - (1 << 128) if s >> 127 else s
                    lo = int(np.float64(float(si) / 16777216.0).view(np.uint64))
                hi = 0
            else:
                lo, hi = s & M64, s >> 64
            if lf & 1:
                lo = hi = 0
            vals += [nn & M64, lo, hi]
            flags |= lf << (2 * l)
        vals += [0, 0, 0] * (cls - len(lanes))
        out[k] = ((k, *vals, flags), total)
    return out


def accumulated(out_rows, cls, tau):
    acc = {}
    for r in out_rows:
        if int(r["time"]) > tau:
            continue
        key = (int(r["key"]),) + tuple(int(x) & M64 for l in range(cls) for x in r["lanes"][l].tolist()) + (int(r["flags"]),)
        acc[key] = acc.get(key, 0) + int(r["diff"])
    assert all(d in (0, 1) for d in acc.values()), "an output row with multiplicity other than 1"
    return {k for k, d in acc.items() if d == 1}


def export_totals(export, tau):
    """Per key, the accumulated total word of the main arrangement's rows with time <= tau."""
    tot = {}
    for r in export:
        if int(r["time"]) <= tau:
            tot[int(r["key"])] = s64(tot.get(int(r["key"]), 0) + int(r["total"]))
    return {k: t for k, t in tot.items() if t != 0}


# values that repeat (so pairs accumulate, vanish and come back), including i64 extremes whose distinct sums
# overflow i64 and words whose bit-fields have the sign bit set
POOL = np.array(
    [0, 1, 2, 7, 2**63 - 1, 2**63 - 2, 2**63, 2**63 + 5, 2**64 - 1, 0xFFFFF, 0x80000, 0x123456789ABCDEF0, 0xF0F0F0F0F0F0F0F0],
    dtype=np.uint64,
)


def distinct_activations(rng, in_words, steps=8, keys=12):
    """Activations over a small value pool: the same pair at several times of a batch, diffs of both signs
    (negative multiplicities), retractions of earlier rows, rows at times past the batch's upper."""
    dt = np.dtype([(f"w{i}", "<u8") for i in range(in_words)])
    live, t = [], 0
    for step in range(steps):
        n = int(rng.integers(1, 200))
        a = np.zeros(n, dtype=dt)
        a["w0"] = rng.integers(0, keys, size=n, dtype=np.uint64)
        for src in range(1, in_words - 2):
            a[f"w{src}"] = POOL[rng.integers(0, len(POOL), size=n)]
        a[f"w{in_words - 2}"] = rng.integers(t, t + 4, size=n, dtype=np.uint64)  # t + 3: sealed next step
        a[f"w{in_words - 1}"] = rng.choice(np.array([-2, -1, 1, 1, 2, 3], dtype=np.int64), size=n).view(np.uint64)
        if live and step % 2 == 1:
            old = np.concatenate(live)
            pk = old[rng.random(len(old)) < 0.5].copy()
            pk[f"w{in_words - 1}"] = (-pk[f"w{in_words - 1}"].view(np.int64)).view(np.uint64)
            pk[f"w{in_words - 2}"] = rng.integers(t, t + 3, size=len(pk), dtype=np.uint64)
            a = np.concatenate([a, pk])
            live = []
        else:
            live.append(a.copy())
        t += 3
        yield a, t


DISTINCT_SETS = {
    "r32_all_distinct": (32, [(I64 | D, VAL1, 0, 64, False), (I64 | D, VAL1, 0, 20, True)]),
    "r40_mixed": (40, [(I64, VAL1, 0, 64, False), (I64 | D, VAL2, 0, 64, False), (I64 | D, VAL1, 8, 16, True)]),
    "r32_one_distinct": (32, [(I64 | D, VAL1, 0, 64, False)]),
    "r40_one_distinct": (40, [(I64 | D, VAL2, 60, 4, True)]),
    "r40_eight_four": (
        40,
        [(I64, VAL1, 0, 64, False), (I64 | D, VAL1, 0, 64, False), (F64, VAL2, 0, 64, False), (I64 | D, VAL2, 0, 64, False),
         (I64, VAL1, 3, 17, True), (I64 | D, VAL1, 60, 4, True), (I64, VAL2, 32, 32, False), (I64 | D, VAL2, 0, 8, True)],
    ),
}


@pytest.mark.parametrize("name", sorted(DISTINCT_SETS))
def test_distinct_lanes_are_group_by_of_accumulated_input(oracle, name):
    in_rb, lanes = DISTINCT_SETS[name]
    in_words = in_rb // 8
    r = ReduceLanesDistinct(oracle, lanes, in_rb)
    rng = np.random.default_rng(3 + len(name))
    seen, outs = [], []
    for a, upper in distinct_activations(rng, in_words):
        seen.append(a)
        outs.append(r.step(a, upper))
        rows, out = np.concatenate(seen), np.concatenate(outs)
        export = r.export()
        for tau in range(upper - 3, upper):
            want = expected(rows, lanes, in_words, r.cls, tau)
            assert accumulated(out, r.cls, tau) == {row for row, _ in want.values()}, (name, tau)
            # the arrangement's total word follows the reference's rule
            assert export_totals(export, tau) == {k: t for k, (_, t) in want.items() if t != 0}, (name, tau)


def _rows(in_words, rows):
    dt = np.dtype([(f"w{i}", "<u8") for i in range(in_words)])
    a = np.zeros(len(rows), dtype=dt)
    for i, r in enumerate(rows):
        for j, x in enumerate(r):
            a[i][f"w{j}"] = np.int64(x).view(np.uint64) if isinstance(x, int) and x < 0 else np.uint64(x)
    return a


def test_presence_within_one_batch(oracle):
    """A pair that vanishes and comes back at later times of one batch, the same pair at several times, a
    negative multiplicity (present), and a value whose distinct sum with another overflows i64."""
    lanes = [(I64, VAL1, 0, 64, False), (I64 | D, VAL1, 0, 64, False)]
    r = ReduceLanesDistinct(oracle, lanes, 32)
    big = 2**63 - 1
    rows = _rows(4, [
        (1, 5, 0, 1), (1, 5, 1, -1), (1, 5, 2, 1), (1, 5, 2, 1),  # 5: present, gone, back (multiplicity 2)
        (1, big, 0, 1), (1, big - 1, 1, 1),  # distinct sum 2^64 - 3: past i64
        (2, 9, 1, -1),  # negative multiplicity: present, counted once
    ])
    r.step(rows, 3)
    pe = r.pair_export(1)
    assert [tuple(int(x) for x in p.tolist()) for p in pe] == [
        (1, 5, 0, 1), (1, 5, 1, -1), (1, 5, 2, 2), (1, big - 1, 1, 1), (1, big, 0, 1), (2, 9, 1, -1)]
    ex = {(int(e["key"]), int(e["time"])): e for e in r.export()}
    # key 1 at time 1: plain diff -1 + 1 (big - 1 arrives), pair 5 vanishes (-1), big - 1 appears (+1)
    assert int(ex[(1, 1)]["total"]) == 0 and int(ex[(1, 1)]["lanes"][1]["non_nulls"]) == 0
    got = {}
    for o in r.step(np.zeros(0, dtype=rows.dtype), 4):
        got[int(o["key"])] = o
    rows_all = rows
    want = expected(rows_all, lanes, 4, 2, 3)
    (k1, _), (k2, _) = want[1], want[2]
    # key 1: count(DISTINCT) = 3 (5, big, big - 1), sum(DISTINCT) = 5 + 2^64 - 3 as i128
    assert k1[4] == 3 and k1[5] | (k1[6] << 64) == 5 + 2 * big - 1
    # key 2: the plain total is -1, the pair adds +1: total 0 with non-zero lanes -> both lanes' error flags
    assert k2[4] == 1 and k2[-1] == 0b1010
    assert got == {}


def test_one_distinct_lane_on_unique_pairs_equals_the_plain_lane(oracle):
    """Every (key, value) at most once and never retracted: the distinct lane's rows are the plain lane's."""
    rng = np.random.default_rng(5)
    r, p = ReduceLanesDistinct(oracle, [(I64 | D, VAL1, 0, 64, False)], 32), ReduceLanesDistinct(oracle, [(I64, VAL1, 0, 64, False)], 32)
    used, t = set(), 0
    for _ in range(5):
        n = 300
        a = np.zeros(n, dtype=oracle.R32)
        a["key"] = rng.integers(0, 30, size=n, dtype=np.uint64)
        a["val"] = rng.integers(-(2**62), 2**62, size=n, dtype=np.int64).view(np.uint64)
        a["time"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        a["diff"] = 1
        keep = [(k, v) not in used and not used.add((k, v)) for k, v in zip(a["key"].tolist(), a["val"].tolist())]
        a = a[np.array(keep)]
        t += 3
        assert r.step(a, t).tobytes() == p.step(a, t).tobytes()
    assert r.export().tobytes() == p.export().tobytes()


def load_fixture():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "sqllogictest_distinct_aggs.json")))


def run_fixture_case(make_op, case):
    """One fixture case through one operator: returns the row of the single group."""
    vals = case["rows"]
    lanes = [(I64 | (D if c["distinct"] else 0), VAL1, 0, 64, True) for c in case["columns"]]
    rows = np.zeros(len(vals), dtype=np.dtype([("key", "<u8"), ("val", "<u8"), ("time", "<u8"), ("diff", "<i8")]))
    rows["val"] = np.array(vals, dtype=np.int64).view(np.uint64)
    rows["diff"] = 1
    op = make_op(lanes)
    (o,) = op.step(rows, 1)
    got = []
    for l, c in enumerate(case["columns"]):
        cnt, s = int(o["lanes"][l]["count"]), int(np.int64(o["lanes"][l]["sum_lo"]))
        got.append({"count": cnt, "sum": s, "avg": s / cnt}[c["agg"]])
    return got


def test_fixture_cases_through_one_operator(oracle):
    fx = load_fixture()
    for case in fx["cases"]:
        got = run_fixture_case(lambda lanes: ReduceLanesDistinct(oracle, lanes, 32), case)
        assert got == case["expect"], case["query"]
