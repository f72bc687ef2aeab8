"""The monotonic MIN / MAX reduce's CPU restatement (tests/monotonic_oracle.py): pinned against the
definition at every time, against the independent oracle's MIN / MAX reduce, against hand-written cases
and against the reference's printed SQL answers; plus the header's row widths."""
import json
import os
import re

import numpy as np
import pytest

from monotonic_oracle import AGG_MAX, AGG_MIN, M64, ReduceMonotonic, order_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAL1, VAL2 = 1, 2
R16 = np.dtype([("key", "<u8"), ("diff", "<i8")])
R32 = np.dtype([("key", "<u8"), ("val", "<u8"), ("time", "<u8"), ("diff", "<i8")])
R40 = np.dtype([("key", "<u8"), ("val1", "<u8"), ("val2", "<u8"), ("time", "<u8"), ("diff", "<i8")])


def rows32(tuples):
    a = np.zeros(len(tuples), dtype=R32)
    for i, (k, v, t, d) in enumerate(tuples):
        a[i] = (k, v & M64, t, d)
    return a


def rows40(tuples):
    a = np.zeros(len(tuples), dtype=R40)
    for i, (k, v1, v2, t, d) in enumerate(tuples):
        a[i] = (k, v1 & M64, v2 & M64, t, d)
    return a


def tl(a):
    """rows as plain tuples (sub-array fields as tuples)"""
    return [tuple(tuple(int(y) for y in x) if isinstance(x, np.ndarray) else int(x) for x in r) for r in a.tolist()]


def accumulate(coll, out, n_lanes):
    for r in out:
        k = (int(r["key"]), tuple(int(x) for x in r["vals"][:n_lanes]))
        coll[k] = coll.get(k, 0) + int(r["diff"])
        if coll[k] == 0:
            del coll[k]


def as_map(coll):
    got = {}
    for (k, v), d in coll.items():
        assert d == 1 and k not in got, (k, v, d)
        got[k] = v
    return got


def random_lanes(rng, n, r40):
    lanes = []
    for _ in range(n):
        bits = int(rng.choice([1, 8, 16, 32, 63, 64]))
        shift = int(rng.integers(0, 64 - bits + 1))
        lanes.append((int(rng.choice([AGG_MIN, AGG_MAX])), int(rng.choice([VAL1, VAL2])) if r40 else VAL1, shift, bits,
                      bool(rng.integers(0, 2))))
    return lanes


def expected(lanes, accepted, key):
    vals = []
    for l, lane in enumerate(lanes):
        vs = [v[l] for v in accepted[key]]
        pick = min if lane[0] == AGG_MIN else max
        vals.append(pick(vs, key=lambda x: order_key(lane, x)))
    return tuple(vals)


@pytest.mark.parametrize("seed", range(6))
def test_definition_at_every_time(seed):
    """At every time the accumulated output is GROUP BY MIN / MAX over the accepted rows so far, and the
    error count at each time is the number of rejected rows there."""
    from monotonic_oracle import lane_value

    rng = np.random.default_rng(seed)
    r40 = seed % 2 == 1
    n_lanes = [1, 3, 4, 5, 8, 2][seed]
    lanes = random_lanes(rng, n_lanes, r40)
    mc = seed >= 3
    op = ReduceMonotonic(lanes, 40 if r40 else 32, mc)
    coll, accepted = {}, {}
    for t in range(8):
        n = 200
        w = rng.integers(0, 2**63, size=(n, 5 if r40 else 4), dtype=np.uint64) * np.uint64(2) + rng.integers(
            0, 2, size=(n, 5 if r40 else 4), dtype=np.uint64)
        w[:, 0] = rng.integers(0, 30, size=n, dtype=np.uint64)
        w[:, -2] = t
        w[:, -1] = rng.choice([1, 1, 1, 2, 0, -1], size=n).astype(np.int64).view(np.uint64)
        if mc:  # some +1 / -1 pairs that cancel before ensure_monotonic
            w[n // 2:n // 2 + 20] = w[:20]
            w[n // 2:n // 2 + 20, -1] = np.int64(-1).astype(np.uint64) * np.ones(20, dtype=np.uint64)
            w[:20, -1] = 1
        rows = w.view(R40 if r40 else R32).reshape(-1)
        out, errs = op.step(rows, t + 1)
        accumulate(coll, out, n_lanes)
        # the definition
        data = {}
        for r in w.tolist():
            d = (r[0],) + tuple(lane_value(l, r) for l in lanes)
            x = r[-1] - (1 << 64) if r[-1] >> 63 else r[-1]
            if mc:
                data[d] = data.get(d, 0) + x
            else:
                data.setdefault(d, []).append(x)
        bad = 0
        for d, xs in data.items():
            for x in ([xs] if mc else xs):
                if mc and x == 0:
                    continue
                if x > 0:
                    accepted.setdefault(d[0], []).append(d[1:])
                else:
                    bad += 1
        assert [(int(e["key"]), int(e["diff"])) for e in errs] == ([(t, bad)] if bad else [])
        assert as_map(coll) == {k: expected(lanes, accepted, k) for k in accepted}
        assert all(int(r["diff"]) in (1, -1) for r in out)
        keys = [tuple(int(x) for x in r.tolist()[:-1]) for r in out.view(np.uint64).reshape(len(out), -1)]
        assert keys == sorted(keys) and len(set(keys)) == len(keys)


def test_one_unsigned_lane_equals_the_bucketed_min_max(oracle):
    """Insert-only input: one unsigned lane is value for value the oracle's MIN / MAX (u64 order),
    including keys with more than 32 live values."""
    rng = np.random.default_rng(7)
    for kind in (AGG_MIN, AGG_MAX):
        mono = ReduceMonotonic([(kind, VAL1, 0, 64, False)])
        old = oracle.Reduce(kind)
        got, want = {}, {}
        for t in range(10):
            n = 500
            r = np.zeros(n, dtype=oracle.R32)
            r["key"] = rng.integers(0, 20, size=n)
            r["val"] = rng.integers(0, 2**64, size=n, dtype=np.uint64)
            r["val"][:5] = [0, M64, 1, M64 - 1, 2**63]
            r["time"] = t
            r["diff"] = rng.integers(1, 3, size=n)
            out, errs = mono.step(r.view(R32), t + 1)
            assert len(errs) == 0
            accumulate(got, out, 1)
            for o in old.step(r, t + 1):
                assert int(o["flags"]) == 0
                k = (int(o["key"]), (int(o["sum_lo"]),))
                want[k] = want.get(k, 0) + int(o["diff"])
                if want[k] == 0:
                    del want[k]
            assert as_map(got) == as_map(want)


def test_plus_minus_one_at_one_time():
    lanes = [(AGG_MAX, VAL1, 0, 64, False)]
    a = ReduceMonotonic(lanes)
    out, errs = a.step(rows32([(1, 5, 0, 1), (1, 5, 0, -1)]), 1)
    assert tl(out) == [(1, (5, 0, 0, 0), 0, 1)] and tl(errs) == [(0, 1)]
    b = ReduceMonotonic(lanes, must_consolidate=True)
    out, errs = b.step(rows32([(1, 5, 0, 1), (1, 5, 0, -1)]), 1)
    assert len(out) == 0 and len(errs) == 0
    assert len(b.export()) == 0


def test_non_positive_diffs_each_count_once():
    op = ReduceMonotonic([(AGG_MIN, VAL1, 0, 64, True)])
    out, errs = op.step(rows32([(1, 4, 3, 0), (1, 2, 3, -3), (2, 7, 3, 2), (2, 9, 4, -1)]), 5)
    assert tl(errs) == [(3, 2), (4, 1)]
    assert tl(out) == [(2, (7, 0, 0, 0), 3, 1)]


def test_a_key_with_only_rejected_rows_has_no_output():
    op = ReduceMonotonic([(AGG_MAX, VAL1, 0, 64, False)], must_consolidate=True)
    out, errs = op.step(rows32([(9, 1, 0, -1), (9, 2, 0, -2)]), 1)
    assert len(out) == 0 and tl(errs) == [(0, 2)] and len(op.export()) == 0


@pytest.mark.parametrize("bits", [1, 32, 64])
def test_signed_and_unsigned_order(bits):
    """The field's top bit set: the largest value unsigned, a negative one signed."""
    top = 1 << (bits - 1)
    lanes = [(AGG_MAX, VAL1, 0, bits, False), (AGG_MAX, VAL1, 0, bits, True),
             (AGG_MIN, VAL1, 0, bits, False), (AGG_MIN, VAL1, 0, bits, True)]
    op = ReduceMonotonic(lanes)
    out, _ = op.step(rows32([(1, top, 0, 1), (1, 0, 0, 1)]), 1)
    neg = M64 ^ (top - 1)  # the top bit sign-extended
    assert tl(out) == [(1, (top, 0, 0, neg), 0, 1)]


def test_extremes():
    i64_min, u64_max = 1 << 63, M64
    lanes = [(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 64, False), (AGG_MAX, VAL1, 0, 64, True),
             (AGG_MIN, VAL1, 0, 64, False)]
    op = ReduceMonotonic(lanes)
    out, _ = op.step(rows32([(1, i64_min, 0, 1), (1, u64_max, 0, 1), (1, 5, 0, 1)]), 1)
    assert tl(out) == [(1, (i64_min, u64_max, 5, 5), 0, 1)]
    # the arrangement words: MIN of INT64_MIN encodes as all ones, MAX(u64::MAX) as all ones,
    # MAX(5) signed as 5 ^ 2^63, MIN(5) unsigned as ~5
    assert tl(op.export()) == [(1, 0, (M64, M64, 5 ^ (1 << 63), M64 ^ 5))]


def test_later_rows_that_do_not_change_the_extremum_are_silent():
    op = ReduceMonotonic([(AGG_MAX, VAL1, 0, 64, False), (AGG_MIN, VAL1, 0, 64, False)])
    op.step(rows32([(1, 5, 0, 1), (1, 1, 0, 1)]), 1)
    out, _ = op.step(rows32([(1, 3, 1, 1), (1, 4, 1, 2)]), 2)
    assert len(out) == 0
    out, _ = op.step(rows32([(1, 6, 2, 1)]), 3)
    assert tl(out) == [(1, (5, 1, 0, 0), 2, -1), (1, (6, 1, 0, 0), 2, 1)]


def test_compaction_merges_by_max():
    op = ReduceMonotonic([(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL2, 0, 8, False)], 40)
    op.step(rows40([(1, 5, 0x1ff, 0, 1), (2, -4, 3, 0, 1)]), 1)
    op.step(rows40([(1, -7, 2, 1, 1), (1, 9, 0x17, 1, 1)]), 2)
    assert len(op.export(0)) == 3
    (row1, row2) = tl(op.export(5))
    enc = op.encode
    assert row1 == (1, 5, tuple(enc([(-7) & M64, 0xff])))
    assert row2 == (2, 5, tuple(enc([(-4) & M64, 3])))


def test_sql_count_min_sum_max_through_one_operator():
    """aggregates.slt's count_min_sum_max (insert-only input): MIN(b) and MAX(b) as one two-lane operator."""
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "sqllogictest_join_reduce.json")))
    cases = {c["shape"]: c for c in fx["cases"]}
    t = fx["tables"]["t"]["rows"]
    op = ReduceMonotonic([(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 64, True)])
    out, errs = op.step(rows32([(a, b, 0, 1) for a, b in t]), 1)
    assert len(errs) == 0
    got = sorted((int(r["key"]), int(np.int64(r["vals"][0])), int(np.int64(r["vals"][1]))) for r in out)
    assert got == sorted((k, mn, mx) for k, _, mn, _, mx in cases["count_min_sum_max"]["expect"])


def test_row_widths_match_header_and_dtypes():
    from materialize_b200 import _ffi

    src = open(os.path.join(ROOT, "include", "mzgpu.h")).read()
    table = {4 if lanes == "1-4" else 8: (int(a), int(o))
             for lanes, a, o in re.findall(r"^\s*\*\s+(1-4|5-8)\s+(\d+) B:.*?(\d+) B:", src, re.M)}
    assert table == _ffi.MONO_ROW_BYTES == {4: (48, 56), 8: (112, 88)}
    for c, (arr_b, out_b) in table.items():
        assert (_ffi.RMONO[c].itemsize, _ffi.MONO_OUT[c].itemsize) == (arr_b, out_b)
        assert int(re.search(rf"#define MZGPU_ROW_RMONO{c} (\d+)", src).group(1)) == arr_b
        assert int(re.search(rf"#define MZGPU_ROW_MONO_OUT{c} (\d+)", src).group(1)) == out_b
    # every width means one thing
    used = {16, 32, 40, 64, 80, 128, 224, 416, 96, 144, 240}
    widths = [w for pair in table.values() for w in pair]
    assert not used & set(widths) and len(set(widths)) == 4
