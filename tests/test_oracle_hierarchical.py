"""The hierarchical MIN / MAX reduce's CPU restatement (tests/hierarchical_oracle.py): pinned against the
per-key definition at every time, against the independent oracle's one-column MIN / MAX reduce, against the
monotonic restatement on insert-only input, against hand-written cases and against the reference's printed
SQL answers; plus the header's row widths."""
import json
import os
import re

import numpy as np
import pytest

from hierarchical_oracle import ReduceHierarchical, key_value, masks
from monotonic_oracle import AGG_MAX, AGG_MIN, M64, ReduceMonotonic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAL1, VAL2 = 1, 2
R32 = np.dtype([("key", "<u8"), ("val", "<u8"), ("time", "<u8"), ("diff", "<i8")])
R40 = np.dtype([("key", "<u8"), ("val1", "<u8"), ("val2", "<u8"), ("time", "<u8"), ("diff", "<i8")])


def rows_of(tuples, iw):
    a = np.zeros(len(tuples), dtype=R32 if iw == 4 else R40)
    if len(tuples):
        a.view(np.uint64).reshape(len(tuples), iw)[:] = np.array([[x & M64 for x in t] for t in tuples],
                                                                  dtype=np.uint64)
    return a


def random_lanes(rng, n, r40):
    lanes = []
    for _ in range(n):
        bits = int(rng.choice([1, 8, 16, 32, 63, 64]))
        shift = int(rng.integers(0, 64 - bits + 1))
        lanes.append((int(rng.choice([AGG_MIN, AGG_MAX])), int(rng.choice([VAL1, VAL2])) if r40 else VAL1, shift, bits,
                      bool(rng.integers(0, 2))))
    return lanes


def random_history(rng, iw, times, keys=12, per_time=30, negatives=True):
    """(key, val1[, val2], time, diff) tuples: inserts, retractions of earlier rows, and (if asked) retractions
    of rows never inserted, which drive counts negative until a later insert repairs them"""
    hist, live = [], []
    for t in range(times):
        for _ in range(per_time):
            u = rng.random()
            if live and u < 0.35:
                r = live.pop(int(rng.integers(0, len(live))))
                hist.append(r[:-2] + (t, -1))
            elif negatives and u < 0.45:
                v = tuple(int(x) for x in rng.integers(0, 2**64, size=iw - 3, dtype=np.uint64))
                hist.append((int(rng.integers(0, keys)),) + v + (t, -1))
                hist.append((hist[-1][0],) + v + (t + int(rng.integers(1, 4)), 1))  # the repair, later
            else:
                if rng.random() < 0.5 and live:  # a value some key already holds
                    v = live[int(rng.integers(0, len(live)))][1:-2]
                else:
                    v = tuple(int(x) for x in rng.choice([0, 1, 2**63, M64, int(rng.integers(0, 2**63))],
                                                          size=iw - 3))
                r = (int(rng.integers(0, keys)),) + v + (t, int(rng.integers(1, 3)))
                hist.append(r)
                live.append(r)
    return hist


def accumulate_upto(out, errs, t, n_lanes):
    coll, err = {}, {}
    for r in out:
        if int(r["time"]) <= t:
            k = (int(r["key"]), tuple(int(x) for x in r["vals"][:n_lanes]))
            coll[k] = coll.get(k, 0) + int(r["diff"])
    for r in errs:
        if int(r["time"]) <= t:
            err[int(r["key"])] = err.get(int(r["key"]), 0) + int(r["diff"])
    got = {}
    for (k, v), d in coll.items():
        if d == 0:
            continue
        assert d == 1 and k not in got, (k, v, d)
        got[k] = v
    assert all(d in (0, 1) for d in err.values()), err
    return got, {k for k, d in err.items() if d == 1}


def definition(lanes, iw, hist, t):
    m = masks(lanes)
    mask = (m[1], m[2])[: iw - 3]
    live = {}
    for r in hist:
        if r[-2] <= t:
            v = tuple(x & mm for x, mm in zip(r[1:-2], mask))
            live.setdefault(r[0], {})
            live[r[0]][v] = live[r[0]].get(v, 0) + r[-1]
    rows, errs = {}, set()
    for k, l in live.items():
        res = key_value(lanes, l, k)
        if res is not None and res[0] == "row":
            rows[k] = res[1]
        elif res is not None:
            errs.add(k)
    return rows, errs


@pytest.mark.parametrize("seed", range(8))
def test_definition_at_every_time(seed):
    """At every time the accumulated output is, per key, every lane's MIN / MAX over the live masked rows while
    every count is positive, and the accumulated errors are exactly the keys with a negative count."""
    rng = np.random.default_rng(seed)
    iw = 5 if seed % 2 else 4
    n = 1 + seed % 8
    lanes = random_lanes(rng, n, iw == 5)
    hist = random_history(rng, iw, 10)
    op = ReduceHierarchical(lanes, iw * 8)
    outs, errs = [], []
    for lo in range(0, 14, 2):  # two times per activation, rows of later times held back
        o, e = op.step(rows_of([r for r in hist if lo <= r[-2] < lo + 2], iw), lo + 2)
        outs.append(o)
        errs.append(e)
        keys = [tuple(int(x) for x in r.tolist()[:-1]) for r in o.view(np.uint64).reshape(len(o), o.dtype.itemsize // 8)]
        assert keys == sorted(keys) and len(set(keys)) == len(keys)
        assert all(int(x["diff"]) != 0 for x in o) and all(int(x["val"]) == 0 for x in e)
    out, err = np.concatenate(outs), np.concatenate(errs)
    assert any(int(x["diff"]) == -1 for x in err), "the history should repair a negative count"
    for t in range(14):
        assert accumulate_upto(out, err, t, n) == definition(lanes, iw, hist, t), t


def test_one_unsigned_lane_equals_the_one_column_min_max(oracle):
    """One unsigned full-word VAL1 lane over R32 input is value for value the oracle's MIN / MAX (which is
    pinned to the reference), including keys with more than 32 live values; with negative counts the keys in
    the error state are exactly those whose one-column output row carries the error flag."""
    rng = np.random.default_rng(11)
    for negatives in (False, True):
        for kind in (AGG_MIN, AGG_MAX):
            hist = random_history(rng, 4, 8, keys=6, per_time=60, negatives=negatives)
            op = ReduceHierarchical([(kind, VAL1, 0, 64, False)])
            old = oracle.Reduce(kind)
            got, want, gerr, werr = {}, {}, {}, {}
            saw_errors = False
            for t in range(12):
                o, e = op.step(rows_of([r for r in hist if r[-2] == t], 4), t + 1)
                saw_errors = saw_errors or len(e) > 0
                for r in o:
                    k = (int(r["key"]), int(r["vals"][0]))
                    got[k] = got.get(k, 0) + int(r["diff"])
                for r in e:
                    gerr[int(r["key"])] = gerr.get(int(r["key"]), 0) + int(r["diff"])
                for r in old.step(rows_of([r for r in hist if r[-2] == t], 4).view(oracle.R32), t + 1):
                    if int(r["flags"]) & 2:
                        werr[int(r["key"])] = werr.get(int(r["key"]), 0) + int(r["diff"])
                    else:
                        k = (int(r["key"]), int(r["sum_lo"]))
                        want[k] = want.get(k, 0) + int(r["diff"])
                clean = lambda d: {k: v for k, v in d.items() if v != 0}
                assert clean(got) == clean(want) and clean(gerr) == clean(werr), (negatives, kind, t)
            assert max(sum(1 for r in hist if r[0] == k) for k in range(6)) > 32
            assert saw_errors == negatives


@pytest.mark.parametrize("iw", [4, 5])
def test_insert_only_equals_the_monotonic_restatement(iw):
    rng = np.random.default_rng(3 + iw)
    lanes = random_lanes(rng, 6, iw == 5)
    hier, mono = ReduceHierarchical(lanes, iw * 8), ReduceMonotonic(lanes, iw * 8)
    for t in range(6):
        rows = rows_of([(int(rng.integers(0, 30)),) + tuple(int(x) for x in rng.integers(0, 2**64, size=iw - 3,
                                                                                          dtype=np.uint64))
                        + (t, int(rng.integers(1, 3))) for _ in range(80)], iw)
        (a, ea), (b, eb) = hier.step(rows, t + 1), mono.step(rows, t + 1)
        assert a.tobytes() == b.tobytes() and len(ea) == len(eb) == 0


def test_rows_that_differ_in_unread_bits_cancel():
    lanes = [(AGG_MAX, VAL1, 0, 8, False)]
    op = ReduceHierarchical(lanes)
    out, errs = op.step(rows_of([(1, 0x105, 0, 1), (1, 0x205, 0, -1), (2, 0x7, 0, 1)], 4), 1)
    assert [(int(r["key"]), int(r["vals"][0]), int(r["diff"])) for r in out] == [(2, 7, 1)] and len(errs) == 0
    assert op.export().tolist() == [[2, 7, 0, 1]]
    # the same pair at different times: +1 at 1 (MAX 5), gone at 2
    out, errs = op.step(rows_of([(1, 0x105, 1, 1), (1, 0x205, 2, -1)], 4), 3)
    assert [(int(r["key"]), int(r["vals"][0]), int(r["time"]), int(r["diff"])) for r in out] == [(1, 5, 1, 1),
                                                                                                 (1, 5, 2, -1)]


def test_retracting_the_extremum_and_repairing_a_negative_count():
    lanes = [(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 64, True)]
    op = ReduceHierarchical(lanes)
    out, errs = op.step(rows_of([(1, -3, 0, 1), (1, 4, 0, 1), (1, 9, 0, 1)], 4), 1)
    assert [tuple(int(np.int64(x)) for x in r["vals"][:2]) for r in out] == [(-3, 9)]
    out, errs = op.step(rows_of([(1, 9, 1, -1), (1, 7, 2, -1)], 4), 3)
    assert [(tuple(int(np.int64(x)) for x in r["vals"][:2]), int(r["time"]), int(r["diff"])) for r in out] == [
        ((-3, 4), 1, 1), ((-3, 4), 2, -1), ((-3, 9), 1, -1)]
    assert [(int(r["key"]), int(r["time"]), int(r["diff"])) for r in errs] == [(1, 2, 1)]
    out, errs = op.step(rows_of([(1, 7, 3, 1)], 4), 4)
    assert [(tuple(int(np.int64(x)) for x in r["vals"][:2]), int(r["diff"])) for r in out] == [((-3, 4), 1)]
    assert [(int(r["key"]), int(r["time"]), int(r["diff"])) for r in errs] == [(1, 3, -1)]


def test_sql_count_min_sum_max_zipped_with_the_lanes(oracle):
    """aggregates.slt's count_min_sum_max: MIN(b) and MAX(b) from this restatement, zipped by key with COUNT(b)
    and SUM(b) from the lanes restatement, against the reference's printed answers."""
    from lanes_oracle import ReduceLanes

    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "sqllogictest_join_reduce.json")))
    cases = {c["shape"]: c for c in fx["cases"]}
    t = fx["tables"]["t"]["rows"]
    rows = rows_of([(a, b, 0, 1) for a, b in t], 4)
    mm, errs = ReduceHierarchical([(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 64, True)]).step(rows, 1)
    cs = ReduceLanes(oracle, [(0, VAL1, 0, 64, True)], 32).step(rows.view(oracle.R32), 1)
    a = {int(r["key"]): (int(np.int64(r["vals"][0])), int(np.int64(r["vals"][1]))) for r in mm}
    b = {int(r["key"]): (int(r["lanes"][0]["count"]), int(np.int64(r["lanes"][0]["sum_lo"]))) for r in cs}
    assert len(errs) == 0 and a.keys() == b.keys()
    got = sorted((k, b[k][0], a[k][0], b[k][1], a[k][1]) for k in a)
    assert got == sorted(tuple(r) for r in cases["count_min_sum_max"]["expect"])


def test_row_widths_match_header():
    from materialize_b200 import _ffi

    src = open(os.path.join(ROOT, "include", "mzgpu.h")).read()
    sec = src[src.index("---- hierarchical MIN / MAX reduce"):]
    assert "MZGPU_ROW_MONO_OUT4 (56 B, 1-4 lanes)" in sec and "MZGPU_ROW_MONO_OUT8 (88 B, 5-8 lanes)" in sec
    assert {c: _ffi.MONO_OUT[c].itemsize for c in (4, 8)} == {4: 56, 8: 88}
    for c in (4, 8):
        assert int(re.search(rf"#define MZGPU_ROW_MONO_OUT{c} (\d+)", src).group(1)) == _ffi.MONO_OUT[c].itemsize
    assert ReduceHierarchical([(AGG_MIN, VAL1, 0, 64, False)] * 5, 40).out_dtype.itemsize == 88
    assert ReduceHierarchical([(AGG_MIN, VAL1, 0, 64, False)] * 4).out_dtype.itemsize == 56
