"""The multi-column accumulable reduce restated on the CPU (tests/lanes_oracle.py: build_accumulable
over several aggregates, one arrangement, one output row per key), pinned by its definition, by the
one-column kind of the oracle it generalizes, and by the reference-held sqllogictest answers; plus
the lane row layouts."""
import json
import os
import re

import numpy as np
import pytest
from lanes_oracle import ReduceLanes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64, M128 = (1 << 64) - 1, (1 << 128) - 1
I64, F64 = 0, 1
VAL1, VAL2 = 1, 2


def s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def pick(row_words, lane):
    kind, src, shift, bits, sx = lane
    w = (row_words[src] >> shift) & ((1 << bits) - 1)
    if kind == I64 and sx and bits < 64 and (w >> (bits - 1)) & 1:
        w |= M64 ^ ((1 << bits) - 1)
    return w


def f64_fixed(x):
    """(x * 2^24) as i128 with Rust's saturating cast (reduce.rs:1528)."""
    y = x * 16777216.0
    if y >= 2.0**127:
        return (1 << 127) - 1
    if y <= -(2.0**127):
        return -(1 << 127)
    return int(y)


def expected(rows, lanes, in_words, cls, tau):
    """GROUP BY key of the input rows with time <= tau: per lane (count, sum, flags), finalized as
    finalize_accum does; keys whose whole accumulation is zero have no row."""
    acc = {}
    for r in rows:
        w = [int(x) for x in r.tolist()]
        if w[in_words - 2] > tau:
            continue
        d = s64(w[in_words - 1])
        a = acc.setdefault(w[0], [0] + [[0, 0, 0, 0, 0] for _ in lanes])
        a[0] += d
        for l, lane in enumerate(lanes):
            v = pick(w, lane)
            x = a[1 + l]
            x[0] += d
            if lane[0] == F64:
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
    out = set()
    for k, a in acc.items():
        total = s64(a[0])
        lanes_w = [[s64(x[0]), x[1] & M128, s64(x[2]), s64(x[3]), s64(x[4])] for x in a[1:]]
        if total == 0 and all(x[0] == 0 and x[1] == 0 and x[2] == 0 and x[3] == 0 and x[4] == 0 for x in lanes_w):
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
        out.add((k, *vals, flags))
    return out


def accumulated(out_rows, cls, tau):
    """The output collection at tau: the corrections with time <= tau, summed per row."""
    acc = {}
    for r in out_rows:
        if int(r["time"]) > tau:
            continue
        key = (int(r["key"]),) + tuple(int(x) & M64 for l in range(cls) for x in r["lanes"][l].tolist()) + (int(r["flags"]),)
        acc[key] = acc.get(key, 0) + int(r["diff"])
    assert all(d in (0, 1) for d in acc.values()), "an output row with multiplicity other than 1"
    return {k for k, d in acc.items() if d == 1}


def activations(rng, lanes, in_words, steps=8, keys=40):
    """Activations with retractions, wrapping diffs, NaN / +-inf / 1e300 floats and i128 overflow."""
    dt = np.dtype([(f"w{i}", "<u8") for i in range(in_words)])
    live, t = [], 0
    for step in range(steps):
        n = int(rng.integers(1, 300))
        a = np.zeros(n, dtype=dt)
        a["w0"] = rng.integers(0, keys, size=n, dtype=np.uint64)
        for src in range(1, in_words - 2):
            words = rng.integers(0, 2**64, size=n, dtype=np.uint64)
            f = (rng.integers(-(10**9), 10**9, size=n).astype(np.float64) / 7.0).view(np.uint64)
            sp = rng.integers(0, 12, size=n)
            fl = f.view(np.float64).copy()
            fl[sp == 0], fl[sp == 1], fl[sp == 2], fl[sp == 3] = np.nan, np.inf, -np.inf, 1e300
            big = np.where(rng.random(n) < 0.5, np.uint64(2**63 - 1), np.uint64(2**63))  # i64 extremes: i128 overflow
            has_f64 = any(l[0] == F64 and l[1] == src for l in lanes)
            v = fl.view(np.uint64) if has_f64 else words
            if not has_f64:
                v = np.where(rng.random(n) < 0.2, big, v)
            a[f"w{src}"] = v
        a[f"w{in_words - 2}"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        d = rng.integers(1, 4, size=n).astype(np.int64)
        d[rng.random(n) < 0.05] = np.int64(2**62)  # diffs that wrap i64 when summed
        a[f"w{in_words - 1}"] = d.view(np.uint64)
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


LANE_SETS = {
    "r40_i64_f64": (40, [(I64, VAL1, 0, 64, False), (F64, VAL2, 0, 64, False)]),
    "r32_bitfields": (32, [(I64, VAL1, 0, 20, True), (I64, VAL1, 20, 20, False), (I64, VAL1, 40, 24, True)]),
    "r40_eight": (
        40,
        [(I64, VAL1, 0, 64, False), (F64, VAL2, 0, 64, False), (I64, VAL1, 3, 17, True), (I64, VAL1, 32, 32, False),
         (I64, VAL1, 63, 1, True), (I64, VAL1, 8, 40, False), (I64, VAL1, 0, 1, False), (I64, VAL1, 56, 8, True)],
    ),
}


@pytest.mark.parametrize("name", sorted(LANE_SETS))
def test_lanes_output_is_group_by_of_accumulated_input(oracle, name):
    in_rb, lanes = LANE_SETS[name]
    in_words = in_rb // 8
    r = ReduceLanes(oracle, lanes, in_rb)
    rng = np.random.default_rng(len(name))
    seen, outs = [], []
    for a, upper in activations(rng, lanes, in_words):
        seen.append(a)
        outs.append(r.step(a, upper))
        rows, out = np.concatenate(seen), np.concatenate(outs)
        for tau in range(upper - 3, upper):
            assert accumulated(out, r.cls, tau) == expected(rows, lanes, in_words, r.cls, tau), (name, tau)


@pytest.mark.parametrize("kind", [I64, F64])
def test_one_lane_equals_the_one_column_kind(oracle, kind):
    rng = np.random.default_rng(90 + kind)
    lanes = [(kind, VAL1, 0, 64, False)]
    r, old = ReduceLanes(oracle, lanes, 32), oracle.Reduce(kind)
    for a, upper in activations(rng, lanes, 4):
        a32 = a.view(oracle.R32)
        got, want = r.step(a32, upper), old.step(a32, upper)
        assert got.dtype.itemsize == want.dtype.itemsize == 64
        assert got.tobytes() == want.tobytes()


def test_fixture_cases_through_one_lanes_operator(oracle):
    """global_sums (two summed columns and an average) and the COUNT / SUM columns of
    count_min_sum_max, each through ONE operator, against the reference's printed answers."""
    fx = json.load(open(os.path.join(ROOT, "tests", "golden", "sqllogictest_join_reduce.json")))
    cases = {c["shape"]: c for c in fx["cases"]}
    t = fx["tables"]["t"]["rows"]
    rows = np.zeros(len(t), dtype=oracle.R40)
    rows["key"], rows["val1"], rows["val2"], rows["time"], rows["diff"] = 0, [a for a, _ in t], [b for _, b in t], 0, 1
    r = ReduceLanes(oracle, [(I64, VAL1, 0, 64, True), (I64, VAL2, 0, 64, True)], 40)
    (o,) = r.step(rows, 1)
    (ca, sa, _), (cb, sb, _) = (tuple(int(np.int64(x)) for x in o["lanes"][l].tolist()) for l in range(2))
    assert ca == cb == len(t) and int(o["flags"]) == 0 and int(o["diff"]) == 1
    assert [[1, sa, sb, sa / ca]] == cases["global_sums"]["expect"]

    g = np.zeros(len(t), dtype=oracle.R32)
    g["key"], g["val"], g["time"], g["diff"] = [a for a, _ in t], [b for _, b in t], 0, 1
    out = ReduceLanes(oracle, [(I64, VAL1, 0, 64, True)], 32).step(g, 1)
    got = sorted((int(o["key"]), int(o["lanes"][0]["count"]), int(np.int64(o["lanes"][0]["sum_lo"]))) for o in out)
    want = sorted((k, c, s) for k, c, _, s, _ in cases["count_min_sum_max"]["expect"])
    assert got == want


def test_lane_row_widths_match_header_and_dtypes():
    from materialize_b200 import _ffi

    src = open(os.path.join(ROOT, "include", "mzgpu.h")).read()
    table = {int(c): (int(a), int(o)) for c, a, o in re.findall(r"^\s*\*\s+([1248])\s+(\d+) B\b.*?(\d+) B\b", src, re.M)}
    assert table == _ffi.LANE_ROW_BYTES == {1: (80, 64), 2: (128, 96), 4: (224, 144), 8: (416, 240)}
    for c, (arr_b, out_b) in table.items():
        arr, out = _ffi.RACC_LANES[c], _ffi.ROUT_LANES[c]
        assert (arr.itemsize, out.itemsize) == (arr_b, out_b)
        assert arr_b == 16 * ((8 * (3 + 6 * c) + 15) // 16) and out_b >= 8 * (3 * c + 4) and out_b % 16 == 0
        assert arr.fields["lanes"][1] == 24 and out.fields["flags"][1] == 8 + 24 * c
        assert out.fields["time"][1] == 16 + 24 * c and out.fields["diff"][1] == 24 + 24 * c
        assert int(re.search(rf"#define MZGPU_ROW_RACC{c} (\d+)", src).group(1)) == arr_b if c > 1 else True
        assert int(re.search(rf"#define MZGPU_ROW_ROUT{c} (\d+)", src).group(1)) == out_b if c > 1 else True
    # every width means one thing: no output width is an arrangement width or another row width
    outs = {o for _, o in table.values()} - {64}
    assert not outs & ({a for a, _ in table.values()} | {16, 32, 40})
    # class 1 has the one-column rows' bytes
    assert _ffi.RACC_LANES[1].itemsize == _ffi.RACC.itemsize and _ffi.ROUT_LANES[1].itemsize == _ffi.ROUT.itemsize
    import ctypes as C

    assert C.sizeof(_ffi.AccumLane) == 12
