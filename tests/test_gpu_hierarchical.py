"""The hierarchical MIN / MAX reduce on the GPU, byte for byte against its CPU restatement
(tests/hierarchical_oracle.py) on the table and wide-key paths, both sides of the single-pass bound, agreement
with the one-column MIN / MAX operators and the monotonic operator, the SQL answers, the creation errors, and
the 40-byte arrangement rows against the plain arrangement reference."""
import json
import os

import numpy as np
import pytest

import arrangement_ref as ref
from hierarchical_oracle import ReduceHierarchical
from monotonic_oracle import AGG_MAX, AGG_MIN, M64, ReduceMonotonic

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
VAL1, VAL2 = 1, 2
E_INVALID, E_UNSUPPORTED = -1, -4


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


def same(got, want):
    assert got.dtype.itemsize == want.dtype.itemsize
    assert len(got) == len(want), (len(got), len(want))
    nw = want.dtype.itemsize // 8
    g, w = got.view(np.uint64).reshape(len(got), nw), want.view(np.uint64).reshape(len(want), nw)
    if g.tobytes() != w.tobytes():
        bad = int(np.flatnonzero(np.any(g != w, axis=1))[0])
        raise AssertionError(f"row {bad} of {len(w)}: got {g[bad].tolist()}, want {w[bad].tolist()}")


class Trace:
    def __init__(self, ctx):
        self.ctx = ctx

    def __enter__(self):
        self.ctx.profile(True)
        return self

    def __exit__(self, *exc):
        try:
            if exc[0] is None:
                self.kernels = {k.strip("()") for k in self.ctx.profile_report()}
        finally:
            self.ctx.profile(False)

    def ran(self, prefix):
        return any(k.startswith(prefix) for k in self.kernels)


LANES = {
    # MIN and MAX of the same field, signed and unsigned, narrow fields
    3: [(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 64, True), (AGG_MIN, VAL1, 0, 16, False)],
    8: [(AGG_MIN if l % 2 else AGG_MAX, VAL1, 8 * (l // 2), 64 - 8 * (l // 2), l % 3 == 0) for l in range(8)],
}


def r40_lanes(lanes):
    return [(k, VAL2 if i % 2 else VAL1, s, b, sx) for i, (k, _, s, b, sx) in enumerate(lanes)]


def gpu_op(mz, ctx, lanes, iw):
    return mz.ReduceHierarchical(ctx, [mz.accum_lane(k, s, sh, b, sx) for k, s, sh, b, sx in lanes], iw * 8)


def to_rows(mz, w, iw):
    w = np.ascontiguousarray(np.array(w, dtype=np.uint64).reshape(-1, iw))
    return w.view(mz.R40 if iw == 5 else mz.R32).reshape(-1)


class History:
    """Random updates with retractions: inserts (values drawn from a small pool per key, so values repeat),
    retractions of live rows (extrema included), retractions of rows never inserted (a negative count, repaired
    a few times later), at several times per activation."""

    def __init__(self, rng, iw, keys, pool=40):
        self.rng, self.iw, self.keys = rng, iw, keys
        self.pool = rng.integers(0, M64, size=(pool, iw - 3), dtype=np.uint64, endpoint=True)
        self.pool[:4] = np.array([0, M64, 1 << 63, (1 << 63) - 1], dtype=np.uint64)[:, None]
        self.live = []
        self.later = []

    def batch(self, n, lo, hi):
        rng, out = self.rng, [r for r in self.later if lo <= r[-2] < hi]
        self.later = [r for r in self.later if r[-2] >= hi]
        for _ in range(n):
            t = int(rng.integers(lo, hi))
            u = rng.random()
            if self.live and u < 0.35:
                r = self.live.pop(int(rng.integers(0, len(self.live))))
                out.append(r[:-2] + [t, M64])
            elif u < 0.40:
                k = int(rng.integers(0, self.keys))
                v = [int(x) for x in self.pool[int(rng.integers(0, len(self.pool)))]]
                out.append([k] + v + [t, M64])
                self.later.append([k] + v + [hi + int(rng.integers(0, 4)), 1])
            else:
                k = int(min(rng.zipf(1.3), self.keys) - 1)
                v = [int(x) for x in self.pool[int(rng.integers(0, len(self.pool)))]]
                r = [k] + v + [t, int(rng.integers(1, 3))]
                out.append(r)
                self.live.append(r)
        return out


@pytest.mark.parametrize("n_lanes", [3, 8])
@pytest.mark.parametrize("iw", [4, 5])
def test_matches_restatement(mz, ctx, n_lanes, iw):
    """Zipf keys with retractions, negative counts and repairs, three times per activation, logical compaction
    every fourth activation: corrections, errors and the arrangement byte for byte."""
    rng = np.random.default_rng(n_lanes * 10 + iw)
    lanes = r40_lanes(LANES[n_lanes]) if iw == 5 else LANES[n_lanes]
    g, o = gpu_op(mz, ctx, lanes, iw), ReduceHierarchical(lanes, iw * 8)
    h = History(rng, iw, 300)
    saw_err = 0
    for step in range(24):
        lo = 3 * step
        rows = to_rows(mz, h.batch(int(rng.choice([0, 5, 400, 3000])), lo, lo + 3), iw)
        out, errs = g.step(rows, lo + 3)
        want_out, want_errs = o.step(rows, lo + 3)
        same(out, want_out)
        same(errs, want_errs)
        saw_err |= len(errs) > 0
        if step % 4 == 3:
            since = max(0, lo - 5)
            g.input_trace().set_logical_compaction(since)
            got = g.input_trace().export()
            same(got, o.export(since).view(got.dtype).reshape(-1))
    assert saw_err
    ctx.sync()


def test_wide_keys_and_table_overflow(mz, ctx):
    """Keys with 31, 32 and 33 distinct live rows; a key that outgrows the 32-entry table while the new batch's
    times replay; the current extremum retracted; a key emptied and refilled; a deep spine merged under
    compaction."""
    lanes = [(AGG_MIN, VAL1, 0, 64, False), (AGG_MAX, VAL1, 0, 64, False), (AGG_MAX, VAL1, 0, 32, True)]
    g, o = gpu_op(mz, ctx, lanes, 4), ReduceHierarchical(lanes)
    rng = np.random.default_rng(9)

    def run(rows, upper):
        rows = to_rows(mz, rows, 4)
        a, b = g.step(rows, upper), o.step(rows, upper)
        same(a[0], b[0])
        same(a[1], b[1])

    run([[k, 1000 * k + v, 0, 1] for k, n in ((1, 31), (2, 32), (3, 33)) for v in range(n)], 1)
    # key 4: 30 prior values; 6 new ones over three times of one batch push it past the table
    run([[4, v, 1, 1] for v in range(30)], 2)
    run([[4, 100 + v, 2 + v % 3, 1] for v in range(6)] + [[4, 0, 3, M64]], 5)
    # retract every key's extremum, then empty key 1 and refill it
    run([[k, 1000 * k + n - 1, 5, M64] for k, n in ((1, 31), (2, 32), (3, 33))] + [[4, 105, 6, M64]], 7)
    run([[1, 1000 + v, 7, M64] for v in range(30)], 8)
    run([[1, 5, 9, 1], [1, 9, 9, 1]], 10)
    # a deep spine: many small batches, compaction lagging behind
    for t in range(10, 60):
        k = int(rng.integers(1, 5))
        run([[k, int(rng.integers(0, 2**64, dtype=np.uint64)), t, 1], [k, 1000 * k + int(rng.integers(0, 33)), t,
                                                                       1 if rng.random() < 0.6 else M64]], t + 1)
        if t % 7 == 0:
            g.input_trace().set_logical_compaction(t - 3)
    g.input_trace().set_logical_compaction(56)
    got = g.input_trace().export()
    same(got, o.export(56).view(got.dtype).reshape(-1))


def test_device_input_and_empty_batches(mz, ctx):
    lanes = r40_lanes(LANES[8])
    g, o = gpu_op(mz, ctx, lanes, 5), ReduceHierarchical(lanes, 40)
    h = History(np.random.default_rng(4), 5, 50)
    out, errs = mz.DeviceRows(ctx, 88), mz.DeviceRows(ctx, 32)
    want_o, want_e = [], []
    for step in range(8):
        rows = to_rows(mz, h.batch(0 if step in (2, 5) else 500, 2 * step, 2 * step + 2), 5)
        g.step_dev(mz.DeviceRows(ctx, 40).upload(rows), 2 * step + 2, out, errs)
        a, b = o.step(rows, 2 * step + 2)
        want_o.append(a)
        want_e.append(b)
    same(out.download(), np.concatenate(want_o))
    same(errs.download(), np.concatenate(want_e))
    a, b = g.step(to_rows(mz, [], 5), 100)
    assert len(a) == 0 and len(b) == 0


def big_batch(mz, n_keys, extra):
    """n_keys keys with two inserts each (MAX of an unsigned word), then `extra` rows of keys above them."""
    rng = np.random.default_rng(n_keys)
    w = np.zeros((2 * n_keys, 4), dtype=np.uint64)
    w[:, 0] = np.repeat(np.arange(n_keys, dtype=np.uint64), 2)
    w[:, 1] = rng.integers(0, M64, size=2 * n_keys, dtype=np.uint64, endpoint=True)
    w[:, 3] = 1
    want = np.zeros((n_keys, 4), dtype=np.uint64)
    want[:, 0] = np.arange(n_keys, dtype=np.uint64)
    want[:, 1] = np.maximum(w[0::2, 1], w[1::2, 1])
    want[:, 3] = 1
    return w, want, [[n_keys + k, v, 0, d] for k, v, d in extra]


@pytest.mark.parametrize("two_pass", [False, True])
def test_both_sides_of_the_single_pass_bound(mz, ctx, two_pass):
    """A batch past MZ_BOUND_MAX_ROWS / 2 rows takes the two-pass form and gives the same rows."""
    lanes = [(AGG_MAX, VAL1, 0, 64, False)]
    n_keys = (25_165_824 // 2) + (8 if two_pass else -8)
    extra = [(0, 5, 1), (0, 7, 1), (1, 3, M64), (2, 4, M64), (2, 4, 1), (3, 9, 1), (3, 9, M64)]
    w, want, tail = big_batch(mz, n_keys, extra)
    o = ReduceHierarchical(lanes)
    tail_out, tail_err = o.step(to_rows(mz, tail, 4), 1)
    g = gpu_op(mz, ctx, lanes, 4)
    with Trace(ctx) as t:
        out, errs = g.step(to_rows(mz, np.concatenate([w, np.array(tail, dtype=np.uint64).reshape(-1, 4)]), 4), 1)
    assert t.ran("k_hier_corrections<") == two_pass and t.ran("k_hier_corrections_lb") != two_pass, t.kernels
    wo = np.zeros((n_keys, 7), dtype=np.uint64)
    wo[:, 0], wo[:, 1], wo[:, 6] = want[:, 0], want[:, 1], 1
    same(out, np.concatenate([wo.view(out.dtype).reshape(-1), tail_out]))
    same(errs, tail_err)
    ctx.sync()


def test_operator_kernels_by_name(mz, ctx):
    """an activation runs the mask and the single-pass corrections kernel"""
    g = gpu_op(mz, ctx, [(AGG_MAX, VAL1, 0, 64, False)], 4)
    with Trace(ctx) as t:
        g.step(to_rows(mz, [[k % 100, k, 0, 1] for k in range(5000)], 4), 1)
    assert t.ran("k_monotonic_mask") and t.ran("k_hier_corrections_lb"), t.kernels


@pytest.mark.parametrize("kind", [AGG_MIN, AGG_MAX])
def test_agrees_with_one_column_operators(mz, ctx, kind):
    """Two unsigned full-word lanes over R40 input against two one-column MIN / MAX operators fed the projections
    (key, val1) and (key, val2): value for value, wide groups included, no errors without negative counts."""
    rng = np.random.default_rng(kind + 40)
    lanes = [(kind, VAL1, 0, 64, False), (kind, VAL2, 0, 64, False)]
    g = gpu_op(mz, ctx, lanes, 5)
    ones = [mz.ReduceAccumulable(ctx, kind) for _ in range(2)]
    got, want = {}, [{}, {}]
    live = []
    for t in range(10):
        rows = []
        for _ in range(4000):
            if live and rng.random() < 0.3:
                r = live.pop(int(rng.integers(0, len(live))))
                rows.append(r[:3] + [t, M64])
            else:
                r = [int(min(rng.zipf(1.2), 200)), int(rng.integers(0, 2**64, dtype=np.uint64)),
                     int(rng.integers(0, 64)), t, 1]
                rows.append(r)
                live.append(r)
        rows = to_rows(mz, rows, 5)
        out, errs = g.step(rows, t + 1)
        assert len(errs) == 0
        for r in out:
            k = (int(r["key"]), int(r["vals"][0]), int(r["vals"][1]))
            got[k] = got.get(k, 0) + int(r["diff"])
        for l, op in enumerate(ones):
            p = np.zeros(len(rows), dtype=mz.R32)
            p["key"], p["val"], p["time"], p["diff"] = rows["key"], rows["val1" if l == 0 else "val2"], t, rows["diff"]
            for r in op.step(p, t + 1):
                assert int(r["flags"]) == 0
                want[l][int(r["key"])] = want[l].get(int(r["key"]), 0) + int(r["diff"]) * (int(r["sum_lo"]) + 1)
        cur = {k[0]: (k[1], k[2]) for k, d in got.items() if d}
        assert len(cur) == sum(1 for d in got.values() if d)
        for l in range(2):
            assert {k: v[l] + 1 for k, v in cur.items()} == {k: s for k, s in want[l].items() if s}
    assert max(np.bincount([r[0] for r in live])) > 32


def test_agrees_with_monotonic_on_insert_only_input(mz, ctx):
    rng = np.random.default_rng(8)
    lanes = r40_lanes(LANES[3])
    g, m = gpu_op(mz, ctx, lanes, 5), mz.ReduceMonotonic(ctx, [mz.accum_lane(*l) for l in lanes], 40)
    for t in range(6):
        w = np.zeros((20_000, 5), dtype=np.uint64)
        w[:, 0] = rng.integers(0, 3000, size=len(w))
        w[:, 1:3] = rng.integers(0, M64, size=(len(w), 2), dtype=np.uint64, endpoint=True)
        w[:, 3], w[:, 4] = t, rng.integers(1, 3, size=len(w))
        rows = to_rows(mz, w, 5)
        (a, ea), (b, eb) = g.step(rows, t + 1), m.step(rows, t + 1)
        same(a, b)
        assert len(ea) == len(eb) == 0


def test_sql_count_min_sum_max_zipped_with_lanes(mz, ctx):
    fx = json.load(open(os.path.join(HERE, "golden", "sqllogictest_join_reduce.json")))
    cases = {c["shape"]: c for c in fx["cases"]}
    t = fx["tables"]["t"]["rows"]
    rows = np.zeros(len(t), dtype=mz.R32)
    rows["key"], rows["val"], rows["time"], rows["diff"] = [a for a, _ in t], [b for _, b in t], 0, 1
    mm, errs = gpu_op(mz, ctx, [(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 64, True)], 4).step(rows, 1)
    cs = mz.ReduceLanes(ctx, [mz.accum_lane(mz.AGG_COUNT_SUM_I64, VAL1, sign_extend=True)]).step(rows, 1)
    a = {int(r["key"]): (int(np.int64(r["vals"][0])), int(np.int64(r["vals"][1]))) for r in mm}
    b = {int(r["key"]): (int(r["lanes"][0]["count"]), int(np.int64(r["lanes"][0]["sum_lo"]))) for r in cs}
    assert len(errs) == 0 and a.keys() == b.keys()
    got = sorted((k, b[k][0], a[k][0], b[k][1], a[k][1]) for k in a)
    assert got == sorted(tuple(r) for r in cases["count_min_sum_max"]["expect"])


def test_creation_errors_leave_the_context_usable(mz, ctx):
    lane = mz.accum_lane(AGG_MAX, VAL1)
    bad = [
        ([], 32),
        ([lane] * 9, 32),
        ([mz.accum_lane(mz.AGG_COUNT_SUM_I64, VAL1)], 32),
        ([mz.accum_lane(AGG_MAX | mz.ACCUM_DISTINCT, VAL1)], 32),
        ([mz.accum_lane(AGG_MAX, VAL2)], 32),
        ([mz.accum_lane(AGG_MAX, VAL1, 60, 8)], 32),
        ([mz.accum_lane(AGG_MAX, VAL1, 0, 0)], 32),
        ([lane], 48),
        ([mz.accum_lane(AGG_MIN | mz.MONO_F64, VAL1), mz.accum_lane(0, VAL1)], 32),
    ]
    for lanes, irb in bad:
        with pytest.raises(mz.MzGpuError) as e:
            mz.ReduceHierarchical(ctx, lanes, irb)
        assert e.value.status == E_INVALID, (lanes, irb)
    for lanes in ([mz.accum_lane(AGG_MIN | mz.MONO_F64, VAL1)], [lane, mz.accum_lane(AGG_MAX | mz.MONO_F64, VAL1)]):
        with pytest.raises(mz.MzGpuError) as e:
            mz.ReduceHierarchical(ctx, lanes)
        assert e.value.status == E_UNSUPPORTED
    out, errs = mz.ReduceHierarchical(ctx, [lane]).step(np.array([(1, 2, 0, 1), (3, 4, 0, -1)], dtype=mz.R32), 1)
    assert [r[:1] + r[-2:] for r in (tuple(int(x) for x in w) for w in out.view(np.uint64).reshape(-1, 7))] == [
        (1, 0, 1)]
    assert errs.tolist() == [(3, 0, 0, 1)]


def test_r40_spine_builds_merges_and_exports(mz, ctx):
    """40-byte rows as an arrangement: batch build, merge under compaction, spine export against the plain
    consolidation of tests/arrangement_ref.py."""
    rng = np.random.default_rng(40)

    def gen(n, t0, t1):
        w = np.zeros((n, 5), dtype=np.uint64)
        w[:, 0] = rng.integers(0, 2000, size=n)
        w[:, 1] = rng.integers(0, 8, size=n)
        w[:, 2] = rng.integers(0, 4, size=n)
        w[:, 3] = rng.integers(t0, t1, size=n)
        w[:, 4] = rng.choice(np.array([1, 2, M64], dtype=np.uint64), size=n)
        return w

    for n in (3000, 300_000):
        a, b = gen(n, 0, 10), gen(n, 10, 20)
        ba, bb = mz.Batch.build(ctx, to_rows(mz, a, 5), 0, 10), mz.Batch.build(ctx, to_rows(mz, b, 5), 10, 20)
        assert ref.words(ba.rows(), 40).tobytes() == ref.consolidate(a).tobytes()
        for since in (0, 15):
            m = ba.merge(bb, since)
            assert ref.words(m.rows(), 40).tobytes() == ref.merge(a, b, since).tobytes()
        s = mz.Spine(ctx, 40)
        s.insert(ba)
        s.insert(bb)
        s.set_logical_compaction(12)
        assert ref.words(s.export(), 40).tobytes() == ref.merge(a, b, 12).tobytes()
