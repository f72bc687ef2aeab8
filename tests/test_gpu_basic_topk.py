"""The basic TopK on the GPU, byte for byte against its restatement (tests/basic_topk_oracle.py): output, errors,
the input arrangement and the summed negatives over Zipf histories with retractions; wide keys, deep spines and
the error state; device input; both forms of the window kernel; agreement with the TopK and monotonic TopK
operators; the sqllogictest answers; and the creation and I/O errors."""
import ctypes as C
from collections import Counter, defaultdict

import numpy as np
import pytest

from basic_topk_oracle import NO_LIMIT, BasicTopKDefinition
from test_gpu_monotonic_topk import LANES, VAL1, r32_lanes, same, tuples, u, words, zipf_keys
from test_oracle_basic_topk import city_rows, golden

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
BOUND_ROWS = 48 << 20  # the single-pass form's output bound (rows of one activation)


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


class History:
    """Input batches with retractions: new rows (a third of them ties on small values), ~10 % retractions of
    earlier rows (a retracted row can go negative), ~1 % re-inserts that repair them, two times per batch."""

    def __init__(self, rng, r40, n_keys=3000, small_vals=False):
        self.rng, self.r40, self.n_keys, self.small = rng, r40, n_keys, small_vals
        self.pool = np.zeros((0, 3), dtype=np.uint64)

    def batch(self, mz, n, t, keys=None, retract=0.1, repair=0.01):
        rng, iw = self.rng, 5 if self.r40 else 4
        w = np.zeros((n, iw), dtype=np.uint64)
        w[:, 0] = zipf_keys(rng, n, self.n_keys) if keys is None else keys
        for c in range(1, iw - 2):
            if self.small:
                w[:, c] = rng.integers(0, 32, size=n, dtype=np.uint64)
            else:
                w[:, c] = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
                w[: n // 3, c] = rng.integers(0, 40, size=n // 3, dtype=np.uint64)
        d = rng.integers(1, 4, size=n).astype(np.int64)
        if len(self.pool) and n:
            for frac, sign in ((retract, -1), (repair, 1)):
                m = rng.random(n) < frac
                pick = self.pool[rng.integers(0, len(self.pool), size=int(m.sum()))]
                w[m, 0] = pick[:, 0]
                w[m, 1] = pick[:, 1]
                if self.r40:
                    w[m, 2] = pick[:, 2]
                d[m] = sign
        ins = d > 0
        new = np.zeros((int(ins.sum()), 3), dtype=np.uint64)
        new[:, 0], new[:, 1] = w[ins, 0], w[ins, 1]
        if self.r40:
            new[:, 2] = w[ins, 2]
        self.pool = np.concatenate([self.pool, new])
        w[:, iw - 2] = t + rng.integers(0, 2, size=n, dtype=np.uint64)
        w[:, iw - 1] = d.view(np.uint64)
        return w.view(mz.R40 if self.r40 else mz.R32).reshape(-1)


def out_words(rows, r40):
    return [(k, v1, v2, t, u(d)) if r40 else (k, v1, t, u(d)) for k, v1, v2, t, d in rows]


def err_words(errs):
    return [(k, z, t, u(d)) for k, z, t, d in errs]


def arr_words(rows):
    return [r[:7] + (u(r[7]), 0) for r in rows]


def summed_negatives(g):
    acc = Counter()
    for k, _, _, d in words(g.negatives_trace().export(), 4).tolist():
        acc[k] += int(np.uint64(d).astype(np.int64))
    return {k: c for k, c in acc.items() if c}


def make(mz, ctx, lanes, limit, offset, r40):
    return mz.TopKBasic(ctx, [mz.order_lane(s, sh, b, sx, d) for s, sh, b, sx, d in lanes], limit, offset,
                        40 if r40 else 32)


def check_step(g, o, rows, upper, r40):
    out, errs = g.step(rows, upper)
    want_out, want_errs = o.step(tuples(rows, r40))
    same(out, out_words(want_out, r40), 5 if r40 else 4)
    same(errs, err_words(want_errs), 4)
    return want_out, want_errs


@pytest.mark.parametrize("limit", [0, 1, 3, 40, NO_LIMIT])
@pytest.mark.parametrize("offset", [0, 2, 50])
@pytest.mark.parametrize("r40", [False, True])
def test_matches_restatement(mz, ctx, limit, offset, r40):
    """32 activations of Zipf(0.9) keys with retractions and logical compaction advancing: output, errors, the
    input arrangement and the summed negatives byte for byte; 0, 1 and 3 lanes by parameter."""
    n_lanes = (0, 1, 3)[(limit % 7 + offset) % 3]
    lanes = LANES[n_lanes] if r40 else r32_lanes(LANES[n_lanes])
    rng = np.random.default_rng(limit % 1000 * 31 + offset * 7 + r40)
    g = make(mz, ctx, lanes, limit, offset, r40)
    o = BasicTopKDefinition(lanes, limit, offset, 40 if r40 else 32)
    h = History(rng, r40)
    n_err = 0
    for a in range(32):
        t = 2 * a
        n = int(rng.choice([0, 60, 1500, 4000]))
        _, errs = check_step(g, o, h.batch(mz, n, t), t + 2, r40)
        n_err += len(errs)
        if a % 4 == 3:
            since = max(0, t - 6)
            g.input_trace().set_logical_compaction(since)
            same(g.input_trace().export(), arr_words(o.input_rows(since)), 9)
            assert summed_negatives(g) == o.negatives()
    assert n_err > 0
    ctx.sync()


def test_wide_keys_deep_spine_and_the_error_state(mz, ctx):
    """Eight keys with groups far wider than the window, no compaction (a deep spine), and keys that enter the
    error state, stay in it across activations and leave it."""
    lanes = r32_lanes(LANES[1])
    rng = np.random.default_rng(3)
    g = make(mz, ctx, lanes, 3, 2, False)
    o = BasicTopKDefinition(lanes, 3, 2)
    h = History(rng, False, n_keys=8)
    states = defaultdict(list)
    for a in range(40):
        keys = rng.integers(0, 8, size=3000, dtype=np.uint64)
        repair = a % 10 == 9
        rows = h.batch(mz, 3000, 2 * a, keys=keys, retract=0 if repair else 0.08, repair=0.04)
        if repair:  # every negative count repaired: the keys in the error state leave it
            fix = [(k, sk[3], 2 * a + 1, -c) for k, acc in o.acc.items() for sk, c in acc.items() if c < 0]
            rows = np.concatenate([rows, np.array(fix, dtype=mz.R32)])
        _, errs = check_step(g, o, rows, 2 * a + 2, False)
        for k, _, t, d in errs:
            states[k].append(d)
    assert summed_negatives(g) == o.negatives()
    assert sum(1 for v in states.values() if len(v) >= 3 and v[:3] == [1, -1, 1]) >= 2, states
    assert g.input_trace().size()["batches"] >= 2


def test_device_input_and_empty_batches(mz, ctx):
    lanes = LANES[3]
    rng = np.random.default_rng(4)
    g = make(mz, ctx, lanes, 3, 0, True)
    o = BasicTopKDefinition(lanes, 3, 0, 40)
    h = History(rng, True, n_keys=200)
    out, errs = mz.DeviceRows(ctx, 40), mz.DeviceRows(ctx, 32)
    want_out, want_errs = [], []
    for a in range(12):
        n = 0 if a % 3 == 1 else 2000
        rows = h.batch(mz, n, 2 * a)
        g.step_dev(mz.DeviceRows(ctx, 40).upload(rows), 2 * a + 2, out, errs)
        wo, we = o.step(tuples(rows, True))
        want_out += wo
        want_errs += we
    same(out.download(), out_words(want_out, True), 5)
    same(errs.download(), err_words(want_errs), 4)


@pytest.mark.parametrize("limit,n,two_pass", [(1000, 24_000, False), (1000, 26_000, True), (NO_LIMIT, 5000, True)])
def test_single_pass_bound_and_the_two_pass_form(mz, ctx, limit, n, two_pass):
    """2 * limit output rows per new row: under 48 Mi rows the look-back kernel runs, past it (and always
    without a limit) the two-pass kernels."""
    from test_gpu_monotonic import Trace

    assert (2 * limit * n > BOUND_ROWS or limit == NO_LIMIT) == two_pass
    lanes = r32_lanes(LANES[1])
    rng = np.random.default_rng(8)
    g = make(mz, ctx, lanes, limit, 2, False)
    o = BasicTopKDefinition(lanes, limit, 2)
    h = History(rng, False, n_keys=6)
    for a in range(3):
        rows = h.batch(mz, n, 2 * a, keys=rng.integers(0, 6, size=n, dtype=np.uint64))
        with Trace(ctx) as tr:
            check_step(g, o, rows, 2 * a + 2, False)
        assert tr.ran("k_topk_basic_explode"), tr.kernels
        assert tr.ran("k_topk_basic_lb") != two_pass and any(k.startswith("k_topk_basic<") for k in tr.kernels) == two_pass, tr.kernels
    g.input_trace().set_logical_compaction(6)
    same(g.input_trace().export(), arr_words(o.input_rows(6)), 9)


def test_agrees_with_topk_operator(mz, ctx):
    """One unsigned full-width lane over R32, windows of at most 32 distinct values, no negative counts: the
    accumulated window rows agree with mzgpu_topk_new's, whose output carries the value in sum_lo."""
    rng = np.random.default_rng(11)
    for limit, offset, desc in ((3, 0, True), (3, 2, False)):
        g = make(mz, ctx, [(VAL1, 0, 64, False, desc)], limit, offset, False)
        old = mz.TopK(ctx, limit, offset, desc)
        h = History(rng, False, n_keys=2000, small_vals=True)
        live = Counter()
        got, want = Counter(), Counter()
        for t in range(6):
            rows = h.batch(mz, 20_000, 2 * t, retract=0.1 if t else 0, repair=0)
            rows["time"] = 2 * t  # one time per batch, so that the array order below is the time order
            for r in rows:  # keep every count non-negative: a retraction of a row not live becomes an insert
                kv = (int(r["key"]), int(r["val"]))
                if live[kv] + int(r["diff"]) < 0:
                    r["diff"] = 1
                live[kv] += int(r["diff"])
            out, errs = g.step(rows, 2 * t + 2)
            assert len(errs) == 0
            for r in out:
                got[(int(r["key"]), int(r["val"]))] += int(r["diff"])
            for r in old.step(rows, 2 * t + 2):
                want[(int(r["key"]), int(r["sum_lo"]))] += int(r["diff"])
            assert {k: d for k, d in got.items() if d} == {k: d for k, d in want.items() if d}


@pytest.mark.parametrize("limit", [1, 3, NO_LIMIT])
def test_agrees_with_monotonic_topk(mz, ctx, limit):
    """Insert-only input, offset 0: the same changes as the monotonic operator."""
    rng = np.random.default_rng(12 + limit % 100)
    lanes = LANES[3]
    g = make(mz, ctx, lanes, limit, 0, True)
    m = mz.TopKMonotonic(ctx, [mz.order_lane(s, sh, b, sx, d) for s, sh, b, sx, d in lanes], limit, 40)
    h = History(rng, True, n_keys=500)
    for t in range(6):
        rows = h.batch(mz, 5000, 2 * t, retract=0, repair=0)
        out, errs = g.step(rows, 2 * t + 2)
        mout, _ = m.step(rows, 2 * t + 2)
        assert len(errs) == 0
        assert out.tobytes() == mout.tobytes()


def test_sqllogictest_answers(mz, ctx):
    fx = golden()
    for case in fx["per_group"]:
        rows, states, names = city_rows(fx, case)
        g = make(mz, ctx, [(VAL1, 0, 64, False, case["descending"])], case["limit"], 0, True)
        out, errs = g.step(np.array([(k, p, c, t, d) for k, p, c, t, d in rows], dtype=mz.R40), 1)
        assert len(errs) == 0 and (out["diff"] == 1).all()
        got = sorted((states[int(r["key"])], names[int(r["val2"])]) for r in out)
        assert got == sorted(tuple(x) for x in case["answer"]), case["name"]
    for case in fx["global"]:
        stages = [make(mz, ctx, [(VAL1, 0, 64, False, False)], s["limit"], s["offset"], False) for s in case["stages"]]
        final = Counter()

        def feed(vals, t, d):
            rows = np.array([(0, x, t, d) for x in vals], dtype=mz.R32)
            for st in stages:
                rows, errs = st.step(rows, t + 1)
                assert len(errs) == 0
            for r in rows:
                final[int(r["val"])] += int(r["diff"])
            return sorted(v for v, c in final.items() if c)

        assert feed(case["t"], 0, 1) == case["answer"], case["name"]
        assert feed(case["t"][:3], 1, -1) == [x + 3 for x in case["answer"]]
        assert feed(case["t"][:3], 2, 1) == case["answer"]
        assert feed([], 3, 1) == case["answer"]


def test_creation_and_io_errors_leave_the_context_usable(mz, ctx):
    from materialize_b200 import _ffi as F

    lane = mz.order_lane(VAL1)

    def new(order, limit=1, offset=0, irb=32, null_order=False):
        arr = (F.OrderLane * max(1, len(order)))()
        for i, (src, sh, b, sx, d, f64) in enumerate(order):
            arr[i].sign_extend, arr[i].descending, arr[i].flags = int(sx), int(d), F.ORDER_F64 if f64 else 0
            arr[i].field = F.Field(src, sh, b, 0)
        h = C.c_void_p(0)
        st = F.lib.mzgpu_topk_basic_new(ctx.h, irb, None if null_order else arr, len(order), limit, offset,
                                        C.byref(h))
        return st, h.value

    for order, irb, null_order in [
        ([lane], 48, False),
        ([lane] * 4, 32, False),
        ([mz.order_lane(2)], 32, False),
        ([mz.order_lane(VAL1, 60, 8)], 32, False),
        ([mz.order_lane(VAL1, 0, 0)], 32, False),
        ([lane], 32, True),
    ]:
        st, h = new(order, 1, 0, irb, null_order)
        assert st == E_INVALID and not h, (order, irb)
    for order, limit, offset in (([lane], -1, 0), ([mz.order_lane(VAL1, f64=True)], 1, 0),
                                 ([lane], 10, (1 << 63) - 10), ([lane], 1 << 62, 1 << 62)):
        st, h = new(order, limit, offset)
        assert st == E_UNSUPPORTED and not h, (order, limit, offset)
    st, h = new([lane], NO_LIMIT, (1 << 64) - 1)  # no limit: any offset
    assert st == 0 and h
    F.lib.mzgpu_reduce_free(h)
    st, h = new([lane], 9, (1 << 63) - 10)  # offset + limit == INT64_MAX
    assert st == 0 and h
    F.lib.mzgpu_reduce_free(h)

    g = make(mz, ctx, [], 1, 0, False)
    rows = np.array([(1, 2, 0, 1), (1, 1, 0, 1)], dtype=mz.R32)
    for ob, eb in ((40, 32), (32, 16), (32, 40)):
        out, errs = mz.DeviceRows(ctx, ob), mz.DeviceRows(ctx, eb)
        st = F.lib.mzgpu_topk_basic(g.h, rows.ctypes.data, len(rows), F.MEM_HOST, 1, out.h, errs.h)
        assert st == E_INVALID
    same_buf = mz.DeviceRows(ctx, 32)
    assert F.lib.mzgpu_topk_basic(g.h, rows.ctypes.data, len(rows), F.MEM_HOST, 1, same_buf.h, same_buf.h) == E_INVALID
    assert F.lib.mzgpu_topk_basic_buf(g.h, mz.DeviceRows(ctx, 40).h, 1, mz.DeviceRows(ctx, 32).h,
                                      mz.DeviceRows(ctx, 32).h) == E_INVALID
    out, errs = g.step(rows, 1)
    assert out.tolist() == [(1, 1, 0, 1)] and len(errs) == 0
