"""The monotonic TopK on the GPU, byte for byte against its definition (tests/monotonic_topk_oracle.py):
output, errors and the window arrangement; the 72-byte window rows on every kernel path against a plain
reference of their SUM arithmetic; agreement with the TopK operator; the testdrive answers; and the
creation errors."""
import ctypes as C
import itertools
import json
import os
from collections import Counter

import numpy as np
import pytest

from monotonic_topk_oracle import M64, NO_LIMIT, TopKDefinition

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


def words(a, nw):
    return np.ascontiguousarray(a).view(np.uint64).reshape(-1, nw)


def same(got, want, nw):
    g = words(got, nw)
    w = np.asarray(want, dtype=np.uint64).reshape(-1, nw)
    assert g.shape == w.shape, (g.shape, w.shape)
    if g.tobytes() != w.tobytes():
        bad = int(np.flatnonzero(np.any(g != w, axis=1))[0])
        raise AssertionError(f"row {bad} of {len(w)}: got {g[bad].tolist()}, want {w[bad].tolist()}")


def u(x):
    return x & M64


def zipf_keys(rng, n, nk, s=0.9):
    p = 1.0 / np.arange(1, nk + 1) ** s
    return rng.choice(nk, size=n, p=p / p.sum()).astype(np.uint64)


def gen_rows(mz, rng, n, r40, t, keys, neg=True, small_vals=False):
    iw = 5 if r40 else 4
    w = np.zeros((n, iw), dtype=np.uint64)
    w[:, 0] = keys
    for c in range(1, iw - 2):
        if small_vals:
            w[:, c] = rng.integers(0, 32, size=n, dtype=np.uint64)  # the TopK operator takes <= 32 values per key
        else:
            w[:, c] = rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True)
            w[: n // 3, c] = rng.integers(0, 40, size=n // 3, dtype=np.uint64)  # ties and repeats
    w[:, iw - 2] = t + rng.integers(0, 2, size=n, dtype=np.uint64)  # two times per activation
    d = rng.choice([1, 1, 1, 1, 2, 3, 7, 0, -1], size=n) if neg else rng.integers(1, 4, size=n)
    w[:, iw - 1] = d.astype(np.int64).view(np.uint64)
    return w.view(mz.R40 if r40 else mz.R32).reshape(-1)


def tuples(rows, r40):
    w = words(rows, 5 if r40 else 4)
    if r40:
        return [(int(a), int(b), int(c), int(t), int(np.int64(np.uint64(d)))) for a, b, c, t, d in w]
    return [(int(a), int(b), 0, int(t), int(np.int64(np.uint64(d)))) for a, b, t, d in w]


def out_words(out, r40):
    return [(k, v1, v2, t, u(d)) if r40 else (k, v1, t, u(d)) for k, v1, v2, t, d in out]


def window_words(rows):
    return [r[:7] + (u(r[7]), 0) for r in rows]


LANES = {
    0: [],
    1: [(VAL1, 0, 64, False, True)],  # ORDER BY val1 DESC: latest per key
    3: [(VAL1, 0, 4, False, False), (VAL2, 0, 64, True, True), (VAL1, 4, 60, True, False)],
}


def make(mz, ctx, lanes, limit, r40, must):
    return mz.TopKMonotonic(ctx, [mz.order_lane(s, sh, b, sx, d) for s, sh, b, sx, d in lanes], limit,
                            40 if r40 else 32, must)


def r32_lanes(lanes):
    return [(VAL1,) + lane[1:] for lane in lanes]


@pytest.mark.parametrize("limit", [0, 1, 3, 40, NO_LIMIT])
@pytest.mark.parametrize("n_lanes", [0, 1, 3])
@pytest.mark.parametrize("r40", [False, True])
def test_matches_definition(mz, ctx, limit, n_lanes, r40):
    """Zipf(0.9) keys over 32 activations with logical compaction advancing: output, errors and the window
    arrangement byte for byte."""
    must = (n_lanes + r40) % 2 == 1
    lanes = LANES[n_lanes] if r40 else r32_lanes(LANES[n_lanes])
    rng = np.random.default_rng(limit % 1000 * 31 + n_lanes * 3 + r40)
    g = make(mz, ctx, lanes, limit, r40, must)
    o = TopKDefinition(lanes, limit, 40 if r40 else 32, must)
    for a in range(32):
        t = 2 * a
        n = int(rng.choice([1, 60, 1500, 6000]))
        rows = gen_rows(mz, rng, n, r40, t, zipf_keys(rng, n, 3000))
        if must and n > 10:  # +1 / -1 pairs that cancel, and pairs that leave -1
            rows[n // 2 : n // 2 + 5] = rows[:5]
            rows[:5]["diff"] = 1
            rows[n // 2 : n // 2 + 5]["diff"] = -1
        out, errs = g.step(rows, t + 2)
        want_out, want_errs = o.step(tuples(rows, r40))
        same(out, out_words(want_out, r40), 5 if r40 else 4)
        same(errs, [(tt, c) for tt, c in want_errs], 2)
        if a % 4 == 3:
            since = max(0, t - 6)
            g.input_trace().set_logical_compaction(since)
            same(g.input_trace().export(), window_words(o.window(since)), 9)
    ctx.sync()


@pytest.mark.parametrize("limit", [1, 3])
def test_compacted_window_is_the_live_window(mz, ctx, limit):
    lanes = r32_lanes(LANES[1])
    rng = np.random.default_rng(100 + limit)
    g = make(mz, ctx, lanes, limit, False, False)
    o = TopKDefinition(lanes, limit)
    for t in range(24):
        rows = gen_rows(mz, rng, 20_000, False, 2 * t, zipf_keys(rng, 20_000, 2000), neg=False)
        g.step(rows, 2 * t + 2)
        o.step(tuples(rows, False))
        g.input_trace().set_logical_compaction(2 * t + 2)
    # idle timestamps: each inserts an empty batch, which fuels the spine's merges
    tr, upper = g.input_trace(), 48
    want = o.window()
    for _ in range(64):
        if tr.size()["updates"] == len(want):
            break
        upper += 1
        g.step(np.zeros(0, dtype=mz.R32), upper)
        tr.set_logical_compaction(upper)
        tr.exert(1 << 40)
    same(tr.export(), window_words(o.window(upper)), 9)
    assert max(Counter(r[0] for r in want).values()) <= limit
    assert tr.size()["updates"] == len(want), (tr.size(), len(want))


def test_wide_window_and_the_two_pass_form(mz, ctx):
    """LIMIT 1000 on a few wide keys, and a batch past the single-pass bound (1001 rows per new row beyond
    48 Mi rows): the two-pass kernels run."""
    from test_gpu_monotonic import Trace  # the profiling helper of the monotonic tests

    lanes = r32_lanes(LANES[1])
    rng = np.random.default_rng(7)
    g = make(mz, ctx, lanes, 1000, False, False)
    o = TopKDefinition(lanes, 1000)
    for t, n in enumerate([3000, 5000, 100_000, 200]):
        rows = gen_rows(mz, rng, n, False, 2 * t, rng.integers(0, 4, size=n, dtype=np.uint64), neg=False)
        with Trace(ctx) as tr:
            out, errs = g.step(rows, 2 * t + 2)
        want_out, _ = o.step(tuples(rows, False))
        same(out, out_words(want_out, False), 4)
        assert len(errs) == 0
        two_pass = n * 1001 > 48 << 20
        assert tr.ran("k_topk_window") and tr.ran("k_topk_window_lb") != two_pass, tr.kernels
    g.input_trace().set_logical_compaction(8)
    same(g.input_trace().export(), window_words(o.window(8)), 9)


def test_agrees_with_topk_operator(mz, ctx):
    """Insert-only R32 batches, top 3 by val1 descending: the accumulated window values agree with
    mzgpu_topk_new's, whose output carries the ordering value."""
    rng = np.random.default_rng(11)
    g = make(mz, ctx, [(VAL1, 0, 64, False, True)], 3, False, False)
    old = mz.TopK(ctx, 3, 0, True)
    got, want = Counter(), Counter()
    for t in range(6):
        n = 20_000
        rows = gen_rows(mz, rng, n, False, 2 * t, zipf_keys(rng, n, 2000), neg=False, small_vals=True)
        rows["diff"] = 1
        out, errs = g.step(rows, 2 * t + 2)
        assert len(errs) == 0
        for r in out:
            got[(int(r["key"]), int(r["val"]))] += int(r["diff"])
        for r in old.step(rows, 2 * t + 2):
            want[(int(r["key"]), int(r["sum_lo"]))] += int(r["diff"])
        assert {k: d for k, d in got.items() if d} == {k: d for k, d in want.items() if d}


def test_testdrive_answers(mz, ctx):
    cases = json.load(open(os.path.join(HERE, "golden", "testdrive_monotonic_topk.json")))["cases"]
    for case in cases:
        flip = case["flip_sign"]
        enc = (lambda v: u(v) ^ (1 << 63)) if flip else u
        g = make(mz, ctx, [(VAL1, 0, 64, bool(sx), bool(d)) for sx, d in case["order"]], case["limit"], False,
                 False)
        acc = Counter()
        for i, (ingest, expect) in enumerate(zip(case["ingest"], case["expect"])):
            rows = np.array([(k, enc(v), t, 1) for k, v, t in ingest], dtype=mz.R32)
            out, errs = g.step(rows, i + 2)
            assert len(errs) == 0
            for r in out:
                acc[(int(r["key"]), int(r["val"]))] += int(r["diff"])
            got = sorted(itertools.chain.from_iterable([kv] * c for kv, c in acc.items() if c))
            assert got == sorted((k, enc(v)) for k, v in expect), case["name"]


def test_operator_kernels_by_name(mz, ctx):
    from test_gpu_monotonic import Trace

    g = make(mz, ctx, r32_lanes(LANES[1]), 1, False, False)
    rng = np.random.default_rng(5)
    rows = gen_rows(mz, rng, 5000, False, 0, zipf_keys(rng, 5000, 100))
    with Trace(ctx) as t:
        g.step(rows, 2)
    assert t.ran("k_topk_explode") and t.ran("k_topk_window_lb"), t.kernels


def test_creation_errors_leave_the_context_usable(mz, ctx):
    from materialize_b200 import _ffi as F

    lane = mz.order_lane(VAL1)

    def new(order, limit=1, irb=32, null_order=False):
        arr = (F.OrderLane * max(1, len(order)))()
        for i, (src, sh, b, sx, d, f64) in enumerate(order):
            arr[i].sign_extend, arr[i].descending, arr[i].flags = int(sx), int(d), F.ORDER_F64 if f64 else 0
            arr[i].field = F.Field(src, sh, b, 0)
        h = C.c_void_p(0)
        st = F.lib.mzgpu_topk_monotonic_new(ctx.h, irb, None if null_order else arr, len(order), limit, 0,
                                            C.byref(h))
        return st, h.value

    for order, limit, irb, null_order in [
        ([lane], 1, 48, False),
        ([lane] * 4, 1, 32, False),
        ([mz.order_lane(VAL2)], 1, 32, False),
        ([mz.order_lane(VAL1, 60, 8)], 1, 32, False),
        ([mz.order_lane(VAL1, 0, 0)], 1, 32, False),
        ([lane], 1, 32, True),
    ]:
        st, h = new(order, limit, irb, null_order)
        assert st == E_INVALID and not h, (order, limit, irb)
    for order, limit in (([lane], -1), ([mz.order_lane(VAL1, f64=True)], 1), ([lane, mz.order_lane(VAL1, f64=True)], 3)):
        st, h = new(order, limit)
        assert st == E_UNSUPPORTED and not h, (order, limit)
    # a malformed lane after a float64 one is still E_INVALID
    st, h = new([mz.order_lane(VAL1, f64=True), mz.order_lane(VAL1, 0, 0)])
    assert st == E_INVALID and not h
    g = make(mz, ctx, [], 1, False, False)
    out, errs = g.step(np.array([(1, 2, 0, 1), (1, 1, 0, 1)], dtype=mz.R32), 1)
    assert out.tolist() == [(1, 1, 0, 1)] and len(errs) == 0


# ------------------------------------------------------------------ 72-byte rows on every kernel path
CODES = {0: "lsd/merge", 1: "msd-warp", 2: "msd-cta", 3: "lsd(overflow)", 4: "fast-msd(64-bit)", 5: "fast-msd(128-bit)"}
RB, NW = 72, 9


def gen_arr(rng, n, key_bits=16, word_bits=4, time_bits=3):
    """window rows: key, five words of `word_bits` bits, time, a small diff of either sign, pad 0"""
    w = np.zeros((n, NW), dtype=np.uint64)
    w[:, 0] = rng.integers(0, 1 << key_bits, size=n, dtype=np.uint64)
    for c in range(1, 6):
        w[:, c] = (rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True) if word_bits >= 64
                   else rng.integers(0, 1 << word_bits, size=n, dtype=np.uint64))
    w[:, 6] = rng.integers(0, 1 << time_bits, size=n, dtype=np.uint64) if time_bits else 0
    w[:, 7] = rng.integers(-2, 3, size=n).astype(np.int64).view(np.uint64)
    return w


def ref_consolidate(w, since=0):
    """per (key, o0..o2, val1, val2, max(time, since)): the wrapping sum of the diffs, zeros dropped,
    sorted (the ND = 2 SUM arithmetic: the pad word stays zero)"""
    w = w.copy()
    w[:, 6] = np.maximum(w[:, 6], np.uint64(since))
    order = np.lexsort(tuple(w[:, c] for c in range(6, -1, -1)))
    w = w[order]
    if len(w) == 0:
        return w
    head = np.ones(len(w), dtype=bool)
    head[1:] = np.any(w[1:, :7] != w[:-1, :7], axis=1)
    starts = np.flatnonzero(head)
    out = w[starts].copy()
    with np.errstate(over="ignore"):
        out[:, 7] = np.add.reduceat(w[:, 7], starts)
    out[:, 8] = 0
    return out[out[:, 7] != 0]


def rows_of(w):
    from materialize_b200 import _ffi as F

    return np.ascontiguousarray(w).view(F.DTYPES[RB]).reshape(-1)


def check(got, want):
    g = words(got, NW)
    assert g.shape == want.shape and g.tobytes() == want.tobytes(), (g.shape, want.shape)


def consolidate_dev(mz, ctx, w):
    d = mz.DeviceRows(ctx, RB).upload(rows_of(w))
    d.consolidate()
    return d.download()


@pytest.mark.parametrize("word_bits,codes", [(4, {4}), (14, {5})])
def test_fast_msd(mz, ctx, word_bits, codes):
    from test_gpu_monotonic import Trace

    rng = np.random.default_rng(word_bits)
    w = gen_arr(rng, 60_000, word_bits=word_bits)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, w)
    t.only_fused(RB, codes, n=len(w))
    check(got, ref_consolidate(w))


def test_exact_msd_and_lsd_after_overflow(mz, ctx):
    """Clumped rows overflow the fast path's buckets: the exact MSD path (or the radix passes) runs; with
    full-width words every key word varies and the composite needs seven radix rounds."""
    from test_gpu_monotonic import Trace

    rng = np.random.default_rng(3)
    w = gen_arr(rng, 40_000, key_bits=18)
    for gi in range(20):
        w[gi * 400 : (gi + 1) * 400, :7] = w[gi * 400, :7]
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, w)
    t.only_fused(RB, {2, 3}, n=len(w))
    check(got, ref_consolidate(w))
    w = gen_arr(rng, 300_000, key_bits=64, word_bits=64, time_bits=0)
    w[:, 6] = rng.integers(0, M64, size=len(w), dtype=np.uint64)
    w[1000:2000] = w[:1000]
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, w)
    t.only_fused(RB, {0, 3}, n=len(w))
    check(got, ref_consolidate(w))


def test_merge_as_sort_and_fused_merge_path(mz, ctx):
    from test_gpu_monotonic import Trace

    rng = np.random.default_rng(20)
    for na, nb, codes in ((40_000, 30_000, {2, 3, 4, 5}), (700_000, 500_000, {0})):
        a = gen_arr(rng, na, key_bits=17, time_bits=6)
        b = gen_arr(rng, nb, key_bits=17, time_bits=6)
        b[:, 6] += np.uint64(64)
        b[:5000, :6] = a[:5000, :6]
        ba, bb = mz.Batch.build(ctx, rows_of(a), 0, 64), mz.Batch.build(ctx, rows_of(b), 64, 200)
        ra, rbb = ref_consolidate(a), ref_consolidate(b)
        for since in (0, 90, 1 << 40):
            with Trace(ctx) as t:
                m = ba.merge(bb, since)
                check(m.rows(), ref_consolidate(np.concatenate([ra, rbb]), since))
            t.only_fused(RB, codes, n=len(ra) + len(rbb))


def test_bulk_sort_consolidate_and_merge(mz, ctx):
    """Past 2M rows: sort.cu + consolidate.cu and merge.cu."""
    from test_gpu_monotonic import Trace

    rng = np.random.default_rng(30)
    w = gen_arr(rng, 2_200_000, key_bits=12, word_bits=3, time_bits=1)
    w[:50_000, 1:6] = rng.integers(0, M64, size=(50_000, 5), dtype=np.uint64)  # seven varying words
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, w)
    assert t.fused == [] and t.ran("k_rs_onesweep") and t.ran("k_segsum"), (t.fused, t.kernels)
    check(got, ref_consolidate(w))
    w1 = gen_arr(rng, 1_600_000, key_bits=30, time_bits=3)
    w2 = gen_arr(rng, 1_500_000, key_bits=30, time_bits=3)
    w2[:100_000, :7] = w1[:100_000, :7]
    w2[:, 6] += np.uint64(3)
    b1, b2 = mz.Batch.build(ctx, rows_of(w1), 0, 9), mz.Batch.build(ctx, rows_of(w2), 9, 20)
    r1, r2 = ref_consolidate(w1), ref_consolidate(w2)
    assert len(b1) + len(b2) > 2 * 1024 * 1024
    with Trace(ctx) as t:
        m = b1.merge(b2, 5)
        check(m.rows(), ref_consolidate(np.concatenate([r1, r2]), 5))
    assert t.fused == [] and t.ran("k_merge_tiles"), (t.fused, t.kernels)


@pytest.mark.parametrize("n", [30_000, 2_200_000])
def test_seal_split(mz, ctx, n):
    """A batcher seal ships the rows below `upper` and keeps the rest for the next seal (fused and bulk)."""
    rng = np.random.default_rng(40 + n)
    w = gen_arr(rng, n, key_bits=20, word_bits=6, time_bits=3)
    b = mz.Batcher(ctx, RB)
    b.push_container(rows_of(w))
    check(b.seal(4).rows(), ref_consolidate(w[w[:, 6] < 4]))
    check(b.seal(8).rows(), ref_consolidate(w[w[:, 6] >= 4]))
