"""The monotonic MIN / MAX reduce on the GPU, byte for byte against its CPU restatement
(tests/monotonic_oracle.py), the max-semigroup arrangement rows on every kernel path, agreement with the
bucketed MIN / MAX operator, and the creation errors."""
import ctypes as C
import json
import os

import numpy as np
import pytest

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


def zipf_keys(rng, n, nk, s=0.9):
    p = 1.0 / np.arange(1, nk + 1) ** s
    return rng.choice(nk, size=n, p=p / p.sum()).astype(np.uint64)


def gen_rows(mz, rng, n, r40, t, keys, neg=True):
    iw = 5 if r40 else 4
    w = np.zeros((n, iw), dtype=np.uint64)
    w[:, 0] = keys
    for c in range(1, iw - 2):
        w[:, c] = rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True)
        w[: n // 50, c] = rng.choice(np.array([0, M64, 1 << 63, (1 << 63) - 1], dtype=np.uint64), size=n // 50)
    w[:, iw - 2] = t
    d = rng.choice([1, 1, 1, 1, 2, 3, 0, -1], size=n) if neg else rng.integers(1, 3, size=n)
    w[:, iw - 1] = d.astype(np.int64).view(np.uint64)
    return w.view(mz.R40 if r40 else mz.R32).reshape(-1)


LANE_SETS = {
    1: [(AGG_MAX, VAL1, 0, 64, False)],
    3: [(AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 0, 32, True), (AGG_MIN, VAL1, 32, 32, False)],
    4: [(AGG_MIN, VAL1, 0, 16, True), (AGG_MAX, VAL1, 16, 1, False), (AGG_MAX, VAL1, 0, 64, True),
        (AGG_MIN, VAL1, 0, 64, False)],
    5: [(AGG_MAX, VAL1, 0, 64, False), (AGG_MIN, VAL1, 0, 64, True), (AGG_MAX, VAL1, 8, 8, True),
        (AGG_MIN, VAL1, 63, 1, False), (AGG_MAX, VAL1, 0, 63, True)],
    8: [(AGG_MIN if l % 2 else AGG_MAX, VAL1, 8 * l, 8 * (8 - l), l % 3 == 0) for l in range(8)],
}


def r40_lanes(lanes):
    """every other lane reads val2"""
    return [(k, VAL2 if i % 2 else VAL1, s, b, sx) for i, (k, _, s, b, sx) in enumerate(lanes)]


@pytest.mark.parametrize("n_lanes", [1, 3, 4, 5, 8])
@pytest.mark.parametrize("r40", [False, True])
@pytest.mark.parametrize("must_consolidate", [False, True])
def test_matches_restatement(mz, ctx, n_lanes, r40, must_consolidate):
    """Zipf(0.9) keys over 32 activations with logical compaction advancing: corrections, errors and the
    arrangement byte for byte."""
    rng = np.random.default_rng(n_lanes * 4 + 2 * r40 + must_consolidate)
    lanes = r40_lanes(LANE_SETS[n_lanes]) if r40 else LANE_SETS[n_lanes]
    g = mz.ReduceMonotonic(ctx, [mz.accum_lane(k, s, sh, b, sx) for k, s, sh, b, sx in lanes], 40 if r40 else 32,
                           must_consolidate)
    o = ReduceMonotonic(lanes, 40 if r40 else 32, must_consolidate)
    for t in range(32):
        n = int(rng.choice([1, 50, 3000, 20000]))
        rows = gen_rows(mz, rng, n, r40, t, zipf_keys(rng, n, 5000))
        if must_consolidate and n > 10:  # +1 / -1 pairs that cancel, and pairs that leave -1
            rows[n // 2 : n // 2 + 5] = rows[:5]
            rows[:5]["diff"] = 1
            rows[n // 2 : n // 2 + 5]["diff"] = -1
        out, errs = g.step(rows, t + 1)
        want_out, want_errs = o.step(rows, t + 1)
        same(out, want_out)
        same(errs, want_errs)
        if t % 4 == 3:
            since = max(0, t - 6)
            g.input_trace().set_logical_compaction(since)
            same(g.input_trace().export(), o.export(since))
    ctx.sync()


# ------------------------------------------------------------------ max-semigroup rows on every path
CODES = {0: "lsd/merge", 1: "msd-warp", 2: "msd-cta", 3: "lsd(overflow)", 4: "fast-msd(64-bit)", 5: "fast-msd(128-bit)"}


class Trace:
    def __init__(self, ctx):
        self.ctx = ctx

    def __enter__(self):
        self.ctx.profile(True)
        return self

    def __exit__(self, *exc):
        from materialize_b200 import _ffi as F

        try:
            if exc[0] is None:
                buf = (C.c_uint64 * (32 * 4096))()
                n = C.c_uint32(0)
                self.ctx.check(F.lib.mzgpu_profile_fused_phases(self.ctx.h, buf, 4096, C.byref(n)))
                a = np.frombuffer(buf, dtype=np.uint64).reshape(-1, 32)[: n.value]
                self.fused = [(int(r[20]), int(r[16]), int(r[21])) for r in a]
                self.kernels = {k.strip("()") for k in self.ctx.profile_report()}
        finally:
            self.ctx.profile(False)

    def ran(self, prefix):
        return any(k.startswith(prefix) for k in self.kernels)

    def only_fused(self, rb, codes, n=None):
        assert len(self.fused) == 1, self.fused
        frb, fn, code = self.fused[0]
        assert frb == rb and code in codes, (self.fused, codes)
        if n is not None:
            assert fn == n, (fn, n)
        return code


NW = {48: 6, 112: 14}
NL = {48: 4, 112: 8}


def gen_arr(rng, rb, n, key_bits=20, time_bits=4):
    """monotonic arrangement rows: lane words anywhere in 64 bits, unused lane words of the class zero"""
    w = np.zeros((n, NW[rb]), dtype=np.uint64)
    w[:, 0] = rng.integers(0, 1 << key_bits, size=n, dtype=np.uint64)
    w[:, 1] = rng.integers(0, 1 << time_bits, size=n, dtype=np.uint64) if time_bits else 0
    w[:, 2 : 2 + NL[rb]] = rng.integers(0, M64, size=(n, NL[rb]), dtype=np.uint64, endpoint=True)
    return w


def ref_consolidate(w, since=0):
    """per (key, max(time, since)): the per-word max of the lane words; sorted; no row ever vanishes"""
    w = w.copy()
    w[:, 1] = np.maximum(w[:, 1], np.uint64(since))
    order = np.lexsort((w[:, 1], w[:, 0]))
    w = w[order]
    if len(w) == 0:
        return w
    head = np.ones(len(w), dtype=bool)
    head[1:] = (w[1:, 0] != w[:-1, 0]) | (w[1:, 1] != w[:-1, 1])
    starts = np.flatnonzero(head)
    out = w[starts].copy()
    out[:, 2:] = np.maximum.reduceat(w[:, 2:], starts, axis=0)
    return out


def rows_of(mz, rb, w):
    from materialize_b200 import _ffi as F

    return np.ascontiguousarray(w).view(F.DTYPES[rb]).reshape(-1)


def words(rows, rb):
    return np.ascontiguousarray(rows).view(np.uint64).reshape(-1, NW[rb])


def check(got, want, rb):
    g = words(got, rb)
    assert g.shape == want.shape and g.tobytes() == want.tobytes(), (g.shape, want.shape)


def consolidate_dev(mz, ctx, rb, w):
    d = mz.DeviceRows(ctx, rb).upload(rows_of(mz, rb, w))
    d.consolidate()
    return d.download()


@pytest.mark.parametrize("rb", [48, 112])
def test_fast_msd(mz, ctx, rb):
    rng = np.random.default_rng(rb)
    w = gen_arr(rng, rb, 60_000, key_bits=16, time_bits=3)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {4, 5}, n=len(w))
    check(got, ref_consolidate(w), rb)
    with Trace(ctx) as t:
        b = mz.Batch.build(ctx, rows_of(mz, rb, w), 0, 9)
        check(b.rows(), ref_consolidate(w), rb)
    t.only_fused(rb, {4, 5})


@pytest.mark.parametrize("rb", [48, 112])
def test_exact_fallback_on_clumped_keys(mz, ctx, rb):
    """A (key, time) with hundreds of rows overflows the fast path's buckets; monotonic rows never take the
    CTA-level path (its shared sums add), so the radix passes run."""
    rng = np.random.default_rng(10 + rb)
    w = gen_arr(rng, rb, 40_000, key_bits=18, time_bits=3)
    for gi in range(20):
        w[gi * 400 : (gi + 1) * 400, :2] = w[gi * 400, :2]
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {3}, n=len(w))
    check(got, ref_consolidate(w), rb)


@pytest.mark.parametrize("rb", [48, 112])
def test_merge_as_sort_and_fused_merge_path(mz, ctx, rb):
    rng = np.random.default_rng(20 + rb)
    for na, nb, codes in ((40_000, 30_000, {2, 3, 4, 5}), (700_000, 500_000, {0})):
        a = gen_arr(rng, rb, na, key_bits=17, time_bits=6)
        b = gen_arr(rng, rb, nb, key_bits=17, time_bits=6)
        b[:, 1] += np.uint64(64)
        b[:5000, 0] = a[:5000, 0]
        ba, bb = mz.Batch.build(ctx, rows_of(mz, rb, a), 0, 64), mz.Batch.build(ctx, rows_of(mz, rb, b), 64, 200)
        ra, rbb = ref_consolidate(a), ref_consolidate(b)
        len(ba), len(bb)
        for since in (0, 90, 1 << 40):
            with Trace(ctx) as t:
                m = ba.merge(bb, since)
                check(m.rows(), ref_consolidate(np.concatenate([ra, rbb]), since), rb)
            t.only_fused(rb, codes, n=len(ra) + len(rbb))


@pytest.mark.parametrize("rb", [48, 112])
def test_bulk_sort_consolidate_and_merge(mz, ctx, rb):
    """Past 2M rows: sort.cu + consolidate.cu (atomicMax segment sums) and merge.cu."""
    rng = np.random.default_rng(30 + rb)
    w = gen_arr(rng, rb, 2_200_000, key_bits=10, time_bits=1)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    assert t.fused == [] and t.ran("k_rs_onesweep") and t.ran("k_segsum"), (t.fused, t.kernels)
    check(got, ref_consolidate(w), rb)
    w1 = gen_arr(rng, rb, 1_300_000, key_bits=30, time_bits=3)
    w2 = gen_arr(rng, rb, 1_200_000, key_bits=30, time_bits=3)
    w2[:100_000, :2] = w1[:100_000, :2]
    w2[:, 1] += np.uint64(3)
    b1, b2 = mz.Batch.build(ctx, rows_of(mz, rb, w1), 0, 9), mz.Batch.build(ctx, rows_of(mz, rb, w2), 9, 20)
    r1, r2 = ref_consolidate(w1), ref_consolidate(w2)
    assert len(b1) + len(b2) > 2 * 1024 * 1024
    with Trace(ctx) as t:
        m = b1.merge(b2, 5)
        check(m.rows(), ref_consolidate(np.concatenate([r1, r2]), 5), rb)
    assert t.fused == [] and t.ran("k_merge_tiles"), (t.fused, t.kernels)


def test_operator_kernels_by_name(mz, ctx):
    """an activation runs the explode and the single-pass corrections kernel"""
    g = mz.ReduceMonotonic(ctx, [mz.accum_lane(AGG_MAX, VAL1)])
    rng = np.random.default_rng(5)
    rows = gen_rows(mz, rng, 5000, False, 0, zipf_keys(rng, 5000, 100))
    with Trace(ctx) as t:
        g.step(rows, 1)
    assert t.ran("k_monotonic_explode") and t.ran("k_monotonic_corrections_lb"), t.kernels


# ------------------------------------------------------------------ agreement and errors
@pytest.mark.parametrize("kind", [AGG_MIN, AGG_MAX])
def test_one_unsigned_lane_equals_min_max_operator(mz, ctx, kind):
    """Insert-only batches: the accumulated output collections agree value for value, keys with more than
    32 live values included."""
    rng = np.random.default_rng(kind)
    g = mz.ReduceMonotonic(ctx, [mz.accum_lane(kind, VAL1)])
    old = mz.ReduceAccumulable(ctx, kind)
    got, want = {}, {}
    for t in range(12):
        n = 20_000
        rows = gen_rows(mz, rng, n, False, t, zipf_keys(rng, n, 2000), neg=False)
        out, errs = g.step(rows, t + 1)
        assert len(errs) == 0
        for r in out:
            k = (int(r["key"]), int(r["vals"][0]))
            got[k] = got.get(k, 0) + int(r["diff"])
        for r in old.step(rows, t + 1):
            assert int(r["flags"]) == 0
            k = (int(r["key"]), int(r["sum_lo"]))
            want[k] = want.get(k, 0) + int(r["diff"])
        assert {k: d for k, d in got.items() if d} == {k: d for k, d in want.items() if d}
    assert max(np.bincount(rows["key"].astype(np.int64))) > 32


def test_sql_count_min_sum_max(mz, ctx):
    fx = json.load(open(os.path.join(HERE, "golden", "sqllogictest_join_reduce.json")))
    cases = {c["shape"]: c for c in fx["cases"]}
    t = fx["tables"]["t"]["rows"]
    rows = np.zeros(len(t), dtype=mz.R32)
    rows["key"], rows["val"], rows["time"], rows["diff"] = [a for a, _ in t], [b for _, b in t], 0, 1
    g = mz.ReduceMonotonic(ctx, [mz.accum_lane(AGG_MIN, VAL1, sign_extend=True),
                                 mz.accum_lane(AGG_MAX, VAL1, sign_extend=True)])
    out, errs = g.step(rows, 1)
    assert len(errs) == 0 and all(int(r["diff"]) == 1 for r in out)
    got = sorted((int(r["key"]), int(np.int64(r["vals"][0])), int(np.int64(r["vals"][1]))) for r in out)
    assert got == sorted((k, mn, mx) for k, _, mn, _, mx in cases["count_min_sum_max"]["expect"])


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
    ]
    for lanes, irb in bad:
        with pytest.raises(mz.MzGpuError) as e:
            mz.ReduceMonotonic(ctx, lanes, irb)
        assert e.value.status == E_INVALID, (lanes, irb)
    for lanes in ([mz.accum_lane(AGG_MIN | mz.MONO_F64, VAL1)],
                  [lane, mz.accum_lane(AGG_MAX | mz.MONO_F64, VAL1)]):
        with pytest.raises(mz.MzGpuError) as e:
            mz.ReduceMonotonic(ctx, lanes)
        assert e.value.status == E_UNSUPPORTED
    # a malformed lane after a float64 one is still E_INVALID
    with pytest.raises(mz.MzGpuError) as e:
        mz.ReduceMonotonic(ctx, [mz.accum_lane(AGG_MIN | mz.MONO_F64, VAL1), mz.accum_lane(0, VAL1)])
    assert e.value.status == E_INVALID
    g = mz.ReduceMonotonic(ctx, [lane])
    out, errs = g.step(np.array([(1, 2, 0, 1)], dtype=mz.R32), 1)
    assert out.tolist()[0][0] == 1 and len(errs) == 0
    # the output rows have no generic meaning
    d = mz.DeviceRows(ctx, 56).upload(out)
    with pytest.raises(mz.MzGpuError) as e:
        d.consolidate()
    assert e.value.status == E_UNSUPPORTED
