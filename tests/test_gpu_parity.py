"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on
the same seeded inputs, bit-exact, plus size-independent properties at large
sizes.  Run with `pytest -m gpu` on an H100."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    c = mz.Context(0)
    yield c
    c.sync()


def rand_r32(rng, n, key_hi, val_hi, time_hi, diff_lo=-3, diff_hi=3, dtype=None):
    a = np.zeros(n, dtype=dtype)
    a["key"] = rng.integers(0, key_hi, size=n, dtype=np.uint64)
    a["val"] = rng.integers(0, val_hi, size=n, dtype=np.uint64)
    a["time"] = rng.integers(0, time_hi, size=n, dtype=np.uint64)
    a["diff"] = rng.integers(diff_lo, diff_hi + 1, size=n, dtype=np.int64)
    return a


def multiset(rows):
    """Order-independent fingerprint of a row array (rows as opaque byte strings, sorted)."""
    if len(rows) == 0:
        return b""
    raw = np.ascontiguousarray(rows).view(np.uint8).reshape(len(rows), rows.dtype.itemsize)
    return np.sort(raw.view(f"V{rows.dtype.itemsize}").ravel()).tobytes()


def same(a, b):
    assert a.dtype == b.dtype
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


# ------------------------------------------------------------------ a1
def test_consolidate_golden_vectors(mz, ctx, oracle):
    vec = json.load(open(os.path.join(HERE, "golden", "consolidate_vectors.json")))
    for case in vec["chunker_u64"]["cases"]:
        rows = oracle.rows(oracle.R32, [(d, 0, t, r) for d, t, r in case["input"]])
        want = oracle.rows(oracle.R32, [(d, 0, t, r) for d, t, r in case["expected"]])
        same(ctx.consolidate(rows), want)
    for case in vec["chunker_keyval"]["cases"]:
        rows = oracle.rows(oracle.R32, [tuple(r) for r in case["input"]])
        want = oracle.rows(oracle.R32, [tuple(r) for r in case["expected"]])
        same(ctx.consolidate(rows), want)
    # cross_batch_consolidation: 100_000 x (42, 0, +1) -> (42, 0, 100000)
    rows = oracle.rows(oracle.R32, [(42, 0, 0, 1)] * 100000)
    same(ctx.consolidate(rows), oracle.rows(oracle.R32, [(42, 0, 0, 100000)]))
    # consolidates_on_threshold: +1/-1 pairs cancel completely
    rows = oracle.rows(oracle.R32, [(7, 0, 0, 1), (7, 0, 0, -1)] * 3000)
    assert len(ctx.consolidate(rows)) == 0
    # emits_multiple_containers: 300_000 distinct rows come back sorted
    rows = oracle.rows(oracle.R32, [(d, 0, 0, 1) for d in range(300000)])
    rng = np.random.default_rng(0)
    same(ctx.consolidate(rows[rng.permutation(len(rows))]), rows)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 4096, 4097, 100000, 1 << 20])
@pytest.mark.parametrize("key_bits", [4, 20, 64])
def test_consolidate_r16_matches_oracle(mz, ctx, oracle, n, key_bits):
    rng = np.random.default_rng(n * 131 + key_bits)
    a = np.zeros(n, dtype=oracle.R16)
    hi = (1 << key_bits) - 1
    a["key"] = rng.integers(0, hi, size=n, dtype=np.uint64, endpoint=True)
    a["diff"] = rng.integers(-3, 4, size=n, dtype=np.int64)
    same(ctx.consolidate(a), oracle.consolidate(a))


@pytest.mark.parametrize(
    "n,key_hi,val_hi,time_hi",
    [
        (0, 1, 1, 1),
        (1, 5, 5, 3),
        (1000, 5, 5, 3),  # heavy collisions (the proptest ranges of batcher.rs:1134-1137)
        (100000, 1000, 1 << 40, 1),
        (100000, 1 << 62, 3, 1 << 33),
        (300000, 2**64 - 1, 2**64 - 1, 7),  # > 64 composite bits: multi-round sort
        (1 << 20, 1 << 20, 4, 2),
    ],
)
def test_consolidate_r32_matches_oracle(mz, ctx, oracle, n, key_hi, val_hi, time_hi):
    rng = np.random.default_rng(n + 7)
    a = rand_r32(rng, n, key_hi, val_hi, time_hi, dtype=oracle.R32)
    same(ctx.consolidate(a), oracle.consolidate(a))


@pytest.mark.parametrize("hot_keys,per_key", [(50, 400), (4, 3000), (2000, 7), (1, 20000)])
def test_consolidate_clumped_keys(mz, ctx, oracle, hot_keys, per_key):
    """Keys arrive in clumps (many rows share the leading key bits): exercises the warp-bucket, the
    CTA bucket-unit and the radix fall-back paths of the fused kernel, which must all agree."""
    rng = np.random.default_rng(hot_keys * 7 + per_key)
    n = hot_keys * per_key
    a = np.zeros(n, dtype=oracle.R32)
    a["key"] = np.repeat(rng.integers(0, 1 << 40, size=hot_keys, dtype=np.uint64), per_key)
    a["val"] = rng.integers(0, 1 << 20, size=n, dtype=np.uint64)
    a["time"] = rng.integers(0, 3, size=n, dtype=np.uint64)
    a["diff"] = rng.integers(-2, 3, size=n, dtype=np.int64)
    rng.shuffle(a)
    same(ctx.consolidate(a), oracle.consolidate(a))
    # and through a seal that keeps part of the rows
    gb, ob = mz.Batcher(ctx, 32), oracle.Batcher(32)
    gb.push_container(a)
    ob.push(a)
    g, o = gb.seal(2), ob.seal(2)
    same(g.rows(), o.rows())
    assert gb.frontier() == ob.frontier()
    g2, o2 = gb.seal(mz.FRONTIER_EMPTY), ob.seal(mz.FRONTIER_EMPTY)
    same(g2.rows(), o2.rows())


def test_consolidate_wrapping_diffs(mz, ctx, oracle):
    a = oracle.rows(oracle.R16, [(1, 2**63 - 1), (1, 1), (2, -(2**63)), (2, -(2**63)), (3, 5)])
    same(ctx.consolidate(a), oracle.consolidate(a))
    assert ctx.consolidate(a).tolist() == [(1, -(2**63)), (3, 5)]


def test_consolidate_other_row_shapes(mz, ctx, oracle):
    rng = np.random.default_rng(5)
    n = 50000
    a = np.zeros(n, dtype=oracle.R40)
    a["key"] = rng.integers(0, 50, size=n, dtype=np.uint64)
    a["val1"] = rng.integers(0, 4, size=n, dtype=np.uint64)
    a["val2"] = rng.integers(0, 4, size=n, dtype=np.uint64)
    a["time"] = rng.integers(0, 3, size=n, dtype=np.uint64)
    a["diff"] = rng.integers(-2, 3, size=n, dtype=np.int64)
    same(ctx.consolidate(a), oracle.consolidate(a))
    r = rand_r32(rng, n, 300, 1 << 62, 4, dtype=oracle.R32)
    r["val"] = rng.integers(-(2**62), 2**62, size=n, dtype=np.int64).astype(np.uint64)
    acc = oracle.explode(r, 0)
    same(ctx.consolidate(acc), oracle.consolidate(acc))
    out = oracle.finalize(oracle.consolidate(acc), 0)
    out["time"] = rng.integers(0, 3, size=len(out), dtype=np.uint64)
    out["diff"] = rng.integers(-1, 2, size=len(out), dtype=np.int64)
    both = np.concatenate([out, out])
    same(ctx.consolidate(both), oracle.consolidate(both))


def test_consolidate_large_properties(mz, ctx):
    """BASELINE-size properties: sortedness, preserved per-key sums, idempotence."""
    rng = np.random.default_rng(11)
    n = 10_000_000
    a = np.zeros(n, dtype=mz.R16)
    a["key"] = rng.integers(0, 1 << 22, size=n, dtype=np.uint64)
    a["diff"] = rng.integers(-3, 4, size=n, dtype=np.int64)
    out = ctx.consolidate(a)
    assert np.all(out["key"][1:] > out["key"][:-1])
    assert np.all(out["diff"] != 0)
    sums = np.bincount(a["key"].astype(np.int64), weights=a["diff"].astype(np.float64), minlength=1 << 22)
    assert np.array_equal(np.nonzero(sums)[0].astype(np.uint64), out["key"])
    assert np.array_equal(sums[out["key"].astype(np.int64)].astype(np.int64), out["diff"])
    same(ctx.consolidate(out), out)


def test_arrange_join_full_size_properties(mz, ctx):
    """BASELINE configs[1] at full size (2 x 10 M rows, uniform keys): the oracle cannot run this in
    seconds, so the join is pinned by size-independent properties -- per-key output counts are the
    product of the inputs' per-key counts, the value columns' checksums follow by linearity, and the
    consolidated output is sorted with unit diffs (row-index values make every output row distinct)."""
    from materialize_b200 import harness

    n = 10_000_000
    a, b = harness.gen_cfg2(ctx, 1, n, n), harness.gen_cfg2(ctx, 2, n, n)
    ha, hb = a.download(), b.download()
    ba, bb = mz.Batcher(ctx, 32), mz.Batcher(ctx, 32)
    ba.push_device(a)
    bb.push_device(b)
    xa, xb = ba.seal(1), bb.seal(1)
    sa, sb = mz.Spine(ctx, 32), mz.Spine(ctx, 32)
    j = mz.JoinCore(ctx, sa, sb)
    sa.insert(xa)
    j.push(0, xa, 0)
    sb.insert(xb)
    j.push(1, xb, 0)
    j.work()
    out = j.results()
    ka, kb = ha["key"].astype(np.int64), hb["key"].astype(np.int64)
    ca, cb = np.bincount(ka, minlength=n), np.bincount(kb, minlength=n)
    assert len(out) == int((ca * cb).sum())
    assert np.array_equal(np.bincount(out["key"].astype(np.int64), minlength=n), ca * cb)
    va = np.bincount(ka, weights=ha["val"].astype(np.float64), minlength=n).astype(np.int64)
    vb = np.bincount(kb, weights=hb["val"].astype(np.float64), minlength=n).astype(np.int64)
    assert int(out["val1"].astype(np.int64).sum()) == int((va * cb).sum())
    assert int(out["val2"].astype(np.int64).sum()) == int((vb * ca).sum())
    assert np.all(out["diff"] == 1) and np.all(out["time"] == 0)
    # (a work item is joined in slices of 1M probe rows, each slice's results consolidated on its own:
    # the whole result is sorted and duplicate-free once consolidated)
    outc = ctx.consolidate(out)
    assert len(outc) == len(out)
    k, v1, v2 = outc["key"], outc["val1"], outc["val2"]
    lt = (k[:-1] < k[1:]) | ((k[:-1] == k[1:]) & ((v1[:-1] < v1[1:]) | ((v1[:-1] == v1[1:]) & (v2[:-1] < v2[1:]))))
    assert np.all(lt)


def test_reduce_full_size_properties(mz, ctx):
    """BASELINE configs[3] at full size (100 M rows, 1 M Zipf(0.9) keys): COUNT and SUM per key
    against numpy's bincount of the same rows, one output row per live key, sorted by key."""
    from materialize_b200 import harness

    n, nk = 100_000_000, 1_000_000
    w = 1.0 / np.power(np.arange(1, nk + 1, dtype=np.float64), 0.9)
    cdf = np.cumsum(w / w.sum())
    cdf[-1] = 1.0
    d = harness.gen_cfg4(ctx, 3, n, cdf)
    h = d.download()
    r = mz.ReduceAccumulable(ctx, mz.AGG_COUNT_SUM_I64)
    out = r.step_dev(d, 1).download()
    del d
    keys = h["key"].astype(np.int64)
    hi = int(keys.max()) + 1
    cnt = np.bincount(keys, minlength=hi)
    sums = np.bincount(keys, weights=h["val"].astype(np.int64).astype(np.float64), minlength=hi)
    assert np.abs(sums).max() < 2.0**53  # float64 accumulation of these integers is exact
    live = np.nonzero(cnt)[0]
    assert np.array_equal(out["key"].astype(np.int64), live)
    assert np.array_equal(out["count"], cnt[live])
    assert np.array_equal(out["sum_lo"].astype(np.int64), sums[live].astype(np.int64))
    assert np.all(out["sum_hi"] == np.where(sums[live] < 0, -1, 0))
    assert np.all(out["diff"] == 1) and np.all(out["flags"] == 0)


@pytest.mark.parametrize("agg_kind", [0, 1])
def test_reduce_incremental_full_size(mz, ctx, agg_kind):
    """BASELINE configs[3] in its incremental regime at full size (SURVEY 8d: 100 batches of 1 M
    rows, 1 M Zipf(0.9) keys, half of every batch retracting rows of the batch before): the CPU
    oracle cannot run 100 M rows in seconds, so the operator is pinned by the property that
    defines it -- at every timestamp, the accumulated output corrections are exactly GROUP BY
    (COUNT, SUM) of the accumulated input -- checked with numpy on host copies of the batches.
    i64 sums are compared exactly; f64 sums (kind 1) are compared exactly in the operator's 2^24
    fixed point (the reference accumulates floats as (x * 2^24) as i128), i.e. with tolerance 0,
    inside the 1e-6 relative tolerance north_star allows."""
    from materialize_b200 import harness

    nb, per, nk = 100, 1_000_000, 1_000_000
    w = 1.0 / np.power(np.arange(1, nk + 1, dtype=np.float64), 0.9)
    cdf = np.cumsum(w / w.sum())
    cdf[-1] = 1.0
    r = mz.ReduceAccumulable(ctx, agg_kind)
    cnt = np.zeros(nk + 1, dtype=np.int64)
    tot = np.zeros(nk + 1, dtype=np.float64)  # sums of small integers: exact in float64
    o_cnt = np.zeros(nk + 1, dtype=np.int64)
    o_sum = np.zeros(nk + 1, dtype=np.float64)
    prev = None
    for b in range(nb):
        fresh = harness.gen_cfg4(ctx, 5, per // 2, cdf, as_f64=(agg_kind == 1), first=b * (per // 2), t=b, diff=1)
        batch = mz.DeviceRows(ctx, 32)
        batch.append_buf(fresh)
        if prev is not None:  # retract the rows the previous batch added
            batch.append_buf(harness.gen_cfg4(ctx, 5, per // 2, cdf, as_f64=(agg_kind == 1), first=(b - 1) * (per // 2), t=b, diff=-1))
        h = batch.download()
        out = r.step_dev(batch, b + 1).download()
        prev = fresh
        keys = h["key"].astype(np.int64)
        d = h["diff"].astype(np.int64)
        if agg_kind == 1:  # the operator's fixed point: (x * 2^24) as i128, truncating (reduce.rs:1528)
            vals = np.trunc(h["val"].view(np.float64) * 2.0**24)
        else:
            vals = h["val"].astype(np.int64).astype(np.float64)
        cnt += np.bincount(keys, weights=d.astype(np.float64), minlength=nk + 1).astype(np.int64)
        tot += np.bincount(keys, weights=d * vals, minlength=nk + 1)
        # fold the corrections in: output row (key, count, sum) with diff +-1
        ok = out["key"].astype(np.int64)
        od = out["diff"].astype(np.int64)
        assert np.all(out["flags"] == 0) and np.all(out["time"] == b)
        if agg_kind == 1:  # finalized f64 sums: back to fixed-point units (exact: multiples of 2^-24 below 2^29)
            osum = out["sum_lo"].view(np.float64) * 2.0**24
        else:
            # i128 sums that fit i64 here: the low word read as two's complement, the high word its sign
            lo64 = out["sum_lo"].astype(np.int64)
            assert np.array_equal(out["sum_hi"].astype(np.int64), np.where(lo64 < 0, -1, 0))
            osum = lo64.astype(np.float64)
        o_cnt += np.bincount(ok, weights=(od * out["count"].astype(np.int64)).astype(np.float64), minlength=nk + 1).astype(np.int64)
        o_sum += np.bincount(ok, weights=od * osum, minlength=nk + 1)
        if b % 10 == 9 or b == nb - 1:
            assert np.array_equal(o_cnt, cnt), b
            assert np.array_equal(o_sum, tot), b
    assert np.abs(tot).max() < 2.0**52
    assert int(cnt.sum()) == per // 2  # everything but the last half batch has been retracted


# ------------------------------------------------------------- a2 - a5
def test_batcher_seal_matches_oracle(mz, ctx, oracle):
    rng = np.random.default_rng(21)
    gb, ob = mz.Batcher(ctx, 32), oracle.Batcher(32)
    lower = 0
    for step, upper in enumerate([3, 3, 5, 9, mz.FRONTIER_EMPTY]):
        for _ in range(int(rng.integers(0, 6))):
            n = int(rng.integers(0, 5000))
            a = rand_r32(rng, n, 200, 5, 10, dtype=oracle.R32)
            a["time"] += np.uint64(lower)  # only times >= the sealed frontier may arrive
            gb.push_container(a)
            ob.push(a)
        assert len(gb) == len(ob) or True  # chain shapes differ; contents are compared at seal
        g, o = gb.seal(upper), ob.seal(upper)
        same(g.rows(), o.rows())
        assert g.desc() == o.desc()
        assert g.keys() == o.keys()
        assert gb.frontier() == ob.frontier()
        if upper != mz.FRONTIER_EMPTY:
            lower = upper


def test_seal_many_matches_single_seals(mz, ctx, oracle):
    """mzgpu_batcher_seal_many: k arrangements sealed by one frontier advance in one launch give the
    batches, kept rows and frontiers of k separate seals (and of the oracle's batchers)."""
    rng = np.random.default_rng(31)
    sizes = [30000, 0, 7000, 90000, 1]
    gbs = [mz.Batcher(ctx, 32) for _ in sizes]
    obs = [oracle.Batcher(32) for _ in sizes]
    t = 0
    for rnd in range(4):
        for gb, ob, n in zip(gbs, obs, sizes):
            a = rand_r32(rng, n, 1 << (8 + 4 * rnd), 1 << 20, 1, dtype=oracle.R32)
            a["time"] = rng.integers(t, t + 4, size=n, dtype=np.uint64)  # some rows stay behind the frontier
            gb.push_container(a)
            ob.push(a)
        t += 2
        got = mz.seal_many(gbs, t)
        for g, gb, ob in zip(got, gbs, obs):
            o = ob.seal(t)
            same(g.rows(), o.rows())
            assert g.desc() == o.desc()
            assert gb.frontier() == ob.frontier()


def test_batch_merge_matches_oracle(mz, ctx, oracle):
    rng = np.random.default_rng(22)
    for since in (0, 2, 4, 100):
        a = rand_r32(rng, 20000, 300, 4, 4, dtype=oracle.R32)
        b = rand_r32(rng, 30000, 300, 4, 4, dtype=oracle.R32)
        b["time"] += np.uint64(4)
        g = mz.Batch.build(ctx, a, 0, 4).merge(mz.Batch.build(ctx, b, 4, 8), since)
        o = oracle.Batch.build(a, 0, 4).merge(oracle.Batch.build(b, 4, 8), since)
        same(g.rows(), o.rows())
        assert g.desc() == o.desc() == (0, 8, since)
        assert g.keys() == o.keys()
    # golden merger vectors (batcher.rs:1016-1093)
    vec = json.load(open(os.path.join(HERE, "golden", "consolidate_vectors.json")))
    for case in vec["merger_keyval"]["cases"]:
        c1 = oracle.rows(oracle.R32, [tuple(r) for ch in case["chain1"] for r in ch])
        c2 = oracle.rows(oracle.R32, [tuple(r) for ch in case["chain2"] for r in ch])
        g = mz.Batch.build(ctx, c1, 0, 1).merge(mz.Batch.build(ctx, c2, 1, 2), 0)
        same(g.rows(), oracle.rows(oracle.R32, [tuple(r) for r in case["expected"]]))


def test_batch_merge_long_collapsed_runs(mz, ctx, oracle):
    """advance_by(since) collapsing hundreds / thousands of times of one (key, val): runs longer than a merge
    tile's slack take k_mrg_tiles' single-thread walk and move tile boundaries across whole tiles; cancelling
    runs drop out.  The cases live in tools/merge_long_runs_check.py (also a stand-alone GPU check)."""
    import importlib.util

    spec = importlib.util.spec_from_file_location(
        "merge_long_runs_check", os.path.join(os.path.dirname(HERE), "tools", "merge_long_runs_check.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lines = []
    assert mod.run(mz, ctx, oracle, log=lines.append), "\n".join(lines)


# ----------------------------------------------------------- a6, a14
def test_spine_structure_and_contents_match_oracle(mz, ctx, oracle):
    rng = np.random.default_rng(23)
    gs, os_ = mz.Spine(ctx, 32), oracle.Spine(32, 1, gate_physical=True)
    t = 0
    for step in range(40):
        n = int(rng.choice([0, 1, 3, 50, 700, 5000]))
        a = rand_r32(rng, n, 500, 3, 1, dtype=oracle.R32)
        a["time"] = t
        g = mz.Batch.build(ctx, a, t, t + 1)
        o = oracle.Batch.build(a, t, t + 1)
        gs.insert(g)
        os_.insert(o)
        t += 1
        if step % 3 != 2:  # physical compaction lags on some steps: batches stay pending
            gs.set_physical_compaction(t)
            os_.set_physical_compaction(t)
        if step % 5 == 4:
            gs.set_logical_compaction(t - 1)
            os_.set_logical_compaction(t - 1)
        if step % 7 == 6:
            e = gs.exert_logic(16)
            assert e == os_.exert_logic(16)
            if e:
                assert gs.exert(e) == os_.exert(e)
        assert gs.layers() == os_.layers(), step
        assert gs.read_upper() == os_.read_upper()
        assert gs.num_batches_through(t) == os_.num_batches_through(t)
    same(gs.export(), os_.export())


# ----------------------------------------------------------------- a8 / a5
def test_batched_cursor_matches_the_oracle_batch(mz, ctx, oracle):
    """Cursor surface (a8): seek_key for many keys at once, step_key in pages, map_times over runs.
    A host-side cursor built from these calls walks the batch exactly as the oracle's OrdValBatch
    cursor does (same keys, same (val, time, diff) sequence per key)."""
    rng = np.random.default_rng(410)
    a = rand_r32(rng, 60000, 5000, 40, 6, dtype=oracle.R32)
    a["key"] *= np.uint64(0x9E3779B97F4A7C15 >> 20)  # spread over the u64 range, gaps between keys
    gb, ob = mz.Batch.build(ctx, a, 0, 6), oracle.Batch.build(a, 0, 6)
    rows = ob.rows()
    same(gb.rows(), rows)
    keys = np.unique(rows["key"])
    # seek: present keys, absent keys (gaps), below the first, beyond the last
    probe = np.concatenate([keys[::7], keys[::11] + np.uint64(1), [0, keys[0], keys[-1], keys[-1] + np.uint64(1), (1 << 64) - 1]]).astype(np.uint64)
    runs = gb.seek_keys(probe)
    for k, r in zip(probe.tolist(), runs):
        lo = int(np.searchsorted(rows["key"], np.uint64(k), side="left"))
        if lo == len(rows):
            assert int(r["len"]) == 0
            continue
        found = int(rows["key"][lo])
        hi = int(np.searchsorted(rows["key"], np.uint64(found), side="right"))
        assert (int(r["key"]), int(r["first"]), int(r["len"])) == (found, lo, hi - lo)
    assert len(gb.seek_keys(np.zeros(0, dtype=np.uint64))) == 0
    # step_key paging covers every distinct key once, in order, with its run
    pages, at = [], 0
    while True:
        pg = gb.key_page(at, 777)
        if len(pg) == 0:
            break
        pages.append(pg)
        at += len(pg)
    allk = np.concatenate(pages)
    assert allk["key"].tolist() == keys.tolist() and at == gb.keys()
    assert int(allk["len"].sum()) == len(rows)
    assert (allk["first"][1:] == allk["first"][:-1] + allk["len"][:-1]).all()
    # map_times over runs: the rows of a few key runs (and of several consecutive runs at once)
    for r in allk[:: max(1, len(allk) // 40)]:
        same(gb.rows_range(int(r["first"]), int(r["len"])), rows[int(r["first"]) : int(r["first"]) + int(r["len"])])
    same(gb.rows_range(int(allk["first"][3]), int(allk["len"][3:9].sum())), rows[int(allk["first"][3]) : int(allk["first"][9])])
    with pytest.raises(mz.MzGpuError):
        gb.rows_range(len(rows) - 1, 5)
    # an empty batch: every seek is at the end
    eb = mz.Batch.build(ctx, a[:0], 6, 7)
    assert int(eb.seek_keys(np.array([5], dtype=np.uint64))["len"][0]) == 0 and len(eb.key_page(0, 10)) == 0


def test_builder_push_done_matches_batch_build(mz, ctx, oracle):
    """Builder::{push, done} (a5): chunks pushed in any order seal into the batch the oracle builds
    from the same updates; the builder is reusable; sizes are reported per arrangement."""
    rng = np.random.default_rng(411)
    a = rand_r32(rng, 30000, 900, 12, 4, dtype=oracle.R32)
    bld = mz.Builder(ctx, 32, capacity=1000)
    for chunk in np.array_split(a, 7):
        bld.push(chunk)
    gb = bld.done(0, 4)
    ob = oracle.Batch.build(a, 0, 4)
    same(gb.rows(), ob.rows())
    assert gb.desc() == (0, 4, 0) and gb.keys() == ob.keys()
    # reuse, device-resident chunk, empty batch
    b2 = rand_r32(rng, 5000, 100, 3, 1, dtype=oracle.R32)
    b2["time"] += 4
    bld.push_buf(mz.DeviceRows(ctx, 32).upload(b2))
    g2 = bld.done(4, 5)
    same(g2.rows(), oracle.Batch.build(b2, 4, 5).rows())
    assert len(bld.done(5, 6)) == 0
    gs = mz.Spine(ctx, 32)
    gs.insert(gb)
    gs.insert(g2)
    gs.set_physical_compaction(5)
    sz = gs.size()
    assert sz["updates"] == len(gb) + len(g2) or sz["batches"] == 1  # (merged or not, nothing lost)
    assert sz["size_bytes"] >= 32 * sz["updates"] and sz["capacity_bytes"] >= sz["size_bytes"] - 16 * (gb.keys() + g2.keys())
    assert sz["allocations"] >= 2 * sz["batches"] and sz["batches"] >= 1


def test_join_core_yields_inside_a_work_item(mz, ctx, oracle):
    """mzgpu_join_core_work_until: a deadline in the past stops after ONE slice of one work item
    (the yield point inside a work item); repeated calls finish the work and the result equals
    the oracle's."""
    import time

    rng = np.random.default_rng(412)
    n = (1 << 20) + 50000  # more than one slice (every row distinct: nothing consolidates away)
    a = np.zeros(n, dtype=oracle.R32)
    a["key"] = rng.integers(0, 200000, size=n, dtype=np.uint64)
    a["val"] = np.arange(n, dtype=np.uint64) * np.uint64(16)
    a["diff"] = 1
    b = a[:70000].copy()
    b["val"] += np.uint64(3)
    g1, g2 = mz.Spine(ctx, 32), mz.Spine(ctx, 32)
    o1, o2 = oracle.Spine(32, 1, True), oracle.Spine(32, 1, True)
    ga, gbb = mz.Batch.build(ctx, a, 0, 1), mz.Batch.build(ctx, b, 0, 1)
    oa, obb = oracle.Batch.build(a, 0, 1), oracle.Batch.build(b, 0, 1)
    g2.insert(gbb)
    o2.insert(obb)
    gj, oj = mz.JoinCore(ctx, g1, g2), oracle.Join(o1, o2)
    g1.insert(ga)
    o1.insert(oa)
    gj.push(0, ga, 0)
    oj.push(0, oa, 0)
    calls, done = 0, False
    while not done:
        done = gj.work_until(1 << 62, 1)  # deadline long past: one slice per call
        calls += 1
        assert calls < 10
    assert calls >= 2  # the single work item took more than one call
    oj.work()
    same(oracle.consolidate(gj.results()), oracle.consolidate(oj.results()))
    # a generous deadline finishes in one call
    gj2 = mz.JoinCore(ctx, g1, g2)
    assert gj2.work_until(1 << 62, time.monotonic_ns() + 60_000_000_000)


# ----------------------------------------------------------------- a9
def brute_join(a, b, cap):
    """All pairs per key: (key, v1, v2, max(t1, t2, cap), d1*d2), consolidated by the caller."""
    out = []
    by_key = {}
    for r in b.tolist():
        by_key.setdefault(r[0], []).append(r)
    for k, v1, t1, d1 in a.tolist():
        for _, v2, t2, d2 in by_key.get(k, ()):
            out.append((k, v1, v2, max(t1, t2, cap), d1 * d2))
    return out


def test_join_core_matches_oracle_and_bruteforce(mz, ctx, oracle):
    rng = np.random.default_rng(24)
    g1, g2 = mz.Spine(ctx, 32), mz.Spine(ctx, 32)
    o1, o2 = oracle.Spine(32, 1, True), oracle.Spine(32, 1, True)
    gj, oj = mz.JoinCore(ctx, g1, g2), oracle.Join(o1, o2)
    all_a, all_b = [], []
    for t in range(6):
        for side, (gs, os_, acc) in enumerate([(g1, o1, all_a), (g2, o2, all_b)]):
            n = int(rng.integers(0, 3000))
            a = rand_r32(rng, n, 400, 6, 1, dtype=oracle.R32)
            a["time"] = t
            acc.append(a)
            gb, ob = mz.Batch.build(ctx, a, t, t + 1), oracle.Batch.build(a, t, t + 1)
            gs.insert(gb)
            os_.insert(ob)
            gj.push(side, gb, t)
            oj.push(side, ob, t)
        gj.work()
        oj.work()
    got = oracle.consolidate(gj.results())
    want = oracle.consolidate(oj.results())
    same(got, want)
    A, B = np.concatenate(all_a), np.concatenate(all_b)
    brute = oracle.consolidate(oracle.rows(oracle.R40, brute_join(oracle.consolidate(A), oracle.consolidate(B), 0)))
    same(got, brute)


def test_join_core_with_closure(mz, ctx, oracle):
    rng = np.random.default_rng(25)
    cl_args = dict(
        key_fields=[(0, 0, 64, 0)],
        val_fields=[(1, 0, 8, 0), (2, 0, 8, 8)],
        filters=[(2, 0, 3, "ne", 0)],
    )
    gcl, ocl = mz.make_closure(**cl_args), oracle.make_closure(**cl_args)
    g1, g2 = mz.Spine(ctx, 32), mz.Spine(ctx, 32)
    o1, o2 = oracle.Spine(32, 1, True), oracle.Spine(32, 1, True)
    gj, oj = mz.JoinCore(ctx, g1, g2, gcl), oracle.Join(o1, o2, ocl)
    for t in range(3):
        for side, (gs, os_) in enumerate([(g1, o1), (g2, o2)]):
            a = rand_r32(rng, 2000, 300, 200, 1, dtype=oracle.R32)
            a["time"] = t
            gb, ob = mz.Batch.build(ctx, a, t, t + 1), oracle.Batch.build(a, t, t + 1)
            gs.insert(gb)
            os_.insert(ob)
            gj.push(side, gb, t)
            oj.push(side, ob, t)
    gj.work()
    oj.work()
    same(oracle.consolidate(gj.results()), oracle.consolidate(oj.results()))


def test_linear_join_two_stages_matches_oracle_and_bruteforce(mz, ctx, oracle):
    """Row L: a linear join plan (src/compute/src/render/join/linear_join.rs:327-527) of three
    inputs -- stage 1 joins A and B by k1, its result is re-arranged by the next stage's key k2
    (the "JoinStage" arrangement: Batcher -> seal -> Spine) and stage 2 joins it with C by k2 --
    run incrementally over several timestamps with retractions.  The GPU operators and the
    oracle's produce the same stage-1 and final collections, and the accumulated final collection
    equals the brute-force three-way join of the accumulated inputs."""
    rng = np.random.default_rng(33)
    # A: (k1, a)   B: (k1, k2 << 20 | b)   C: (k2, c)
    cl1 = dict(key_fields=[(2, 20, 10, 0)], val_fields=[(1, 0, 20, 0), (2, 0, 20, 20)])  # key' = k2, val' = a | b << 20
    cl2 = dict(key_fields=[(0, 0, 10, 0)], val_fields=[(1, 0, 40, 0), (2, 0, 20, 40)])  # val'' = a | b << 20 | c << 40
    g = dict(A=mz.Spine(ctx, 32), B=mz.Spine(ctx, 32), S=mz.Spine(ctx, 32), C=mz.Spine(ctx, 32))
    o = dict(A=oracle.Spine(32, 1, True), B=oracle.Spine(32, 1, True), S=oracle.Spine(32, 1, True), C=oracle.Spine(32, 1, True))
    gj1, oj1 = mz.JoinCore(ctx, g["A"], g["B"], mz.make_closure(**cl1)), oracle.Join(o["A"], o["B"], oracle.make_closure(**cl1))
    gj2, oj2 = mz.JoinCore(ctx, g["S"], g["C"], mz.make_closure(**cl2)), oracle.Join(o["S"], o["C"], oracle.make_closure(**cl2))
    gstage, ostage = mz.Batcher(ctx, 32), oracle.Batcher(32)
    acc = dict(A=[], B=[], C=[])
    g1_seen = o1_seen = g2_seen = o2_seen = 0
    for t in range(6):
        ins = {}
        for name, (kh, n) in dict(A=(60, 500), B=(60, 400), C=(40, 300)).items():
            x = np.zeros(n, dtype=oracle.R32)
            x["key"] = rng.integers(0, kh, size=n, dtype=np.uint64)
            x["val"] = rng.integers(0, 50, size=n, dtype=np.uint64)
            if name == "B":
                x["val"] |= rng.integers(0, 40, size=n, dtype=np.uint64) << np.uint64(20)
            x["time"] = t
            x["diff"] = rng.integers(-1, 3, size=n)
            if t >= 2 and acc[name]:  # retract some of what an earlier timestamp added
                old = acc[name][t - 2][:100].copy()
                old["time"] = t
                old["diff"] = -old["diff"]
                x = np.concatenate([x, old])
            ins[name] = x
            acc[name].append(x)
        # stage 1
        for side, name in enumerate(("A", "B")):
            gb, ob = mz.Batch.build(ctx, ins[name], t, t + 1), oracle.Batch.build(ins[name], t, t + 1)
            g[name].insert(gb)
            o[name].insert(ob)
            gj1.push(side, gb, t)
            oj1.push(side, ob, t)
        gj1.work()
        oj1.work()
        gr, orr = gj1.results(), oj1.results()
        g_new, o_new = gr[g1_seen:], orr[o1_seen:]
        g1_seen, o1_seen = len(gr), len(orr)
        same(oracle.consolidate(g_new), oracle.consolidate(o_new))
        # the stage arrangement ("JoinStage"): re-arrange the running result by k2
        gstage.push_container(g_new)
        ostage.push(o_new)
        gsb, osb = gstage.seal(t + 1), ostage.seal(t + 1)
        same(gsb.rows(), osb.rows())
        g["S"].insert(gsb)
        o["S"].insert(osb)
        gj2.push(0, gsb, t)
        oj2.push(0, osb, t)
        gc, oc = mz.Batch.build(ctx, ins["C"], t, t + 1), oracle.Batch.build(ins["C"], t, t + 1)
        g["C"].insert(gc)
        o["C"].insert(oc)
        gj2.push(1, gc, t)
        oj2.push(1, oc, t)
        gj2.work()
        oj2.work()
        gr2, or2 = gj2.results(), oj2.results()
        same(oracle.consolidate(gr2[g2_seen:]), oracle.consolidate(or2[o2_seen:]))
        g2_seen, o2_seen = len(gr2), len(or2)
        for sp in list(g.values()) + list(o.values()):
            sp.set_physical_compaction(t + 1)
    # accumulated final collection (times collapsed) == brute-force three-way join
    final = gj2.results().copy()
    final["time"] = 0
    final = oracle.consolidate(final)
    A, B, Cc = (np.concatenate(acc[n]) for n in ("A", "B", "C"))
    for x in (A, B, Cc):
        x["time"] = 0
    A, B, Cc = oracle.consolidate(A), oracle.consolidate(B), oracle.consolidate(Cc)
    by_b, by_c = {}, {}
    for k, v, _, d in B.tolist():
        by_b.setdefault(k, []).append((v >> 20, v & 0xFFFFF, d))
    for k, v, _, d in Cc.tolist():
        by_c.setdefault(k, []).append((v, d))
    want = {}
    for k1, a, _, da in A.tolist():
        for k2, b, db in by_b.get(k1, ()):
            for c, dc in by_c.get(k2, ()):
                key = (k2, a | (b << 20) | (c << 40))
                want[key] = want.get(key, 0) + da * db * dc
    want = sorted((k, v, 0, d) for (k, v), d in want.items() if d != 0)
    assert [tuple(r) for r in final.tolist()] == want


def test_linear_join_plan_operator_matches_oracle_composition(mz, ctx, oracle):
    """Row L through the boundary's plan descriptor: `mzgpu_linear_join_{new, step}` renders a two-stage
    LinearJoinPlan (source A; stage 0: lookup B by k1, closure re-keys by k2; stage 1: lookup C by k2; a final
    closure that filters and projects) itself -- key preparation, the "JoinStage" arrangements, mz_join_core per
    stage (src/compute/src/render/join/linear_join.rs:230-527) -- and produces, activation by activation, the
    collection the same plan composed by hand from the oracle's operators produces; accumulated, that is the
    brute-force three-way join behind the final closure."""
    rng = np.random.default_rng(34)
    ident = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 64, 0)])
    cl1 = dict(key_fields=[(2, 20, 10, 0)], val_fields=[(1, 0, 20, 0), (2, 0, 20, 20)])  # key' = k2, val' = a | b << 20
    cl2 = dict(key_fields=[(0, 0, 10, 0)], val_fields=[(1, 0, 40, 0), (2, 0, 20, 40)])  # val'' = a | b << 20 | c << 40
    fin = dict(key_fields=[(0, 0, 10, 0)], val_fields=[(1, 20, 40, 0)], filters=[(1, 0, 20, "lt", 40)])  # a < 40; keep b, c
    gB, gC = mz.Spine(ctx, 32), mz.Spine(ctx, 32)
    lj = mz.LinearJoin(ctx, [(gB, mz.make_closure(**ident), mz.make_closure(**cl1)), (gC, mz.make_closure(**ident), mz.make_closure(**cl2))],
                       final_closure=mz.make_closure(**fin))
    o = dict(A=oracle.Spine(32, 1, True), B=oracle.Spine(32, 1, True), S=oracle.Spine(32, 1, True), C=oracle.Spine(32, 1, True))
    oj1 = oracle.Join(o["A"], o["B"], oracle.make_closure(**cl1))
    oj2 = oracle.Join(o["S"], o["C"], oracle.make_closure(**cl2))
    ostage = oracle.Batcher(32)
    acc = dict(A=[], B=[], C=[])
    o1_seen = o2_seen = 0
    got_all = []
    for t in range(7):
        ins = {}
        for name, (kh, n) in dict(A=(60, 500), B=(60, 400), C=(40, 300)).items():
            x = np.zeros(n if not (name == "C" and t == 3) else 0, dtype=oracle.R32)  # C is silent at t = 3
            x["key"] = rng.integers(0, kh, size=len(x), dtype=np.uint64)
            x["val"] = rng.integers(0, 50, size=len(x), dtype=np.uint64)
            if name == "B":
                x["val"] |= rng.integers(0, 40, size=len(x), dtype=np.uint64) << np.uint64(20)
            x["time"] = t
            x["diff"] = rng.integers(-1, 3, size=len(x))
            if t >= 2 and len(acc[name][t - 2]):
                old = acc[name][t - 2][:100].copy()
                old["time"] = t
                old["diff"] = -old["diff"]
                x = np.concatenate([x, old])
            ins[name] = x
            acc[name].append(x)
        # the oracle's composition of the same plan
        for side, name in enumerate(("A", "B")):
            ob = oracle.Batch.build(ins[name], t, t + 1)
            o[name].insert(ob)
            oj1.push(side, ob, t)
        oj1.work()
        orr = oj1.results()
        o_new, o1_seen = orr[o1_seen:], len(orr)
        ostage.push(o_new)
        osb = ostage.seal(t + 1)
        o["S"].insert(osb)
        oj2.push(0, osb, t)
        oc = oracle.Batch.build(ins["C"], t, t + 1)
        o["C"].insert(oc)
        oj2.push(1, oc, t)
        oj2.work()
        or2 = oj2.results()
        want = oracle.consolidate(oracle.map_rows(or2[o2_seen:], oracle.make_closure(**fin)))
        o2_seen = len(or2)
        # the operator: the lookup batches go into the caller's arrangements, then one activation
        gb, gc = mz.Batch.build(ctx, ins["B"], t, t + 1), mz.Batch.build(ctx, ins["C"], t, t + 1)
        gB.insert(gb)
        gC.insert(gc)
        got = lj.step(ins["A"], [gb, gc], t + 1)
        same(oracle.consolidate(got), want)
        got_all.append(got)
        for sp in o.values():
            sp.set_physical_compaction(t + 1)
    final = np.concatenate(got_all)
    final["time"] = 0
    final = oracle.consolidate(final)
    A, B, Cc = (np.concatenate(acc[n]) for n in ("A", "B", "C"))
    for x in (A, B, Cc):
        x["time"] = 0
    A, B, Cc = oracle.consolidate(A), oracle.consolidate(B), oracle.consolidate(Cc)
    by_b, by_c = {}, {}
    for k, v, _, d in B.tolist():
        by_b.setdefault(k, []).append((v >> 20, v & 0xFFFFF, d))
    for k, v, _, d in Cc.tolist():
        by_c.setdefault(k, []).append((v, d))
    want = {}
    for k1, a, _, da in A.tolist():
        if a >= 40:
            continue
        for k2, b, db in by_b.get(k1, ()):
            for c, dc in by_c.get(k2, ()):
                key = (k2, b | (c << 20))
                want[key] = want.get(key, 0) + da * db * dc
    want = sorted((k, v, 0, d) for (k, v), d in want.items() if d != 0)
    assert [tuple(r) for r in final.tolist()] == want
    # plans the descriptor cannot hold are refused at render time
    with pytest.raises(mz.MzGpuError):
        mz.LinearJoin(ctx, [])
    with pytest.raises(mz.MzGpuError):
        mz.LinearJoin(ctx, [(gB, mz.make_closure(**ident), mz.make_closure(**cl1))] * 7)


# ---------------------------------------------------------------- a10
@pytest.mark.parametrize("cmp_mode", [0, 1])
def test_half_join_matches_oracle(mz, ctx, oracle, cmp_mode):
    rng = np.random.default_rng(26 + cmp_mode)
    gs, os_ = mz.Spine(ctx, 32), oracle.Spine(32, 1, True)
    for t in range(5):
        a = rand_r32(rng, 4000, 500, 1 << 20, 1, dtype=oracle.R32)
        a["time"] = t
        gs.insert(mz.Batch.build(ctx, a, t, t + 1))
        os_.insert(oracle.Batch.build(a, t, t + 1))
        gs.set_physical_compaction(t + 1)
        os_.set_physical_compaction(t + 1)
    stream = rand_r32(rng, 6000, 600, 1 << 20, 6, dtype=oracle.R32)
    cl_args = dict(
        key_fields=[(2, 0, 10, 0)],
        val_fields=[(1, 0, 20, 0), (2, 10, 10, 20), (0, 0, 10, 40)],
        filters=[(2, 0, 20, "lt", 900000)],
    )
    for closure_args in (None, cl_args):
        gcl = mz.make_closure(**closure_args) if closure_args else None
        ocl = oracle.make_closure(**closure_args) if closure_args else None
        got = mz.half_join(ctx, stream, gs, cmp_mode, gcl)
        want = oracle.half_join(stream, os_, cmp_mode, ocl)
        same(got, want)


def test_half_join_many_matches_single_half_joins(mz, ctx, oracle):
    """mzgpu_half_join_many: independent half joins of one stage in one launch; requests naming the
    same output form a chain and append in request order (the concatenated outputs of the delta
    paths' last stage) -- row for row what the single calls produce."""
    rng = np.random.default_rng(77)
    spines = []
    for sp in range(3):
        gs = mz.Spine(ctx, 32)
        for t in range(3 + sp):
            a = rand_r32(rng, 3000, 400 + 100 * sp, 1 << 20, 1, dtype=oracle.R32)
            a["time"] = t
            gs.insert(mz.Batch.build(ctx, a, t, t + 1))
            gs.set_physical_compaction(t + 1)
        spines.append(gs)
    streams = [rand_r32(rng, n, 600, 1 << 20, 8, dtype=oracle.R32) for n in (5000, 1, 777)]
    cl = mz.make_closure(key_fields=[(2, 0, 10, 0)], val_fields=[(1, 0, 20, 0), (2, 10, 10, 20)], filters=[(2, 0, 20, "lt", 900000)])
    closures = [None, cl, cl]
    cmps = [mz.HALFJOIN_LE, mz.HALFJOIN_LT, mz.HALFJOIN_LE]
    devs = [mz.DeviceRows(ctx, 32).upload(s) for s in streams]
    # (a) three independent outputs, (b) chain of two + one apart, (c) one chain of three
    for layout in ([0, 1, 2], [0, 0, 1], [0, 0, 0]):
        outs = [mz.DeviceRows(ctx, 32) for _ in range(3)]
        want = [mz.DeviceRows(ctx, 32) for _ in range(3)]
        # something already in the buffers: appends must start behind it
        for o, w in zip(outs, want):
            o.upload(streams[1])
            w.upload(streams[1])
        mz.half_join_many(ctx, [(devs[j], spines[j], cmps[j], closures[j], outs[layout[j]]) for j in range(3)])
        for j in range(3):
            mz.half_join_dev(ctx, devs[j], spines[j], cmps[j], closures[j], False, want[layout[j]])
        for o, w in zip(outs, want):
            same(o.download(), w.download())


def test_delta_first_stage_many_matches_separate_operators(mz, ctx, oracle):
    """mzgpu_delta_first_stage_many = update_stream (as_of skip + initial closure) then half_join,
    for one and for several paths, including paths that share the output collection."""
    rng = np.random.default_rng(78)
    spines, batches = [], []
    for sp in range(3):
        gs = mz.Spine(ctx, 32)
        for t in range(2 + sp):
            a = rand_r32(rng, 3000, 400, 1 << 20, 1, dtype=oracle.R32)
            a["time"] = t
            gs.insert(mz.Batch.build(ctx, a, t, t + 1))
            gs.set_physical_compaction(t + 1)
        spines.append(gs)
        b = rand_r32(rng, (4000, 2, 900)[sp], 500, 1 << 20, 3, dtype=oracle.R32)
        batches.append(mz.Batch.build(ctx, b, 0, 3))
    init = mz.make_closure(key_fields=[(1, 0, 9, 0)], val_fields=[(0, 0, 20, 0)], filters=[(1, 0, 20, "lt", 800000)])
    stage = mz.make_closure(key_fields=[(2, 0, 10, 0)], val_fields=[(1, 0, 20, 0), (2, 10, 10, 20)])
    inits = [init, None, init]
    skips = [mz.FRONTIER_EMPTY, 0, 1]
    cmps = [mz.HALFJOIN_LE, mz.HALFJOIN_LT, mz.HALFJOIN_LE]
    for k, layout in ((1, [0]), (3, [0, 1, 2]), (3, [0, 0, 0]), (2, [0, 0])):
        outs = [mz.DeviceRows(ctx, 32) for _ in range(3)]
        want = [mz.DeviceRows(ctx, 32) for _ in range(3)]
        mz.delta_first_stage_many(
            ctx, [(batches[j], inits[j], skips[j], spines[j], cmps[j], stage, outs[layout[j]]) for j in range(k)]
        )
        for j in range(k):
            stream = mz.update_stream_dev(ctx, batches[j], inits[j], skips[j])
            mz.half_join_dev(ctx, stream, spines[j], cmps[j], stage, False, want[layout[j]])
        for o, w in zip(outs, want):
            same(o.download(), w.download())


def test_update_stream_and_map_rows(mz, ctx, oracle):
    rng = np.random.default_rng(28)
    a = rand_r32(rng, 5000, 100, 1 << 12, 3, dtype=oracle.R32)
    cl_args = dict(key_fields=[(1, 0, 6, 0)], val_fields=[(0, 0, 64, 0)], filters=[(1, 6, 6, "ge", 10)])
    gcl, ocl = mz.make_closure(**cl_args), oracle.make_closure(**cl_args)
    gb, ob = mz.Batch.build(ctx, a, 0, 3), oracle.Batch.build(a, 0, 3)
    for skip in (mz.FRONTIER_EMPTY, 0, 1):
        same(mz.update_stream(ctx, gb, gcl, skip), oracle.update_stream(ob, ocl, skip))
        same(mz.update_stream(ctx, gb, None, skip), oracle.update_stream(ob, None, skip))
    same(mz.map_rows(ctx, a, gcl), oracle.map_rows(a, ocl))


def test_gpu_operators_reproduce_sqllogictest_answers(mz, ctx, oracle):
    """The reference-held SQL answers (tests/golden/sqllogictest_join_reduce.json: joins.slt /
    aggregates.slt, integer-only cases) computed with the GPU operators through the C ABI."""
    import sql_golden as sg

    fx = sg.load()
    gops, oops = sg.GpuOps(mz, ctx), sg.OracleOps(oracle)
    for case in fx["cases"]:
        if case["shape"] == "sum_of_nulls":
            continue  # NULL inputs are outside the ABI's fixed-width subset (pinned on finalize_accum, CPU suite)
        got = sg.norm(sg.evaluate(gops, case, fx["tables"]))
        assert got == sg.norm([tuple(r) for r in case["expect"]]), (case["name"], case["cite"], got)
        assert got == sg.norm(sg.evaluate(oops, case, fx["tables"]))


def test_malformed_closures_are_rejected_at_plan_time(mz, ctx):
    """Closure descriptors are caller data: counts beyond the descriptor, shifts >= 64, zero-width
    fields, unknown sources / operators / expression kinds never reach a kernel (mzgpu.h: E_INVALID
    for malformed descriptors, E_UNSUPPORTED for plans outside the subset)."""
    from materialize_b200 import _ffi as F

    a = rand_r32(np.random.default_rng(5), 64, 100, 100, 3, dtype=mz.R32)
    good = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 64, 0)])

    def bad(mutate):
        c = mz.make_closure(**good)
        mutate(c)
        return c

    cases = [
        (bad(lambda c: setattr(c, "n_key_fields", 7)), F.E_UNSUPPORTED),
        (bad(lambda c: setattr(c, "n_val_fields", 100)), F.E_UNSUPPORTED),
        (bad(lambda c: setattr(c, "n_filters", 5)), F.E_UNSUPPORTED),
        (bad(lambda c: setattr(c, "expr_kind", 9)), F.E_UNSUPPORTED),
        (bad(lambda c: setattr(c.key_fields[0], "shift", 64)), F.E_INVALID),
        (bad(lambda c: setattr(c.key_fields[0], "bits", 0)), F.E_INVALID),
        (bad(lambda c: setattr(c.key_fields[0], "bits", 65)), F.E_INVALID),
        (bad(lambda c: setattr(c.val_fields[0], "dst_shift", 64)), F.E_INVALID),
        (bad(lambda c: setattr(c.val_fields[0], "src", 3)), F.E_INVALID),
    ]
    flt = mz.make_closure(filters=[(0, 0, 8, "ge", 1)], **good)
    flt.filters[0].op = 6
    cases.append((flt, F.E_UNSUPPORTED))
    gb = mz.Batch.build(ctx, a, 0, 3)
    gs = mz.Spine(ctx, 32)
    gs.insert(gb)
    for c, code in cases:
        for call in (
            lambda: mz.map_rows(ctx, a, c),
            lambda: mz.update_stream(ctx, gb, c),
            lambda: mz.half_join(ctx, a, gs, mz.HALFJOIN_LE, c),
            lambda: mz.JoinCore(ctx, gs, gs, c),
        ):
            with pytest.raises(mz.MzGpuError) as e:
                call()
            assert e.value.status == code, (e.value.status, code)
    # the context is still usable (nothing sticky)
    same(mz.map_rows(ctx, a, mz.make_closure(**good)), mz.map_rows(ctx, a, mz.make_closure(**good)))


# ----------------------------------------------------------- a11, a12
@pytest.mark.parametrize("agg_kind", [0, 1])
def test_reduce_accumulable_matches_oracle(mz, ctx, oracle, agg_kind):
    rng = np.random.default_rng(29 + agg_kind)
    gr, orr = mz.ReduceAccumulable(ctx, agg_kind), oracle.Reduce(agg_kind)
    live = []
    t = 0
    for step in range(8):
        n = int(rng.integers(1, 4000))
        a = np.zeros(n, dtype=oracle.R32)
        a["key"] = rng.integers(0, 300, size=n, dtype=np.uint64)
        if agg_kind == 0:
            a["val"] = rng.integers(-(10**6), 10**6, size=n, dtype=np.int64).astype(np.uint64)
        else:
            v = rng.integers(-(10**6), 10**6, size=n).astype(np.float64) / 7.0
            special = rng.integers(0, 200, size=n)
            v[special == 0] = np.nan
            v[special == 1] = np.inf
            v[special == 2] = -np.inf
            v[special == 3] = 1e300
            a["val"] = v.view(np.uint64)
        a["time"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        a["diff"] = 1
        # retract roughly half of what is live
        if live and step % 2 == 1:
            old = np.concatenate(live)
            pick = old[rng.random(len(old)) < 0.5].copy()
            pick["diff"] = -1
            pick["time"] = rng.integers(t, t + 3, size=len(pick), dtype=np.uint64)
            a = np.concatenate([a, pick])
            live = []
        else:
            live.append(a.copy())
        t += 3
        got, want = gr.step(a, t), orr.step(a, t)
        same(got, want)
    # the accumulated arrangement matches too
    same(gr.input_trace().export(), oracle.consolidate(gr.input_trace().export()))


@pytest.mark.parametrize("agg_kind", [2, 3])
def test_reduce_distinct_and_threshold_match_oracle(mz, ctx, oracle, agg_kind):
    """ReducePlan::Distinct (reduce.rs:264-334) and ThresholdPlan::Basic (threshold.rs:33-77) as
    instances of the same reduce operator: multiplicities go negative, return to zero, recover."""
    rng = np.random.default_rng(50 + agg_kind)
    gr, orr = mz.ReduceAccumulable(ctx, agg_kind), oracle.Reduce(agg_kind)
    t = 0
    for step in range(10):
        n = int(rng.integers(1, 5000))
        a = np.zeros(n, dtype=oracle.R32)
        a["key"] = rng.integers(0, 400, size=n, dtype=np.uint64)
        a["val"] = rng.integers(0, 1 << 30, size=n, dtype=np.uint64)  # ignored by both plans
        a["time"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        a["diff"] = rng.integers(-3, 4, size=n, dtype=np.int64)
        t += 3
        same(gr.step(a, t), orr.step(a, t))


@pytest.mark.parametrize("agg_kind", [4, 5])
def test_reduce_min_max_match_oracle(mz, ctx, oracle, agg_kind):
    """MIN / MAX: the hierarchical reduce's result (reduce.rs:796-1135): values retract, the
    extremum moves both ways, groups empty out and come back, negative counts give the error row."""
    rng = np.random.default_rng(70 + agg_kind)
    gr, orr = mz.ReduceAccumulable(ctx, agg_kind), oracle.Reduce(agg_kind)
    t = 0
    saw_err = False
    for step in range(12):
        n = int(rng.integers(1, 6000))
        a = np.zeros(n, dtype=oracle.R32)
        a["key"] = rng.integers(0, 500, size=n, dtype=np.uint64)
        a["val"] = rng.integers(0, 14, size=n, dtype=np.uint64) * np.uint64(0x1234567890ABCDEF)
        a["time"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        a["diff"] = rng.integers(-1, 3, size=n, dtype=np.int64)
        t += 3
        got, want = gr.step(a, t), orr.step(a, t)
        same(got, want)
        saw_err = saw_err or bool((want["flags"] == 2).any())
    assert saw_err


@pytest.mark.parametrize(
    "limit,offset,desc", [(1, 0, False), (3, 0, True), (2, 1, False), (None, 2, True), (0, 0, False), (40, 0, False)]
)
def test_topk_matches_oracle(mz, ctx, oracle, limit, offset, desc):
    """TopK per key (top_k.rs:215-248, 521-673): windows shift as values arrive and retract, offsets
    eat multiplicities, limits cut inside a value's copies, negative counts give the error row."""
    rng = np.random.default_rng(90 + (limit or 0) + offset)
    gr = mz.TopK(ctx, limit, offset, desc)
    orr = oracle.TopK(-1 if limit is None else limit, offset, desc)
    t = 0
    for step in range(10):
        n = int(rng.integers(1, 5000))
        a = np.zeros(n, dtype=oracle.R32)
        a["key"] = rng.integers(0, 400, size=n, dtype=np.uint64)
        a["val"] = rng.integers(0, 12, size=n, dtype=np.uint64) * np.uint64(0x0123456789ABCDEF)
        a["time"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        a["diff"] = rng.integers(-1, 3, size=n, dtype=np.int64)
        t += 3
        same(gr.step(a, t), orr.step(a, t))


@pytest.mark.parametrize("agg_kind", [4, 5])
def test_reduce_min_max_wide_groups_match_oracle(mz, ctx, oracle, agg_kind):
    """Groups with 10^3 .. 10^5 distinct live values (the reference's bucketed reduction tree,
    reduce.rs:796-1135, exists for these): values arrive over several batches and timestamps, the
    extremum is retracted and comes back, whole prefixes of the value range cancel, a negative
    count appears and is repaired.  Narrow keys in the same batches keep the table path."""
    rng = np.random.default_rng(700 + agg_kind)
    gr, orr = mz.ReduceAccumulable(ctx, agg_kind), oracle.Reduce(agg_kind)
    widths = {11: 1000, 12: 20000, 13: 100000}
    t = 0
    live = {k: np.zeros(0, dtype=np.uint64) for k in widths}
    broken = {}
    for step in range(7):
        parts = []
        for k, wdt in widths.items():
            n = wdt // 4 if step < 4 else wdt // 50
            v = rng.integers(0, 1 << 40, size=n, dtype=np.uint64)
            x = np.zeros(n, dtype=oracle.R32)
            x["key"], x["val"], x["diff"] = k, v, 1
            x["time"] = rng.integers(t, t + 2, size=n, dtype=np.uint64)
            parts.append(x)
            live[k] = np.concatenate([live[k], v])
            if step in (2, 4, 5) and len(live[k]):
                # retract the current extremum's neighbourhood (the smallest / largest 5 %) ...
                srt = np.sort(live[k])
                cut = srt[: len(srt) // 20] if agg_kind == 4 else srt[-(len(srt) // 20) :]
                y = np.zeros(len(cut), dtype=oracle.R32)
                y["key"], y["val"], y["diff"], y["time"] = k, cut, -1, t + 1
                parts.append(y)
                live[k] = np.setdiff1d(live[k], cut)
            if step == 3:
                # ... and one value (far from the extremum) more often than it was inserted: the
                # error row, repaired at step 4
                broken[k] = live[k].max() if agg_kind == 4 else live[k].min()
                z = np.zeros(1, dtype=oracle.R32)
                z["key"], z["val"], z["diff"], z["time"] = k, broken[k], -2, t
                parts.append(z)
            if step == 4:
                z = np.zeros(1, dtype=oracle.R32)
                z["key"], z["val"], z["diff"], z["time"] = k, broken[k], 2, t
                parts.append(z)
        nar = rand_r32(rng, 3000, 300, 9, 1, dtype=oracle.R32)
        nar["key"] += np.uint64(1000)
        nar["time"] = t
        nar["diff"] = rng.integers(-1, 3, size=len(nar))
        parts.append(nar)
        a = np.concatenate(parts)
        t += 2
        got, want = gr.step(a, t), orr.step(a, t)
        same(got, want)
        if step == 3:
            assert (want["flags"][np.isin(want["key"], list(widths))] == 2).any()


def test_topk_wide_groups_match_oracle(mz, ctx, oracle):
    """TopK on groups of thousands of distinct values: limits up to 32 take any group width (the
    window is found by the value-ordered merge of the key's runs); a window wider than 32
    distinct values on a wide group is reported as unsupported, never wrong."""
    rng = np.random.default_rng(720)
    for limit, offset, desc in ((1, 0, False), (5, 3, True), (32, 100, False)):
        gr, orr = mz.TopK(ctx, limit, offset, desc), oracle.TopK(limit, offset, desc)
        t = 0
        for step in range(4):
            n = 6000
            a = np.zeros(n, dtype=oracle.R32)
            a["key"] = rng.integers(0, 3, size=n, dtype=np.uint64)
            a["val"] = rng.integers(0, 4000, size=n, dtype=np.uint64)
            a["time"] = rng.integers(t, t + 2, size=n, dtype=np.uint64)
            a["diff"] = rng.integers(0, 3, size=n) if step != 2 else -rng.integers(0, 2, size=n)
            t += 2
            same(gr.step(a, t), orr.step(a, t))
    priv = mz.Context(0)  # (the report is deferred and poisons the context, hence a private one)
    a = np.zeros(100, dtype=oracle.R32)
    a["key"], a["val"], a["diff"] = 7, np.arange(100), 1
    with pytest.raises(mz.MzGpuError) as e:
        mz.TopK(priv, 40, 0, False).step(a, 1)
    assert e.value.status == -4  # MZGPU_E_UNSUPPORTED


def test_reduce_large_i128_sums(mz, ctx, oracle):
    """i128 accumulation with carries: sums far beyond i64."""
    a = np.zeros(40000, dtype=oracle.R32)
    a["key"] = np.arange(40000) % 3
    a["val"] = np.uint64(2**63 - 1)
    a["time"] = 0
    a["diff"] = 3
    gr, orr = mz.ReduceAccumulable(ctx, 0), oracle.Reduce(0)
    got, want = gr.step(a, 1), orr.step(a, 1)
    same(got, want)
    assert int(got["sum_hi"][0]) > 0
    a["diff"] = -3
    a["time"] = 1
    same(gr.step(a, 2), orr.step(a, 2))


# ------------------------------------------------------------ edge cases
def test_empty_inputs_everywhere(mz, ctx, oracle):
    """Zero-row inputs through every entry point (empty containers are routine in timely)."""
    e32 = np.zeros(0, dtype=oracle.R32)
    e16 = np.zeros(0, dtype=oracle.R16)
    same(ctx.consolidate(e32), e32)
    same(ctx.consolidate(e16), e16)
    gb, ob = mz.Batcher(ctx, 32), oracle.Batcher(32)
    gb.push_container(e32)
    ob.push(e32)
    g, o = gb.seal(3), ob.seal(3)
    same(g.rows(), o.rows())
    assert len(g) == 0 and g.desc() == o.desc() and gb.frontier() == ob.frontier() == mz.FRONTIER_EMPTY
    gs, os_ = mz.Spine(ctx, 32), oracle.Spine(32, 1, True)
    gs.insert(g)
    os_.insert(o)
    gs.set_physical_compaction(3)
    os_.set_physical_compaction(3)
    assert gs.layers() == os_.layers()
    # probes: empty stream against a non-empty trace, non-empty stream against an empty trace
    rng = np.random.default_rng(41)
    a = rand_r32(rng, 500, 50, 1 << 10, 1, dtype=oracle.R32)
    a["time"] = 3
    same(mz.half_join(ctx, a, gs, 0), oracle.half_join(a, os_, 0))
    gs.insert(mz.Batch.build(ctx, a, 3, 4))
    os_.insert(oracle.Batch.build(a, 3, 4))
    same(mz.half_join(ctx, e32, gs, 1), oracle.half_join(e32, os_, 1))
    same(mz.update_stream(ctx, g), oracle.update_stream(o))
    same(mz.map_rows(ctx, e32, None), e32)
    # reduce: an activation without input, then one whose input cancels completely
    gr, orr = mz.ReduceAccumulable(ctx, 0), oracle.Reduce(0)
    same(gr.step(e32, 1), orr.step(e32, 1))
    b = rand_r32(rng, 300, 20, 1 << 10, 1, dtype=oracle.R32)
    b["time"] = 1
    b["diff"] = 1
    c = b.copy()
    c["diff"] = -1
    both = np.concatenate([b, c])
    same(gr.step(both, 2), orr.step(both, 2))
    assert len(ctx.consolidate(both)) == 0
    same(gr.step(b, 3), orr.step(b, 3))
    # merge of two empty batches, and of an empty with a non-empty one
    m1 = mz.Batch.build(ctx, e32, 0, 1).merge(mz.Batch.build(ctx, e32, 1, 2), 0)
    assert len(m1) == 0 and m1.desc() == (0, 2, 0)
    m2 = mz.Batch.build(ctx, e32, 0, 1).merge(mz.Batch.build(ctx, a, 1, 4), 2)
    o2 = oracle.Batch.build(e32, 0, 1).merge(oracle.Batch.build(a, 1, 4), 2)
    same(m2.rows(), o2.rows())


def test_extreme_values_and_single_rows(mz, ctx, oracle):
    """u64 extremes in every key word, i64 extremes and wrapping in the diffs, one-row inputs."""
    M = 2**64 - 1
    rows = [(0, 0, 0, 1), (M, M, 7, -1), (M, 0, 7, 2**63 - 1), (M, 0, 7, 2**63 - 1), (0, M, 0, -(2**63)),
            (0, M, 0, -(2**63)), (1, 1, 1, 5), (1, 1, 1, -5), (M - 1, M - 1, 6, 3)]
    a = oracle.rows(oracle.R32, rows)
    same(ctx.consolidate(a), oracle.consolidate(a))
    one = oracle.rows(oracle.R32, [(M, M, 5, -7)])
    same(ctx.consolidate(one), one)
    g, o = mz.Batch.build(ctx, a, 0, 8), oracle.Batch.build(a, 0, 8)
    same(g.rows(), o.rows())
    assert g.keys() == o.keys()
    gs, os_ = mz.Spine(ctx, 32), oracle.Spine(32, 1, True)
    gs.insert(g)
    os_.insert(o)
    stream = oracle.rows(oracle.R32, [(M, 9, 8, 2), (0, 9, 8, -3), (5, 9, 8, 1), (M - 1, 9, 8, 2**62)])
    for cmp_mode in (0, 1):
        same(mz.half_join(ctx, stream, gs, cmp_mode), oracle.half_join(stream, os_, cmp_mode))
    r16 = oracle.rows(oracle.R16, [(M, 1), (0, -1), (M, -1), (0, 2**63 - 1), (0, 2**63 - 1), (7, 0)])
    same(ctx.consolidate(r16), oracle.consolidate(r16))


def test_hash_index_collisions(mz, ctx, oracle):
    """Many distinct keys packed into few hash slots' neighbourhoods (long linear-probe chains):
    a batch of dense keys 0..n-1 fills its open-addressing table to the 0.5 load factor; every key
    and a comparable number of absent keys are probed."""
    rng = np.random.default_rng(43)
    n = 70000
    a = np.zeros(n, dtype=oracle.R32)
    a["key"] = np.arange(n, dtype=np.uint64) * np.uint64(1 << 20)  # same low bits: the mixer must spread them
    a["val"] = rng.integers(0, 1 << 30, size=n, dtype=np.uint64)
    a["diff"] = 1
    gs, os_ = mz.Spine(ctx, 32), oracle.Spine(32, 1, True)
    gs.insert(mz.Batch.build(ctx, a, 0, 1))
    os_.insert(oracle.Batch.build(a, 0, 1))
    stream = np.zeros(2 * n, dtype=oracle.R32)
    stream["key"] = np.concatenate([a["key"], a["key"] + np.uint64(1)])
    stream["val"] = np.arange(2 * n, dtype=np.uint64)
    stream["time"] = 1
    stream["diff"] = 1
    rng.shuffle(stream)
    same(mz.half_join(ctx, stream, gs, 0), oracle.half_join(stream, os_, 0))


# ------------------------------------------ device-resident operator chaining
def test_chained_operators_no_readback(mz, ctx, oracle):
    """arrange -> update_stream -> half_join x2 -> reduce with every intermediate in a device
    buffer (the *_buf entry points): same output as the oracle, and the host waits for the
    device only a handful of times for the whole chain."""
    rng = np.random.default_rng(31)
    n = 6000
    look1 = rand_r32(rng, 5000, 800, 1 << 16, 1, dtype=oracle.R32)
    look2 = rand_r32(rng, 7000, 1 << 16, 1 << 10, 1, dtype=oracle.R32)
    look1["time"] = 0
    look2["time"] = 0
    gs1, os1 = mz.Spine(ctx, 32), oracle.Spine(32, 1, True)
    gs2, os2 = mz.Spine(ctx, 32), oracle.Spine(32, 1, True)
    for gs, os_, rows in ((gs1, os1, look1), (gs2, os2, look2)):
        gs.insert(mz.Batch.build(ctx, rows, 0, 1))
        os_.insert(oracle.Batch.build(rows, 0, 1))
        gs.set_physical_compaction(1)
        os_.set_physical_compaction(1)
    # stage 1 keeps the key, stage 2 re-keys by the low 16 bits of the looked-up value
    cl1 = dict(key_fields=[(2, 0, 16, 0)], val_fields=[(1, 0, 20, 0)])
    cl2 = dict(key_fields=[(0, 0, 8, 0)], val_fields=[(2, 0, 10, 0), (1, 0, 20, 10)])
    g1, o1 = mz.make_closure(**cl1), oracle.make_closure(**cl1)
    g2, o2 = mz.make_closure(**cl2), oracle.make_closure(**cl2)
    gb, ob = mz.Batcher(ctx, 32), oracle.Batcher(32)
    gr, orr = mz.ReduceAccumulable(ctx, 0), oracle.Reduce(0)
    ctx.sync()
    for t in (1, 2, 3):
        upd = rand_r32(rng, n, 800, 1 << 20, 1, dtype=oracle.R32)
        upd["time"] = t
        dev = mz.DeviceRows(ctx, 32).upload(upd)
        s0 = ctx.stats()["host_syncs"]
        gb.push_buf(dev)
        batch = gb.seal_lazy(t + 1)
        stream = mz.update_stream_dev(ctx, batch)
        j1 = mz.half_join_dev(ctx, stream, gs1, mz.HALFJOIN_LE, g1)
        j2 = mz.half_join_dev(ctx, j1, gs2, mz.HALFJOIN_LT, g2)
        out = gr.step_dev(j2, t + 1)
        enqueue_syncs = ctx.stats()["host_syncs"] - s0
        got = out.download()
        # oracle, operator by operator
        ob.push(upd)
        obatch = ob.seal(t + 1)
        ws = oracle.update_stream(obatch, None, mz.FRONTIER_EMPTY)
        w1 = oracle.half_join(ws, os1, 0, o1)
        w2 = oracle.half_join(w1, os2, 1, o2)
        want = orr.step(w2, t + 1)
        same(got, want)
        # enqueueing the whole chain waits at most twice (the probes' fan-out bounds need the
        # lengths of freshly sealed batches; nothing else)
        assert enqueue_syncs <= 2, enqueue_syncs


# -------------------------------------------------- the whole Q3 dataflow
@pytest.mark.parametrize("peers", [1, 2, 3, 8, 16])
def test_exchange_partition_kernels_route_like_the_oracle(mz, ctx, oracle, peers):
    """The Exchange pact's device half (exchange.cu: k_part_count_many / offsets / scatter_many, the
    kernels mzgpu_exchange_many launches) on ONE GPU for several cluster sizes: every row lands in
    the group of worker hash(key) % peers (arrange.rs:116, columnar.rs:227-237; the oracle's
    mzo_route), groups are in worker order with the reported counts, nothing lost or duplicated --
    for R32 and RACC buffers of different sizes in one round."""
    rng = np.random.default_rng(300 + peers)
    a = rand_r32(rng, 70001, 1 << 40, 1 << 30, 4, dtype=mz.R32)
    b = rand_r32(rng, 513, 50, 7, 2, dtype=mz.R32)  # few keys: some workers get nothing
    c = np.zeros(20000, dtype=mz.RACC)
    c["key"] = rng.integers(0, 1 << 63, size=len(c), dtype=np.uint64)
    c["time"] = rng.integers(0, 5, size=len(c), dtype=np.uint64)
    c["total"] = rng.integers(-5, 5, size=len(c), dtype=np.int64)
    c["acc_lo"] = rng.integers(0, 1 << 62, size=len(c), dtype=np.uint64)
    e = np.zeros(0, dtype=mz.R32)
    ins = [a, b, c, e]
    bufs = [mz.DeviceRows(ctx, x.dtype.itemsize).upload(x) for x in ins]
    res = mz.partition_many(ctx, bufs, peers)
    for x, (rows, counts) in zip(ins, res):
        dest = np.array([oracle.lib().mzo_route(int(k), peers) for k in x["key"]], dtype=np.int64)
        assert counts == [int((dest == p).sum()) for p in range(peers)]
        assert len(rows) == len(x)
        at = 0
        for p in range(peers):
            grp = rows[at : at + counts[p]]
            at += counts[p]
            want = x[dest == p]
            assert multiset(grp) == multiset(want)
            assert all(mz.route(int(k), peers) == p for k in grp["key"][:50])


@pytest.mark.parametrize("peers", [2, 4])
def test_exchange_over_peer_memory_on_one_gpu(mz, oracle, peers):
    """The peer-memory exchange (k_p2p_scatter / k_p2p_gather: partition + delivery in one kernel,
    flags and counts in the landing zones, compaction on the receiver) with every worker running
    on ONE GPU (zones mapped in-process): several rounds, R32 and RACC buffers of uneven sizes,
    an empty buffer, a worker that sends nothing -- every destination receives exactly the rows
    the oracle's routing function sends it, grouped by source worker in worker order."""
    rng = np.random.default_rng(500 + peers)
    ctxs = [mz.Context(0, w, peers) for w in range(peers)]
    mz.p2p_connect_local(ctxs, 40000, 80)
    for rnd in range(5):
        ins = []
        for w in range(peers):
            n1 = 0 if (w == 1 and rnd == 2) else int(rng.integers(1, 30000))
            a = rand_r32(rng, n1, 1 << 40, 1 << 30, 4, dtype=mz.R32)
            b = np.zeros(int(rng.integers(0, 9000)), dtype=mz.RACC)
            b["key"] = rng.integers(0, 1 << 63, size=len(b), dtype=np.uint64)
            b["total"] = rng.integers(-5, 5, size=len(b), dtype=np.int64)
            e = np.zeros(0, dtype=mz.R32)
            ins.append([a, b, e])
        dev = [[mz.DeviceRows(c, x.dtype.itemsize).upload(x) for x in ins[w]] for w, c in enumerate(ctxs)]
        outs = [[mz.DeviceRows(c, x.dtype.itemsize) for x in ins[w]] for w, c in enumerate(ctxs)]
        for w, c in enumerate(ctxs):
            mz.exchange_p2p_send(c, dev[w])
        for w, c in enumerate(ctxs):
            mz.exchange_p2p_recv(c, outs[w], None if rnd % 2 else [200000, 200000, 10])
        for d in range(peers):
            for e in range(3):
                got = outs[d][e].download()
                at = 0
                for s_ in range(peers):
                    x = ins[s_][e]
                    dest = np.array([oracle.lib().mzo_route(int(k), peers) for k in x["key"]], dtype=np.int64)
                    want = x[dest == d]
                    assert multiset(got[at : at + len(want)]) == multiset(want), (rnd, d, e, s_)
                    at += len(want)
                assert at == len(got)
    for c in ctxs:
        c.sync()
        c.close()


def test_device_correction_buffer_matches_oracle(mz, ctx, oracle):
    """CorrectionV2 on the device (f3): the same random sequence of insert / insert_negated /
    advance_since / consolidate_at_since / updates_before drives the oracle's chain-of-chunks
    restatement and the GPU buffer; every read returns the same rows in the same (time, data)
    order, at update-batch sizes as well as in the small."""
    EMPTY = mz.FRONTIER_EMPTY
    for seed, scale in ((1, 1), (2, 1), (3, 400)):
        rng = np.random.default_rng(600 + seed)
        g, o = mz.Correction(ctx), oracle.Correction(3.0, 64)
        since = 0
        for step in range(50):
            op = rng.integers(0, 10)
            if op < 5:
                n = int(rng.integers(0, 90)) * scale
                a = np.zeros(n, dtype=oracle.R32)
                a["key"] = rng.integers(0, 40 * scale, size=n, dtype=np.uint64)
                a["val"] = rng.integers(0, 3, size=n, dtype=np.uint64)
                a["time"] = rng.integers(max(0, since - 3), since + 12, size=n, dtype=np.uint64)
                a["diff"] = rng.integers(-2, 3, size=n)
                neg = bool(rng.integers(0, 2))
                if rng.integers(0, 2):
                    g.insert(a, neg)
                else:
                    g.insert_buf(mz.DeviceRows(ctx, 32).upload(a), neg)
                o.insert(a, neg)
            elif op < 7:
                since += int(rng.integers(0, 4))
                g.advance_since(since)
                o.advance_since(since)
            elif op < 8:
                g.consolidate_at_since()
                o.consolidate_at_since()
            else:
                upper = max(since + int(rng.integers(-1, 8)), 0)
                same(g.updates_before(upper), o.updates_before(upper))
        same(g.updates_before(EMPTY), o.updates_before(EMPTY))
        assert len(g) == len(o.updates_before(EMPTY))
        # what was written comes back negated: the buffer empties; the empty since discards
        rest = o.updates_before(EMPTY)
        g.insert(rest, negate=True)
        assert len(g.updates_before(EMPTY)) == 0 and len(g) == 0
        g.advance_since(EMPTY)
        g.insert(rest)
        assert len(g.updates_before(EMPTY)) == 0


def _column_rows(oracle, rng, n, row_keys):
    a = np.zeros(n, dtype=oracle.R32)
    if row_keys:
        for f in ("key", "val"):
            lens = rng.integers(0, 8, size=n, dtype=np.uint64)
            body = rng.integers(0, 1 << 56, size=n, dtype=np.uint64)
            keep = np.where(lens == 0, np.uint64(0), ~((np.uint64(1) << (np.uint64(56) - np.uint64(8) * lens)) - np.uint64(1)) & np.uint64((1 << 56) - 1))
            a[f] = (lens << np.uint64(56)) | (body & keep)
    else:
        a["key"] = rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * 2 + 1
        a["val"] = rng.integers(0, 1 << 40, size=n, dtype=np.uint64)
    a["time"] = rng.integers(0, 50, size=n, dtype=np.uint64)
    a["diff"] = rng.integers(-3, 4, size=n)
    return a


@pytest.mark.parametrize("layout", [0, 1, 2])
@pytest.mark.parametrize("n", [0, 1, 255, 4097, 200_000])
def test_column_wire_format_matches_oracle(mz, ctx, oracle, layout, n):
    """f4: a serialized `Column` (columnar.rs:54-222) decoded on the device gives the oracle's rows, and rows
    encoded on the device give the oracle's bytes, word for word -- ((u64, u64), u64, i64), (u64, i64) and
    ((Row, Row), Timestamp, Diff) with Rows of 0..7 bytes."""
    rng = np.random.default_rng(900 + 10 * layout + n % 97)
    a = _column_rows(oracle, rng, n, layout == 2)
    words = oracle.column_encode(layout, a)
    dev = mz.column_decode(ctx, layout, words)
    got = dev.download()
    if layout == 1:
        assert got.dtype.itemsize == 16
        assert got["key"].tobytes() == a["key"].tobytes() and got["diff"].tobytes() == a["diff"].tobytes()
    else:
        assert got.tobytes() == oracle.column_rows(layout, words).tobytes() == a.tobytes()
    # decode appends: a second container lands behind the first
    mz.column_decode(ctx, layout, words, out=dev)
    assert len(dev) == 2 * n
    assert dev.download()[n:].tobytes() == got.tobytes()
    # encode: the same bytes back (a sub-range too)
    assert mz.column_encode(dev, layout, 0, n).tobytes() == words.tobytes()
    if n > 10:
        sub = mz.column_encode(dev, layout, 3, n - 7)
        assert sub.tobytes() == oracle.column_encode(layout, a[3 : n - 4]).tobytes()
    assert mz._ffi.lib.mzgpu_column_length_in_words(layout, n, int((a["key"] >> np.uint64(56)).sum()) if layout == 2 else 0,
                                                     int((a["val"] >> np.uint64(56)).sum()) if layout == 2 else 0) == len(words)


@pytest.mark.parametrize("layout", [0, 1, 2])
def test_column_builder_matches_oracle(mz, ctx, oracle, layout):
    """ColumnBuilder (builder.rs:28-111) over a device buffer: the same containers, cut at the same rows, as
    pushing the rows one at a time through the oracle's builder; decoding them all restores the rows."""
    rng = np.random.default_rng(950 + layout)
    n = 400_000
    a = _column_rows(oracle, rng, n, layout == 2)
    want = oracle.column_builder(layout, a)
    dev = mz.DeviceRows(ctx, 16 if layout == 1 else 32)
    if layout == 1:
        r16 = np.zeros(n, dtype=mz.R16)
        r16["key"], r16["diff"] = a["key"], a["diff"]
        dev.upload(r16)
    else:
        dev.upload(a)
    got = mz.column_build(dev, layout)
    assert len(got) == len(want) >= 3
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    back = mz.DeviceRows(ctx, dev.row_bytes)
    for g in got:
        mz.column_decode(ctx, layout, g, out=back)
    assert back.download().tobytes() == dev.download().tobytes()
    if layout != 2:
        assert mz._ffi.lib.mzgpu_column_ship_rows(layout) == len(oracle.column_rows(layout, want[0]))


def test_column_rejects_what_it_cannot_hold(mz, ctx, oracle):
    """Malformed indexes are MZGPU_E_INVALID, a Row longer than 7 bytes is MZGPU_E_UNSUPPORTED, and neither
    appends anything."""
    F = mz._ffi
    rng = np.random.default_rng(970)
    a = _column_rows(oracle, rng, 1000, True)
    words = oracle.column_encode(2, a)
    out = mz.DeviceRows(ctx, 32).upload(a[:5])
    for mutate in (lambda w: w.__setitem__(0, 48), lambda w: w.__setitem__(6, 8 * len(w) + 8), lambda w: w.__setitem__(3, w[3] + 8)):
        bad = words.copy()
        mutate(bad)
        with pytest.raises(mz.MzGpuError) as e:
            mz.column_decode(ctx, 2, bad, out=out)
        assert e.value.status == F.E_INVALID
    # bounds that run backwards are found on the device
    bad = words.copy()
    bad[7 + 10] = bad[7 + 9] - 1 if bad[7 + 9] else 999999
    with pytest.raises(mz.MzGpuError) as e:
        mz.column_decode(ctx, 2, bad, out=out)
    assert e.value.status == F.E_INVALID
    # an eight-byte Row
    one = np.array([5], dtype="<u8").tobytes()
    long_row = oracle.col_encode_slices([np.array([8], dtype="<u8").tobytes(), b"12345678", np.array([0], dtype="<u8").tobytes(), b"", one, one])
    with pytest.raises(mz.MzGpuError) as e:
        mz.column_decode(ctx, 2, long_row, out=out)
    assert e.value.status == F.E_UNSUPPORTED
    with pytest.raises(mz.MzGpuError):
        mz.column_decode(ctx, 0, words, out=out)  # six slices are not a four-slice container
    assert out.download().tobytes() == a[:5].tobytes()


def test_batch_walk_into_columns(mz, ctx, oracle):
    """walk_cursor (context.rs:1299-1355) over a sealed batch into containers: the whole batch in fuel-sized
    pieces, and one key's rows after seek_key."""
    rng = np.random.default_rng(980)
    a = rand_r32(rng, 30_000, 2000, 50, 3, 1, 3, dtype=mz.R32)
    gb = mz.Batcher(ctx, 32)
    gb.push_container(a)
    batch = gb.seal(3)
    rows = batch.rows()
    pieces, first = [], 0
    while True:
        words, n = mz.batch_walk_column(batch, 0, first=first, fuel=7001)
        pieces.append(oracle.column_rows(0, words))
        first += n
        if n < 7001:
            break
    assert np.concatenate(pieces).tobytes() == rows.tobytes()
    key = int(rows["key"][len(rows) // 2])
    words, n = mz.batch_walk_column(batch, 0, key=key)
    assert oracle.column_rows(0, words).tobytes() == rows[rows["key"] == key].tobytes() and n == (rows["key"] == key).sum()
    words, n = mz.batch_walk_column(batch, 0, key=(1 << 63) + 12345)
    assert n == 0 and len(oracle.column_rows(0, words)) == 0


def test_q3_dataflow_matches_oracle(mz, ctx, oracle):
    """Hydration + update batches through the C++ harness (delta join, 3 paths x 2
    half_joins, reduce) vs the CPU oracle dataflow on the same seeded inputs."""
    from materialize_b200 import harness

    args = dict(seed=7, n_customer=3000, n_orders=30000, n_part=4000, per_batch=500)
    g = harness.Q3Dataflow(ctx, **args)
    o = oracle.Q3(workers=2, **args)
    g.hydrate()
    o.hydrate()
    same(oracle.consolidate(g.out_rows()), o.drain())
    g.clear_out()
    for b in range(6):
        rows = g.stage_batch(b, g.time())
        _, orows = o.step(b)
        assert rows == orows
        # the device generator and the host generator produce the same multiset
        same(oracle.consolidate(g.staged(3)), oracle.consolidate(o.inputs(3)))
        g.step()
        same(oracle.consolidate(g.out_rows()), o.drain())
        g.clear_out()


def test_device_generators_match_host(mz, ctx, oracle):
    from materialize_b200 import harness

    same(harness.gen_cfg1(ctx, 1, 5000, 20).download(), oracle.gen_cfg1(1, 5000, 20))
    same(harness.gen_cfg1(ctx, 1, 5000, 64).download(), oracle.gen_cfg1(1, 5000, 64))
    same(harness.gen_cfg2(ctx, 2, 5000, 10**7).download(), oracle.gen_cfg2(2, 5000, 10**7))
    cdf = oracle.zipf_cdf(0.9, 10000)
    same(harness.gen_cfg4(ctx, 3, 5000, cdf).download(), oracle.gen_cfg4(3, 0, 5000, cdf))
    same(harness.gen_cfg4(ctx, 3, 5000, cdf, as_f64=True).download(), oracle.gen_cfg4(3, 0, 5000, cdf, True))
