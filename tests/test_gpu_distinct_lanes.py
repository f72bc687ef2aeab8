"""COUNT(DISTINCT x) / SUM(DISTINCT x) lanes (MZGPU_ACCUM_DISTINCT) on the GPU: byte for byte against the
CPU restatement (output, main arrangement, pair arrangements), against the plain lane they reduce to on
unique pairs, reference-held answers through one operator, a full-size run against numpy, and rejections."""
import numpy as np
import pytest

from distinct_lanes_oracle import ReduceLanesDistinct
from test_oracle_distinct_lanes import D, DISTINCT_SETS, I64, VAL1, VAL2, distinct_activations, load_fixture, run_fixture_case

pytestmark = pytest.mark.gpu

F64 = 1


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    # the full-size run's 50 M-row step peaks at about 42 GB of device memory: this module runs before the
    # modules that keep their contexts (and their cached blocks) alive, and hands its own back when it ends
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


def same_bytes(a, b):
    assert a.dtype.itemsize == b.dtype.itemsize
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


def gpu_op(mz, ctx, lanes, in_rb):
    return mz.ReduceLanes(ctx, [mz.accum_lane(*l) for l in lanes], in_rb)


@pytest.mark.parametrize("name", sorted(DISTINCT_SETS))
def test_distinct_lanes_match_restatement(mz, ctx, oracle, name):
    in_rb, lanes = DISTINCT_SETS[name]
    g, o = gpu_op(mz, ctx, lanes, in_rb), ReduceLanesDistinct(oracle, lanes, in_rb)
    rng = np.random.default_rng(17 + len(name))
    for a, upper in distinct_activations(rng, in_rb // 8, steps=10, keys=300):
        same_bytes(g.step(a, upper), o.step(a, upper))
        same_bytes(g.input_trace().export(), o.export())
        for l, lane in enumerate(lanes):
            if lane[0] & D:
                same_bytes(g.distinct_trace(l).export(), o.pair_export(l))
            else:
                assert g.distinct_trace(l) is None
    assert g.distinct_trace(len(lanes)) is None


def test_one_distinct_lane_on_unique_pairs_is_the_plain_lane(mz, ctx):
    """Every (key, value) at most once, never retracted: the distinct lane is byte-identical to the same lane
    without the flag, output and arrangement."""
    rng = np.random.default_rng(23)
    d, p = mz.ReduceLanes(ctx, [mz.accum_lane(I64 | D, VAL1)], 32), mz.ReduceLanes(ctx, [mz.accum_lane(I64, VAL1)], 32)
    t = 0
    for step in range(6):
        n = 50_000
        a = np.zeros(n, dtype=mz.R32)
        a["key"] = rng.integers(0, 2000, size=n, dtype=np.uint64)
        # unique values: a step's block of a bijection of [0, 2^40) (an odd multiplier), made signed
        v = ((np.arange(n, dtype=np.int64) + step * n) * 0x9E3779B1) & (2**40 - 1)
        a["val"] = (v - 2**39).view(np.uint64)
        a["time"] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        a["diff"] = 1
        t += 3
        same_bytes(d.step(a, t), p.step(a, t))
    same_bytes(d.input_trace().export(), p.input_trace().export())


def test_fixture_cases_through_one_gpu_operator(mz, ctx):
    for case in load_fixture()["cases"]:
        got = run_fixture_case(lambda lanes: gpu_op(mz, ctx, lanes, 32), case)
        assert got == case["expect"], case["query"]


def test_distinct_rejections_leave_the_context_usable(mz, ctx):
    E_INVALID, E_UNSUPPORTED = -1, -4
    for lanes, status in [
        ([mz.accum_lane(F64 | D, VAL1)], E_UNSUPPORTED),  # which floats are one value is not pinned
        ([mz.accum_lane(I64, VAL1), mz.accum_lane(F64 | D, VAL1)], E_UNSUPPORTED),
        ([mz.accum_lane(I64 | 0x200, VAL1)], E_INVALID),  # unknown bit
        ([mz.accum_lane(I64 | D | 0x200, VAL1)], E_INVALID),
        ([mz.accum_lane(2 | D, VAL1)], E_INVALID),  # DISTINCT is not a lane kind, with or without the bit
        ([mz.accum_lane(I64 | D, VAL2)], E_INVALID),  # no val2 in R32
    ]:
        with pytest.raises(mz.MzGpuError) as e:
            mz.ReduceLanes(ctx, lanes, 32)
        assert e.value.status == status, lanes
    r = mz.ReduceLanes(ctx, [mz.accum_lane(I64 | D, VAL1), mz.accum_lane(I64, VAL1)], 32)
    a = np.zeros(3, dtype=mz.R32)
    a["key"], a["val"], a["diff"] = 1, [4, 4, 6], 1
    (o,) = r.step(a, 1)
    assert [int(x) for x in o["lanes"][0].tolist()] == [2, 10, 0] and int(o["lanes"][1]["count"]) == 3
    assert len(ctx.consolidate(np.zeros(4, dtype=mz.R32))) == 0


def _zipf_cdf(nk):
    w = 1.0 / np.power(np.arange(1, nk + 1, dtype=np.float64), 0.9)
    cdf = np.cumsum(w / w.sum())
    cdf[-1] = 1.0
    return cdf


def test_distinct_full_size_against_numpy(mz, ctx):
    """50 M R40 rows: a plain int64 lane (val1) and a distinct lane (val2) over about 10^7 distinct (key, value)
    pairs of 1 M Zipf(0.9) keys, then incremental batches of which half retract earlier rows.  After every
    step the operator's accumulated output equals per-key COUNT / SUM and COUNT(DISTINCT) / SUM(DISTINCT)
    computed with numpy."""
    rng = np.random.default_rng(31)
    n_pairs, n = 10_000_000, 50_000_000
    pair_key = np.searchsorted(_zipf_cdf(1_000_000), rng.random(n_pairs)).astype(np.uint64)
    # distinct values by construction (an odd multiplier is a bijection of [0, 2^34)), signed; every per-key
    # sum stays below 2^53, so numpy's float64 bincount is exact
    pair_val = ((np.arange(n_pairs, dtype=np.int64) * 0x9E3779B1) & (2**34 - 1)) - 2**33
    r = mz.ReduceLanes(ctx, [mz.accum_lane(I64, VAL1), mz.accum_lane(I64 | D, VAL2)], 40)

    def rows_of(idx, v1, t, d):
        a = np.zeros(len(idx), dtype=mz.R40)
        a["key"], a["val1"], a["val2"], a["time"], a["diff"] = pair_key[idx], v1.view(np.uint64), pair_val[idx].view(np.uint64), t, d
        return a

    live_idx = rng.integers(0, n_pairs, size=n, dtype=np.int64)
    live_v1 = rng.integers(-(2**30), 2**30, size=n, dtype=np.int64)
    outs = [r.step(rows_of(live_idx, live_v1, 0, 1), 1)]
    print("distinct full size: device_bytes_peak after the 50 M-row step", ctx.stats()["device_bytes_peak"])
    check_state(outs, live_idx, live_v1, pair_key, pair_val, n_pairs)
    for step in range(1, 4):
        m = 1_000_000
        fresh_idx = rng.integers(0, n_pairs, size=m // 2, dtype=np.int64)
        fresh_v1 = rng.integers(-(2**30), 2**30, size=m // 2, dtype=np.int64)
        back = np.unique(rng.integers(0, len(live_idx), size=m // 2))
        batch = np.concatenate([rows_of(fresh_idx, fresh_v1, step, 1), rows_of(live_idx[back], live_v1[back], step, -1)])
        outs.append(r.step(batch, step + 1))
        keep = np.ones(len(live_idx), dtype=bool)
        keep[back] = False
        live_idx = np.concatenate([live_idx[keep], fresh_idx])
        live_v1 = np.concatenate([live_v1[keep], fresh_v1])
        check_state(outs, live_idx, live_v1, pair_key, pair_val, n_pairs)
    print("distinct full size: device_bytes_peak", ctx.stats()["device_bytes_peak"])


def check_state(outs, live_idx, live_v1, pair_key, pair_val, n_pairs):
    # the operator's current output: per key, the row of its last correction if that added a row
    out = np.concatenate(outs)
    step = np.concatenate([np.full(len(o), i) for i, o in enumerate(outs)])
    order = np.lexsort((out["diff"], step, out["key"]))  # within a key and step the retraction comes first
    out, step = out[order], step[order]
    last = np.r_[out["key"][1:] != out["key"][:-1], True]
    cur = out[last & (out["diff"] == 1)]
    # numpy: plain COUNT / SUM over the live rows, distinct COUNT / SUM over the live pairs
    keys = pair_key[live_idx].astype(np.int64)
    hi = int(pair_key.max()) + 1
    cnt = np.bincount(keys, minlength=hi)
    sums = np.bincount(keys, weights=live_v1.astype(np.float64), minlength=hi)
    assert np.abs(sums).max() < 2.0**53
    sums = sums.astype(np.int64)
    present = np.bincount(live_idx, minlength=n_pairs) > 0
    pk = pair_key[present].astype(np.int64)
    dcnt = np.bincount(pk, minlength=hi)
    dsum = np.bincount(pk, weights=pair_val[present].astype(np.float64), minlength=hi)
    assert np.abs(dsum).max() < 2.0**53
    dsum = dsum.astype(np.int64)
    live = np.nonzero(cnt)[0]
    assert np.array_equal(cur["key"].astype(np.int64), live)
    assert np.all(cur["flags"] == 0)
    l0, l1 = cur["lanes"][:, 0], cur["lanes"][:, 1]
    assert np.array_equal(l0["count"], cnt[live]) and np.array_equal(l0["sum_lo"].view(np.int64), sums[live])
    assert np.array_equal(l0["sum_hi"], np.where(sums[live] < 0, -1, 0))
    assert np.array_equal(l1["count"], dcnt[live]) and np.array_equal(l1["sum_lo"].view(np.int64), dsum[live])
    assert np.array_equal(l1["sum_hi"], np.where(dsum[live] < 0, -1, 0))
