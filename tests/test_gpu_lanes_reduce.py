"""The multi-column accumulable reduce (mzgpu_reduce_lanes_*) on the GPU: bit-exact against the CPU
oracle and against the one-column kinds it generalizes, reference-held answers through one
operator, full-size properties at every new row width, and descriptor rejections."""
import json
import os

import numpy as np
import pytest

from lanes_oracle import ReduceLanes
from test_oracle_reduce_lanes import F64, I64, LANE_SETS, VAL1, VAL2, accumulated, activations

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    # this module's 100 M-row seal needs about 50 GB of device memory: it runs before the modules that
    # keep their contexts (and their cached blocks) alive, and hands its own back when it ends
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


def same_bytes(a, b):
    assert a.dtype.itemsize == b.dtype.itemsize
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


def accumulable_sequence(oracle, agg_kind):
    """The 8 activations of test_gpu_parity.py::test_reduce_accumulable_matches_oracle."""
    rng = np.random.default_rng(29 + agg_kind)
    live, t = [], 0
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
        yield a, t


@pytest.mark.parametrize("agg_kind", [0, 1])
def test_one_lane_is_byte_identical_to_the_one_column_kind(mz, ctx, oracle, agg_kind):
    lanes_op = mz.ReduceLanes(ctx, [mz.accum_lane(agg_kind)], 32)
    old = mz.ReduceAccumulable(ctx, agg_kind)
    for a, upper in accumulable_sequence(oracle, agg_kind):
        same_bytes(lanes_op.step(a, upper), old.step(a, upper))
    same_bytes(lanes_op.input_trace().export(), old.input_trace().export())


@pytest.mark.parametrize("name", sorted(LANE_SETS))
def test_lanes_match_oracle(mz, ctx, oracle, name):
    in_rb, lanes = LANE_SETS[name]
    g = mz.ReduceLanes(ctx, [mz.accum_lane(k, s, sh, b, sx) for k, s, sh, b, sx in lanes], in_rb)
    o = ReduceLanes(oracle, lanes, in_rb)
    rng = np.random.default_rng(7 * len(name))
    for a, upper in activations(rng, lanes, in_rb // 8, steps=10, keys=500):
        same_bytes(g.step(a, upper), o.step(a, upper))
    same_bytes(g.input_trace().export(), o.export())


def test_lanes_match_single_lane_operators(mz, ctx):
    """Per lane, the accumulated output of one 8-lane operator equals what a one-lane operator on the
    same column accumulates, at every step."""
    in_rb, lanes = LANE_SETS["r40_eight"]
    g = mz.ReduceLanes(ctx, [mz.accum_lane(*l) for l in lanes], in_rb)
    singles = [mz.ReduceLanes(ctx, [mz.accum_lane(*l)], in_rb) for l in lanes]
    rng = np.random.default_rng(11)
    outs, souts = [], [[] for _ in lanes]
    for a, upper in activations(rng, lanes, in_rb // 8, steps=10, keys=500):
        outs.append(g.step(a, upper))
        for j, s in enumerate(singles):
            souts[j].append(s.step(a, upper))
        whole = accumulated(np.concatenate(outs), 8, upper)
        for j in range(len(lanes)):
            mine = {(r[0], *r[1 + 3 * j : 4 + 3 * j], (r[-1] >> (2 * j)) & 3) for r in whole}
            theirs = accumulated(np.concatenate(souts[j]), 1, upper)
            assert mine == theirs, j


def test_fixture_cases_through_one_gpu_lanes_operator(mz, ctx):
    fx = json.load(open(os.path.join(HERE, "golden", "sqllogictest_join_reduce.json")))
    cases = {c["shape"]: c for c in fx["cases"]}
    t = fx["tables"]["t"]["rows"]
    rows = np.zeros(len(t), dtype=mz.R40)
    rows["key"], rows["val1"], rows["val2"], rows["time"], rows["diff"] = 0, [a for a, _ in t], [b for _, b in t], 0, 1
    r = mz.ReduceLanes(ctx, [mz.accum_lane(I64, VAL1), mz.accum_lane(I64, VAL2)], 40)
    (o,) = r.step(rows, 1)
    (ca, sa, _), (cb, sb, _) = (tuple(int(np.int64(x)) for x in o["lanes"][l].tolist()) for l in range(2))
    assert ca == cb == len(t) and int(o["flags"]) == 0 and int(o["diff"]) == 1
    assert [[1, sa, sb, sa / ca]] == cases["global_sums"]["expect"]

    g = np.zeros(len(t), dtype=mz.R32)
    g["key"], g["val"], g["time"], g["diff"] = [a for a, _ in t], [b for _, b in t], 0, 1
    out = mz.ReduceLanes(ctx, [mz.accum_lane(I64, VAL1)], 32).step(g, 1)
    got = sorted((int(o["key"]), int(o["lanes"][0]["count"]), int(np.int64(o["lanes"][0]["sum_lo"]))) for o in out)
    assert got == sorted((k, c, s) for k, c, _, s, _ in cases["count_min_sum_max"]["expect"])


def _zipf_cdf(nk):
    w = 1.0 / np.power(np.arange(1, nk + 1, dtype=np.float64), 0.9)
    cdf = np.cumsum(w / w.sum())
    cdf[-1] = 1.0
    return cdf


@pytest.mark.parametrize("n,lanes", [(100_000_000, 2), (10_000_000, 8)])
def test_lanes_full_size_properties(mz, ctx, n, lanes):
    """BASELINE configs[3] (1 M Zipf(0.9) keys) through one lanes operator: lane 0 sums the whole
    value, the others bit-fields of it; COUNT and SUM per key against numpy's bincount.  100 M rows
    at 2 lanes and 10 M rows at 8 run the bulk seal, merges and corrections at 128 and 416 bytes."""
    from materialize_b200 import harness

    d = harness.gen_cfg4(ctx, 3, n, _zipf_cdf(1_000_000))
    h = d.download()
    picks = [(0, 64)] + [(4 * j, 12) for j in range(1, lanes)]
    r = mz.ReduceLanes(ctx, [mz.accum_lane(I64, VAL1, s, b, b < 64) for s, b in picks], 32)
    out = r.step_dev(d, 1).download()
    del d
    keys = h["key"].astype(np.int64)
    hi = int(keys.max()) + 1
    cnt = np.bincount(keys, minlength=hi)
    live = np.nonzero(cnt)[0]
    assert np.array_equal(out["key"].astype(np.int64), live)
    assert np.all(out["diff"] == 1) and np.all(out["flags"] == 0)
    v = h["val"]
    for j, (s, b) in enumerate(picks):
        col = v.astype(np.int64) if b == 64 else ((v >> np.uint64(s)) & np.uint64((1 << b) - 1)).astype(np.int64)
        if b < 64:
            col = np.where(col >= 1 << (b - 1), col - (1 << b), col)
        sums = np.bincount(keys, weights=col.astype(np.float64), minlength=hi)
        assert np.abs(sums).max() < 2.0**53
        lane = out["lanes"][:, j]
        assert np.array_equal(lane["count"], cnt[live]), j
        assert np.array_equal(lane["sum_lo"].astype(np.int64), sums[live].astype(np.int64)), j
        assert np.all(lane["sum_hi"] == np.where(sums[live] < 0, -1, 0)), j


def test_malformed_descriptors_are_rejected(mz, ctx):
    E_INVALID = -1
    ok = mz.accum_lane(I64, VAL1)
    bad = [
        (32, [mz.accum_lane(7, VAL1)]),  # kind
        (32, [mz.accum_lane(2, VAL1)]),  # DISTINCT is not a lane kind
        (32, [mz.accum_lane(I64, VAL2)]),  # no val2 in R32
        (40, [mz.accum_lane(I64, 0)]),  # the key is not a value column
        (40, [mz.accum_lane(I64, 3)]),
        (32, [mz.accum_lane(I64, VAL1, 0, 0)]),  # zero width
        (32, [mz.accum_lane(I64, VAL1, 60, 8)]),  # past the word
        (32, [mz.accum_lane(I64, VAL1, 64, 1)]),
        (32, [mz.accum_lane(F64, VAL1, 0, 32)]),  # partial-word float
        (32, [mz.accum_lane(F64, VAL1, 8, 56)]),
        (32, []),  # no lanes
        (32, [ok] * 9),  # more than 8
        (48, [ok]),  # input width
        (80, [ok]),
    ]
    for in_rb, lanes in bad:
        with pytest.raises(mz.MzGpuError) as e:
            mz.ReduceLanes(ctx, lanes, in_rb)
        assert e.value.status == E_INVALID, (in_rb, lanes)
    # a wrong input or output buffer width on a good operator
    r = mz.ReduceLanes(ctx, [ok, ok, ok], 32)  # class 4: 144-byte output
    rows = mz.DeviceRows(ctx, 32).upload(np.zeros(1, dtype=mz.R32))
    for in_buf, out_rb in [(rows, 64), (rows, 96), (mz.DeviceRows(ctx, 40), 144)]:
        with pytest.raises(mz.MzGpuError) as e:
            r.step_dev(in_buf, 1, mz.DeviceRows(ctx, out_rb))
        assert e.value.status == E_INVALID
    # the one-column entry points do not take a lanes operator
    with pytest.raises(mz.MzGpuError):
        mz.ReduceAccumulable.step(r, np.zeros(1, dtype=mz.R32), 1)
    # lanes output rows have no consolidation (their width has no row meaning in the generic kernels)
    out = r.step_dev(rows, 1)
    st = mz._ffi.lib.mzgpu_buf_consolidate(out.h)
    assert st == -4  # MZGPU_E_UNSUPPORTED
    # nothing sticky: the context and the operator keep working
    good = r.step(np.zeros(0, dtype=mz.R32), 2)
    assert len(good) == 0
    assert len(ctx.consolidate(np.zeros(4, dtype=mz.R32))) == 0
