"""The multi-column reduces on the GPU -- lanes (mzgpu_reduce_lanes_*), COUNT / SUM(DISTINCT) lanes, HAVING
and monotonic MIN / MAX -- against their restatements (tests/lanes_oracle.py, distinct_lanes_oracle.py,
having_oracle.py, monotonic_oracle.py) and, past the single-pass bound, the NumPy expectations of
tests/lanes_paths_ref.py, on every lane class and kernel path.

As in test_gpu_reduce_paths.py, every activation's output is compared byte for byte and in order as the
operator returned it; the input arrangement (and the pair arrangements of distinct lanes) after each
sequence; each case asserts the kernels it must and must not reach and the data precondition it relies on
(a run stored with slot length 0, more than 8 prior batches, a pair batch that consolidates to nothing).
The paths reached, the module's wall time and its device and host memory peaks are printed at the end
(pytest -s).  Kernel names are those of the profile report, which does not name the class: the notes
add it."""
import resource
import time

import numpy as np
import pytest

import lanes_paths_ref as R
from distinct_lanes_oracle import ACCUM_DISTINCT as D
from distinct_lanes_oracle import ReduceLanesDistinct
from having_oracle import ReduceLanesHaving, cmp, num, sum_
from lanes_oracle import ReduceLanes
from monotonic_oracle import ReduceMonotonic
from test_gpu_monotonic import ref_consolidate
from test_gpu_reduce_paths import Trace, _dev_input, _filler, _key_rows, same, trace_batches, words, zero_slot_batch

pytestmark = pytest.mark.gpu

I64, F64, VAL1 = R.I64, R.F64, 1
M64 = R.M64
PATHS = set()
PEAK = {}
BOUND = 48 << 20  # MZ_BOUND_MAX_ROWS: two output rows per batch row, so 24 Mi rows run in one pass
LOOSE = (24 << 20) + 40_000
LB = "k_corrections_lb<C>"
LB_HV = "k_corrections_lb_having<C>"
TWO = ("k_corrections<", "k_corrections_having<")
MONO_LB = "k_monotonic_corrections_lb"
MONO_TWO = ("k_monotonic_corrections<C,_false>", "k_monotonic_corrections<C,_true>")


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    t0 = time.time()
    c = mz.Context(0)
    yield c
    c.sync()
    PEAK["module context"] = c.stats()["device_bytes_peak"]
    c.close()
    print("\nlanes paths reached:")
    for p in sorted(PATHS):
        print(f"  {p}")
    print(f"wall time {time.time() - t0:.0f} s; host peak {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss >> 20} GiB")
    for k, v in sorted(PEAK.items()):
        print(f"device_bytes_peak {k}: {v / 2**30:.1f} GiB")


def note(cls, t=None, what=""):
    for k in sorted(t.kernels if t is not None else ()):
        if k.startswith(("k_corrections", "k_monotonic_corrections", "k_distinct_presence", "k_scan_tiles")):
            PATHS.add(f"C={cls} {k}")
    if what:
        PATHS.add(f"C={cls} {what}")


def private(mz, name, fn):
    """fn(ctx) on a context of its own, closed afterwards; its device peak is reported."""
    c = mz.Context(0)
    try:
        return fn(c)
    finally:
        c.sync()
        PEAK[name] = c.stats()["device_bytes_peak"]
        c.close()


def as_in(mz, w):
    return np.ascontiguousarray(w).view(mz.R40 if w.shape[1] == 5 else mz.R32).reshape(-1)


def gen(rng, keys, times, iw, diffs, small=False):
    """(n, iw) input words: random value words (the last one float64 bits, f64_words), or, with small,
    integers in [-2^40, 2^40)."""
    n = len(keys)
    w = np.zeros((n, iw), dtype=np.uint64)
    w[:, 0], w[:, iw - 2] = keys, times
    w[:, iw - 1] = np.asarray(diffs, dtype=np.int64).view(np.uint64)
    if small:
        w[:, 1 : iw - 2] = rng.integers(-(2**40), 2**40, size=(n, iw - 3)).view(np.uint64)
    else:
        w[:, 1 : iw - 3] = rng.integers(0, 2**64, size=(n, iw - 4), dtype=np.uint64)
        w[:, iw - 3] = R.f64_words(rng, n)
    return w


def lanes_op(mz, ctx, lanes, iw, having=None):
    return mz.ReduceLanes(ctx, [mz.accum_lane(*l) for l in lanes], 8 * iw, having=having)


def step(mz, g, o, w, upper):
    """One activation through both: the GPU's rows as returned, against the restatement's."""
    want = o.step(w, upper)
    same(g.step(as_in(mz, w), upper), words(want))
    return want


def step_dev(mz, ctx, g, o, w, upper, filler=1000):
    """The same through step_dev, with rows whose count is known on the device only."""
    buf, held = _dev_input(mz, ctx, w, _filler(filler, upper + 5), upper + 5)
    want = o.step(held, upper)
    same(g.step_dev(buf, upper).download(), words(want))
    return want


def same_arrangement(g, o):
    same(words(g.input_trace().export()), words(o.export()))


# ------------------------------------------------------------------ lanes
LANE_COUNTS = [1, 2, 3, 4, 5, 8]
MID, LAST = 600, 1 << 40
FIXED = [11, 4099, 9001, 15999]  # keys with a row in every activation of a "more than 8 batches" sequence


def hot_rows(rng, iw, t0, small=False):
    """Prior rows: 3000 over keys below 1200 and 1500 distinct times of each of MID and LAST (the last key
    of the batch): both runs are stored with slot length 0."""
    keys = np.r_[rng.integers(0, 1200, 3000), np.full(1500, MID), np.full(1500, LAST)].astype(np.uint64)
    times = np.r_[rng.integers(t0, t0 + 100, 3000), np.arange(t0, t0 + 1500), np.arange(t0, t0 + 1500)]
    return gen(rng, keys, times, iw, np.ones(len(keys), np.int64), small)


def check_hot_slots(mz, ctx, g, sp=None):
    for key, last in ((MID, False), (LAST, True)):
        _, keys = zero_slot_batch(mz, ctx, g, key, sp)
        assert (keys.max() == key) == last and keys.min() < key


def decreasing(rng, iw, t, top, pool, fixed, small=False):
    """Activations of 2^top down to 1 rows at one time each (distinct keys from `pool`), then two of one row,
    each with a row of every key of `fixed` as well: the spine keeps one batch per layer, so later
    activations see more than 8 prior batches, and the fixed keys they probe are held in every one."""
    pool = np.setdiff1d(pool, fixed)
    for e in list(range(top, -1, -1)) + [0, 0]:
        n = 1 << e
        keys = np.r_[rng.choice(pool, size=n, replace=False), fixed].astype(np.uint64)
        yield gen(rng, keys, np.full(len(keys), t), iw, rng.choice([-2, -1, 1, 2, 3], size=len(keys)), small), t + 1
        t += 1


def deep_keys(mz, ctx, g, keys, sp=None):
    """The keys of `keys` held in a batch at index 8 or later of the input trace (or of the spine sp): the
    second group of GROUP = 8 hash slots that prior_sum fetches at once."""
    keys = np.unique(np.asarray(keys, dtype=np.uint64))
    held = set()
    for b in trace_batches(mz, ctx, g, sp)[8:]:
        for run in b.seek_keys(keys):
            if run["len"] > 0 and run["key"] in keys:
                held.add(int(run["key"]))
    return held


def with_fixed(rng, w, iw, fixed, t0):
    """w and a row of every fixed key, so that the first batch holds them too."""
    return np.concatenate([w, gen(rng, fixed, np.full(len(fixed), t0), iw, np.ones(len(fixed), np.int64))])


def run_decreasing(mz, ctx, g, steps, fixed, expect, sp_of=lambda g: None):
    """Runs the activations of `decreasing` through `steps` (w, upper) -> the Trace of the step; `expect`
    checks each Trace.  Before each activation records how many batches the trace holds and which fixed keys
    (all probed by it) sit in a batch at index 8 or later.  Returns (max batches, activations probing a
    fixed key there)."""
    seen, deep = [], 0
    for w, upper in steps:
        sp = sp_of(g)
        seen.append((sp if sp is not None else g.input_trace()).size()["batches"])
        deep += bool(deep_keys(mz, ctx, g, fixed, sp))
        expect(w, upper)
    assert max(seen) > 8 and deep >= 2, (seen, deep)
    return max(seen), deep


def hot_probe(rng, iw, t, small=False):
    """100 times of MID and LAST, each a +1 row and a -1 row of other values: the count stays, the sums move,
    so each time retracts and re-adds the key's row (200 corrections of one key sorted by one thread)."""
    k = np.repeat(np.array([MID, LAST], np.uint64), 200)
    times = np.tile(np.repeat(np.arange(t, t + 100), 2), 2)
    return gen(rng, k, times, iw, np.tile([1, -1], 200), small)


@pytest.mark.parametrize("iw", [4, 5])
@pytest.mark.parametrize("n_lanes", LANE_COUNTS)
def test_lanes_hot_keys_and_many_prior_batches(mz, ctx, oracle, n_lanes, iw):
    """prior_sum<C> over runs with slot length 0 (a middle key and the last key of a batch) and over more
    than 8 prior batches (GROUP = 8 slots fetched at once); walk_key's sort of 200 corrections of one key."""
    rng = np.random.default_rng(3000 + 10 * n_lanes + iw)
    lanes = R.two_pass_lanes(n_lanes, iw)
    cls = R.lane_class(n_lanes)
    g, o = lanes_op(mz, ctx, lanes, iw), ReduceLanes(oracle, lanes, 8 * iw)
    fixed = FIXED + [MID, LAST]
    step(mz, g, o, with_fixed(rng, hot_rows(rng, iw, 0), iw, FIXED, 0), 1500)

    def expect(w, upper):
        with Trace(ctx) as t:
            step(mz, g, o, w, upper)
        t.only(LB, never=TWO)

    seen, deep = run_decreasing(mz, ctx, g, decreasing(rng, iw, 1500, 13, np.arange(1 << 14), fixed), fixed, expect)
    check_hot_slots(mz, ctx, g)
    with Trace(ctx) as t:
        out = step(mz, g, o, hot_probe(rng, iw, 2000), 2100)
    t.only("k_explode", LB, never=TWO)
    assert int((out["key"] == MID).sum()) > 150
    same_arrangement(g, o)
    note(cls, t, f"prior_sum: slot length 0 (middle and last key), {seen} prior batches (keys probed in batch 8+ "
                 f"by {deep} activations); 200 corrections of one key")


def test_lanes_edge_values(mz, ctx, oracle):
    """A class-8 operator with 6 lanes (2 unused): bit-fields at the ends of the word (shift 63 with 1 bit,
    signed and unsigned; shift 0 with 64 bits; a sign-extended 32-bit field at 0x80000000), i64 diffs at the
    extremes (the 128-bit sums wrap), a float64 lane with NaN, +-inf, 1e300 (saturation), -0.0 and sums on a
    rounding tie, and a DISTINCT lane of bits 8-15.  Both flags of a lane l > 0: bit 2l + 1 (a non-zero
    accumulation while total == 0) and bit 2l (the lane's accumulation is zero while total > 0).  With plain
    lanes only, bit 2l cannot be set: every row adds its diff to both the total and each lane's non_nulls, so
    they are equal.  The DISTINCT lane's present pairs add to the total alone, which makes it reachable."""
    for iw in (4, 5):
        lanes = [(I64, 1, 63, 1, True), (I64, 1, 63, 1, False), (I64, 1, 0, 64, False), (I64, 1, 0, 32, True),
                 (F64, iw - 3, 0, 64, False), (I64 | D, 1, 8, 8, False)]
        g, o = lanes_op(mz, ctx, lanes, iw), ReduceLanesDistinct(oracle, lanes, 8 * iw)
        ints = [0, 1, 0x80000000, 0x7FFFFFFF, 1 << 63, (1 << 63) - 1, M64, 0xFFFFFFFF]
        b = lambda x: int(np.float64(x).view(np.uint64))  # noqa: E731
        floats = [b(x) for x in (np.nan, np.inf, -np.inf, 1e300, -1e300, -0.0, 0.0, 2.0**93, 2.0**40, 2.0**-24,
                                 2.0**36, 5e-324, 2.5)] + [0x7FF0000000000123]
        diffs = [1, -1, 3, -3, (1 << 63) - 1, -(1 << 63)]
        spec = []
        for i in range(max(len(ints), len(floats))):
            x, f = ints[i % len(ints)], floats[i % len(floats)]
            vals = [x, f] if iw == 5 else [x if i % 2 else f]
            for j, d in enumerate(diffs):
                spec.append([100 + 8 * i + j, *vals, j % 3, d & M64])
                spec.append([7, *vals, j % 3, (d if j < 4 else 1) & M64])
        # rounding edges of the float lane, one key each (2^117 + 2^64 is a tie; + 1 rounds up)
        for k, xs in ((1, [2.0**93, 2.0**40]), (2, [2.0**93, 2.0**40, 2.0**-24]), (3, [-1e300, -1e300])):
            spec += [[k, *([0, b(x)] if iw == 5 else [b(x)]), 0, 1] for x in xs]
        # key 9: total 0 (the DISTINCT lane sees value 0 at +1 and -1: absent), lane 2 (64 bits) non-zero
        spec += [[9, *([5, b(1.0)] if iw == 5 else [5]), 0, 1], [9, *([3, b(2.0)] if iw == 5 else [3]), 0, M64]]
        # key 10: the DISTINCT lane holds values 1 (+1) and 2 (-1), so total = 2; lanes 0, 1 (bit 63) and 4 (a
        # zero or subnormal float) accumulate nothing
        spec += [[10, *([0x100, 0] if iw == 5 else [0x100]), 0, 1], [10, *([0x200, 0] if iw == 5 else [0x200]), 0, M64]]
        w = np.array(spec, dtype=np.uint64)
        first = step(mz, g, o, w, 3)
        flags = {int(r["key"]): int(r["flags"]) for r in first}
        assert flags[9] & (1 << 5), flags[9]
        assert flags[10] & (1 << 2) and flags[10] & (1 << 8) and not flags[10] & (1 << 4), flags[10]
        back = w[np.random.default_rng(iw).random(len(w)) < 0.5].copy()
        back[:, iw - 1] = (-back[:, iw - 1].view(np.int64)).view(np.uint64)
        back[:, iw - 2] = 3
        step(mz, g, o, back, 4)
        again = np.concatenate([w, back])
        again[:, iw - 2] = 5
        with Trace(ctx) as t:
            out = step(mz, g, o, again, 6)
        t.only("k_explode", LB, never=TWO)
        assert len(out) > 100
        same_arrangement(g, o)
        same(words(g.distinct_trace(5).export()), words(o.pair_export(5)))
    note(8, t, "edge values: bit-fields at the word's ends, i64 extremes, f64 NaN / inf / saturation / ties, "
               "flags 2l and 2l+1 of lanes l > 0")


def test_lanes_loose_device_bound(mz, oracle):
    """A few thousand rows in a device buffer whose bound is past the single-pass bound at C = 2: reduce_main
    reads the length back and runs the single-pass form."""
    rng = np.random.default_rng(3100)
    lanes = R.two_pass_lanes(2, 4)

    def run(c):
        g, o = lanes_op(mz, c, lanes, 4), ReduceLanes(oracle, lanes, 32)
        w = gen(rng, rng.integers(0, 700, 4000), np.zeros(4000), 4, rng.choice([-1, 1, 2], 4000))
        buf, held = _dev_input(mz, c, w, _filler(LOOSE, 9), 9)
        before = c.stats()["rows_in"]
        with Trace(c) as t:
            got = g.step_dev(buf, 1).download()
        assert c.stats()["rows_in"] - before >= LOOSE > BOUND // 2 > len(held)
        same(got, words(o.step(held, 1)))
        t.only("k_explode", LB, never=TWO)
        same_arrangement(g, o)
        note(2, t, f"loose device bound ({LOOSE} rows) resolved to {len(held)} rows, single pass")

    private(mz, "lanes loose bound", run)


# ------------------------------------------------------------------ DISTINCT lanes
def byte_lanes(order, plain):
    """Distinct lanes reading byte order[j] of val (byte 0 first in the list only if order says so), and
    with plain, a plain 64-bit lane of val at the end."""
    return [(I64 | D, VAL1, 8 * b, 8, False) for b in order] + ([(I64, VAL1, 0, 64, True)] if plain else [])


def rep(b):
    return np.asarray(b, dtype=np.uint64) * np.uint64(0x0101010101010101)


@pytest.mark.parametrize("n_distinct,plain", [(2, True), (3, False), (3, True), (8, False)])
def test_distinct_lanes_jobs_slots_and_prior_batches(mz, ctx, oracle, n_distinct, plain):
    """Through step_dev with device-only counts (k_distinct_pairs writes the job lengths):
    - prior pair runs of 1280 (value, time) rows (slot length 0), a middle key and the last key, then a
      batch that changes the presence of values at the start, middle and end of the runs and of absent values
      before the start, in a gap and past the end;
    - more than 8 prior pair batches, with keys probed in the batches past the eighth;
    - presence toggled 0 -> 1 -> 0 -> 1 in one batch, and negative multiplicities;
    - an activation in which byte 0's lane cancels to nothing while the others do not: one k_distinct_presence
      launch over jobs of different lengths, none a multiple of 256, the empty job between non-empty ones."""
    order = [1, 0, 2, 3, 4, 5, 6, 7][:n_distinct]
    lanes = byte_lanes(order, plain)
    cls = R.lane_class(len(lanes))
    a_lane = order.index(0)
    rng = np.random.default_rng(3200 + 10 * n_distinct + plain)
    g, o = lanes_op(mz, ctx, lanes, 4), ReduceLanesDistinct(oracle, lanes, 32)
    # prior: random rows, and 64 values (4, 6, ..., 130) x 20 times of MID and LAST (every lane sees the same
    # byte): runs of 1280 pair rows, which the seal's index stores with slot length 0
    hk = np.repeat(np.array([MID, LAST], np.uint64), 1280)
    hv = rep(np.tile(np.repeat(4 + 2 * np.arange(64), 20), 2))
    ht = np.tile(np.arange(20), 128)
    w = np.zeros((2000 + 2560, 4), np.uint64)
    w[:2000, 0] = rng.integers(0, 300, 2000)
    w[:2000, 1] = rng.integers(0, 2**64, 2000, dtype=np.uint64) & rep(0x0F)
    w[:2000, 2] = rng.integers(0, 10, 2000)
    w[:2000, 3] = rng.choice([-1, 1, 2], 2000).astype(np.int64).view(np.uint64)
    w[2000:, 0], w[2000:, 1], w[2000:, 2], w[2000:, 3] = hk, hv, ht, 1

    def rows_of(keys, t):
        w = np.zeros((len(keys), 4), np.uint64)
        w[:, 0] = keys
        w[:, 1] = rng.integers(0, 2**64, len(keys), dtype=np.uint64) & rep(0x0F)
        w[:, 2], w[:, 3] = t, rng.choice([-1, 1, 2], len(keys)).astype(np.int64).view(np.uint64)
        return w

    step_dev(mz, ctx, g, o, np.concatenate([w, rows_of(FIXED, 0)]), 20)
    for l in range(n_distinct):
        check_hot_slots(mz, ctx, g, g.distinct_trace(l))

    # more than 8 prior pair batches, each holding the FIXED keys (not MID or LAST)
    def steps():
        for i, e in enumerate(list(range(10, -1, -1)) + [0, 0]):
            yield np.concatenate([rows_of(rng.choice(np.arange(1000, 3000), size=1 << e, replace=False), 20 + i),
                                  rows_of(FIXED, 20 + i)]), 21 + i

    def expect(w, upper):
        with Trace(ctx) as tr:
            step_dev(mz, ctx, g, o, w, upper)
        tr.only("k_distinct_presence<C>")

    seen, deep = run_decreasing(mz, ctx, g, steps(), FIXED, expect, lambda g: g.distinct_trace(0))
    t = 33
    # presence changes on the hot runs (4, 68, 130 present; 1, 33, 200 absent: before the start, in a gap, past
    # the end), a toggle, a negative count
    vals = (1, 4, 33, 68, 130, 200)
    spec = []
    for k in (MID, LAST):
        for v in vals:
            m = o.pair_mult[0].get((k, v), 0)
            spec.append((k, v, t, -m if m else 1))
    spec += [(5000, 3, t, 1), (5000, 3, t + 1, -1), (5000, 3, t + 2, 2), (5001, 4, t, -1)]
    w = np.array([(k, int(rep(v)), tt, d & M64) for k, v, tt, d in spec], dtype=np.uint64)
    for k in (MID, LAST):
        assert {v for v in vals if o.pair_mult[0].get((k, v), 0)} == {4, 68, 130}
    for l in range(n_distinct):  # the runs this activation probes are still stored with slot length 0
        check_hot_slots(mz, ctx, g, g.distinct_trace(l))
    with Trace(ctx) as tr:
        out = step_dev(mz, ctx, g, o, w, t + 3)
    tr.only("k_distinct_presence<C>")
    assert int((out["key"] == 5000).sum()) >= 3
    t += 3
    # the cancelling activation: pairs (k, x, +1), (k, y, -1) with the same byte 0 and other bytes drawn from
    # ranges that differ per lane
    rng = np.random.default_rng(3250)
    P = 700
    x = np.zeros(P, np.uint64)
    y = np.zeros(P, np.uint64)
    b0 = rng.integers(0, 256, P).astype(np.uint64)
    for j in range(1, 8):
        x |= rng.integers(0, 2 + 9 * j, P).astype(np.uint64) << np.uint64(8 * j)
        y |= rng.integers(0, 2 + 9 * j, P).astype(np.uint64) << np.uint64(8 * j)
    keys = rng.integers(10_000, 10_300, P).astype(np.uint64)
    w = np.zeros((2 * P, 4), np.uint64)
    w[:, 0] = np.r_[keys, keys]
    w[:, 1] = np.r_[x | b0, y | b0]
    w[:, 2] = t
    w[:, 3] = np.r_[np.ones(P, np.int64), -np.ones(P, np.int64)].view(np.uint64)
    with Trace(ctx) as tr:
        out = step_dev(mz, ctx, g, o, w, t + 1)
    tr.only("k_distinct_presence<C>")
    assert tr.launches["k_distinct_presence<C>"] == 1, tr.launches
    lens = []
    for l in range(n_distinct):
        pe = words(g.distinct_trace(l).export())
        same(pe, words(o.pair_export(l)))
        lens.append(int((pe[:, 2] == np.uint64(t)).sum()))
    assert lens[a_lane] == 0 and all(n % 256 for n in lens[:a_lane] + lens[a_lane + 1 :]), lens
    assert len(set(lens)) == len(lens) and max(lens) > 256, lens
    # keys new in this activation: lane A (l > 0) holds nothing while the others' pairs make total > 0 (bit 2A)
    assert a_lane > 0 and any(int(r["flags"]) & (1 << (2 * a_lane)) for r in out if int(r["diff"]) == 1)
    same_arrangement(g, o)
    note(cls, tr, f"distinct: {n_distinct} lanes{' + plain' if plain else ''}, jobs {lens}, pair slot length 0, "
                  f"{seen} prior pair batches (keys probed in batch 8+ by {deep} activations)")


# ------------------------------------------------------------------ HAVING
def test_having_class8_toggles_on_hot_key_and_many_prior_batches(mz, ctx, oracle):
    """C = 8, single pass, SUM(lane 6) > 0: MID and LAST (slot length 0 in a prior batch) switch between
    visible and invisible at each of 100 times of one batch, after more than 8 prior batches."""
    rng = np.random.default_rng(3300)
    lanes = R.two_pass_lanes(8, 5)
    preds = [[sum_(6), num(0), cmp("gt")]]
    g, o = lanes_op(mz, ctx, lanes, 5, mz.having(*preds)), ReduceLanesHaving(oracle, lanes, 40, preds)
    fixed = FIXED + [MID, LAST]
    step(mz, g, o, with_fixed(rng, hot_rows(rng, 5, 0, small=True), 5, FIXED, 0), 1500)

    def expect(w, upper):
        with Trace(ctx) as t:
            step(mz, g, o, w, upper)
        t.only(LB_HV, never=TWO + (LB,))

    seen, deep = run_decreasing(mz, ctx, g, decreasing(rng, 5, 1500, 12, np.arange(1 << 13), fixed, small=True),
                                fixed, expect)
    check_hot_slots(mz, ctx, g)
    spec = []
    for k in (MID, LAST):
        acc = o.acc[k][7][1]
        s = acc - (1 << 128) if acc >> 127 else acc
        for i in range(100):
            v = (-s + 1) if s <= 0 else (-s - 1)  # the sum alternates between +1 and -1
            s += v
            spec.append([k, v & M64, 0, 2000 + i, 1])
    with Trace(ctx) as t:
        out = step(mz, g, o, np.array(spec, dtype=np.uint64), 2100)
    t.only(LB_HV, never=TWO + (LB,))
    assert int(((out["key"] == MID) & (out["diff"] == 1)).sum()) >= 49
    same_arrangement(g, o)
    note(8, t, f"HAVING: visibility toggled at 100 times of a slot-length-0 key, {seen} prior batches "
               f"(keys probed in batch 8+ by {deep} activations)")


# ------------------------------------------------------------------ monotonic MIN / MAX
def mono_op(mz, ctx, lanes, iw, must_consolidate=False):
    return mz.ReduceMonotonic(ctx, [mz.accum_lane(*l) for l in lanes], 8 * iw, must_consolidate)


def mono_step(mz, g, o, w, upper):
    want, werr = o.step(w, upper)
    out, errs = g.step(as_in(mz, w), upper)
    same(out, words(want))
    same(errs, words(werr))
    return want


def mono_arrangement(g, o):
    same(words(g.input_trace().export()), words(o.export()))


@pytest.mark.parametrize("iw", [4, 5])
@pytest.mark.parametrize("cls", [4, 8])
def test_mono_two_pass(mz, cls, iw):
    """25.2 M distinct keys over two activations (the second gives half of the keys fresh values, the others
    repeat theirs): k_monotonic_corrections<C, false / true> and k_scan_tiles; the full output against
    lanes_paths_ref and every row of 2000 sampled keys of the arrangement."""
    n = 25_200_000
    assert 2 * n > BOUND
    rng = np.random.default_rng(3400 + cls + iw)
    lanes = R.two_pass_lanes(cls, iw, mono=True)
    w1, w2, fresh = R.mono_input(rng, n, iw)

    def run(c):
        g = mono_op(mz, c, lanes, iw)
        first, second, _ = R.two_pass_expect("mono", lanes, w1, w2)
        for w, upper, want in ((w1, 1, first), (w2, 2, second)):
            with Trace(c) as t:
                out, errs = g.step(as_in(mz, w), upper)
            assert len(errs) == 0
            same(out, want)
            t.only(*MONO_TWO, "k_scan_tiles", never=(MONO_LB,))
        assert 0 < len(np.unique(second[:, 0])) <= fresh.sum()
        assert g.input_trace().size()["updates"] == 2 * n
        pick = np.sort(rng.choice(n, size=2000, replace=False))
        same(_key_rows(mz, c, g, w1[pick, 0], merge=ref_consolidate), R.two_pass_arrangement("mono", lanes, w1, w2, pick))
        note(cls, t, f"monotonic two-pass ({n} keys, R{8 * iw})")
        del g

    private(mz, f"mono two-pass C={cls} R{8 * iw}", run)


@pytest.mark.parametrize("cls", [4, 8])
def test_mono_loose_device_bound_runs_two_pass(mz, cls):
    """A few thousand rows in a device buffer bounded past 24 Mi rows, after a real prior activation:
    monotonic_dev checks the bound it is given (it does not read the length back), so the two-pass kernels
    run; the output is the restatement's."""
    rng = np.random.default_rng(3500 + cls)
    lanes = R.two_pass_lanes(cls, 4, mono=True)

    def run(c):
        g, o = mono_op(mz, c, lanes, 4), ReduceMonotonic(lanes, 32)
        mono_step(mz, g, o, gen(rng, rng.integers(0, 700, 3000), np.zeros(3000), 4, np.ones(3000, np.int64)), 1)
        w = gen(rng, rng.integers(0, 900, 4000), rng.integers(1, 8, 4000), 4, rng.choice([1, 1, 2, 0, -1], 4000))
        buf, held = _dev_input(mz, c, w, _filler(LOOSE, 9), 9)
        want, werr = o.step(held, 9)
        with Trace(c) as t:
            out, errs = g.step_dev(buf, 9)
        same(out.download(), words(want))
        same(errs.download(), words(werr))
        assert len(werr) > 0 and len(want) > 1000
        t.only(*MONO_TWO, never=(MONO_LB,))
        mono_arrangement(g, o)
        note(cls, t, f"monotonic loose device bound ({LOOSE} rows, {len(held)} real): two-pass, prior arranged")

    private(mz, f"mono loose bound C={cls}", run)


@pytest.mark.parametrize("iw", [4, 5])
@pytest.mark.parametrize("cls", [4, 8])
def test_mono_hot_keys_and_many_prior_batches(mz, ctx, cls, iw):
    """mono_prior over runs with slot length 0 (MID and LAST; the run's last row holds an extremum the other
    rows do not) and over more than 8 prior batches; mono_walk's sort of 200 corrections of one key."""
    rng = np.random.default_rng(3600 + cls + iw)
    lanes = R.two_pass_lanes(cls, iw, mono=True)
    g, o = mono_op(mz, ctx, lanes, iw), ReduceMonotonic(lanes, 8 * iw)
    w = hot_rows(rng, iw, 0)
    w[:, iw - 1] = 1
    hot = (w[:, 0] == MID) | (w[:, 0] == LAST)
    w[hot, 1 : iw - 2] = np.uint64(0x5555555555555555)
    w[hot & (w[:, iw - 2] == 1499), 1 : iw - 2] = rng.integers(0, 2**64, size=(2, iw - 3), dtype=np.uint64)
    mono_step(mz, g, o, with_fixed(rng, w, iw, FIXED, 0), 1500)
    for k in (MID, LAST):  # precondition: the run's last row changes the key's accumulation
        assert o.acc[k] != [int(R.field(w[hot & (w[:, 0] == k)][:1], l, True)[0]) for l in lanes]

    def expect(w, upper):
        w[:, iw - 1] = np.where(w[:, iw - 1].view(np.int64) > 0, w[:, iw - 1], np.uint64(1))
        with Trace(ctx) as t:
            mono_step(mz, g, o, w, upper)
        t.only(MONO_LB, never=MONO_TWO)

    # (MID and LAST stay out of these: the last row of their slot-length-0 runs is the one above)
    seen, deep = run_decreasing(mz, ctx, g, decreasing(rng, iw, 1500, 13, np.arange(1 << 14), FIXED), FIXED, expect)
    check_hot_slots(mz, ctx, g)
    w = hot_probe(rng, iw, 2000)
    w[:, iw - 1] = 1
    w[:, 1] = np.uint64(M64 - 1000) + np.tile(np.repeat(np.arange(100, dtype=np.uint64), 2), 2)  # lane 0 (MAX) rises
    with Trace(ctx) as t:
        out = mono_step(mz, g, o, w, 2100)
    t.only(MONO_LB, never=MONO_TWO)
    assert int((out["key"] == MID).sum()) == 200
    mono_arrangement(g, o)
    note(cls, t, f"mono_prior: slot length 0 (middle and last key), {seen} prior batches (keys probed in batch 8+ "
                 f"by {deep} activations); 200 corrections of one key")


# lanes that leave bits 0-7 and 48-63 of val unread: rows that differ only there are one row to consolidate_named_if
CONSOLIDATE_LANES = {4: [(R.AGG_MAX, 1, 8, 16, False), (R.AGG_MIN, 1, 32, 8, True), (R.AGG_MAX, 1, 40, 8, False)]}
CONSOLIDATE_LANES[8] = CONSOLIDATE_LANES[4] + [(R.AGG_MIN, 1, 8, 8, False), (R.AGG_MAX, 1, 24, 8, True)]


@pytest.mark.parametrize("cls", [4, 8])
def test_mono_must_consolidate_with_device_counts(mz, ctx, cls):
    """must_consolidate through step_dev with device-only counts.  Pairs of rows that differ only in bits no
    lane reads -- (k, v | 1, t, +1) with (k, v | 2, t, -1), which cancel, and with (k, v | 2, t, -2), which
    leave -1 -- stay two rows in the input buffer and fold only in the operator's masked consolidation.  The
    corrections and the error collection match the restatement, and differ from those of an operator without
    must_consolidate on the same input (which keeps the +1 row and reports the negative one)."""
    rng = np.random.default_rng(3700 + cls)
    lanes = CONSOLIDATE_LANES[cls]
    assert R.mono_class(len(lanes)) == cls
    g, o = mono_op(mz, ctx, lanes, 4, True), ReduceMonotonic(lanes, 32, True)
    g0, o0 = mono_op(mz, ctx, lanes, 4, False), ReduceMonotonic(lanes, 32, False)
    for s in range(6):
        n, p = 3000, 300
        t0, upper, skip = 2 * s, 2 * s + 2, 2 * s + 7
        w = gen(rng, rng.integers(0, 400, n), rng.integers(t0, upper, n), 4, rng.choice([1, 1, 2, -1], n))
        w[:, 1] = rng.integers(0, 2**64, n, dtype=np.uint64) & np.uint64(~0xF & M64)
        pair = w[:p].copy()
        w[:p, 1] |= np.uint64(1)
        w[:p, 3] = 1
        pair[:, 1] |= np.uint64(2)
        pair[:, 3] = np.where(np.arange(p) < p // 2, -1, -2).astype(np.int64).view(np.uint64)
        w = np.concatenate([w, pair])
        outs = []
        for op, ref in ((g, o), (g0, o0)):
            buf, held = _dev_input(mz, ctx, w, _filler(500, skip), skip)
            assert len(held) == n + p  # no two rows of the buffer are equal: the pairs stay two rows
            want, werr = ref.step(held, upper)
            with Trace(ctx) as t:
                out, errs = op.step_dev(buf, upper)
            out, errs = out.download(), errs.download()
            same(out, words(want))
            same(errs, words(werr))
            t.only(MONO_LB, never=MONO_TWO)
            outs.append((out.tobytes(), errs.tobytes()))
        assert outs[0][0] != outs[1][0] and outs[0][1] != outs[1][1]
    mono_arrangement(g, o)
    mono_arrangement(g0, o0)
    note(cls, t, "monotonic must_consolidate with device-only counts (folds rows that differ in unread bits)")
