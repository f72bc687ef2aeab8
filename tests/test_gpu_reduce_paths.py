"""The one-column reduce on the GPU -- COUNT/SUM over int64 and float64, DISTINCT, threshold (kinds 0-3),
MIN / MAX (4, 5) and TopK (6) -- against the plain reference of tests/reduce_ref.py, on every path the
reduce kernels can take.

Every activation's output is compared byte for byte and in order, as the operator returned it (not
consolidated by the test), with the reference's consolidated rows: that also checks that the
accumulable kinds' corrections leave the kernel consolidated.  After each sequence the input
arrangement (`input_trace().export()`, times advanced to its logical compaction frontier) is compared
with the reference's.  Each case asserts the kernels it must reach and those it must not from the
profile report, and the data precondition it relies on (how many distinct live values a key has, a
run stored with length 0 in a batch's hash slot, how many prior batches an activation saw) from the
reference state or from the input trace's batches.  The paths reached are printed at the end of the
module (pytest -s).

Kernel names are those of the profile report: the one-column operator launches the lane kernels with
C = 1, reported as k_corrections_lb<C>, k_corrections<C, false / true>.

The cases past the single-pass bounds (two-pass accumulable, MIN / TopK refusals) build batches of up
to 25.2 M rows on private contexts; they check the output (against vectorised NumPy references), not
the arrangement."""
import ctypes as C

import numpy as np
import pytest

import arrangement_ref as aref
import reduce_ref as ref
from test_ref_reduce import activations, f64_values

pytestmark = pytest.mark.gpu

M64 = ref.M64
FE = ref.FE
REACHED = set()
E_UNSUPPORTED = -4
# MZ_BOUND_MAX_ROWS (host.cu): the single-pass form writes at most per_row output rows per row of the
# sealed batch into one buffer of at most 48 Mi rows; per_row = 2 for kinds 0-5 and 2 * min(limit, 32) + 2
# for TopK (LIMIT NULL counts as 32).  The bound is checked against the batch's len_ub and, when that does
# not fit, against its length read back: the refusals below apply to the actual row count.
BOUND = 48 << 20


def single_pass_rows(per_row):
    return BOUND // per_row


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
    print("\nreduce paths reached:")
    for p in sorted(REACHED):
        print(f"  {p}")


class Trace:
    """Profiling over a block: the names of every kernel launched in it, and each one's launch count."""

    def __init__(self, ctx):
        self.ctx = ctx

    def __enter__(self):
        self.ctx.profile(True)
        self.ctx.profile_report()
        return self

    def __exit__(self, *exc):
        try:
            if exc[0] is None:
                self.launches = {k.strip("()"): v["launches"] for k, v in self.ctx.profile_report().items()}
                self.kernels = set(self.launches)
        finally:
            self.ctx.profile(False)

    def ran(self, prefix):
        return any(k.startswith(prefix) for k in self.kernels)

    def only(self, *prefixes, never=()):
        """Every prefix ran and none of `never` did; the reduce kernels that ran are noted."""
        for p in prefixes:
            assert self.ran(p), (p, self.kernels)
        for p in never:
            assert not self.ran(p), (p, self.kernels)
        for k in self.kernels:
            if k.startswith(("k_explode", "k_corrections", "k_minmax_lb", "k_scan_tiles")):
                REACHED.add(k)


def note(path):
    REACHED.add(path)


ACC_SINGLE = dict(never=("k_corrections<", "k_minmax_lb"))
MM = dict(never=("k_explode", "k_corrections"))


# ------------------------------------------------------------------ helpers
def words(a):
    return np.ascontiguousarray(a).view(np.uint64).reshape(len(a), a.dtype.itemsize // 8)


def r32(mz, w):
    return aref.as_rows(np.asarray(w, dtype=np.uint64).reshape(-1, 4), mz.R32)


def rows(spec):
    """(n, 4) u64 words from (key, val, time, diff) tuples (diffs signed)."""
    a = np.zeros((len(spec), 4), dtype=np.uint64)
    for i, row in enumerate(spec):
        for j, x in enumerate(row):
            a[i, j] = np.uint64(int(x) & M64)
    return a


def same(got, want):
    got = words(got) if got.dtype.names else got
    assert len(got) == len(want), (len(got), len(want))
    if got.tobytes() != want.tobytes():
        bad = int(np.flatnonzero(np.any(got != want, axis=1))[0])
        raise AssertionError(f"row {bad} of {len(want)}: got {got[bad].tolist()}, want {want[bad].tolist()}")


def new_op(mz, ctx, kind, limit=None, offset=0, desc=False):
    g = mz.TopK(ctx, limit, offset, desc) if kind == ref.TOPK else mz.ReduceAccumulable(ctx, kind)
    return g, ref.make(kind, limit, offset, desc)


def step(mz, g, r, w, upper):
    """One activation through both; the GPU's rows as returned, against the reference's."""
    want = r.step(w, upper)
    same(g.step(r32(mz, w), upper), want)
    return want


def same_arrangement(g, r):
    tr = g.input_trace()
    same(tr.export(), r.export(tr.get_logical_compaction()))


def trace_batches(mz, ctx, g, sp=None):
    """The batches of g's input trace (or of the spine sp), oldest first (each retained, so they outlive
    later merges)."""
    sp = sp if sp is not None else g.input_trace()
    arr = (C.c_void_p * 128)()
    n = C.c_uint32(0)
    ctx.check(mz._ffi.lib.mzgpu_spine_batches_through(sp.h, sp.read_upper(), arr, 128, C.byref(n)))
    out = []
    for i in range(n.value):
        mz._ffi.lib.mzgpu_batch_retain(arr[i])
        out.append(mz.Batch(ctx, C.c_void_p(arr[i]), sp.row_bytes))
    return out


def slot_len(b, key):
    """The run length field of `key`'s slot in batch b's index (None when the key is absent)."""
    slots, _, _ = b.index()
    s = np.ascontiguousarray(slots).view(np.uint64).reshape(-1, 2)
    hit = np.flatnonzero((s[:, 0] == np.uint64(key)) & (s[:, 1] != 0))
    return None if len(hit) == 0 else int(s[hit[0], 1]) >> 44


def zero_slot_batch(mz, ctx, g, key, sp=None):
    """A batch of the input trace (or of the spine sp) holding `key` with run length 0 in its slot, and
    that batch's keys."""
    for b in trace_batches(mz, ctx, g, sp):
        if slot_len(b, key) == 0:
            return b, np.unique(words(b.rows())[:, 0])
    raise AssertionError(f"no batch stores key {key} with slot length 0")


# ------------------------------------------------------------------ accumulable, single pass
@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_accumulable_sequences(mz, ctx, kind):
    """30+ activations of Zipf keys with retractions (groups empty out and come back), an empty
    activation, one whose input cancels completely, and rows at times near 2^64 - 2 that wait in the
    batcher until the last activations ship them."""
    rng = np.random.default_rng(1000 + kind)
    g, r = new_op(mz, ctx, kind)
    late = rows([(3, 5, M64 - 2, 1), (3, 7, M64 - 3, 2), (1 << 40, 9, M64 - 2, -1), (1, 0, M64 - 3, 1)])
    n_out = 0
    for i, (w, upper) in enumerate(activations(rng, kind, 32, 500)):
        if i == 3:
            w = np.concatenate([w, late])
        if i == 7:
            w = w[:0]
        if i == 11:
            neg = w.copy()
            neg[:, 3] = (-neg[:, 3].view(np.int64)).view(np.uint64)
            w = np.concatenate([w, neg])
        with Trace(ctx) as t:
            n_out += len(step(mz, g, r, w, upper))
        if len(w) and i != 11:
            t.only("k_explode", "k_corrections_lb<C>", **ACC_SINGLE)
        if i == 7:  # (the batcher's held rows are sealed again: a batch bound, no rows)
            t.only(never=("k_explode", "k_corrections<"))
    for upper in (M64 - 2, FE):
        with Trace(ctx) as t:
            step(mz, g, r, rows([]), upper)
        t.only("k_corrections_lb<C>", never=("k_explode", "k_corrections<"))
    assert n_out > 1000
    same_arrangement(g, r)
    note(f"kind {kind}: 34 activations (empty, cancelling, times up to 2^64 - 2)")


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("where", ["middle", "last"])
def test_hot_key_run_with_slot_length_zero(mz, ctx, kind, where):
    """A key with 1500 distinct times in one activation: its run is stored with length 0 in the slot
    (any seal or merge of that batch: the index records runs shorter than 1024, or of 64 rows or
    fewer), so prior_sum scans the run to its end when the next activation probes the key."""
    rng = np.random.default_rng(1100 + kind + (where == "last"))
    g, r = new_op(mz, ctx, kind)
    hot = 600 if where == "middle" else 5000
    w = np.zeros((3000, 4), dtype=np.uint64)
    w[:, 0] = rng.integers(0, 1200, size=3000, dtype=np.uint64)
    w[:, 2] = rng.integers(0, 100, size=3000, dtype=np.uint64)
    w[:, 3] = 1
    h = np.zeros((1500, 4), dtype=np.uint64)
    h[:, 0], h[:, 2], h[:, 3] = hot, np.arange(1500, dtype=np.uint64), 1
    vals = f64_values(rng, 4500) if kind == 1 else rng.integers(-(2**62), 2**62, size=4500, dtype=np.int64).view(np.uint64)
    w = np.concatenate([w, h])
    w[:, 1] = vals
    step(mz, g, r, w, 1500)
    b, keys = zero_slot_batch(mz, ctx, g, hot)
    assert (keys.max() == hot) == (where == "last") and keys.min() < hot
    probe = rows([(hot, 3, 1600, 1), (int(keys[0]), 4, 1601, 1), (hot, 5, 1602, -1)])
    with Trace(ctx) as t:
        assert len(step(mz, g, r, probe, 1700)) >= 2
    t.only("k_explode", "k_corrections_lb<C>", **ACC_SINGLE)
    same_arrangement(g, r)
    note(f"prior_sum: run of 1500 rows with slot length 0 ({where} key of its batch)")


def test_more_than_eight_prior_batches(mz, ctx):
    """Activations of decreasing size (distinct (key, time) rows: 2^15 down to 1) leave one batch per
    spine layer: more than 8 prior batches, which prior_sum reads in groups of 8 hash slots (GROUP = 8).
    Keys come from one pool, so the activations probe keys held in many prior batches."""
    rng = np.random.default_rng(1200)
    g, r = new_op(mz, ctx, 0)
    seen = []
    t = 0
    for e in list(range(15, -1, -1)) + [0, 0]:
        n = 1 << e
        w = np.zeros((n, 4), dtype=np.uint64)
        w[:, 0] = rng.choice(1 << 16, size=n, replace=False).astype(np.uint64)
        w[:, 1] = rng.integers(-1000, 1000, size=n).astype(np.int64).view(np.uint64)
        w[:, 2] = t
        w[:, 3] = rng.integers(-2, 3, size=n).astype(np.int64).view(np.uint64)
        seen.append(g.input_trace().size()["batches"])
        with Trace(ctx) as tr:
            step(mz, g, r, w, t + 1)
        tr.only("k_corrections_lb<C>", **ACC_SINGLE)
        t += 1
    assert max(seen) > 8, seen
    same_arrangement(g, r)
    note(f"prior_sum: up to {max(seen)} prior batches (more than GROUP = 8)")


# ------------------------------------------------------------------ edge values
def _edge_case(mz, ctx, kind, values, seed):
    """Each value under its own key and in a shared key, with diffs +-1, +-3 and the i64 extremes,
    over three activations (inserted, partly retracted, the rest retracted)."""
    rng = np.random.default_rng(seed)
    g, r = new_op(mz, ctx, kind)
    diffs = [1, -1, 3, -3, (1 << 63) - 1, -(1 << 63)]
    spec = []
    for i, v in enumerate(values):
        for j, d in enumerate(diffs):
            spec.append((100 + 8 * i + j, v, j % 3, d))
            spec.append((7, v, j % 3, d if j < 4 else 1))
    w = rows(spec)
    step(mz, g, r, w, 3)
    back = w[rng.random(len(w)) < 0.5].copy()
    back[:, 3] = (-back[:, 3].view(np.int64)).view(np.uint64)
    back[:, 2] = 3
    step(mz, g, r, back, 4)
    with Trace(ctx) as t:
        step(mz, g, r, np.concatenate([w, back]) * np.array([1, 1, 0, 1], dtype=np.uint64) + np.array([0, 0, 5, 0], dtype=np.uint64), 6)
    t.only("k_explode", "k_corrections_lb<C>", **ACC_SINGLE)
    same_arrangement(g, r)
    return g, r


def test_f64_edge_values(mz, ctx):
    b = ref.bits
    ulp39 = 2.0**-13
    values = [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308,
              2.0**39 - ulp39 / 2, 2.0**39, 2.0**39 + ulp39, -(2.0**39 + ulp39),
              2.0**60, -(2.0**60), 1e20, -1e20, 2.0**100, -(2.0**100), 2.0**92 + 2.0**40,
              2.0**103 - 2.0**50, 2.0**103, -(2.0**103), 1e300, -1e300,
              float("inf"), float("-inf")]
    vb = [b(x) for x in values] + [0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000123, 0xFFFFFFFFFFFFFFFF]
    _edge_case(mz, ctx, 1, vb, 1300)
    # sums on the rounding edges, one key each (the rows of an activation share one time)
    g, r = new_op(mz, ctx, 1)
    cases = {
        1: [2.0**93, 2.0**40],  # 2^117 + 2^64: a tie, to even (2^93)
        2: [2.0**93, 2.0**40, 2.0**-24],  # ... + 1: the sticky bit rounds up
        3: [2.0**36, 2.0**-17 + 2.0**-24],  # 2^60 + 129 below 2^64: rounds up (not toward zero)
        4: [-(2.0**100), 2.0**100, 1.0],  # the [2^116, 2^127) branch and its negation cancel exactly
        5: [-1e300, -1e300],  # saturated twice: wraps
        6: [-1e300],  # -2^127 converts exactly
        7: [-(2.0**60), 2.0**60 + 2.0**8],
    }
    spec = [(k, b(x), 0, 1) for k, xs in cases.items() for x in xs]
    spec += [(8, b(float("inf")), 0, 1), (8, b(0.0), 0, -1)]  # net zero: only pos_infs is left (flag bit 1)
    spec += [(9, b(float("nan")), 0, 1), (9, b(2.5), 0, -1)]
    with Trace(ctx) as t:
        out = step(mz, g, r, rows(spec), 1)
    t.only("k_explode", "k_corrections_lb<C>", **ACC_SINGLE)
    got = {int(row[0]): row for row in out.tolist()}
    assert got[1][2] == b(2.0**93) and got[2][2] == b((2.0**117 + 2.0**65) / 2.0**24)
    assert got[3][2] == b((2.0**60 + 256) / 2.0**24) and got[4][2] == b(1.0) and got[6][2] == b(-(2.0**103))
    assert got[8][4] == 2 and got[8][2] == ref.PINF_BITS and got[9][4] == 2
    same_arrangement(g, r)
    note("f64 fixed point: both conversion branches, saturation, ties, sticky bit, flag bit 1 via pos_infs")


def test_i64_edge_values(mz, ctx):
    g, r = _edge_case(mz, ctx, 0, [(1 << 63) - 1, -((1 << 63) - 1), 1 << 63, 0, 1, M64], 1400)
    # sums wrapping past 2^127
    spec = [(1, (1 << 63) - 1, 7, (1 << 63) - 1)] * 3 + [(1, 1 << 63, 7, -(1 << 63))] * 2
    out = step(mz, g, r, rows(spec), 8)
    assert len(out) > 0
    same_arrangement(g, r)
    note("i64: extreme values times extreme diffs, sums wrapping at 2^128")


# ------------------------------------------------------------------ accumulable, two-pass
def _two_pass_expect(kind, keys, v1, v2, back):
    """Activation outputs for one row per key at time 0 (value v1, diff 1), then at time 1 either its
    retraction (back) or a second row (v2, diff 1); exact sums of integers or multiples of 2^-24."""
    n = len(keys)

    def sums(v):
        if kind == 1:
            return (v.astype(np.float64) / 2.0**24).view(np.uint64), np.zeros(len(v), np.uint64)
        return v.view(np.uint64), (v >> 63).view(np.uint64)

    def block(k, count, v, t, d):
        w = np.zeros((len(k), 8), dtype=np.uint64)
        w[:, 0] = k
        if kind in (0, 1):
            w[:, 1] = count
            w[:, 2], w[:, 3] = sums(v)
        elif kind == 2:
            w[:, 1] = 1
        w[:, 5] = t
        w[:, 6] = np.uint64(d & M64)
        return w

    order = np.argsort(keys)
    first = block(keys, 1, v1, 0, 1)[order]
    stay = ~back
    parts = [block(keys[back], 1, v1[back], 1, -1)]
    if kind in (0, 1):
        parts += [block(keys[stay], 1, v1[stay], 1, -1), block(keys[stay], 2, v1[stay] + v2[stay], 1, 1)]
    elif kind == 3:
        parts += [block(keys[stay], 0, v1[stay], 1, 1)]
    second = np.concatenate(parts)
    second = second[np.lexsort([second[:, 1], second[:, 0]])]
    assert n == len(first)
    return first, second


def _key_rows(mz, ctx, g, keys, merge=aref.consolidate):
    """The input trace's rows of `keys`, found through each batch's cursor (seek_keys), merged by `merge`
    (which takes (n, words) u64 rows; the default sums a one-word diff)."""
    keys = np.unique(np.asarray(keys, dtype=np.uint64))
    parts = []
    for b in trace_batches(mz, ctx, g):
        for run in b.seek_keys(keys):
            if run["len"] > 0 and run["key"] in keys:
                parts.append(words(b.rows_range(int(run["first"]), int(run["len"]))))
    nw = g.input_trace().row_bytes // 8
    return merge(np.concatenate(parts) if parts else np.zeros((0, nw), dtype=np.uint64))


def _two_pass_arrangement(kind, keys, v1, v2, back):
    """The mzgpu_racc rows the two activations of the two-pass case leave for `keys`: (key, 0) with
    diff 1 and value v1, (key, 1) with the retraction of v1 or a second row of value v2."""
    def block(t, d, v):
        w = np.zeros((len(keys), 10), dtype=np.uint64)
        w[:, 0], w[:, 1], w[:, 2] = keys, t, d.view(np.uint64)
        if kind in (0, 1):  # (kind 1: the values are v / 2^24, so the accumulator is v itself)
            acc = d * v
            w[:, 3], w[:, 4], w[:, 5] = d.view(np.uint64), acc.view(np.uint64), (acc >> 63).view(np.uint64)
        return w

    one = np.ones(len(keys), dtype=np.int64)
    w = np.concatenate([block(0, one, v1), block(1, np.where(back, -one, one), np.where(back, v1, v2))])
    return w[np.lexsort([w[:, 1], w[:, 0]])]


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_two_pass_past_the_single_pass_bound(mz, kind):
    """A batch of more than 24 Mi distinct (key, time) rows: 2 x rows exceeds the single-pass bound
    (48 Mi output rows), so k_corrections<C, false / true> and k_scan_tiles run; the second activation
    retracts half of the keys and adds a row to the others (their prior sums are read back)."""
    n = single_pass_rows(2) + 34_176  # 25,200,000
    rng = np.random.default_rng(1500 + kind)
    keys = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(2**40 - 1)
    v1 = rng.integers(-(2**40), 2**40, size=n, dtype=np.int64)
    v2 = rng.integers(-(2**40), 2**40, size=n, dtype=np.int64)
    back = rng.random(n) < 0.5
    first, second = _two_pass_expect(kind, keys, v1, v2, back)

    def vals(v):
        return (v.astype(np.float64) / 2.0**24).view(np.uint64) if kind == 1 else v.view(np.uint64)

    a = np.zeros(n, dtype=mz.R32)
    a["key"], a["val"], a["time"], a["diff"] = keys, vals(v1), 0, 1
    b = a.copy()
    b["time"] = 1
    b["diff"] = np.where(back, -1, 1)
    b["val"] = np.where(back, a["val"], vals(v2))
    c = mz.Context(0)
    try:
        g = mz.ReduceAccumulable(c, kind)
        for rows_, upper, want in ((a, 1, first), (b, 2, second)):
            with Trace(c) as t:
                got = g.step(rows_, upper)
            same(got, want)
            t.only("k_explode", "k_corrections<C,_false>", "k_corrections<C,_true>", "k_scan_tiles",
                   never=("k_corrections_lb", "k_minmax_lb"))
        # the input arrangement: its row count, and every row of 2000 sampled keys (a full export of
        # 50 M accumulator rows would take 4 GB on each side)
        assert g.input_trace().size()["updates"] == 2 * n
        pick = np.sort(rng.choice(n, size=2000, replace=False))
        same(_key_rows(mz, c, g, keys[pick]), _two_pass_arrangement(kind, keys[pick], v1[pick], v2[pick], back[pick]))
        del g
    finally:
        c.close()
    note(f"kind {kind}: two-pass corrections ({n} rows per activation)")


# ------------------------------------------------------------------ MIN / MAX
def _live(r, k):
    return len(r.live(k))


@pytest.mark.parametrize("kind", [4, 5])
def test_minmax_table_and_stream(mz, ctx, kind):
    """Keys with 31, 32 and 33 distinct live values in the prior batches; a key that first overflows the
    32-entry table while the new batch's times are replayed; values inserted and cancelled across prior
    batches (dead entries reused); the u64 edge values; error rows that appear and are repaired on the
    table path and on the stream path.  Wide keys take a new extremum at a later time of the batch."""
    rng = np.random.default_rng(1600 + kind)
    g, r = new_op(mz, ctx, kind)
    lo_first = kind == 4
    K31, K32, K33, KREPLAY, KDEAD, KEDGE, KERR, KWERR = 31, 32, 33, 40, 50, 60, 70, 80

    def vals(k, n, base=1000, t=0):
        return [(k, (base + 7 * i) << 20, t, 1) for i in range(n)]

    narrow = [(1000 + i, int(v) << 40, 0, int(d)) for i, v, d in
              zip(rng.integers(0, 300, 2000), rng.integers(0, 9, 2000), rng.integers(-1, 3, 2000))]
    a1 = vals(K31, 20) + vals(K32, 20) + vals(K33, 20) + vals(KREPLAY, 32) + vals(KDEAD, 20) + vals(KWERR, 40)
    a1 += [(KEDGE, v, 0, 1) for v in (0, (1 << 63) - 1, 1 << 63, M64)] + [(KERR, 5, 0, 1)] + narrow
    step(mz, g, r, rows(a1), 1)
    # second prior batch: the rest of the widths; KDEAD cancels its 10 smallest values (which the table
    # meets first) and adds 20 larger ones
    a2 = vals(K31, 11, 5000, 1) + vals(K32, 12, 5000, 1) + vals(K33, 13, 5000, 1)
    a2 += [(KDEAD, (1000 + 7 * i) << 20, 1, -1) for i in range(10)] + [(KDEAD, (9000 + i) << 20, 1, 1) for i in range(20)]
    step(mz, g, r, rows(a2), 2)
    assert [_live(r, k) for k in (K31, K32, K33, KREPLAY)] == [31, 32, 33, 32]
    # KDEAD: 40 distinct values, 30 live; its cancellations precede its new values in value order
    assert _live(r, KDEAD) == 30 and len(r.counts[KDEAD]) == 40
    ext = 1 if lo_first else M64 - 1  # a new extremum
    mid = 3000 << 20
    # K31 reaches 32 values (the table is full) and then 33 at a later time; K32 retracts a value and
    # takes a new one (the dead entry is reused: 32 entries, still the table); K33 and KWERR are on the
    # stream from the start and take a new extremum at a later time than a middle value
    a3 = [(K31, mid, 2, 1), (K31, ext, 3, 1), (K32, 1000 << 20, 2, -1), (K32, ext, 3, 1)]
    for k in (K33, KDEAD, KWERR):
        a3 += [(k, mid + k, 2, 1), (k, ext, 3, 1)]
    a3 += [(KREPLAY, mid, 2, 1), (KREPLAY, ext, 3, 1), (KREPLAY, mid + 1, 4, 1)]  # the 33rd value arrives at time 2
    a3 += [(KEDGE, M64, 2, -1), (KEDGE, 0, 3, -1), (KERR, 6, 2, -1), (KWERR, 1000 << 20, 2, -3)]
    with Trace(ctx) as t:
        out = step(mz, g, r, rows(a3), 5)
    t.only("k_minmax_lb", **MM)
    errs = {int(row[0]) for row in out.tolist() if row[4] == 2 and row[6] == 1}
    assert errs == {KERR, KWERR}, errs
    assert _live(r, K31) == 33 and _live(r, K32) == 32 and _live(r, KREPLAY) == 35
    a4 = [(KERR, 6, 5, 1), (KWERR, 1000 << 20, 6, 2), (K32, ext, 5, -1), (K33, ext, 6, -1)]
    with Trace(ctx) as t:
        out = step(mz, g, r, rows(a4), 7)
    t.only("k_minmax_lb", **MM)
    assert {int(row[0]) for row in out.tolist() if row[4] == 2 and row[6] == M64} == {KERR, KWERR}
    same_arrangement(g, r)
    note("k_minmax_lb: 31 / 32 / 33 live values, overflow during replay, dead-entry reuse, error rows")


@pytest.mark.parametrize("kind", [4, 5])
def test_minmax_wide_runs_with_slot_length_zero(mz, ctx, kind):
    """Wide keys whose runs are stored with slot length 0 (1100 rows), as the first and as the last key
    of their batch: mm_runs finds the end of each run by binary search."""
    rng = np.random.default_rng(1700 + kind)
    g, r = new_op(mz, ctx, kind)
    first, last = 10, 1 << 50
    w = [(first, int(v), int(t), 1) for v, t in zip(rng.integers(1, 1 << 62, 1100), rng.integers(0, 4, 1100))]
    w += [(last, int(v), int(t), 1) for v, t in zip(rng.integers(1, 1 << 62, 1100), rng.integers(0, 4, 1100))]
    w += [(int(k), int(v), 0, 1) for k, v in zip(rng.integers(20, 5000, 3000), rng.integers(0, 1 << 62, 3000))]
    step(mz, g, r, rows(w), 4)
    for key, pos in ((first, 0), (last, -1)):
        b, keys = zero_slot_batch(mz, ctx, g, key)
        assert keys[pos] == key
    top = max(r.live(last)) if kind == 5 else min(r.live(last))
    a = [(first, 5, 4, 1), (first, M64 - 3, 5, 1), (last, top, 4, -1), (last, 1 << 61, 6, 1), (77, 3, 5, 1)]
    with Trace(ctx) as t:
        out = step(mz, g, r, rows(a), 8)
    t.only("k_minmax_lb", **MM)
    assert len(out) >= 4
    same_arrangement(g, r)
    note("k_minmax_lb: wide runs with slot length 0 (first and last key of the batch)")


# ------------------------------------------------------------------ TopK
TOPK_SHAPES = [(0, 0, False), (1, 0, True), (1, 2, False), (31, 3, False), (32, 0, True), (32, 5, False),
               (None, 10, False), (None, 10, True)]


@pytest.mark.parametrize("limit,offset,desc", TOPK_SHAPES)
def test_topk_table_and_stream(mz, ctx, limit, offset, desc):
    """Narrow keys (at most 12 distinct values, counts up to 3: the table; limits cut inside a value's
    copies, offsets past a group's total multiplicity, negative counts) and wide keys with 34-40 live
    values of count 1 (the stream: at most 41 live at any time, so with offset 10 the window stays
    within 32 distinct values), one of which goes
    negative and is repaired."""
    rng = np.random.default_rng(1800 + (limit or 99) * 7 + offset + desc)
    g, r = new_op(mz, ctx, ref.TOPK, limit, offset, desc)
    wide = {2000 + i: set() for i in range(5)}
    fresh = iter(range(1, 1 << 20))
    t = 0
    for s in range(7):
        n = 1500
        w = [(int(k), int(v) * 0x0123456789ABCDEF, int(tt), int(d)) for k, v, tt, d in
             zip(rng.integers(0, 150, n), rng.integers(0, 12, n), rng.integers(t, t + 3, n), rng.integers(-1, 4, n))]
        w += [(150, 5, t, 1)] if s == 0 else []  # total multiplicity 1 (below the offsets)
        for k, live in wide.items():
            if s > 0:
                assert _live(r, k) > 32
                for v in rng.choice(sorted(live), size=3, replace=False).tolist():
                    live.discard(v)
                    w.append((k, v << 8, t + 1, -1))
            while len(live) < 34 + int(rng.integers(0, 5)):
                v = next(fresh)
                live.add(v)
                w.append((k, v << 8, int(rng.integers(t, t + 3)), 1))
        if s == 3:
            w.append((2000, 7, t + 2, -1))  # negative count on the stream path
        if s == 4:
            w.append((2000, 7, t, 1))
        t += 3
        with Trace(ctx) as tr:
            out = step(mz, g, r, rows(w), t)
        tr.only("k_minmax_lb", **MM)
        if s == 3:
            assert any(row[0] == 2000 and row[4] == 2 and row[6] == 1 for row in out.tolist())
    assert all(len(r.counts.get(k, {})) <= 12 for k in range(150))
    same_arrangement(g, r)
    note(f"k_minmax_lb (TopK): limit {limit}, offset {offset}, {'desc' if desc else 'asc'}, table and stream")


def test_topk_window_of_32_and_33_distinct_values(mz, ctx):
    """On a group of 40 distinct values, a window of exactly 32 distinct values matches; one of 33 is
    reported MZGPU_E_UNSUPPORTED (the report poisons its context, hence a private one)."""
    w = rows([(7, v, 0, 1) for v in range(40)] + [(8, v, 0, 2) for v in range(10)])
    for limit, offset in ((32, 0), (None, 8), (32, 7)):
        g, r = new_op(mz, ctx, ref.TOPK, limit, offset)
        with Trace(ctx) as t:
            out = step(mz, g, r, w, 1)
        t.only("k_minmax_lb", **MM)
        assert int((out[:, 0] == 7).sum()) == 32
    for limit, offset in ((33, 0), (None, 7)):
        priv = mz.Context(0)
        try:
            with pytest.raises(mz.MzGpuError) as e:
                mz.TopK(priv, limit, offset).step(r32(mz, w), 1)
            assert e.value.status == E_UNSUPPORTED
        finally:
            priv.close()
    note("TopK: a window of 32 distinct values fits, 33 is reported")


# ------------------------------------------------------------------ single-pass bounds
def _distinct_rows(mz, n, seed):
    rng = np.random.default_rng(seed)
    a = np.zeros(n, dtype=mz.R32)
    a["key"] = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(2**40 - 1)
    a["val"] = rng.integers(0, 2**64, size=n, dtype=np.uint64)
    a["diff"] = 1
    return a


def _one_row_per_key(a):
    w = np.zeros((len(a), 8), dtype=np.uint64)
    w[:, 0], w[:, 2], w[:, 6] = a["key"], a["val"], 1
    return w[np.argsort(w[:, 0])]


def _refused(mz, c, op, a):
    with pytest.raises(mz.MzGpuError) as e:
        op.step(a, 1)
    assert e.value.status == E_UNSUPPORTED, e.value
    # the operator stays dead; the context does not
    with pytest.raises(mz.MzGpuError) as e:
        op.step(a[:3], 2)
    assert e.value.status == E_UNSUPPORTED, e.value
    ok = mz.TopK(c, 1)
    same(ok.step(a[:100], 1), _one_row_per_key(a[:100]))


@pytest.mark.parametrize("limit", [None, 1])
def test_topk_single_pass_bound(mz, limit):
    """TopK's single-pass bound: 48 Mi / (2 min(limit, 32) + 2) rows of the sealed batch -- 762,600 for
    LIMIT NULL, 12 Mi for LIMIT 1.  At the bound the activation runs and matches; one row past it is
    refused with MZGPU_E_UNSUPPORTED."""
    n = single_pass_rows(2 * (32 if limit is None else limit) + 2)
    assert n == (762_600 if limit is None else 12 << 20)
    a = _distinct_rows(mz, n + 1, 1900 + (limit or 0))
    c = mz.Context(0)
    try:
        g = mz.TopK(c, limit)
        with Trace(c) as t:
            same(g.step(a[:n], 1), _one_row_per_key(a[:n]))
        t.only("k_minmax_lb", **MM)
        _refused(mz, c, mz.TopK(c, limit), a)
    finally:
        c.close()
    note(f"TopK LIMIT {limit}: {n} rows single pass, {n + 1} refused")


def test_min_single_pass_bound(mz):
    """MIN / MAX: 24 Mi rows of the sealed batch; 24 Mi + 1 is refused."""
    n = single_pass_rows(2)
    assert n == 24 << 20
    a = _distinct_rows(mz, n + 1, 1950)
    c = mz.Context(0)
    try:
        _refused(mz, c, mz.ReduceAccumulable(c, ref.MIN), a)
    finally:
        c.close()
    note(f"MIN: {n + 1} rows refused")


# ------------------------------------------------------------------ device-resident input
def _dev_input(mz, ctx, w, filler, skip):
    """A device buffer from update_stream_dev: the rows of `w` and `filler` rows at `skip`, which the
    stream drops, so the row count is known on the device only and the buffer's bound counts the
    filler.  Returns the buffer and the rows it holds (the batch's consolidated rows not at skip)."""
    allw = np.concatenate([w, filler]) if len(filler) else w
    b = mz.Batch.build(ctx, r32(mz, allw), 0, skip + 1)
    got = aref.consolidate(w)
    return mz.update_stream_dev(ctx, b, None, skip), got[got[:, 2] != np.uint64(skip)]


def _filler(n, skip, key0=1 << 50):
    f = np.zeros((n, 4), dtype=np.uint64)
    f[:, 0] = np.arange(n, dtype=np.uint64) + np.uint64(key0)
    f[:, 2], f[:, 3] = skip, 1
    return f


@pytest.mark.parametrize("kind", [0, 1, 4, 6])
def test_device_resident_input(mz, ctx, kind):
    """A sample of activations through step_dev, with rows whose count is known only on the device."""
    rng = np.random.default_rng(2000 + kind)
    g, r = new_op(mz, ctx, kind, 3 if kind == ref.TOPK else None)
    out = mz.DeviceRows(ctx, 64)
    want = []
    for i, (w, upper) in enumerate(activations(rng, kind if kind < 4 else ref.MIN, 8, 300)):
        w = w[w[:, 2] < np.uint64(upper)]
        skip = upper + 5
        buf, held = _dev_input(mz, ctx, w, _filler(int(rng.integers(1, 500)), skip), skip)
        with Trace(ctx) as t:
            g.step_dev(buf, upper, out)
        t.only("k_minmax_lb" if kind >= 4 else "k_corrections_lb<C>", never=("k_corrections<",))
        want.append(r.step(held, upper))
    same(out.download(), np.concatenate(want))
    same_arrangement(g, r)
    note(f"kind {kind}: step_dev with device-only row counts")


@pytest.mark.parametrize("kind,limit,loose", [(6, None, 800_000), (4, None, (24 << 20) + 40_000)])
def test_loose_device_bound_runs_single_pass(mz, kind, limit, loose):
    """A few thousand real rows in a device buffer whose bound is past the single-pass bound (the
    filler rows sit at the dropped time): the length is read back and the single-pass form runs.  The
    buffer's length is not read before the step (that would tighten its bound); the bound the operator
    saw is its rows_in count (mzgpu_reduce_accumulable_buf adds the input's bound)."""
    rng = np.random.default_rng(2100 + kind)
    c = mz.Context(0)
    try:
        g, r = new_op(mz, c, kind, limit)
        w = np.zeros((4000, 4), dtype=np.uint64)
        w[:, 0] = rng.integers(0, 700, size=4000, dtype=np.uint64)
        w[:, 1] = rng.integers(0, 20, size=4000, dtype=np.uint64) << np.uint64(40)
        w[:, 3] = rng.integers(-1, 3, size=4000).astype(np.int64).view(np.uint64)
        buf, held = _dev_input(mz, c, w, _filler(loose, 9), 9)
        per_row = 2 if kind != ref.TOPK else 2 * (32 if limit is None else min(limit, 32)) + 2
        before = c.stats()["rows_in"]
        with Trace(c) as t:
            got = g.step_dev(buf, 1).download()
        seen_ub = c.stats()["rows_in"] - before
        assert seen_ub >= loose > single_pass_rows(per_row) > len(held), (seen_ub, loose, len(held))
        same(got, r.step(held, 1))
        t.only("k_minmax_lb", **MM)
        del g, buf
    finally:
        c.close()
    note(f"kind {kind}: loose device bound ({loose} rows) resolved to {len(held)} rows, single pass")
