"""The probe reference (tests/probe_ref.py) pinned against the CPU oracle on shared inputs, and by
hand at the edges: both half-join time filters at t2 == t1 and t2 == t1 +- 1 (and times 0 and
2^64 - 2), every closure part at its limits, the exact output order over three batches, join_core's
meet above both times and its side-1 value swap."""
import numpy as np
import pytest

import arrangement_ref as aref
import probe_ref as ref

M64 = ref.M64
FE = ref.FRONTIER_EMPTY
TMAX = M64 - 1  # the largest time a row can carry


def r32(rows):
    """(n, 4) u64 words from (key, val, time, diff) tuples (diffs as signed ints)."""
    a = np.zeros((len(rows), 4), dtype=np.uint64)
    for i, (k, v, t, d) in enumerate(rows):
        a[i] = (k, v, t, d & M64)
    return a


def as_r32(oracle, w):
    return np.ascontiguousarray(w, dtype=np.uint64).view(oracle.R32).reshape(-1)


def words(a):
    return ref._w(a)


def multiset(w):
    w = words(w)
    return sorted(map(tuple, w.tolist()))


def rand(rng, n, keys, vals, times, unique_vals=False, start=0):
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = rng.integers(0, keys, size=n, dtype=np.uint64)
    w[:, 1] = np.arange(start, start + n, dtype=np.uint64) if unique_vals else rng.integers(0, vals, size=n, dtype=np.uint64)
    w[:, 2] = rng.integers(0, times, size=n, dtype=np.uint64)
    d = rng.integers(1, 4, size=n) * rng.choice([-1, 1], size=n)
    w[:, 3] = d.astype(np.int64).view(np.uint64)
    return w


def trace(oracle, batches):
    """An oracle spine holding `batches` (each [lower, upper) = [i, i + 1)) and the reference's view of
    it: each batch consolidated, in insertion order."""
    sp = oracle.Spine(32, 1, True)
    refb = []
    for i, w in enumerate(batches):
        sp.insert(oracle.Batch.build(as_r32(oracle, w), i, i + 1))
        refb.append(aref.consolidate(w))
    return sp, refb


CL = dict(key_fields=[(2, 0, 10, 0)], val_fields=[(1, 0, 20, 0), (2, 10, 10, 20), (0, 0, 10, 40)], filters=[(2, 0, 20, "lt", 700)])


# ------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("mode", [ref.LE, ref.LT])
@pytest.mark.parametrize("cl", [None, CL])
def test_half_join_matches_oracle(oracle, mode, cl):
    rng = np.random.default_rng(10 + mode)
    # unique lookup values: the oracle sums the diffs of one (stream row, val2) over its times, so the
    # unconsolidated outputs are equal as multisets only when each (key, val2) sits at one time
    batches = [rand(rng, 3000, 400, 0, 6, unique_vals=True, start=3000 * i) for i in range(4)]
    sp, refb = trace(oracle, batches)
    stream = rand(rng, 4000, 450, 1 << 20, 8)
    ocl = oracle.make_closure(**cl) if cl else None
    got = ref.half_join(stream, refb, mode, cl)
    want = oracle.half_join(as_r32(oracle, stream), sp, mode, ocl, consolidate_output=False)
    assert len(got) > 1000
    assert multiset(got) == multiset(want)
    # consolidated, with repeated values (the oracle's per-value sums no longer matter)
    batches = [rand(rng, 3000, 300, 50, 6) for _ in range(3)]
    sp, refb = trace(oracle, batches)
    want = oracle.half_join(as_r32(oracle, stream), sp, mode, ocl, consolidate_output=True)
    assert aref.consolidate(ref.half_join(stream, refb, mode, cl)).tobytes() == words(want).tobytes()


def test_update_stream_and_map_rows_match_oracle(oracle):
    rng = np.random.default_rng(3)
    w = rand(rng, 5000, 100, 1 << 12, 3)
    cl = dict(key_fields=[(1, 0, 6, 0)], val_fields=[(0, 0, 64, 0)], filters=[(1, 6, 6, "ge", 10)])
    ob = oracle.Batch.build(as_r32(oracle, w), 0, 3)
    rows = aref.consolidate(w)
    for skip in (FE, 0, 1, 2):
        for c in (None, cl):
            want = oracle.update_stream(ob, oracle.make_closure(**c) if c else None, skip)
            assert ref.update_stream(rows, c, skip).tobytes() == words(want).tobytes(), (skip, c)
    want = oracle.map_rows(as_r32(oracle, w), oracle.make_closure(**cl))
    assert ref.update_stream(w, cl).tobytes() == words(want).tobytes()


@pytest.mark.parametrize("cl", [None, dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 8, 0), (2, 0, 8, 8)], filters=[(2, 0, 3, "ne", 0)])])
def test_join_core_push_matches_oracle(oracle, cl):
    """Pushes on both sides with capabilities above, between and below the batches' times; every
    work() contribution equals join_core_push of that batch against the other side's batches."""
    rng = np.random.default_rng(5)
    s1, s2 = oracle.Spine(32, 1, True), oracle.Spine(32, 1, True)
    oj = oracle.Join(s1, s2, oracle.make_closure(**cl) if cl else None)
    held = [[], []]
    seen = 0
    for t in range(5):
        for side in (0, 1):
            w = rand(rng, 1500, 200, 6, 1)
            w[:, 2] = t
            ob = oracle.Batch.build(as_r32(oracle, w), t, t + 1)
            (s1, s2)[side].insert(ob)
            cap = [0, t, 1 << 40, t + 3, TMAX][(t + side) % 5]
            oj.push(side, ob, cap)
            want = ref.join_core_push(w, held[1 - side], side, cap, cl)
            held[side].append(aref.consolidate(w))
            oj.work()
            res = words(oj.results())
            assert res[seen:].tobytes() == want.tobytes(), (t, side)
            seen = len(res)


# ------------------------------------------------------------------ time filters
@pytest.mark.parametrize("t1", [0, 1, 7, TMAX])
def test_time_filters_at_the_edges(t1):
    t2s = sorted({t for t in (t1 - 1, t1, t1 + 1, 0, TMAX) if 0 <= t <= TMAX})
    look = r32([(5, i, t, 1) for i, t in enumerate(t2s)])
    stream = r32([(5, 99, t1, 2)])
    for mode, ok in ((ref.LE, lambda t: t <= t1), (ref.LT, lambda t: t < t1)):
        got = ref.half_join(stream, [look], mode)
        want = r32([(5, i, t1, 2) for i, t in enumerate(t2s) if ok(t)])
        assert got.tobytes() == want.tobytes(), (mode, t1)
    got = ref.probe(stream, [look], ref.JOIN, 0)
    assert got[:, 3].tolist() == [max(t1, t) for t in t2s]


# ------------------------------------------------------------------ closures
def test_closure_edges():
    key = np.array([0, 1, M64, 1 << 63, 0x0123456789ABCDEF], dtype=np.uint64)
    v1 = np.array([M64, 0, 5, 3, 0xFEDCBA9876543210], dtype=np.uint64)
    v2 = np.array([7, M64, 1 << 63, 0, 42], dtype=np.uint64)
    # a whole 64-bit field; shift + bits = 64; dst_shift 63
    keep, k, v = ref.closure(dict(key_fields=[(2, 0, 64, 0)], val_fields=[(1, 60, 4, 0), (0, 0, 1, 63)]), key, v1, v2)
    assert keep.all()
    assert k.tolist() == v2.tolist()
    assert v.tolist() == [(int(a) >> 60) | ((int(b) & 1) << 63) for a, b in zip(v1, key)]
    # a * (c - b) wraps at 64 bits
    _, _, v = ref.closure(dict(expr=((0, 0, 64), (2, 0, 64), 3)), key, v1, v2)
    assert v.tolist() == [(int(a) * (3 - int(b))) & M64 for a, b in zip(key, v2)]
    # every compare at rhs 0 and 2^64 - 1
    for op, f in (("eq", lambda x, r: x == r), ("ne", lambda x, r: x != r), ("lt", lambda x, r: x < r),
                  ("le", lambda x, r: x <= r), ("gt", lambda x, r: x > r), ("ge", lambda x, r: x >= r)):
        for rhs in (0, M64):
            keep, _, _ = ref.closure(dict(filters=[(0, 0, 64, op, rhs)]), key, v1, v2)
            assert keep.tolist() == [f(int(x), rhs) for x in key], (op, rhs)
    # a filter that drops everything
    keep, _, _ = ref.closure(dict(filters=[(1, 0, 64, "gt", M64)]), key, v1, v2)
    assert not keep.any()


CLOSURE_EDGES = [
    dict(key_fields=[(2, 0, 64, 0)], val_fields=[(1, 0, 64, 0)]),
    dict(key_fields=[(1, 60, 4, 0), (0, 0, 1, 63)], val_fields=[(2, 32, 32, 0), (0, 63, 1, 32)]),
    dict(key_fields=[(0, 0, 64, 0)], expr=((1, 0, 64), (2, 0, 64), 3)),
    dict(key_fields=[(0, 0, 64, 0)], val_fields=[(2, 0, 64, 0)], filters=[(1, 0, 64, "ge", M64)]),
    dict(key_fields=[(0, 0, 64, 0)], val_fields=[(2, 0, 64, 0)], filters=[(2, 0, 64, "le", 0)]),
    dict(key_fields=[(0, 0, 64, 0)], val_fields=[(2, 0, 64, 0)], filters=[(1, 0, 64, "ne", M64), (2, 0, 64, "lt", M64)]),
    dict(key_fields=[(0, 0, 64, 0)], val_fields=[(2, 0, 64, 0)], filters=[(0, 0, 64, "gt", M64)]),
]


@pytest.mark.parametrize("case", range(len(CLOSURE_EDGES)))
def test_closure_edges_match_oracle(oracle, case):
    """The same closures through the oracle's half join: one stream row per key against one lookup row."""
    cl = CLOSURE_EDGES[case]
    rng = np.random.default_rng(40 + case)
    n = 400
    key = np.unique(rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True))
    n = len(key)
    ext = np.array([0, M64, 1 << 63, 3], dtype=np.uint64)
    v1 = np.concatenate([ext, rng.integers(0, M64, size=n - 4, dtype=np.uint64, endpoint=True)])
    v2 = np.concatenate([ext[::-1], rng.integers(0, M64, size=n - 4, dtype=np.uint64, endpoint=True)])
    look = np.stack([key, v2, np.zeros(n, np.uint64), np.ones(n, np.uint64)], axis=1)
    stream = np.stack([key, v1, np.ones(n, np.uint64), np.ones(n, np.uint64)], axis=1)
    sp, refb = trace(oracle, [look])
    got = ref.half_join(stream, refb, ref.LE, cl)
    want = oracle.half_join(as_r32(oracle, stream), sp, 0, oracle.make_closure(**cl), consolidate_output=False)
    assert multiset(got) == multiset(want)
    keep, _, _ = ref.closure(cl, key, v1, v2)
    assert len(got) == int(keep.sum())


# ------------------------------------------------------------------ by hand
def test_output_order_over_three_batches():
    """Stream order, then batch order, then row order -- not key order, not time order."""
    b0 = r32([(1, 10, 0, 1), (1, 11, 0, 1), (3, 30, 0, 1)])
    b1 = r32([(1, 12, 1, 1), (2, 20, 1, 1)])
    b2 = r32([(1, 13, 2, 1), (1, 14, 2, 1), (3, 31, 2, 1)])
    stream = r32([(3, 0, 5, 1), (1, 1, 5, 1), (9, 2, 5, 1), (1, 3, 2, -1)])
    got = ref.half_join(stream, [b0, b1, b2], ref.LE)
    want = r32([
        (3, 30, 5, 1), (3, 31, 5, 1),
        (1, 10, 5, 1), (1, 11, 5, 1), (1, 12, 5, 1), (1, 13, 5, 1), (1, 14, 5, 1),
        (1, 10, 2, -1), (1, 11, 2, -1), (1, 12, 2, -1), (1, 13, 2, -1), (1, 14, 2, -1),
    ])
    assert got.tobytes() == want.tobytes()
    got = ref.half_join(stream, [b0, b1, b2], ref.LT)
    assert got[7:].tolist() == r32([(1, 10, 2, -1), (1, 11, 2, -1), (1, 12, 2, -1)]).tolist()


def test_join_meet_and_swap():
    look = r32([(4, 40, 3, 2), (4, 41, 9, -1)])
    batch = r32([(4, 7, 5, 3)])
    # meet above both times: every output at meet
    got = ref.probe(batch, [look], ref.JOIN, 20)
    assert got.tolist() == [[4, 7, 40, 20, 6], [4, 7, 41, 20, (-3) & M64]]
    # meet below: max(t1, t2)
    got = ref.probe(batch, [look], ref.JOIN, 4)
    assert got[:, 3].tolist() == [5, 9]
    # side 1: the pushed batch's value is val2, the trace's val1
    got = ref.join_core_push(batch, [look], 1, 0)
    assert got.tolist() == [[4, 40, 7, 5, 6], [4, 41, 7, 9, (-3) & M64]]
    # diff products wrap at 64 bits
    big = r32([(4, 1, 0, -(1 << 63)), (4, 2, 0, (1 << 63) - 1), (4, 3, 0, -1)])
    got = ref.probe(r32([(4, 0, 0, -1)]), [big], ref.JOIN, 0)
    assert got[:, 4].tolist() == [1 << 63, ((1 << 63) + 1) & M64, 1]


def test_update_stream_chain():
    batch = r32([(1, 5, 0, 1), (1, 5, 3, -1), (2, 6, 3, 2)])
    look = r32([(1, 50, 0, 1), (2, 60, 0, 1)])
    init = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 64, 0)], filters=[(1, 0, 64, "ne", 6)])
    prior = r32([(9, 9, 9, 9)])
    outs = ref.half_join_chain(
        [dict(batch=batch, initial=init, skip_time=3, batches=[look], mode=ref.LE, out=0),
         dict(stream=r32([(2, 1, 4, 1)]), batches=[look], mode=ref.LT, out=0),
         dict(batch=batch, skip_time=0, batches=[look], mode=ref.LE, out=1)],
        [prior, None],
    )
    assert outs[0].tolist() == r32([(9, 9, 9, 9), (1, 50, 0, 1), (2, 60, 4, 1)]).tolist()
    assert outs[1].tolist() == r32([(1, 50, 3, -1), (2, 60, 3, 2)]).tolist()
