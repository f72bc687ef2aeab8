"""Consolidation, seal, merge and the hash index on the GPU, at every row width and on every path the
device can pick, against the plain reference of tests/arrangement_ref.py.

Each case drives one set of rows through DeviceRows.consolidate, Batch.build, Batcher.seal /
seal_lazy, Batch.merge or a spine, compares rows, description, key count and batcher frontier with
the reference byte for byte, checks every batch's hash index, and asserts the path it was built to
reach: the fused kernel's per-launch record (profiling on) names the path it took, the kernel names
of the profile report tell the other kernel families apart.  A case that lands on another path fails.
The paths reached are printed at the end of the module (pytest -s)."""
import ctypes as C

import numpy as np
import pytest

import arrangement_ref as ref

pytestmark = pytest.mark.gpu

FE = ref.FRONTIER_EMPTY
M64 = (1 << 64) - 1
ALL = [16, 32, 40, 64, 80, 128, 224, 416]
BATCH = [32, 80, 128, 224, 416]  # widths a Batch / Batcher takes (64-byte rows are reduce outputs only)
WIDE = [128, 224, 416]
CODES = {0: "lsd/merge", 1: "msd-warp", 2: "msd-cta", 3: "lsd(overflow)", 4: "fast-msd(64-bit)", 5: "fast-msd(128-bit)"}
REACHED = set()


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
    print("\npaths reached (row bytes, path):")
    for rb, p in sorted(REACHED):
        print(f"  {rb:4d}  {p}")
    assert not any(p == CODES[1] for _, p in REACHED), "the exact warp-bucket path ran"


class Trace:
    """Profiling over a block: the fused kernel's records (row bytes, rows, path code, inline index
    flag of the fast path) and the names of every kernel launched.  A merge job and an LSD sort both
    record code 0; the case that made the job tells them apart."""

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
                self.fused = [(int(r[20]), int(r[16]), int(r[21]), int(r[22])) for r in a]
                self.kernels = {k.strip("()") for k in self.ctx.profile_report()}
        finally:
            self.ctx.profile(False)

    def ran(self, prefix):
        return any(k.startswith(prefix) for k in self.kernels)

    def only_fused(self, rb, codes, n=None):
        """Exactly one fused launch, at width rb, with a path code in `codes` (and `n` rows)."""
        assert len(self.fused) == 1, self.fused
        frb, fn, code, inline = self.fused[0]
        assert frb == rb and code in codes, (self.fused, codes)
        if n is not None:
            assert fn == n, (fn, n)
        REACHED.add((rb, CODES[code]))
        return code, inline


def note(rb, path):
    REACHED.add((rb, path))


# ------------------------------------------------------------------ inputs
def gen(rng, rb, n, key_bits=20, val_bits=8, time_bits=4, diffs="small", key_base=0):
    """n rows of width rb: key word `key_bits` wide, the other data words `val_bits`, the time
    `time_bits`.  diffs: "small" (|d| <= 3) or "carry" (acc_lo anywhere in 64 bits, so that lane
    sums carry into acc_hi; totals near +-2^62)."""
    nw, nk, nd, tw = ref.LAYOUT[rb]
    w = np.zeros((n, nw), dtype=np.uint64)

    def bits(b):
        if b == 0:
            return np.zeros(n, dtype=np.uint64)
        return rng.integers(0, 1 << b, size=n, dtype=np.uint64) if b < 64 else rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True)

    w[:, 0] = bits(key_bits) + np.uint64(key_base)
    for k in range(1, nk):
        w[:, k] = bits(time_bits if k == tw else val_bits)
    big = diffs == "carry"
    w[:, nk] = (rng.integers(-3, 4, size=n, dtype=np.int64) * (1 << 61 if big else 1)).view(np.uint64)
    for l in range(ref.lanes(nd)):
        b = nk + 1 + 6 * l
        w[:, b] = rng.integers(-2, 3, size=n, dtype=np.int64).view(np.uint64)
        w[:, b + 1] = rng.integers(0, M64, size=n, dtype=np.uint64, endpoint=True) if big else rng.integers(0, 9, size=n, dtype=np.uint64)
        w[:, b + 2] = rng.integers(-2, 3, size=n, dtype=np.int64).view(np.uint64)
        w[:, b + 3] = rng.integers(0, 2, size=n, dtype=np.uint64)
    return w


def hot(rng, rb, w, groups, rows_each):
    """Replace the first groups * rows_each rows by `groups` composite keys repeated rows_each times."""
    nk = ref.LAYOUT[rb][1]
    w = w.copy()
    for g in range(groups):
        w[g * rows_each : (g + 1) * rows_each, :nk] = w[g * rows_each, :nk]
    return w


def dtype_of(mz, rb):
    from materialize_b200 import _ffi as F

    return F.DTYPES[rb]


def rows_of(mz, rb, w):
    return ref.as_rows(w, dtype_of(mz, rb))


def same(got, want_words):
    got_w = ref.words(got) if len(got) else np.zeros((0, want_words.shape[1]), dtype=np.uint64)
    assert len(got_w) == len(want_words), (len(got_w), len(want_words))
    if got_w.tobytes() != want_words.tobytes():
        bad = int(np.flatnonzero(np.any(got_w != want_words, axis=1))[0])
        raise AssertionError(f"row {bad} of {len(want_words)}: got {got_w[bad].tolist()}, want {want_words[bad].tolist()}")


def check_batch(b, want_words, desc=None):
    rows = b.rows()
    same(rows, want_words)
    slots, n_keys, longest = b.index()
    ref.check_index(want_words, slots, len(slots) - 1, n_keys, longest)
    assert b.keys() == n_keys
    if desc is not None:
        assert b.desc() == desc, (b.desc(), desc)


def consolidate_dev(mz, ctx, rb, w):
    d = mz.DeviceRows(ctx, rb).upload(rows_of(mz, rb, w))
    d.consolidate()
    return d.download()


# ------------------------------------------------------------------ the fused MSD paths
@pytest.mark.parametrize("rb", ALL)
def test_fast_msd_64bit(mz, ctx, rb):
    rng = np.random.default_rng(rb)
    w = gen(rng, rb, 60_000, key_bits=16, val_bits=3, time_bits=3)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {4}, n=len(w))
    same(got, ref.consolidate(w))
    if rb in BATCH:
        with Trace(ctx) as t:
            b = mz.Batch.build(ctx, rows_of(mz, rb, w), 0, 9)
            check_batch(b, ref.consolidate(w), (0, 9, 0))
        t.only_fused(rb, {4})


@pytest.mark.parametrize("rb", [r for r in ALL if r != 16])
def test_fast_msd_128bit(mz, ctx, rb):
    rng = np.random.default_rng(100 + rb)
    if ref.LAYOUT[rb][1] > 2:  # key + one more data word, 40 bits each
        w = gen(rng, rb, 50_000, key_bits=40, val_bits=40, time_bits=0)
        w[:, 2 : ref.LAYOUT[rb][1]] = 0
    else:  # a full-width key word and 20-bit times
        w = gen(rng, rb, 50_000, key_bits=64, time_bits=20)
        w[:3, 0] = np.array([0, M64, M64], dtype=np.uint64)
        w[:3, 1] = np.array([0, 0, (1 << 20) - 1], dtype=np.uint64)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {5}, n=len(w))
    same(got, ref.consolidate(w))


@pytest.mark.parametrize("rb", BATCH)
@pytest.mark.parametrize("many_keys", [False, True])
def test_inline_and_separate_index(mz, ctx, rb, many_keys):
    """The fast path builds the index inline when the bucket bits are all key bits; with two keys
    (one key bit against 9+ bucket bits) the separate index phase builds it."""
    rng = np.random.default_rng(200 + rb + many_keys)
    if many_keys:
        w = gen(rng, rb, 30_000, key_bits=24, val_bits=2, time_bits=2)
    else:
        w = gen(rng, rb, 30_000, key_bits=1, val_bits=24, time_bits=24 if ref.LAYOUT[rb][1] == 2 else 2)
    with Trace(ctx) as t:
        b = mz.Batch.build(ctx, rows_of(mz, rb, w), 0, 99)
        check_batch(b, ref.consolidate(w), (0, 99, 0))
    _, inline = t.only_fused(rb, {4, 5})
    assert inline == (1 if many_keys else 0)
    note(rb, "inline index" if inline else "separate index phase")


def _clumped(rng, rb, n, hot_rows, groups=1):
    w = gen(rng, rb, n, key_bits=18, val_bits=4, time_bits=3)
    return hot(rng, rb, w, groups, hot_rows)


@pytest.mark.parametrize("rb", [16, 32, 40, 64, 80])
def test_exact_msd_cta_units(mz, ctx, rb):
    """One bucket past the warp capacity (128 rows) makes the fast path overflow; every unit of
    eight buckets still fits the CTA sort (LOCAL_MAX: 1024 rows, 256 at 80 bytes)."""
    rng = np.random.default_rng(300 + rb)
    w = _clumped(rng, rb, 20_000, 140 if rb == 80 else 400)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {2}, n=len(w))
    same(got, ref.consolidate(w))
    if rb in BATCH:
        with Trace(ctx) as t:
            b = mz.Batch.build(ctx, rows_of(mz, rb, w), 0, 9)
            check_batch(b, ref.consolidate(w))
        t.only_fused(rb, {2})


@pytest.mark.parametrize("rb", ALL)
def test_lsd_after_overflow(mz, ctx, rb):
    """Clumps past the CTA units (and, at 128-416 bytes, any bucket past 128 rows: 50 hot
    (key, time) pairs x 400 rows) fall through to the radix passes."""
    rng = np.random.default_rng(400 + rb)
    # (the exact path takes at most 4096 buckets: 49 K rows at 80 bytes and more, 196 K below)
    if rb in WIDE:
        w = gen(rng, rb, 40_000, key_bits=20, time_bits=6, diffs="carry")
        w = hot(rng, rb, w, 50, 400)
    else:
        w = _clumped(rng, rb, 40_000 if rb == 80 else 60_000, 2000, groups=2)
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {3}, n=len(w))
    same(got, ref.consolidate(w))
    if rb in BATCH:
        with Trace(ctx) as t:
            b = mz.Batch.build(ctx, rows_of(mz, rb, w), 0, 99)
            check_batch(b, ref.consolidate(w))
        t.only_fused(rb, {3})


@pytest.mark.parametrize("rb", ALL)
def test_fused_lsd(mz, ctx, rb):
    """Past 2^20 rows (and below 2M) the fused kernel sorts by radix passes; at R32 / R40 / ROUT
    also below 2^20 rows once the composite key is wider than 128 bits."""
    rng = np.random.default_rng(500 + rb)
    w = gen(rng, rb, 1_200_000, key_bits=30, val_bits=6, time_bits=5, diffs="carry")
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    t.only_fused(rb, {0}, n=len(w))
    same(got, ref.consolidate(w))
    if ref.LAYOUT[rb][1] > 2:
        w = gen(rng, rb, 40_000, key_bits=64, val_bits=64, time_bits=12)
        w[1000:1100, : ref.LAYOUT[rb][1]] = w[1000, : ref.LAYOUT[rb][1]]
        with Trace(ctx) as t:
            got = consolidate_dev(mz, ctx, rb, w)
        t.only_fused(rb, {0}, n=len(w))
        same(got, ref.consolidate(w))


# ------------------------------------------------------------------ merges at the wide widths
def _batch(mz, ctx, rb, w, lower, upper):
    return mz.Batch.build(ctx, rows_of(mz, rb, w), lower, upper)


@pytest.mark.parametrize("rb", [80] + WIDE)
def test_merge_as_sort(mz, ctx, rb):
    rng = np.random.default_rng(600 + rb)
    a = gen(rng, rb, 40_000, key_bits=14, time_bits=4, diffs="carry")
    b = gen(rng, rb, 30_000, key_bits=14, time_bits=4, diffs="carry")
    b[:5000] = a[:5000]
    b[:5000, 2:] = (-(a[:5000, 2:].view(np.int64))).view(np.uint64)  # cancels partly (not the i128)
    ba, bb = _batch(mz, ctx, rb, a, 0, 10), _batch(mz, ctx, rb, b, 10, 20)
    ra, rbb = ref.consolidate(a), ref.consolidate(b)
    len(ba), len(bb)
    for since in (0, 8, 1000):
        with Trace(ctx) as t:
            m = ba.merge(bb, since)
            check_batch(m, ref.merge(ra, rbb, since), (0, 20, since))
        code, _ = t.only_fused(rb, {2, 3, 4, 5}, n=len(ra) + len(rbb))
        note(rb, f"merge as sort ({CODES[code]})")


@pytest.mark.parametrize("rb", [80] + WIDE)
def test_fused_merge_path(mz, ctx, rb):
    """A merge of 2^18 < n <= 2M rows runs the fused kernel's merge path; since = 0, in the middle
    of the times, and past every time (every time collapses: long runs across tiles)."""
    rng = np.random.default_rng(700 + rb)
    a = gen(rng, rb, 200_000, key_bits=17, time_bits=6, diffs="carry")
    b = gen(rng, rb, 150_000, key_bits=17, time_bits=6, diffs="carry")
    b[:, 1] += np.uint64(64)
    ba, bb = _batch(mz, ctx, rb, a, 0, 64), _batch(mz, ctx, rb, b, 64, 200)
    ra, rbb = ref.consolidate(a), ref.consolidate(b)
    len(ba), len(bb)
    for since in (0, 90, 1 << 40):
        with Trace(ctx) as t:
            m = ba.merge(bb, since)
            check_batch(m, ref.merge(ra, rbb, since), (0, 200, since))
        t.only_fused(rb, {0}, n=len(ra) + len(rbb))
        note(rb, "fused merge path")


@pytest.mark.parametrize("rb", [32, 80, 224])
def test_fused_job_with_a_loose_bound(mz, ctx, rb):
    """A stash whose host bound is past 2M rows while its device count is small: buffers are sized
    by the bound, the work by the count (the record's row count is the actual one)."""
    rng = np.random.default_rng(800 + rb)
    w = gen(rng, rb, 1_500_000, key_bits=10, val_bits=2, time_bits=3)
    d0 = mz.DeviceRows(ctx, rb).upload(rows_of(mz, rb, w))
    d0.consolidate()  # its count stays on the device, its bound is 1.5 M
    acc = mz.DeviceRows(ctx, rb)
    acc.append_buf_at_most(d0, 1_500_000)
    acc.append_buf_at_most(d0, 1_500_000)
    bt = mz.Batcher(ctx, rb)
    bt.push_buf(acc)
    c = ref.consolidate(w)
    with Trace(ctx) as t:
        b = bt.seal_lazy(6)
        shipped, kept, frontier = ref.seal(np.concatenate([c, c]), 6)
        check_batch(b, shipped, (0, 6, 0))
        assert bt.frontier() == frontier
    assert len(t.fused) == 1 and t.fused[0][0] == rb and t.fused[0][1] == 2 * len(c), t.fused
    note(rb, f"loose bound ({CODES[t.fused[0][2]]})")


@pytest.mark.parametrize("rb", [32, 80, 128, 416])
def test_bulk_sort_and_merge(mz, ctx, rb):
    """Past 2M rows: sort.cu + consolidate.cu for a consolidation / build, merge.cu for a merge of
    the wide rows.  Long (key, time) segments span warps and tiles, and their i128 lane sums carry."""
    rng = np.random.default_rng(900 + rb)
    n = 2_200_000
    w = gen(rng, rb, n, key_bits=10, val_bits=1, time_bits=1, diffs="carry")
    with Trace(ctx) as t:
        got = consolidate_dev(mz, ctx, rb, w)
    assert t.fused == [] and t.ran("k_rs_onesweep") and t.ran("k_segsum"), (t.fused, t.kernels)
    note(rb, "bulk sort + segsum")
    want = ref.consolidate(w)
    same(got, want)
    with Trace(ctx) as t:
        b = mz.Batch.build(ctx, rows_of(mz, rb, w), 0, 9)
        check_batch(b, want, (0, 9, 0))
    assert t.ran("k_build_index"), t.kernels
    note(rb, "index.cu")
    if rb == 32:
        return
    w1 = gen(rng, rb, 1_300_000, key_bits=30, time_bits=3, diffs="carry")
    w2 = gen(rng, rb, 1_200_000, key_bits=30, time_bits=3, diffs="carry")
    w2[:100_000, :2] = w1[:100_000, :2]  # rows of A and B that meet
    w2[:, 1] += np.uint64(3)
    b1 = mz.Batch.build(ctx, rows_of(mz, rb, w1), 0, 9)
    b2 = mz.Batch.build(ctx, rows_of(mz, rb, w2), 9, 20)
    r1, r2 = ref.consolidate(w1), ref.consolidate(w2)
    assert len(b1) + len(b2) > 2 * 1024 * 1024  # (exact lengths: the merge is sized by them)
    with Trace(ctx) as t:
        m = b1.merge(b2, 5)
        check_batch(m, ref.merge(r1, r2, 5), (0, 20, 5))
    assert t.fused == [] and t.ran("k_merge_tiles"), (t.fused, t.kernels)
    note(rb, "merge.cu")


@pytest.mark.parametrize("rb", BATCH)
def test_seal_split(mz, ctx, rb):
    """Rows on both sides of `upper`: the batch ships the earlier ones, the batcher keeps the rest
    and reports the smallest kept time; a seal at the empty frontier ships everything."""
    rng = np.random.default_rng(1000 + rb)
    tw = ref.LAYOUT[rb][3]
    bt = mz.Batcher(ctx, rb)
    stash = np.zeros((0, ref.LAYOUT[rb][0]), dtype=np.uint64)
    lower = 0
    for i, upper in enumerate([5, 5, 12, 40, FE]):
        w = gen(rng, rb, 20_000, key_bits=12, time_bits=5, diffs="carry" if i % 2 else "small")
        w[:, tw] += np.uint64(3 * i)
        w[:10, tw] = np.uint64((1 << 64) - 2)  # the largest time a row can carry
        bt.push_container(rows_of(mz, rb, w))
        stash = np.concatenate([stash, w])
        shipped, kept, frontier = ref.seal(stash, upper)
        b = bt.seal(upper) if i % 2 == 0 else bt.seal_lazy(upper)
        check_batch(b, shipped, (lower, upper, 0))
        assert bt.frontier() == frontier, (bt.frontier(), frontier)
        stash, lower = kept, upper
    note(rb, "seal split")


# ------------------------------------------------------------------ mergepath.cu (R32)
def r32(keys, vals, times, diffs):
    n = len(keys)
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0], w[:, 1], w[:, 2] = keys, vals, times
    w[:, 3] = np.asarray(diffs, dtype=np.int64).view(np.uint64)
    return ref.consolidate(w)


def merge32(mz, ctx, a, b, since, lower=0, mid=10, upper=20):
    ba, bb = _batch(mz, ctx, 32, a, lower, mid), _batch(mz, ctx, 32, b, mid, upper)
    with Trace(ctx) as t:
        m = ba.merge(bb, since)
        check_batch(m, ref.merge(a, b, since), (lower, upper, since))
    assert t.fused == [] and t.ran("k_mrg_tiles") and t.ran("k_mrg_index"), (t.fused, t.kernels)
    note(32, "mergepath.cu")
    return m


def distinct(n, start=0, time=0):
    k = np.arange(start, start + n, dtype=np.uint64)
    return r32(k, k * np.uint64(3), np.full(n, time, dtype=np.uint64), np.ones(n))


@pytest.mark.parametrize("na,nb", [(0, 0), (0, 5), (5, 0), (1, 1), (1000, 23), (512, 512), (1024, 1), (1024, 1024), (3, 3_000_000)])
def test_mergepath_sizes(mz, ctx, na, nb):
    rng = np.random.default_rng(na * 7 + nb)
    a = r32(rng.integers(0, 1 << 40, size=na, dtype=np.uint64), rng.integers(0, 9, size=na, dtype=np.uint64),
            rng.integers(0, 5, size=na, dtype=np.uint64), rng.integers(1, 4, size=na))
    b = r32(rng.integers(0, 1 << 40, size=nb, dtype=np.uint64), rng.integers(0, 9, size=nb, dtype=np.uint64),
            rng.integers(5, 9, size=nb, dtype=np.uint64), rng.integers(-3, 0, size=nb))
    for since in (0, 4, FE):
        merge32(mz, ctx, a, b, since)


@pytest.mark.parametrize("past", [1, 255, 256, 257])
def test_mergepath_run_straddles_a_tile(mz, ctx, past):
    """A run of equal (key, val, max(time, since)) rows -- one (key, val) at many times, collapsed
    by since -- crosses the 1024-row diagonal by `past` rows (257: the tile's single-thread path)."""
    run = 37 + past  # + 3 rows of B: the merged run is 40 + past rows from position 984
    a = np.concatenate([distinct(1024 - 40, 0), r32(np.full(run, 5000, np.uint64), np.zeros(run, np.uint64), np.arange(run, dtype=np.uint64), np.ones(run)), distinct(700, 6000)])
    b = np.concatenate([r32(np.full(3, 5000, np.uint64), np.zeros(3, np.uint64), np.arange(3, dtype=np.uint64) + np.uint64(run), np.ones(3)), distinct(400, 9000, 12)])
    m = merge32(mz, ctx, a, b, 1000)
    assert len(m) == (1024 - 40) + 1 + 700 + 400


@pytest.mark.parametrize("where", ["first", "last"])
def test_mergepath_run_swallows_tiles(mz, ctx, where):
    run = 3000  # past two whole tiles
    big = r32(np.full(run, 77_000, np.uint64), np.full(run, 1, np.uint64), np.arange(run, dtype=np.uint64), np.ones(run))
    if where == "first":
        a = np.concatenate([distinct(10, 0), big, distinct(2500, 100_000)])
    else:
        a = np.concatenate([distinct(2500, 0), big])
    b = np.concatenate([r32(np.full(7, 77_000, np.uint64), np.full(7, 1, np.uint64), np.arange(7, dtype=np.uint64) + np.uint64(run), np.full(7, -1)), distinct(300, 200_000, 15)])
    for since in (0, 5000):
        merge32(mz, ctx, a, b, since)


def test_mergepath_runs_cancel(mz, ctx):
    """A and B cancel over whole tiles; in one case the result is empty."""
    rng = np.random.default_rng(5)
    keys = rng.integers(0, M64, size=5000, dtype=np.uint64, endpoint=True)
    a = r32(keys, keys >> np.uint64(7), np.arange(5000, dtype=np.uint64) % np.uint64(3), np.full(5000, 2))
    neg = a.copy()
    neg[:, 3] = (-(a[:, 3].view(np.int64))).view(np.uint64)
    merge32(mz, ctx, a, neg, 0)  # empty
    part = np.concatenate([neg[:1000], neg[3500:]])
    m = merge32(mz, ctx, a, part, 0)
    assert len(m) == 2500
    # cancellation only once since collapses the times
    tshift = neg.copy()
    tshift[:, 2] += np.uint64(10)
    merge32(mz, ctx, a, ref.consolidate(tshift), 20)


def test_mergepath_extreme_values(mz, ctx):
    k = np.array([0, 0, M64, M64, 1, M64 - 1], dtype=np.uint64)
    v = np.array([0, M64, 0, M64, 5, 5], dtype=np.uint64)
    t = np.array([0, (1 << 64) - 2, (1 << 64) - 2, 7, 3, (1 << 63)], dtype=np.uint64)
    a = r32(k, v, t, [1, 2, 3, 4, 5, 6])
    b = r32(k, v, t[::-1].copy(), [-1, -2, 3, -4, 5, 6])
    for since in (0, 5, 1 << 63, (1 << 64) - 2, FE):
        merge32(mz, ctx, a, b, since)


def test_mergepath_device_counts_and_cascades(mz, ctx):
    """Inputs from seal_lazy (lengths on the device, caps looser than the contents), merged, and the
    merge output merged again with no read-back in between."""
    rng = np.random.default_rng(6)
    bt = mz.Batcher(ctx, 32)
    stash = np.zeros((0, 4), dtype=np.uint64)
    batches, refs = [], []
    for i, upper in enumerate([4, 8, 12, 16]):
        w = gen(rng, 32, 30_000, key_bits=11, val_bits=2, time_bits=4)
        w[:, 2] += np.uint64(4 * i)
        bt.push_container(rows_of(mz, 32, w))
        stash = np.concatenate([stash, w])
        shipped, stash, _ = ref.seal(stash, upper)
        batches.append(bt.seal_lazy(upper))
        refs.append(shipped)
    with Trace(ctx) as t:
        m01 = batches[0].merge(batches[1], 2)
        m23 = batches[2].merge(batches[3], 2)
        m = m01.merge(m23, 9)
        check_batch(m, ref.merge(ref.merge(refs[0], refs[1], 2), ref.merge(refs[2], refs[3], 2), 9), (0, 16, 9))
        check_batch(m01, ref.merge(refs[0], refs[1], 2), (0, 8, 2))
    assert t.ran("k_mrg_tiles") and t.fused == [], (t.fused, t.kernels)
    note(32, "mergepath.cu (device counts)")


# ------------------------------------------------------------------ spines
@pytest.mark.parametrize("rb", [80, 128, 416])
def test_spines_share_timestamps(mz, ctx, oracle, rb):
    """Three spines whose inserts share timestamps (their deferred merges share launches), batches
    up to ~300 K rows so that merges cross 2^18 rows; after every step the contents equal the
    reference of everything inserted, advanced to the logical compaction frontier (and at 80 bytes
    the layers equal the oracle's spine)."""
    rng = np.random.default_rng(1100 + rb)
    tw = ref.LAYOUT[rb][3]
    spines = [mz.Spine(ctx, rb) for _ in range(3)]
    inserted = [np.zeros((0, ref.LAYOUT[rb][0]), dtype=np.uint64) for _ in spines]  # consolidated so far
    ospine = oracle.Spine(80, 1, gate_physical=True) if rb == 80 else None
    since = 0
    sizes = [300_000, 1000, 150_000, 5, 0, 280_000, 40_000, 2000, 120_000, 300]
    with Trace(ctx) as tr:
        for t, n in enumerate(sizes):
            for s, (sp, ins) in enumerate(zip(spines, inserted)):
                w = gen(rng, rb, n, key_bits=22, time_bits=0, diffs="carry")
                w[:, tw] = np.uint64(t)
                inserted[s] = np.concatenate([ins, w])
                sp.insert(mz.Batch.build(ctx, rows_of(mz, rb, w), t, t + 1))
                if s == 0 and ospine is not None:
                    ospine.insert(oracle.Batch.build(rows_of(mz, rb, w).view(oracle.RACC), t, t + 1))
                sp.set_physical_compaction(t + 1)
                if ospine is not None and s == 0:
                    ospine.set_physical_compaction(t + 1)
            if t % 3 == 2:
                since = t - 1
                for sp in spines:
                    sp.set_logical_compaction(since)
                if ospine is not None:
                    ospine.set_logical_compaction(since)
            for s, sp in enumerate(spines):
                inserted[s] = ref.consolidate(ref.advance(inserted[s], since))
                same(sp.export(), inserted[s])
            if ospine is not None:
                assert spines[0].layers() == ospine.layers(), t
    merges = [f for f in tr.fused if f[2] == 0 and f[1] > (1 << 18)]  # (the builds take the MSD paths)
    assert merges, [f for f in tr.fused if f[2] == 0]
    note(rb, f"spine merges (largest {max(f[1] for f in merges)} rows)")
