"""The join probes on the GPU -- half_join, update streams, the probe chains of half_join_many /
delta_first_stage_many, and join_core -- against the plain reference of tests/probe_ref.py, on every
path the probe kernels can take.

Traces are pinned: every batch stays pending (physical compaction never advances), so the trace a
reader probes is exactly the batches the test inserted, in order, and unconsolidated output is
compared byte for byte, in order, behind the rows the output buffer already held.  Where the batch
set is not pinned (merged layers, a merge in flight on the side stream) the consolidated output is
compared; join_core is compared one push at a time (each work item's consolidated contribution).
Each case asserts the path it was built to reach from the kernel names of the profile report, and
the index precondition it relies on from Batch.index().  The paths reached are printed at the end
of the module (pytest -s).

Not reached here: k_probe_chains<5> (every half join writes 32-byte rows through a closure, so the
chains never carry R40 rows), k_map_rows<...> (an update stream of more than 2^28 rows) and a probe
of more than MZ_LB_TILES tiles (about 33 M stream rows against 33 or more batches)."""
import numpy as np
import pytest

import arrangement_ref as aref
import probe_ref as ref

pytestmark = pytest.mark.gpu

FE = ref.FRONTIER_EMPTY
M64 = ref.M64
LE, LT = ref.LE, ref.LT
REACHED = set()
CL = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 20, 0), (2, 0, 20, 20)], filters=[(2, 0, 20, "lt", 3 << 18)])
CLJ = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 16, 0), (2, 0, 16, 16)], filters=[(2, 0, 20, "ne", 5)])


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
    print("\nprobe paths reached:")
    for p in sorted(REACHED):
        print(f"  {p}")


class Trace:
    """Profiling over a block: the names of every kernel launched in it."""

    def __init__(self, ctx):
        self.ctx = ctx

    def __enter__(self):
        self.ctx.profile(True)
        return self

    def __exit__(self, *exc):
        try:
            if exc[0] is None:
                self.kernels = {k.strip("()") for k in self.ctx.profile_report()}
        finally:
            self.ctx.profile(False)

    def ran(self, prefix):
        return any(k.startswith(prefix) for k in self.kernels)

    def only(self, *prefixes, never=()):
        """Every prefix ran and none of `never` did."""
        for p in prefixes:
            assert self.ran(p), (p, self.kernels)
        for p in never:
            assert not self.ran(p), (p, self.kernels)


def note(path):
    REACHED.add(path)


def probe_kernels(t):
    for k in t.kernels:
        if k.startswith(("k_probe", "k_map_rows")):
            note(k)


# ------------------------------------------------------------------ inputs
def gen(rng, n, keys, vals=1 << 20, times=(0, 6), key_base=0):
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = rng.integers(0, keys, size=n, dtype=np.uint64) + np.uint64(key_base)
    w[:, 1] = rng.integers(0, vals, size=n, dtype=np.uint64)
    w[:, 2] = rng.integers(times[0], times[1], size=n, dtype=np.uint64)
    w[:, 3] = (rng.integers(1, 4, size=n) * rng.choice([-1, 1], size=n)).astype(np.int64).view(np.uint64)
    return w


def runs(rng, keys, lengths, time=0, val_base=0):
    """Rows of `keys[i]` repeated lengths[i] times with distinct values (one run per key)."""
    k = np.repeat(np.asarray(keys, dtype=np.uint64), lengths)
    w = np.zeros((len(k), 4), dtype=np.uint64)
    w[:, 0] = k
    w[:, 1] = np.arange(len(k), dtype=np.uint64) + np.uint64(val_base)
    w[:, 2] = time
    w[:, 3] = rng.integers(1, 3, size=len(k)).astype(np.uint64)
    return w


def extreme_diffs(w):
    """Three rows with diffs -2^63, 2^63 - 1 and -1: their products wrap."""
    w = w.copy()
    w[:3, 3] = np.array([-(1 << 63), (1 << 63) - 1, -1], dtype=np.int64).view(np.uint64)
    return w


def rows_of(mz, w):
    return aref.as_rows(np.asarray(w, dtype=np.uint64).reshape(-1, 4), mz.R32)


def words(a, nw=4):
    return ref._w(a, nw)


def dev(mz, ctx, w):
    d = mz.DeviceRows(ctx, 32)
    if len(w):
        d.upload(rows_of(mz, w))
    return d


def pending_spine(mz, ctx, ws, lower=0):
    """A spine of one batch per entry of `ws` ([lower + i, lower + i + 1)), all left pending, and the
    reference's view of its trace (each batch consolidated, in order)."""
    sp = mz.Spine(ctx, 32)
    for i, w in enumerate(ws):
        sp.insert(mz.Batch.build(ctx, rows_of(mz, w), lower + i, lower + i + 1))
    return sp, [aref.consolidate(w) for w in ws]


def same(got, want):
    got = words(got, want.shape[1])
    assert len(got) == len(want), (len(got), len(want))
    if got.tobytes() != want.tobytes():
        bad = int(np.flatnonzero(np.any(got != want, axis=1))[0])
        raise AssertionError(f"row {bad} of {len(want)}: got {got[bad].tolist()}, want {want[bad].tolist()}")


def gcl(mz, cl):
    return mz.make_closure(**cl) if cl is not None else None


def half_exact(mz, ctx, stream, sp, refb, mode, cl, prior):
    """half_join_dev (unconsolidated) into a buffer holding `prior`: prior, then the reference's rows."""
    out = dev(mz, ctx, prior)
    mz.half_join_dev(ctx, dev(mz, ctx, stream), sp, mode, gcl(mz, cl), False, out)
    want = np.concatenate([prior, ref.half_join(stream, refb, mode, cl)])
    same(out.download(), want)
    return len(want) - len(prior)


def slot_meta(b, key):
    """(slot index, home slot, run length field) of `key` in batch b's index, or None when absent."""
    slots, _, _ = b.index()
    s = np.ascontiguousarray(slots).view(np.uint64).reshape(-1, 2)
    mask = len(s) - 1
    hit = np.flatnonzero((s[:, 0] == np.uint64(key)) & (s[:, 1] != 0))
    home = int(aref.mix64(np.array([key], dtype=np.uint64))[0]) & mask
    if len(hit) == 0:
        return None
    return int(hit[0]), home, int(s[hit[0], 1]) >> 44


# ------------------------------------------------------------------ more than 8 batches
@pytest.mark.parametrize("cl", [None, CL], ids=["identity", "closure"])
@pytest.mark.parametrize("mode", [LE, LT], ids=["le", "lt"])
@pytest.mark.parametrize("nb", [9, 16, 17, 33, 64])
def test_half_join_many_batches(mz, ctx, nb, mode, cl):
    """9-64 pending batches: the second slot walk, tile rows 128 / 64 / 32 (and, at 33+ batches, more
    than 128 candidates in a warp of four probe rows)."""
    rng = np.random.default_rng(100 + nb * 4 + mode * 2 + (cl is not None))
    ws = [gen(rng, 1200, 3000, times=(i, i + 1)) for i in range(nb)]
    sp, refb = pending_spine(mz, ctx, ws)
    stream = gen(rng, 5000, 3200, times=(0, nb + 2))
    prior = gen(rng, 37, 100)
    with Trace(ctx) as t:
        n = half_exact(mz, ctx, stream, sp, refb, mode, cl, prior)
    assert n > 1000
    t.only("k_probe_lb<4>", never=("k_probe<", "k_probe_chains<"))
    probe_kernels(t)
    note(f"k_probe_lb: {nb} batches, {({9: 128, 16: 128, 17: 64, 33: 32, 64: 32})[nb]} rows per tile")


def test_65_batches_are_unsupported_until_compacted(mz, ctx):
    """A trace of 65 non-empty batches is refused (E_UNSUPPORTED), the output buffer is left as it was
    and the context keeps working; once compaction merges the trace the same probe is right."""
    rng = np.random.default_rng(7)
    ws = [gen(rng, 300, 500, times=(i, i + 1)) for i in range(65)]
    sp, refb = pending_spine(mz, ctx, ws)
    stream = gen(rng, 2000, 520, times=(0, 70))
    prior = gen(rng, 11, 50)
    out = dev(mz, ctx, prior)
    with pytest.raises(mz.MzGpuError) as e:
        mz.half_join_dev(ctx, dev(mz, ctx, stream), sp, LE, None, False, out)
    assert e.value.status == -4, e.value  # MZGPU_E_UNSUPPORTED
    same(out.download(), prior)
    # still usable: a probe of a small trace, then the compacted big one (merges on the main stream
    # while profiling)
    sp1, refb1 = pending_spine(mz, ctx, ws[:2])
    half_exact(mz, ctx, stream, sp1, refb1, LE, None, prior)
    with Trace(ctx) as t:
        sp.set_physical_compaction(FE)
        got = mz.half_join_dev(ctx, dev(mz, ctx, stream), sp, LE, None, False, dev(mz, ctx, prior)).download()
    same(aref.consolidate(words(got)), aref.consolidate(np.concatenate([prior, ref.half_join(stream, refb, LE)])))
    t.only("k_probe_lb<4>")
    note("65 non-empty batches: E_UNSUPPORTED, then correct after compaction")


# ------------------------------------------------------------------ candidate loops and run lengths
@pytest.mark.parametrize("cl", [None, CL], ids=["identity", "closure"])
@pytest.mark.parametrize("mode", [LE, LT], ids=["le", "lt"])
def test_rare_candidate_loops(mz, ctx, mode, cl):
    """Stream keys whose runs hold 5-50 rows, and one key with a 900-row run: far more than 32 * 4
    candidates in a warp (the loops past the register-held candidates, counted and written)."""
    rng = np.random.default_rng(200 + mode * 2 + (cl is not None))
    keys = np.arange(300, dtype=np.uint64) * np.uint64(7)
    lens = rng.integers(5, 51, size=300)
    w0 = np.concatenate([runs(rng, keys, lens, 1), runs(rng, [5000], [900], 2, val_base=1 << 16)])
    w0[:, 2] = rng.integers(0, 4, size=len(w0), dtype=np.uint64)
    w0[:, 1] = rng.permutation(len(w0)).astype(np.uint64)  # values in [0, 2^20): the closure keeps some
    w1 = extreme_diffs(gen(rng, 2000, 2100))
    sp, refb = pending_spine(mz, ctx, [w0, w1])
    b = mz.Batch.build(ctx, rows_of(mz, w0), 0, 1)
    assert slot_meta(b, 5000)[2] == 900  # the run length is in the slot
    stream = gen(rng, 3000, 300, times=(0, 5))
    stream[:, 0] *= np.uint64(7)
    stream[::97, 0] = 5000  # one lane in three warps hits the 900-row run
    stream[:3, 0] = w1[:3, 0]
    stream = extreme_diffs(stream)
    with Trace(ctx) as t:
        half_exact(mz, ctx, stream, sp, refb, mode, cl, gen(rng, 5, 10))
    t.only("k_probe_lb<4>", never=("k_probe<",))
    probe_kernels(t)
    note("k_probe_lb: more than 128 candidates per warp")


def _merged_long_runs(mz, ctx, rng):
    """A batch from the R32 merge-path kernels (mergepath.cu), whose index records runs of 64 rows
    or fewer: runs of 65-1023 rows carry length 0 in the slot."""
    keys = np.arange(120, dtype=np.uint64) * np.uint64(11) + np.uint64(1)
    lens = rng.integers(40, 500, size=120)
    lens[:3] = [65, 1023 - 300, 64]
    a = runs(rng, keys, lens, 0)
    bw = runs(rng, keys[:60], np.full(60, 150), 3, val_base=1 << 18)
    bw[:, 3] = np.uint64(M64)  # -1
    a[: 3, 3] = np.array([-(1 << 63), (1 << 63) - 1, -1], dtype=np.int64).view(np.uint64)
    ra, rb_ = aref.consolidate(a), aref.consolidate(bw)
    ba = mz.Batch.build(ctx, rows_of(mz, a), 0, 3)
    bb = mz.Batch.build(ctx, rows_of(mz, bw), 3, 6)
    with Trace(ctx) as t:
        m = ba.merge(bb, 0)
        len(m)
    t.only("k_mrg_tiles")
    want = aref.merge(ra, rb_, 0)
    lens_m = {int(k): int(n) for k, n in zip(*aref.key_runs(want)[::2])}
    long_keys = [k for k, n in lens_m.items() if 64 < n < 1024]
    assert long_keys and all(slot_meta(m, k)[2] == 0 for k in long_keys[:20])
    return m, want, keys


@pytest.mark.parametrize("cl", [None, CL], ids=["identity", "closure"])
@pytest.mark.parametrize("mode", [LE, LT], ids=["le", "lt"])
def test_run_length_not_in_slot(mz, ctx, mode, cl):
    """probe_slot_resolve's search for the end of a run whose length the index did not record."""
    rng = np.random.default_rng(300 + mode * 2 + (cl is not None))
    m, mrows, keys = _merged_long_runs(mz, ctx, rng)
    sp = mz.Spine(ctx, 32)
    sp.insert(m)
    w2 = gen(rng, 3000, 1400)
    sp.insert(mz.Batch.build(ctx, rows_of(mz, w2), 6, 7))
    refb = [mrows, aref.consolidate(w2)]
    stream = gen(rng, 2500, 120, times=(0, 8))
    stream[:, 0] = stream[:, 0] * np.uint64(11) + np.uint64(1)
    stream[::5, 0] = rng.integers(0, 1400, size=len(stream[::5]), dtype=np.uint64)
    with Trace(ctx) as t:
        half_exact(mz, ctx, stream, sp, refb, mode, cl, gen(rng, 3, 10))
    t.only("k_probe_lb<4>", never=("k_probe<",))
    note("k_probe_lb: run length 0 in the slot (end of run searched)")


@pytest.mark.parametrize("mode", [LE, LT], ids=["le", "lt"])
def test_linear_probing_wraps_past_the_table_end(mz, ctx, mode):
    """Keys whose home slot is one of the table's last three: their chains (and the four-slot
    lookahead) wrap to the start of the table, for keys present and absent."""
    rng = np.random.default_rng(400 + mode)
    n = 1000
    probe_b = mz.Batch.build(ctx, rows_of(mz, runs(rng, np.arange(n, dtype=np.uint64) + np.uint64(10**6), np.ones(n, int))), 0, 1)
    mask = len(probe_b.index()[0]) - 1
    cand = rng.integers(1 << 40, 1 << 62, size=400_000, dtype=np.uint64)
    home = aref.mix64(cand) & np.uint64(mask)
    tail = np.unique(cand[home >= np.uint64(mask - 2)])
    present, absent = tail[:10], tail[10:30]
    filler = cand[(home > np.uint64(40)) & (home < np.uint64(mask - 40))][: n - len(present)]
    keys = np.sort(np.concatenate([present, filler]))
    w = runs(rng, keys, np.ones(len(keys), int), 0)
    sp, refb = pending_spine(mz, ctx, [w])
    b = mz.Batch.build(ctx, rows_of(mz, w), 0, 1)
    assert len(b.index()[0]) - 1 == mask
    metas = [slot_meta(b, int(k)) for k in present]
    assert any(pos < home for pos, home, _ in metas), metas  # a present key's chain wrapped
    s = np.ascontiguousarray(b.index()[0]).view(np.uint64).reshape(-1, 2)
    assert s[0, 1] != 0 and s[mask, 1] != 0  # absent keys' chains run over the end into slot 0
    stream = np.zeros((3000, 4), dtype=np.uint64)
    stream[:, 0] = rng.choice(np.concatenate([present, absent, filler[:200]]), size=3000)
    stream[:, 1] = rng.integers(0, 1 << 20, size=3000, dtype=np.uint64)
    stream[:, 2] = rng.integers(0, 2, size=3000, dtype=np.uint64)
    stream[:, 3] = 1
    with Trace(ctx) as t:
        got = half_exact(mz, ctx, stream, sp, refb, mode, None, np.zeros((0, 4), np.uint64))
    assert got > 0
    t.only("k_probe_lb<4>")
    note("k_probe_lb: linear probing wraps past the table end (hits and misses)")


# ------------------------------------------------------------------ the two-pass form
@pytest.mark.parametrize("cl", [None, CL], ids=["identity", "closure"])
@pytest.mark.parametrize("mode", [LE, LT], ids=["le", "lt"])
def test_two_pass_inexact_fanout(mz, ctx, mode, cl):
    """A run of 1500 rows saturates the batch's longest-run record (1024): the fan-out bound is
    inexact and the exact two-pass form runs (count, read back, write), in the same order."""
    rng = np.random.default_rng(500 + mode * 2 + (cl is not None))
    w0 = np.concatenate([runs(rng, [77], [1500], 0), gen(rng, 2000, 3000, key_base=100)])
    w0[:, 2] = rng.integers(0, 3, size=len(w0), dtype=np.uint64)
    w1 = gen(rng, 2000, 3100, key_base=100)
    sp, refb = pending_spine(mz, ctx, [w0, w1])
    b = mz.Batch.build(ctx, rows_of(mz, w0), 0, 1)
    assert b.index()[2] == 1024 and slot_meta(b, 77)[2] == 0
    stream = gen(rng, 4000, 3100, times=(0, 5), key_base=100)
    stream[::50, 0] = 77
    with Trace(ctx) as t:
        half_exact(mz, ctx, stream, sp, refb, mode, cl, gen(rng, 4, 10))
    t.only("k_probe<4,_false>", "k_probe<4,_true>", never=("k_probe_lb<",))
    probe_kernels(t)
    note("k_probe (two-pass): inexact fan-out")


def test_two_pass_bound_too_large(mz, ctx):
    """n_ub x fan-out past MZ_BOUND_MAX_ROWS (48 Mi rows): a 1000-row run against a 60 K-row stream
    that mostly misses takes the two-pass form although the bound is exact."""
    rng = np.random.default_rng(6)
    w0 = np.concatenate([runs(rng, [9], [1000], 1), gen(rng, 500, 600, key_base=20)])
    sp, refb = pending_spine(mz, ctx, [w0])
    stream = gen(rng, 60_000, 1 << 30, times=(0, 3), key_base=1 << 20)
    stream[::500, 0] = 9
    stream[1::100, 0] = rng.integers(20, 620, size=len(stream[1::100]), dtype=np.uint64)
    for mode, cl in ((LE, None), (LT, CL)):
        with Trace(ctx) as t:
            half_exact(mz, ctx, stream, sp, refb, mode, cl, gen(rng, 2, 10))
        t.only("k_probe<4,_false>", never=("k_probe_lb<",))
    note("k_probe (two-pass): n_ub x fan-out above 48 Mi rows")


# ------------------------------------------------------------------ update streams and chains
def _all_at(rng, n, time):
    w = gen(rng, n, 1000)
    w[:, 2] = time
    return w


def test_empty_device_stream_single_pass(mz, ctx):
    """An update stream whose rows all sit at skip_time: 0 rows on the device, a positive bound on
    the host.  The single-pass probe has no tile and leaves the output's length as it was."""
    rng = np.random.default_rng(8)
    sp, refb = pending_spine(mz, ctx, [gen(rng, 2000, 1000)])
    batch = mz.Batch.build(ctx, rows_of(mz, _all_at(rng, 3000, 4)), 0, 5)
    prior = gen(rng, 9, 10)
    out = dev(mz, ctx, prior)
    with Trace(ctx) as t:
        s = mz.update_stream_dev(ctx, batch, None, 4)
        mz.half_join_dev(ctx, s, sp, LE, None, False, out)
        same(out.download(), prior)
        assert len(s) == 0
    t.only("k_map_rows_lb", "k_probe_lb<4>")
    probe_kernels(t)
    note("k_probe_lb: empty device stream with n_ub > 0 (no tiles)")


def test_update_stream_matches_reference(mz, ctx):
    rng = np.random.default_rng(9)
    w = gen(rng, 6000, 800, times=(0, 4))
    b = mz.Batch.build(ctx, rows_of(mz, w), 0, 4)
    rows = aref.consolidate(w)
    init = dict(key_fields=[(1, 0, 10, 0)], val_fields=[(0, 0, 64, 0)], filters=[(1, 10, 10, "ge", 300)])
    prior = gen(rng, 5, 10)
    for skip in (FE, 0, 3):
        for c in (None, init):
            with Trace(ctx) as t:
                got = mz.update_stream_dev(ctx, b, gcl(mz, c), skip, dev(mz, ctx, prior)).download()
            same(got, np.concatenate([prior, ref.update_stream(rows, c, skip)]))
            t.only("k_map_rows_lb")
    note("k_map_rows_lb")


@pytest.fixture(scope="module")
def chain_traces(mz, ctx):
    """Three pinned traces: 3 batches (256 probe rows per tile), 12 batches (128 rows per tile), and
    one whose 1500-row run makes the fan-out inexact."""
    rng = np.random.default_rng(10)
    a = pending_spine(mz, ctx, [gen(rng, 2500, 1500, times=(i, i + 1)) for i in range(3)])
    b = pending_spine(mz, ctx, [gen(rng, 800, 1500, times=(i, i + 1)) for i in range(12)])
    w = np.concatenate([runs(rng, [5], [1500], 0), gen(rng, 1000, 1500)])
    c = pending_spine(mz, ctx, [w])
    return a, b, c


def _chain_case(mz, ctx, reqs, n_outs, rng, many):
    """Run the requests through half_join_many / delta_first_stage_many into buffers that already
    hold rows, and compare every buffer with the reference's chains."""
    priors = [gen(rng, 3 + i, 10) for i in range(n_outs)]
    outs = [dev(mz, ctx, p) for p in priors]
    with Trace(ctx) as t:
        if many == "half":
            mz.half_join_many(ctx, [(r["dev"], r["sp"], r["mode"], gcl(mz, r.get("closure")), outs[r["out"]]) for r in reqs])
        else:
            mz.delta_first_stage_many(ctx, [(r["gbatch"], gcl(mz, r.get("initial")), r["skip_time"], r["sp"], r["mode"],
                                             gcl(mz, r.get("closure")), outs[r["out"]]) for r in reqs])
        got = [o.download() for o in outs]
    want = ref.half_join_chain(reqs, priors)
    for g, w in zip(got, want):
        same(g, w)
    return t


def test_half_join_many_chains(mz, ctx, chain_traces):
    rng = np.random.default_rng(11)
    (sa, ra), (sb, rb_), (sc, rc) = chain_traces
    big = gen(rng, 6000, 1600, times=(0, 14))
    small = gen(rng, 100, 1600, times=(0, 14))
    empty_src = mz.Batch.build(ctx, rows_of(mz, _all_at(rng, 500, 2)), 0, 3)
    empty = mz.update_stream_dev(ctx, empty_src, None, 2)  # 0 rows on the device, 500 on the host bound

    def req(stream, which, mode, closure, out):
        sp, refb = [(sa, ra), (sb, rb_), (sc, rc)][which]
        return dict(dev=empty if stream is None else dev(mz, ctx, stream),
                    stream=np.zeros((0, 4), np.uint64) if stream is None else stream,
                    sp=sp, batches=refb, mode=mode, closure=closure, out=out)

    # one chain of three: tile rows 256 then 128, an empty job in the middle
    t = _chain_case(mz, ctx, [req(big, 0, LE, CL, 0), req(None, 1, LT, None, 0), req(small, 1, LT, CL, 0)], 1, rng, "half")
    t.only("k_probe_chains<4>", never=("k_probe<", "k_probe_lb<"))
    note("k_probe_chains: tile rows differ inside a chain, an empty job")
    # five requests: launches of three and two; a chain crosses the split
    reqs = [req(big, 0, LE, None, 0), req(small, 1, LE, CL, 0), req(big, 1, LT, None, 0), req(small, 0, LT, CL, 0), req(big, 1, LE, CL, 1)]
    t = _chain_case(mz, ctx, reqs, 2, rng, "half")
    t.only("k_probe_chains<4>", never=("k_probe<",))
    note("k_probe_chains: more than 3 requests (split into launches)")
    # a job with an inexact fan-out: request by request
    t = _chain_case(mz, ctx, [req(big, 0, LE, CL, 0), req(small, 2, LT, None, 0), req(big, 1, LE, None, 1)], 2, rng, "half")
    t.only("k_probe<4,_false>", "k_probe_lb<4>", never=("k_probe_chains<",))
    note("half_join_many one by one (inexact fan-out)")


def test_delta_first_stage_many_chains(mz, ctx, chain_traces):
    """The update stream formed inside the probe (rows at skip_time dropped, the initial closure
    applied), several paths, a request whose rows are all skipped, a chain across the launch split."""
    rng = np.random.default_rng(12)
    (sa, ra), (sb, rb_), _ = chain_traces
    init = dict(key_fields=[(1, 0, 11, 0)], val_fields=[(0, 0, 32, 0)], filters=[(1, 11, 9, "lt", 400)])

    def req(w, which, init_, skip, mode, closure, out):
        sp, refb = [(sa, ra), (sb, rb_)][which]
        gb = mz.Batch.build(ctx, rows_of(mz, w), 0, 14)
        return dict(gbatch=gb, batch=aref.consolidate(w), initial=init_, skip_time=skip, sp=sp, batches=refb,
                    mode=mode, closure=closure, out=out)

    src = gen(rng, 5000, 1 << 20, times=(0, 14))
    near = gen(rng, 3000, 1600, times=(0, 14))
    reqs = [req(src, 0, init, FE, LE, CL, 0), req(_all_at(rng, 700, 6), 1, None, 6, LT, None, 0),
            req(near, 1, None, 3, LT, CL, 0), req(near, 0, init, 13, LE, None, 1)]
    t = _chain_case(mz, ctx, reqs, 2, rng, "delta")
    t.only("k_probe_chains<4>", never=("k_probe<", "k_map_rows"))
    note("k_probe_chains: fused update stream (skip_time, initial closure), a fully skipped request")


# ------------------------------------------------------------------ join_core
@pytest.mark.parametrize("cl", [None, CLJ], ids=["r40", "closure"])
@pytest.mark.parametrize("n1,long_run", [(3, False), (12, True), (40, False)])
def test_join_core_pushes(mz, ctx, n1, long_run, cl):
    """join_core's work items one at a time: the pre-loaded side-1 batch against n1 pending batches
    of trace 1 (values swapped), a side-0 push with the capability above both times, a side-1 push
    with it in between.  Keys clustered in the pushed batches (sorted by key) put hundreds of
    candidates in a warp; a 1500-row run makes the fan-out inexact (the two-pass form, which counts
    whole runs from the slot when there is no closure)."""
    rng = np.random.default_rng(600 + n1 + (cl is not None))
    nw = 4 if cl is not None else 5
    w1 = [gen(rng, 600, 400, vals=1 << 16, times=(i, i + 1)) for i in range(n1)]
    w1[0] = np.concatenate([w1[0], runs(rng, [401], [1500 if long_run else 700], 0, val_base=1 << 17)])
    t1, r1 = pending_spine(mz, ctx, w1)
    w2 = extreme_diffs(gen(rng, 3000, 402, vals=1 << 16, times=(0, 1)))
    w2[:3, 0] = w1[1][:3, 0]
    w2[3:40, 0] = 401
    t2, r2 = pending_spine(mz, ctx, [w2])
    gj = mz.JoinCore(ctx, t1, t2, gcl(mz, cl))
    seen = 0

    def step(want, tag, two_pass):
        nonlocal seen
        with Trace(ctx) as t:
            gj.work()
            got = words(gj.results(), nw)
        same(got[seen:], want)
        seen = len(got)
        assert len(want) > 0, tag
        if two_pass:
            t.only(f"k_probe<{nw},_false>", never=("k_probe_lb<",))
        else:
            t.only(f"k_probe_lb<{nw}>", never=("k_probe<",))
        probe_kernels(t)
        return t

    step(ref.join_core_push(r2[0], r1, 1, 0, cl), "pre-load", long_run)
    cap = 1 << 40
    wb = gen(rng, 2000, 402, vals=1 << 16, times=(n1, n1 + 1))
    bb = mz.Batch.build(ctx, rows_of(mz, wb), n1, n1 + 1)
    t1.insert(bb)
    gj.push(0, bb, cap)
    step(ref.join_core_push(aref.consolidate(wb), r2, 0, cap, cl), "meet above both times", False)
    wc = gen(rng, 2000, 402, vals=1 << 16, times=(1, 2))
    cb = mz.Batch.build(ctx, rows_of(mz, wc), 1, 2)
    t2.insert(cb)
    gj.push(1, cb, n1 // 2)
    step(ref.join_core_push(aref.consolidate(wc), r1 + [aref.consolidate(wb)], 1, n1 // 2, cl), "meet between", long_run)
    note(f"join_core: {'two-pass' if long_run else 'single-pass'}, OUT_NW {nw}, {n1} batches")


# ------------------------------------------------------------------ a merge in flight
def test_half_join_reads_the_inputs_of_a_merge_in_flight(mz, ctx):
    """Physical compaction follows the inserts (as in an arrangement), so inserts start spine merges
    on the side stream; a half join right after each insert reads the merges' inputs.  The batch set
    is not pinned: consolidated output is compared (no profiling: it would move the merges onto the
    main stream)."""
    rng = np.random.default_rng(13)
    sp = mz.Spine(ctx, 32)
    inserted = []
    stream = gen(rng, 4000, 1100, times=(0, 20))
    for t, n in enumerate([3000, 3000, 200, 3000, 5000, 50, 6000, 6000]):
        w = gen(rng, n, 1000, times=(t, t + 1))
        inserted.append(aref.consolidate(w))
        sp.insert(mz.Batch.build(ctx, rows_of(mz, w), t, t + 1))
        sp.set_physical_compaction(t + 1)
        for mode in (LE, LT):
            got = mz.half_join_dev(ctx, dev(mz, ctx, stream), sp, mode, None, False).download()
            same(aref.consolidate(words(got)), aref.consolidate(ref.half_join(stream, inserted, mode)))
    ctx.sync()
    note("half join beside spine merges on the side stream (consolidated; not profiled)")
