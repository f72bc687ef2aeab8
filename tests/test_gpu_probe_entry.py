"""The join-probe entry points -- mzgpu_half_join (host rows), mzgpu_half_join_buf, mzgpu_half_join_many,
mzgpu_delta_first_stage_many and join_core's work -- call by call: the rows counted in, the kernels launched,
the host waits, the bytes copied each way, and the bytes of the output, on every probe form (bounded single
pass, two-pass for an inexact fan-out or a bound past MZ_BOUND_MAX_ROWS, an empty stream, an empty trace),
for a chain across the three-request launch split and for a request that reads an earlier request's output.
Every refusal is checked with its status, the message it leaves and the rows it has already counted.

Each case runs in a context of its own, so that the counters do not depend on what ran before.  The
outputs are checked against the plain reference of tests/probe_ref.py and pinned by hash; the counters
are pinned as the library produced them on an H100."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import arrangement_ref as aref
import probe_ref as ref

pytestmark = pytest.mark.gpu

FE = ref.FRONTIER_EMPTY
LE, LT = ref.LE, ref.LT
E_INVALID, E_UNSUPPORTED = -1, -4
CL = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 20, 0), (2, 0, 20, 20)], filters=[(2, 0, 20, "lt", 3 << 18)])
CLJ = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 16, 0), (2, 0, 16, 16)], filters=[(2, 0, 20, "ne", 5)])
COUNTERS = ("rows_in", "kernel_launches", "host_syncs", "h2d_bytes", "d2h_bytes")

# case -> [(call, (rows_in, kernel_launches, host_syncs, h2d_bytes, d2h_bytes), output hash)]
EXPECTED = {
    "half_join": [
        ("host bounded mode=0 closure=False consolidate=0", (4000, 1, 1, 128000, 272), "c767ea8d7ba9628c"),
        ("buf bounded mode=0 closure=False consolidate=0", (4000, 1, 0, 0, 0), "c767ea8d7ba9628c"),
        ("host bounded mode=0 closure=False consolidate=1", (4000, 3, 0, 128000, 0), "83d8250d7d8e4a1e"),
        ("buf bounded mode=0 closure=False consolidate=1", (4000, 3, 0, 0, 0), "83d8250d7d8e4a1e"),
        ("host bounded mode=1 closure=True consolidate=0", (4000, 1, 0, 128000, 0), "dc344754f6a27f35"),
        ("buf bounded mode=1 closure=True consolidate=0", (4000, 1, 0, 0, 0), "dc344754f6a27f35"),
        ("host bounded mode=1 closure=True consolidate=1", (4000, 3, 0, 128000, 0), "7f5574ae08154b48"),
        ("buf bounded mode=1 closure=True consolidate=1", (4000, 3, 0, 0, 0), "7f5574ae08154b48"),
        ("host bounded empty consolidate=0", (0, 0, 0, 0, 0), "23a0575d174e1336"),
        ("buf bounded empty consolidate=0", (0, 0, 0, 0, 0), "23a0575d174e1336"),
        ("buf bounded device-empty consolidate=0", (500, 1, 0, 0, 0), "23a0575d174e1336"),
        ("buf bounded device-counted consolidate=0", (4000, 1, 0, 0, 0), "1755e6890cb4801b"),
        ("host bounded empty consolidate=1", (0, 0, 0, 0, 0), "ea892b78da4afc10"),
        ("buf bounded empty consolidate=1", (0, 0, 0, 0, 0), "ea892b78da4afc10"),
        ("buf bounded device-empty consolidate=1", (500, 3, 0, 0, 0), "ea892b78da4afc10"),
        ("buf bounded device-counted consolidate=1", (4000, 3, 0, 0, 0), "c480a344b02379bb"),
        ("host inexact mode=0 closure=False consolidate=0", (4000, 3, 1, 128000, 8), "bdac4af7285cd1d0"),
        ("buf inexact mode=0 closure=False consolidate=0", (4000, 3, 1, 0, 8), "bdac4af7285cd1d0"),
        ("host inexact mode=0 closure=False consolidate=1", (4000, 5, 1, 128000, 8), "9529481981bcef72"),
        ("buf inexact mode=0 closure=False consolidate=1", (4000, 5, 1, 0, 8), "9529481981bcef72"),
        ("host inexact mode=1 closure=True consolidate=0", (4000, 3, 1, 128000, 8), "547bcb8ec3a3c20b"),
        ("buf inexact mode=1 closure=True consolidate=0", (4000, 3, 1, 0, 8), "547bcb8ec3a3c20b"),
        ("host inexact mode=1 closure=True consolidate=1", (4000, 5, 1, 128000, 8), "7851bcc9ea6ea880"),
        ("buf inexact mode=1 closure=True consolidate=1", (4000, 5, 1, 0, 8), "7851bcc9ea6ea880"),
        ("host inexact empty consolidate=0", (0, 0, 0, 0, 0), "b0226aaca5ca2810"),
        ("buf inexact empty consolidate=0", (0, 0, 0, 0, 0), "b0226aaca5ca2810"),
        ("buf inexact device-empty consolidate=0", (500, 0, 1, 0, 272), "b0226aaca5ca2810"),
        ("buf inexact device-counted consolidate=0", (4000, 3, 2, 0, 280), "d2eca395adcb8b1b"),
        ("host inexact empty consolidate=1", (0, 0, 0, 0, 0), "45f793f03ecf56cd"),
        ("buf inexact empty consolidate=1", (0, 0, 0, 0, 0), "45f793f03ecf56cd"),
        ("buf inexact device-empty consolidate=1", (500, 0, 1, 0, 272), "45f793f03ecf56cd"),
        ("buf inexact device-counted consolidate=1", (4000, 5, 2, 0, 280), "1b9d3ea83c056f10"),
        ("host wide mode=0 closure=False consolidate=0", (60000, 3, 1, 1920000, 8), "ceac40e282246368"),
        ("buf wide mode=0 closure=False consolidate=0", (60000, 3, 1, 0, 8), "ceac40e282246368"),
        ("host wide mode=0 closure=False consolidate=1", (60000, 5, 1, 1920000, 8), "c72e79ccb0d8e73d"),
        ("buf wide mode=0 closure=False consolidate=1", (60000, 5, 1, 0, 8), "c72e79ccb0d8e73d"),
        ("host wide mode=1 closure=True consolidate=0", (60000, 3, 1, 1920000, 8), "362810a0b270ab4c"),
        ("buf wide mode=1 closure=True consolidate=0", (60000, 3, 1, 0, 8), "362810a0b270ab4c"),
        ("host wide mode=1 closure=True consolidate=1", (60000, 5, 1, 1920000, 8), "486388658247098a"),
        ("buf wide mode=1 closure=True consolidate=1", (60000, 5, 1, 0, 8), "486388658247098a"),
        ("host wide empty consolidate=0", (0, 0, 0, 0, 0), "c3604bcd9c9c6e8a"),
        ("buf wide empty consolidate=0", (0, 0, 0, 0, 0), "c3604bcd9c9c6e8a"),
        ("buf wide device-empty consolidate=0", (500, 1, 0, 0, 0), "c3604bcd9c9c6e8a"),
        ("buf wide device-counted consolidate=0", (4000, 1, 0, 0, 0), "f9a6d02ba5d343b8"),
        ("host wide empty consolidate=1", (0, 0, 0, 0, 0), "e7a9043e81d2f2a8"),
        ("buf wide empty consolidate=1", (0, 0, 0, 0, 0), "e7a9043e81d2f2a8"),
        ("buf wide device-empty consolidate=1", (500, 3, 0, 0, 0), "e7a9043e81d2f2a8"),
        ("buf wide device-counted consolidate=1", (4000, 3, 0, 0, 0), "381af6c405aaded6"),
        ("host empty mode=0 closure=False consolidate=0", (4000, 0, 0, 128000, 0), "cc19b26f0664e17f"),
        ("buf empty mode=0 closure=False consolidate=0", (4000, 0, 0, 0, 0), "cc19b26f0664e17f"),
        ("host empty mode=0 closure=False consolidate=1", (4000, 0, 0, 128000, 0), "7301bc22b9b1dbbf"),
        ("buf empty mode=0 closure=False consolidate=1", (4000, 0, 0, 0, 0), "7301bc22b9b1dbbf"),
        ("host empty mode=1 closure=True consolidate=0", (4000, 0, 0, 128000, 0), "9e979bc08bf32be8"),
        ("buf empty mode=1 closure=True consolidate=0", (4000, 0, 0, 0, 0), "9e979bc08bf32be8"),
        ("host empty mode=1 closure=True consolidate=1", (4000, 0, 0, 128000, 0), "2ccd4e1cdcbf0bce"),
        ("buf empty mode=1 closure=True consolidate=1", (4000, 0, 0, 0, 0), "2ccd4e1cdcbf0bce"),
        ("host empty empty consolidate=0", (0, 0, 0, 0, 0), "27be6409fbacaf2c"),
        ("buf empty empty consolidate=0", (0, 0, 0, 0, 0), "27be6409fbacaf2c"),
        ("buf empty device-empty consolidate=0", (500, 0, 0, 0, 0), "27be6409fbacaf2c"),
        ("buf empty device-counted consolidate=0", (4000, 0, 0, 0, 0), "27be6409fbacaf2c"),
        ("host empty empty consolidate=1", (0, 0, 0, 0, 0), "2320102852d349cc"),
        ("buf empty empty consolidate=1", (0, 0, 0, 0, 0), "2320102852d349cc"),
        ("buf empty device-empty consolidate=1", (500, 0, 0, 0, 0), "2320102852d349cc"),
        ("buf empty device-counted consolidate=1", (4000, 0, 0, 0, 0), "2320102852d349cc"),
    ],
    "half_join_many": [
        ("one request", (6000, 1, 1, 0, 240), "8245f00e1c2e3e99"),
        ("chain of three, an empty job", (6600, 1, 0, 0, 0), "14f7cd565ad6618e"),
        ("five requests, a chain across the launch split", (18200, 2, 0, 0, 0), "fe00cdd27556f87e"),
        ("inexact fan-out: request by request", (12100, 6, 1, 0, 8), "b6ae98b962070769"),
        ("an empty trace: request by request", (6100, 1, 0, 0, 0), "4f0cad58f660b601"),
        ("an empty stream first: request by request", (6600, 6, 1, 0, 8), "d2a1232450c3920b"),
        ("a stream that is an earlier request's output", (204, 4, 2, 3200, 248), "7d47af9c342c9718"),
    ],
    "delta_first_stage_many": [
        ("one source batch", (3000, 1, 1, 0, 240), "d15dee6ef3b64d02"),
        ("four requests, a fully skipped one, a chain across the launch split", (11700, 2, 0, 0, 0), "42ea89bdcf30d574"),
        ("inexact fan-out: update streams, then request by request", (11000, 9, 2, 0, 280), "12660b3dba8316a9"),
        ("an empty trace: request by request", (6000, 3, 0, 0, 0), "000ef74d5e5c8417"),
    ],
    "join_core": [
        ("pre-load closure=False", (0, 2, 2, 0, 352), "343bb65ac706baaf"),
        ("push side 0 closure=False", (0, 2, 2, 0, 352), "36633b943a2f73e2"),
        ("push side 1 closure=False", (0, 2, 2, 0, 352), "e04d7960acacc882"),
        ("pre-load closure=True", (0, 4, 2, 0, 184), "3ad1fabe8db320d3"),
        ("push side 0 closure=True", (0, 2, 2, 0, 352), "55d687d4cd8f4754"),
        ("push side 1 closure=True", (0, 4, 2, 0, 280), "b550844a559c2054"),
        ("pre-load against an empty trace", (0, 0, 0, 0, 0), "e3b0c44298fc1c14"),
    ],
}


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def F():
    from materialize_b200 import _ffi

    return _ffi


@pytest.fixture
def ctx(mz):
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


# ------------------------------------------------------------------ inputs
def gen(rng, n, keys, times=(0, 6), key_base=0):
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = rng.integers(0, keys, size=n, dtype=np.uint64) + np.uint64(key_base)
    w[:, 1] = rng.integers(0, 1 << 20, size=n, dtype=np.uint64)
    w[:, 2] = rng.integers(times[0], times[1], size=n, dtype=np.uint64)
    w[:, 3] = (rng.integers(1, 4, size=n) * rng.choice([-1, 1], size=n)).astype(np.int64).view(np.uint64)
    return w


def run_of(key, n, time=0):
    """n rows of one key with distinct values: a key run of length n."""
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = key
    w[:, 1] = np.arange(n, dtype=np.uint64) + np.uint64(1 << 17)
    w[:, 2] = time
    w[:, 3] = 1
    return w


def all_at(rng, n, time):
    w = gen(rng, n, 1000)
    w[:, 2] = time
    return w


def rows_of(mz, w):
    return aref.as_rows(np.asarray(w, dtype=np.uint64).reshape(-1, 4), mz.R32)


def dev(mz, ctx, w):
    d = mz.DeviceRows(ctx, 32)
    if len(w):
        d.upload(rows_of(mz, w))
    return d


def spine(mz, ctx, ws):
    """A spine of one batch per entry of `ws`, all left pending (compaction never advances), and the
    reference's view of it."""
    sp = mz.Spine(ctx, 32)
    for i, w in enumerate(ws):
        sp.insert(mz.Batch.build(ctx, rows_of(mz, w), i, i + 1))
    return sp, [aref.consolidate(w) for w in ws]


def traces(mz, ctx, rng):
    """bounded: three batches; inexact: a 1500-row run saturates the longest-run record (1024); wide: a
    1000-row run, exact, but past MZ_BOUND_MAX_ROWS against a 60 K-row stream; empty: no batches."""
    return {
        "bounded": spine(mz, ctx, [gen(rng, 2500, 1500, times=(i, i + 1)) for i in range(3)]),
        "inexact": spine(mz, ctx, [np.concatenate([run_of(5, 1500), gen(rng, 1000, 1500)])]),
        "wide": spine(mz, ctx, [np.concatenate([run_of(9, 1000, 1), gen(rng, 500, 600, key_base=20)])]),
        "empty": (mz.Spine(ctx, 32), []),
    }


def gcl(mz, cl):
    return mz.make_closure(**cl) if cl is not None else None


def clp(c):
    return C.byref(c) if c is not None else None


def words(a, nw=4):
    return ref._w(a, nw)


def digest(rows):
    return hashlib.sha256(np.ascontiguousarray(rows).tobytes()).hexdigest()[:16]


class Calls:
    """The counters of each measured call (with the profiler off) and the hash of what it left behind."""

    def __init__(self, ctx):
        self.ctx, self.seen = ctx, []

    def measure(self, label, call, out_rows):
        s0 = self.ctx.stats()
        call()
        s1 = self.ctx.stats()
        got = out_rows()
        self.seen.append((label, tuple(s1[k] - s0[k] for k in COUNTERS), digest(got)))
        return got


def check(case, seen):
    want = EXPECTED[case]
    assert [s[0] for s in seen] == [w[0] for w in want]
    for got, w in zip(seen, want):
        assert got[1] == tuple(w[1]), (got[0], dict(zip(COUNTERS, got[1])), dict(zip(COUNTERS, w[1])))
        assert got[2] == w[2], got[0]


# ------------------------------------------------------------------ single half joins
def case_half_join(mz, F, ctx):
    """mzgpu_half_join (host rows) and mzgpu_half_join_buf, consolidated and not, on every form."""
    rng = np.random.default_rng(1)
    tr = traces(mz, ctx, rng)
    calls = Calls(ctx)
    stream = gen(rng, 4000, 1600, times=(0, 8))
    stream[::50, 0] = 5  # meets the 1500-row run
    wide_stream = gen(rng, 60_000, 1 << 30, times=(0, 3), key_base=1 << 20)
    wide_stream[::500, 0] = 9
    wide_stream[1::100, 0] = rng.integers(20, 620, size=len(wide_stream[1::100]), dtype=np.uint64)
    skipped = mz.Batch.build(ctx, rows_of(mz, all_at(rng, 500, 2)), 0, 3)
    counted = mz.Batch.build(ctx, rows_of(mz, stream), 0, 8)
    for name, (sp, refb) in tr.items():
        s = wide_stream if name == "wide" else stream
        for mode, cl in ((LE, None), (LT, CL)):
            want = ref.half_join(s, refb, mode, cl)
            for cons in (0, 1):
                prior = gen(rng, 7, 10)
                host_rows = rows_of(mz, s)
                out = dev(mz, ctx, prior)
                got = calls.measure(
                    f"host {name} mode={mode} closure={cl is not None} consolidate={cons}",
                    lambda: ctx.check(F.lib.mzgpu_half_join(ctx.h, host_rows.ctypes.data, len(host_rows), F.MEM_HOST,
                                                            sp.h, mode, clp(gcl(mz, cl)), cons, out.h)),
                    out.download)
                check_half(got, prior, want, cons)
                d, out = dev(mz, ctx, s), dev(mz, ctx, prior)
                got = calls.measure(f"buf {name} mode={mode} closure={cl is not None} consolidate={cons}",
                                    lambda: mz.half_join_dev(ctx, d, sp, mode, gcl(mz, cl), bool(cons), out),
                                    out.download)
                check_half(got, prior, want, cons)
        # empty streams: none on the host, none in the buffer, none on the device behind a positive bound;
        # and a stream whose length is still on the device
        for cons in (0, 1):
            prior = gen(rng, 3, 10)
            out = dev(mz, ctx, prior)
            calls.measure(f"host {name} empty consolidate={cons}",
                          lambda: ctx.check(F.lib.mzgpu_half_join(ctx.h, None, 0, F.MEM_HOST, sp.h, LE, None, cons,
                                                                  out.h)), out.download)
            out, d = dev(mz, ctx, prior), mz.DeviceRows(ctx, 32)
            calls.measure(f"buf {name} empty consolidate={cons}",
                          lambda: mz.half_join_dev(ctx, d, sp, LE, None, bool(cons), out), out.download)
            d = mz.update_stream_dev(ctx, skipped, None, 2)
            out = dev(mz, ctx, prior)
            got = calls.measure(f"buf {name} device-empty consolidate={cons}",
                                lambda: mz.half_join_dev(ctx, d, sp, LE, None, bool(cons), out), out.download)
            check_half(got, prior, np.zeros((0, 4), np.uint64), cons)
            d = mz.update_stream_dev(ctx, counted, gcl(mz, CL), FE)
            out = dev(mz, ctx, prior)
            got = calls.measure(f"buf {name} device-counted consolidate={cons}",
                                lambda: mz.half_join_dev(ctx, d, sp, LT, None, bool(cons), out), out.download)
            check_half(got, prior, ref.half_join(ref.update_stream(aref.consolidate(stream), CL), refb, LT), cons)
    return calls.seen


def check_half(got, prior, want, cons):
    got = words(got)
    assert got[: len(prior)].tobytes() == prior.tobytes()
    if cons:
        assert aref.consolidate(got[len(prior):]).tobytes() == aref.consolidate(want).tobytes()
    else:
        assert got[len(prior):].tobytes() == want.tobytes()


# ------------------------------------------------------------------ chains
def many(mz, ctx, calls, label, reqs, n_outs, rng, kind):
    """half_join_many / delta_first_stage_many into buffers that already hold rows; checked against the
    reference's chains."""
    priors = [gen(rng, 3 + i, 10) for i in range(n_outs)]
    outs = [dev(mz, ctx, p) for p in priors]
    if kind == "half":
        call = lambda: mz.half_join_many(  # noqa: E731
            ctx, [(r["dev"], r["sp"], r["mode"], gcl(mz, r.get("closure")), outs[r["out"]]) for r in reqs])
    else:
        call = lambda: mz.delta_first_stage_many(  # noqa: E731
            ctx, [(r["gbatch"], gcl(mz, r.get("initial")), r["skip_time"], r["sp"], r["mode"], gcl(mz, r.get("closure")),
                   outs[r["out"]]) for r in reqs])
    got = calls.measure(label, call, lambda: np.concatenate([words(o.download()) for o in outs]))
    want = ref.half_join_chain(reqs, priors)
    assert got.tobytes() == np.concatenate(want).tobytes()


def case_half_join_many(mz, F, ctx):
    rng = np.random.default_rng(2)
    tr = traces(mz, ctx, rng)
    calls = Calls(ctx)
    big = gen(rng, 6000, 1600, times=(0, 14))
    small = gen(rng, 100, 1600, times=(0, 14))
    small[::9, 0] = 5
    skipped = mz.Batch.build(ctx, rows_of(mz, all_at(rng, 500, 2)), 0, 3)

    def req(stream, which, mode, closure, out):
        sp, refb = tr[which]
        empty = stream is None
        return dict(dev=mz.update_stream_dev(ctx, skipped, None, 2) if empty else dev(mz, ctx, stream),
                    stream=np.zeros((0, 4), np.uint64) if empty else stream, sp=sp, batches=refb, mode=mode,
                    closure=closure, out=out)

    many(mz, ctx, calls, "one request", [req(big, "bounded", LE, CL, 0)], 1, rng, "half")
    many(mz, ctx, calls, "chain of three, an empty job",
         [req(big, "bounded", LE, CL, 0), req(None, "bounded", LT, None, 0), req(small, "bounded", LT, CL, 0)], 1, rng,
         "half")
    many(mz, ctx, calls, "five requests, a chain across the launch split",
         [req(big, "bounded", LE, None, 0), req(small, "bounded", LE, CL, 0), req(big, "bounded", LT, None, 0),
          req(small, "bounded", LT, CL, 0), req(big, "bounded", LE, CL, 1)], 2, rng, "half")
    many(mz, ctx, calls, "inexact fan-out: request by request",
         [req(big, "bounded", LE, CL, 0), req(small, "inexact", LT, None, 0), req(big, "bounded", LE, None, 1)], 2,
         rng, "half")
    many(mz, ctx, calls, "an empty trace: request by request",
         [req(big, "bounded", LE, CL, 0), req(small, "empty", LT, None, 1)], 2, rng, "half")
    many(mz, ctx, calls, "an empty stream first: request by request",
         [req(None, "bounded", LE, CL, 0), req(small, "inexact", LT, None, 0), req(big, "bounded", LE, None, 0)], 1,
         rng, "half")

    # request 2 reads request 1's output, which request 1 has just appended to: request by request
    prior = [gen(rng, 4, 10), gen(rng, 5, 10)]
    mid, last = dev(mz, ctx, prior[0]), dev(mz, ctx, prior[1])
    sp_a, ra = tr["bounded"]
    sp_b, rb_ = tr["inexact"]
    got = calls.measure(
        "a stream that is an earlier request's output",
        lambda: mz.half_join_many(ctx, [(dev(mz, ctx, small), sp_a, LE, gcl(mz, CL), mid), (mid, sp_b, LT, None, last)]),
        lambda: np.concatenate([words(mid.download()), words(last.download())]))
    first = np.concatenate([prior[0], ref.half_join(small, ra, LE, CL)])
    second = np.concatenate([prior[1], ref.half_join(first, rb_, LT)])
    assert got.tobytes() == np.concatenate([first, second]).tobytes()
    return calls.seen


def case_delta_first_stage_many(mz, F, ctx):
    rng = np.random.default_rng(3)
    tr = traces(mz, ctx, rng)
    calls = Calls(ctx)
    init = dict(key_fields=[(1, 0, 11, 0)], val_fields=[(0, 0, 32, 0)], filters=[(1, 11, 9, "lt", 400)])

    def req(w, which, init_, skip, mode, closure, out):
        sp, refb = tr[which]
        return dict(gbatch=mz.Batch.build(ctx, rows_of(mz, w), 0, 14), batch=aref.consolidate(w), initial=init_,
                    skip_time=skip, sp=sp, batches=refb, mode=mode, closure=closure, out=out)

    src = gen(rng, 5000, 1 << 20, times=(0, 14))
    near = gen(rng, 3000, 1600, times=(0, 14))
    near[::40, 0] = 5
    many(mz, ctx, calls, "one source batch", [req(near, "bounded", None, 3, LT, CL, 0)], 1, rng, "delta")
    many(mz, ctx, calls, "four requests, a fully skipped one, a chain across the launch split",
         [req(src, "bounded", init, FE, LE, CL, 0), req(all_at(rng, 700, 6), "bounded", None, 6, LT, None, 0),
          req(near, "bounded", None, 3, LT, CL, 0), req(near, "bounded", init, 13, LE, None, 1)], 2, rng, "delta")
    many(mz, ctx, calls, "inexact fan-out: update streams, then request by request",
         [req(near, "bounded", None, FE, LE, CL, 0), req(near, "inexact", None, 3, LT, None, 0),
          req(src, "bounded", init, 13, LE, None, 1)], 2, rng, "delta")
    many(mz, ctx, calls, "an empty trace: request by request",
         [req(near, "empty", None, FE, LE, CL, 0), req(near, "bounded", None, 3, LT, None, 1)], 2, rng, "delta")
    return calls.seen


# ------------------------------------------------------------------ join_core
def case_join_core(mz, F, ctx):
    """A pre-loaded work item and a push on each side, single-pass (R40) and two-pass (closure, a
    saturated run); and a pre-load against an empty trace."""
    calls = Calls(ctx)
    for cl, long_run in ((None, False), (CLJ, True)):
        rng = np.random.default_rng(4 + long_run)
        nw = 4 if cl is not None else 5
        w1 = [gen(rng, 600, 400, times=(i, i + 1)) for i in range(3)]
        w1[0] = np.concatenate([w1[0], run_of(401, 1500 if long_run else 700)])
        t1, r1 = spine(mz, ctx, w1)
        w2 = gen(rng, 3000, 402, times=(0, 1))
        w2[3:40, 0] = 401
        t2, r2 = spine(mz, ctx, [w2])
        gj = mz.JoinCore(ctx, t1, t2, gcl(mz, cl))
        seen = 0

        def step(label, want):
            nonlocal seen
            got = words(calls.measure(f"{label} closure={cl is not None}", gj.work, gj.results), nw)
            assert got[seen:].tobytes() == want.tobytes(), label
            assert len(want) > 0
            seen = len(got)

        step("pre-load", ref.join_core_push(r2[0], r1, 1, 0, cl))
        wb = gen(rng, 2000, 402, times=(3, 4))
        bb = mz.Batch.build(ctx, rows_of(mz, wb), 3, 4)
        t1.insert(bb)
        gj.push(0, bb, 1 << 40)
        step("push side 0", ref.join_core_push(aref.consolidate(wb), r2, 0, 1 << 40, cl))
        wc = gen(rng, 2000, 402, times=(1, 2))
        cb = mz.Batch.build(ctx, rows_of(mz, wc), 1, 2)
        t2.insert(cb)
        gj.push(1, cb, 1)
        step("push side 1", ref.join_core_push(aref.consolidate(wc), r1 + [aref.consolidate(wb)], 1, 1, cl))
    rng = np.random.default_rng(6)
    empty = mz.Spine(ctx, 32)
    t2, _ = spine(mz, ctx, [gen(rng, 1000, 300)])
    gj = mz.JoinCore(ctx, empty, t2)
    got = calls.measure("pre-load against an empty trace", gj.work, gj.results)
    assert len(got) == 0
    return calls.seen


CASES = {
    "half_join": case_half_join,
    "half_join_many": case_half_join_many,
    "delta_first_stage_many": case_delta_first_stage_many,
    "join_core": case_join_core,
}


@pytest.mark.parametrize("case", list(CASES))
def test_probe_entry_counters(mz, F, ctx, case):
    check(case, CASES[case](mz, F, ctx))


# ------------------------------------------------------------------ refusals
def rows_in(ctx):
    return ctx.stats()["rows_in"]


def last_error(F, ctx):
    return F.lib.mzgpu_last_error(ctx.h).decode()


def refused(F, ctx, call, status, counted=0, msg=None):
    """`call` returns `status`, counts `counted` rows in and leaves `msg` (None: the message as it was)."""
    before_rows, before_msg = rows_in(ctx), last_error(F, ctx)
    assert call() == status
    assert rows_in(ctx) == before_rows + counted
    assert last_error(F, ctx) == (before_msg if msg is None else msg)


def bad_closure(F):
    c = F.Closure()
    c.n_key_fields = 1
    c.expr_kind = 7
    return c


BAD_CLOSURE_MSG = "closure: unknown expression kind 7"


def test_refusals(mz, F, ctx):
    rng = np.random.default_rng(7)
    sp, _ = spine(mz, ctx, [gen(rng, 500, 100)])
    sp40 = mz.Spine(ctx, 40)
    w = gen(rng, 300, 100)
    host = rows_of(mz, w)
    p, n = host.ctypes.data, len(host)
    s0, s1 = dev(mz, ctx, w), dev(mz, ctx, gen(rng, 200, 100))
    out, out2, out40, s40 = mz.DeviceRows(ctx, 32), mz.DeviceRows(ctx, 32), mz.DeviceRows(ctx, 40), mz.DeviceRows(ctx, 40)
    s40.upload(np.zeros(5, dtype=mz.R40))
    bad = bad_closure(F)
    badp = C.byref(bad)
    lib = F.lib

    # mzgpu_half_join (host rows)
    for args in [(p, n, F.MEM_HOST, sp.h, LE, None, 0, out40.h), (p, n, F.MEM_HOST, sp40.h, LE, None, 0, out.h),
                 (p, n, F.MEM_HOST, sp.h, 2, None, 0, out.h), (None, n, F.MEM_HOST, sp.h, LE, None, 0, out.h),
                 (p, n, F.MEM_HOST, None, LE, None, 0, out.h), (p, n, F.MEM_HOST, sp.h, LE, None, 0, None),
                 (p, n, F.MEM_HOST, sp.h, 2, badp, 1, out.h)]:
        refused(F, ctx, lambda: lib.mzgpu_half_join(ctx.h, *args), E_INVALID)
    refused(F, ctx, lambda: lib.mzgpu_half_join(ctx.h, p, n, F.MEM_HOST, sp.h, LE, badp, 0, out.h), E_UNSUPPORTED,
            msg=BAD_CLOSURE_MSG)
    ctx.check(lib.mzgpu_half_join(ctx.h, None, 0, F.MEM_HOST, sp.h, LE, None, 0, out.h))
    assert last_error(F, ctx) == BAD_CLOSURE_MSG  # a call that succeeds leaves the message as it was

    # mzgpu_half_join_buf
    for args in [(s40.h, sp.h, LE, None, 0, out.h), (s0.h, sp40.h, LE, None, 0, out.h), (s0.h, sp.h, LE, None, 0, out40.h),
                 (s0.h, sp.h, 2, None, 0, out.h), (s0.h, sp.h, LE, None, 0, s0.h), (None, sp.h, LE, None, 0, out.h),
                 (s0.h, None, LE, None, 0, out.h), (s0.h, sp.h, LE, None, 0, None), (s0.h, sp.h, LE, badp, 0, s0.h)]:
        refused(F, ctx, lambda: lib.mzgpu_half_join_buf(ctx.h, *args), E_INVALID)
    ctx.check(lib.mzgpu_ctx_sync(ctx.h))
    refused(F, ctx, lambda: lib.mzgpu_half_join_buf(ctx.h, s0.h, sp.h, LT, badp, 1, out.h), E_UNSUPPORTED,
            msg=BAD_CLOSURE_MSG)

    # mzgpu_half_join_many: request j + 1 is checked after request j's rows are counted
    def hjm(reqs, k=None):
        k = len(reqs) if k is None else k
        arr = lambda t, xs: (t * max(1, len(xs)))(*xs)  # noqa: E731
        return lib.mzgpu_half_join_many(
            ctx.h, k, arr(C.c_void_p, [r[0] for r in reqs]), arr(C.c_void_p, [r[1] for r in reqs]),
            arr(C.c_int32, [r[2] for r in reqs]),
            arr(C.c_void_p, [C.cast(C.pointer(r[3]), C.c_void_p) if r[3] is not None else None for r in reqs]),
            arr(C.c_void_p, [r[4] for r in reqs]))

    good = (s0.h, sp.h, LE, None, out.h)
    assert hjm([], 0) == 0
    refused(F, ctx, lambda: hjm([good] * 65), E_INVALID)
    for second in [(s40.h, sp.h, LE, None, out2.h), (s1.h, sp40.h, LE, None, out2.h), (s1.h, sp.h, LE, None, out40.h),
                   (s1.h, sp.h, 5, None, out2.h), (out2.h, sp.h, LE, None, out2.h), (None, sp.h, LE, None, out2.h)]:
        refused(F, ctx, lambda: hjm([good, second]), E_INVALID, counted=len(w))
    refused(F, ctx, lambda: hjm([good, (s1.h, sp.h, LT, bad, out2.h)]), E_UNSUPPORTED, counted=len(w),
            msg=BAD_CLOSURE_MSG)
    refused(F, ctx, lambda: hjm([(s1.h, sp.h, LT, bad, out2.h), good]), E_UNSUPPORTED, msg=BAD_CLOSURE_MSG)

    # mzgpu_delta_first_stage_many
    b0 = mz.Batch.build(ctx, host, 0, 1)
    b40 = mz.Batch.build(ctx, np.zeros(3, dtype=mz.R40), 0, 1)

    def dfs(reqs, k=None):
        k = len(reqs) if k is None else k
        arr = lambda t, xs: (t * max(1, len(xs)))(*xs)  # noqa: E731
        cl = lambda xs: arr(C.c_void_p, [C.cast(C.pointer(c), C.c_void_p) if c is not None else None for c in xs])  # noqa: E731
        return lib.mzgpu_delta_first_stage_many(
            ctx.h, k, arr(C.c_void_p, [r[0] for r in reqs]), cl([r[1] for r in reqs]), arr(C.c_uint64, [FE] * len(reqs)),
            arr(C.c_void_p, [r[2] for r in reqs]), arr(C.c_int32, [r[3] for r in reqs]), cl([r[4] for r in reqs]),
            arr(C.c_void_p, [r[5] for r in reqs]))

    dgood = (b0.h, None, sp.h, LE, None, out.h)
    assert dfs([], 0) == 0
    refused(F, ctx, lambda: dfs([dgood] * 65), E_INVALID)
    for second in [(b40.h, None, sp.h, LE, None, out2.h), (b0.h, None, sp40.h, LE, None, out2.h),
                   (b0.h, None, sp.h, LE, None, out40.h), (b0.h, None, sp.h, 3, None, out2.h),
                   (None, None, sp.h, LE, None, out2.h), (b0.h, None, sp.h, LE, None, None)]:
        refused(F, ctx, lambda: dfs([dgood, second]), E_INVALID, counted=len(b0))
    ctx.check(lib.mzgpu_ctx_sync(ctx.h))
    refused(F, ctx, lambda: dfs([dgood, (b0.h, bad, sp.h, LE, None, out2.h)]), E_UNSUPPORTED, counted=len(b0),
            msg=BAD_CLOSURE_MSG)
    refused(F, ctx, lambda: dfs([dgood, (b0.h, None, sp.h, LE, bad, out2.h)]), E_UNSUPPORTED, counted=len(b0),
            msg=BAD_CLOSURE_MSG)
    # nothing was appended, and the context still works
    assert len(out) == 0 and len(out2) == 0 and len(out40) == 0
    ctx.check(hjm([good]))
    assert len(out) > 0
