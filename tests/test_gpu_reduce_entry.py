"""The step entry points of every reduce-family operator: each of the twelve refuses an operator of another kind,
row widths it does not take and null arguments with MZGPU_E_INVALID and its exact message, without counting rows
or disturbing the operator; and the host form and the buffer form of each operator compute the same output."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

VAL1, VAL2 = 1, 2
E_INVALID = -1

# entry family -> (host-form function, buffer-form function, name in messages or None, error row bytes or 0)
ENTRIES = {
    "accumulable": ("mzgpu_reduce_accumulable", "mzgpu_reduce_accumulable_buf", None, 0),
    "lanes": ("mzgpu_reduce_lanes", "mzgpu_reduce_lanes_buf", "reduce_lanes", 0),
    "monotonic": ("mzgpu_reduce_monotonic", "mzgpu_reduce_monotonic_buf", "reduce_monotonic", 16),
    "hierarchical": ("mzgpu_reduce_hierarchical", "mzgpu_reduce_hierarchical_buf", "reduce_hierarchical", 32),
    "topk_monotonic": ("mzgpu_topk_monotonic", "mzgpu_topk_monotonic_buf", "topk_monotonic", 16),
    "topk_basic": ("mzgpu_topk_basic", "mzgpu_topk_basic_buf", "topk_basic", 32),
}

# operator kind, input row bytes -> its entry family
KINDS = [("accumulable", 32), ("topk", 32)] + [
    (k, rb) for k in ("lanes", "lanes2", "monotonic", "hierarchical", "topk_monotonic", "topk_basic") for rb in (32, 40)
]
FAMILY = {"accumulable": "accumulable", "topk": "accumulable", "lanes": "lanes", "lanes2": "lanes"}


def family(kind):
    return FAMILY.get(kind, kind)


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def F():
    from materialize_b200 import _ffi

    return _ffi


@pytest.fixture(scope="module")
def ctx(mz):
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


def make(mz, ctx, kind, in_rb):
    """A fresh operator of `kind` and the widths of its (out, errs) rows (errs 0: no error buffer)."""
    if kind == "accumulable":
        return mz.ReduceAccumulable(ctx, mz.AGG_COUNT_SUM_I64), 64, 0
    if kind == "topk":
        return mz.TopK(ctx, 2), 64, 0
    val2 = in_rb == 40
    if kind in ("lanes", "lanes2"):
        lanes = [mz.accum_lane(mz.AGG_COUNT_SUM_I64, VAL1)]
        if kind == "lanes2":
            lanes.append(mz.accum_lane(mz.AGG_COUNT_SUM_I64, VAL2 if val2 else VAL1, 0, 16))
        g = mz.ReduceLanes(ctx, lanes, in_rb)
        return g, g.out_row_bytes, 0
    if kind in ("monotonic", "hierarchical"):
        lanes = [mz.accum_lane(mz.AGG_MAX, VAL1), mz.accum_lane(mz.AGG_MIN, VAL2 if val2 else VAL1, 0, 32)]
        g = (mz.ReduceMonotonic if kind == "monotonic" else mz.ReduceHierarchical)(ctx, lanes, in_rb)
        return g, g.out_row_bytes, 16 if kind == "monotonic" else 32
    order = [mz.order_lane(VAL2 if val2 else VAL1, 0, 16)]
    if kind == "topk_monotonic":
        return mz.TopKMonotonic(ctx, order, 2, in_rb), in_rb, 16
    return mz.TopKBasic(ctx, order, 2, 0, in_rb), in_rb, 32


def rows_of(mz, in_rb, t0, seed, n=300):
    rng = np.random.default_rng(seed)
    rows = np.zeros(n, dtype=mz.R40 if in_rb == 40 else mz.R32)
    rows["key"] = rng.integers(0, 40, n)
    rows["val1" if in_rb == 40 else "val"] = rng.integers(0, 1 << 20, n)
    if in_rb == 40:
        rows["val2"] = rng.integers(0, 1 << 20, n)
    rows["time"] = t0 + rng.integers(0, 3, n)
    rows["diff"] = 1
    return rows


def rows_in(ctx):
    return ctx.stats()["rows_in"]


def last_error(F, ctx):
    return F.lib.mzgpu_last_error(ctx.h).decode()


def call_host(F, fam, h, rows, n, out, errs):
    fn = getattr(F.lib, ENTRIES[fam][0])
    args = [h, rows, n, F.MEM_HOST, 3, out]
    return fn(*(args + [errs] if ENTRIES[fam][3] else args))


def call_buf(F, fam, h, rows, out, errs):
    fn = getattr(F.lib, ENTRIES[fam][1])
    args = [h, rows, 3, out]
    return fn(*(args + [errs] if ENTRIES[fam][3] else args))


def host_msg(fam, out_rb, errs_rb):
    name, has_errs = ENTRIES[fam][2], ENTRIES[fam][3]
    if name is None:
        return None
    m = f"{name}: output buffer of {out_rb}-byte rows"
    return m + f" / error buffer of {errs_rb}-byte rows" if has_errs else m


def buf_msg(fam, in_rb, out_rb, errs_rb):
    name, has_errs = ENTRIES[fam][2], ENTRIES[fam][3]
    if name is None:
        return None
    m = f"{name}: input rows of {in_rb} bytes / output rows of {out_rb} bytes"
    return m + f" / error rows of {errs_rb} bytes" if has_errs else m


def refused(F, ctx, call, msg):
    """`call` returns MZGPU_E_INVALID, counts no rows and leaves `msg` (None: the message is left as it was)."""
    before_rows, before_msg = rows_in(ctx), last_error(F, ctx)
    assert call() == E_INVALID
    assert rows_in(ctx) == before_rows
    assert last_error(F, ctx) == (before_msg if msg is None else msg)


def step_outputs(g, rows, upper, dev=None):
    res = g.step_dev(dev, upper) if dev is not None else g.step(rows, upper)
    if not isinstance(res, tuple):
        res = (res,)
    return [r.download().tobytes() if hasattr(r, "download") else r.tobytes() for r in res]


def assert_steps_like_fresh(mz, ctx, g, kind, in_rb):
    """g, after refused calls, steps exactly as an operator that never saw them."""
    fresh = make(mz, ctx, kind, in_rb)[0]
    for t0, seed in ((0, 1), (3, 2)):
        rows = rows_of(mz, in_rb, t0, seed)
        assert step_outputs(g, rows, t0 + 3) == step_outputs(fresh, rows, t0 + 3)


@pytest.mark.parametrize("kind,in_rb", KINDS)
def test_wrong_operator(mz, F, ctx, kind, in_rb):
    g, _, _ = make(mz, ctx, kind, in_rb)
    rows = rows_of(mz, in_rb, 0, 0)
    dev = mz.DeviceRows(ctx, in_rb).upload(rows)
    for fam, (_, _, _, errs_rb) in ENTRIES.items():
        if fam == family(kind):
            continue
        # the widths that entry point takes for this input, so only the operator's kind is wrong
        out_rb = {"accumulable": 64, "lanes": 64, "monotonic": 56, "hierarchical": 56}.get(fam, in_rb)
        out, errs = mz.DeviceRows(ctx, out_rb), mz.DeviceRows(ctx, errs_rb or 16)
        refused(F, ctx, lambda: call_host(F, fam, g.h, rows.ctypes.data, len(rows), out.h, errs.h),
                host_msg(fam, out_rb, errs_rb))
        refused(F, ctx, lambda: call_buf(F, fam, g.h, dev.h, out.h, errs.h), buf_msg(fam, in_rb, out_rb, errs_rb))
        assert len(out) == 0 and len(errs) == 0
    assert_steps_like_fresh(mz, ctx, g, kind, in_rb)


@pytest.mark.parametrize("kind,in_rb", KINDS)
def test_wrong_widths(mz, F, ctx, kind, in_rb):
    g, out_rb, errs_rb = make(mz, ctx, kind, in_rb)
    fam = family(kind)
    rows = rows_of(mz, in_rb, 0, 0)
    other_in = 40 if in_rb == 32 else 32
    dev, dev_other = mz.DeviceRows(ctx, in_rb).upload(rows), mz.DeviceRows(ctx, other_in)
    bad_out = 72 if out_rb != 72 else 64
    cases = [(bad_out, errs_rb)]
    if errs_rb:
        cases.append((out_rb, 16 if errs_rb == 32 else 32))
    for ob, eb in cases:
        out, errs = mz.DeviceRows(ctx, ob), mz.DeviceRows(ctx, eb or 16)
        refused(F, ctx, lambda: call_host(F, fam, g.h, rows.ctypes.data, len(rows), out.h, errs.h),
                host_msg(fam, ob, eb))
        refused(F, ctx, lambda: call_buf(F, fam, g.h, dev.h, out.h, errs.h), buf_msg(fam, in_rb, ob, eb))
    out, errs = mz.DeviceRows(ctx, out_rb), mz.DeviceRows(ctx, errs_rb or 16)
    refused(F, ctx, lambda: call_buf(F, fam, g.h, dev_other.h, out.h, errs.h),
            buf_msg(fam, other_in, out_rb, errs_rb))
    if errs_rb:
        # one buffer as both outputs, also where its width would suit both
        for rb in {out_rb, errs_rb}:
            both = mz.DeviceRows(ctx, rb)
            refused(F, ctx, lambda: call_host(F, fam, g.h, rows.ctypes.data, len(rows), both.h, both.h),
                    host_msg(fam, rb, rb))
            refused(F, ctx, lambda: call_buf(F, fam, g.h, dev.h, both.h, both.h), buf_msg(fam, in_rb, rb, rb))
    assert_steps_like_fresh(mz, ctx, g, kind, in_rb)


@pytest.mark.parametrize("kind,in_rb", KINDS)
def test_null_arguments(mz, F, ctx, kind, in_rb):
    g, out_rb, errs_rb = make(mz, ctx, kind, in_rb)
    fam = family(kind)
    rows = rows_of(mz, in_rb, 0, 0)
    dev = mz.DeviceRows(ctx, in_rb).upload(rows)
    out, errs = mz.DeviceRows(ctx, out_rb), mz.DeviceRows(ctx, errs_rb or 16)
    p, n = rows.ctypes.data, len(rows)
    host = [(None, p, n, out.h, errs.h), (g.h, None, n, out.h, errs.h), (g.h, p, n, None, errs.h)]
    buf = [(None, dev.h, out.h, errs.h), (g.h, None, out.h, errs.h), (g.h, dev.h, None, errs.h)]
    if errs_rb:
        host.append((g.h, p, n, out.h, None))
        buf.append((g.h, dev.h, out.h, None))
    for a in host:
        before = rows_in(ctx)
        assert call_host(F, fam, *a) == E_INVALID, a
        assert rows_in(ctx) == before
    for a in buf:
        before = rows_in(ctx)
        assert call_buf(F, fam, *a) == E_INVALID, a
        assert rows_in(ctx) == before
    assert len(out) == 0 and len(errs) == 0
    assert_steps_like_fresh(mz, ctx, g, kind, in_rb)


@pytest.mark.parametrize("kind,in_rb", KINDS)
def test_host_and_buffer_forms_agree(mz, ctx, kind, in_rb):
    host, buf = make(mz, ctx, kind, in_rb)[0], make(mz, ctx, kind, in_rb)[0]
    nonempty = False
    for t0, seed in ((0, 5), (3, 6), (6, 7)):
        rows = rows_of(mz, in_rb, t0, seed)
        before = rows_in(ctx)
        got_host = step_outputs(host, rows, t0 + 3)
        assert rows_in(ctx) == before + len(rows)
        dev = mz.DeviceRows(ctx, in_rb).upload(rows)
        before = rows_in(ctx)
        got_buf = step_outputs(buf, None, t0 + 3, dev)
        assert rows_in(ctx) == before + len(rows)
        assert got_host == got_buf
        nonempty = nonempty or len(got_host[0]) > 0
    assert nonempty
