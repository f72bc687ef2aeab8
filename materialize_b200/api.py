"""Host-side mirror of the differential-dataflow operator surface, over the C ABI.

Names follow the reference's traits so the parity tests read like its own:

  consolidate / consolidate_updates   differential_dataflow::consolidation
  Batcher.push_container / seal       Batcher (src/timely-util/src/operator.rs:572-633)
  Batch                               Rc<OrdValBatch> (len / description / cursor export)
  Spine (Trace)                       spine_fueled::Spine behind TraceAgent
                                      (insert / exert / set_*_compaction / cursor_through)
  JoinCore                            mz_join_core (src/compute/src/render/join/mz_join_core.rs)
  half_join                           dogs3 half_join (delta_join.rs:401-431)
  ReduceAccumulable                   build_accumulable (src/compute/src/render/reduce.rs:1261)

Everything executes on the GPU through libmzgpu.so; rows cross the boundary as
numpy structured arrays (host memory) or stay in `DeviceRows` (device memory).
"""
import ctypes as C

import numpy as np

from . import _ffi as F
from ._ffi import (  # noqa: F401  (re-exported)
    ACCUM_DISTINCT,
    AGG_COUNT_SUM_F64,
    AGG_DISTINCT,
    AGG_THRESHOLD,
    AGG_MIN,
    AGG_MAX,
    AGG_COUNT_SUM_I64,
    FRONTIER_EMPTY,
    HALFJOIN_LE,
    HALFJOIN_LT,
    R16,
    R32,
    R40,
    RACC,
    ROUT,
    Closure,
    MzGpuError,
)

SRC_KEY, SRC_VAL1, SRC_VAL2 = 0, 1, 2
_CMP = {"eq": 0, "ne": 1, "lt": 2, "le": 3, "gt": 4, "ge": 5}


def make_closure(key_fields=(), val_fields=(), filters=(), expr=None):
    """Build a closure descriptor.  key_fields / val_fields: (src, shift, bits, dst_shift);
    filters: (src, shift, bits, op, rhs); expr: ((src, shift, bits), (src, shift, bits), c) = a * (c - b)."""
    c = F.Closure()
    c.n_key_fields, c.n_val_fields, c.n_filters = len(key_fields), len(val_fields), len(filters)
    for i, f in enumerate(key_fields):
        c.key_fields[i] = F.Field(*f)
    for i, f in enumerate(val_fields):
        c.val_fields[i] = F.Field(*f)
    for i, (src, shift, bits, op, rhs) in enumerate(filters):
        c.filters[i] = F.Filter(F.Field(src, shift, bits, 0), _CMP[op], rhs)
    if expr is not None:
        a, b, k = expr
        c.expr_kind = 1
        c.expr_a = F.Field(a[0], a[1], a[2], 0)
        c.expr_b = F.Field(b[0], b[1], b[2], 0)
        c.expr_c = k
    return c


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _clp(closure):
    return C.byref(closure) if closure is not None else None


class Context:
    """One per timely worker / GPU (mzgpu_ctx)."""

    def __init__(self, device=0, worker_index=0, peers=1):
        h = C.c_void_p()
        st = F.lib.mzgpu_ctx_create(device, worker_index, peers, C.byref(h))
        self.h = h
        if st != F.OK:
            msg = F.lib.mzgpu_last_error(h).decode() if h else "context allocation failed"
            raise MzGpuError(st, msg)
        self.device, self.worker_index, self.peers = device, worker_index, peers

    def check(self, st):
        if st != F.OK:
            raise MzGpuError(st, F.lib.mzgpu_last_error(self.h).decode())

    def sync(self):
        self.check(F.lib.mzgpu_ctx_sync(self.h))

    def stats(self):
        s = F.Stats()
        self.check(F.lib.mzgpu_ctx_stats(self.h, C.byref(s)))
        return {name: int(getattr(s, name)) for name, _ in F.Stats._fields_}

    def stream(self):
        return F.lib.mzgpu_ctx_stream(self.h)

    def profile(self, on=True):
        """Bracket every kernel launch with CUDA events on the ctx stream."""
        self.check(F.lib.mzgpu_profile_enable(self.h, 1 if on else 0))

    def host_times(self):
        """{wait_ns, alloc_ns, allocs, alloc_bytes}: host time spent waiting for the device / in the allocator."""
        out = (C.c_uint64 * 4)()
        self.check(F.lib.mzgpu_ctx_host_times(self.h, out))
        return {"wait_ns": out[0], "alloc_ns": out[1], "allocs": out[2], "alloc_bytes": out[3]}

    def profile_report(self):
        """{kernel: {launches, ms, bytes}} since the last report."""
        buf = C.create_string_buffer(1 << 20)
        self.check(F.lib.mzgpu_profile_report(self.h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            name, launches, ms, nbytes = line.rsplit(" ", 3)
            out[name] = {"launches": int(launches), "ms": float(ms), "bytes": int(nbytes)}
        return out

    def close(self):
        if self.h:
            F.lib.mzgpu_ctx_destroy(self.h)
            self.h = None

    # -- a1
    def consolidate(self, rows):
        """consolidate / consolidate_updates on a host array (R16 or R32); returns the survivors."""
        rows = np.ascontiguousarray(rows).copy()
        n_out = C.c_uint64(0)
        if rows.dtype.itemsize == 16:
            st = F.lib.mzgpu_consolidate_r16(self.h, _ptr(rows), len(rows), F.MEM_HOST, C.byref(n_out))
        elif rows.dtype.itemsize == 32:
            st = F.lib.mzgpu_consolidate_r32(self.h, _ptr(rows), len(rows), F.MEM_HOST, C.byref(n_out))
        else:
            buf = DeviceRows(self, rows.dtype.itemsize)
            buf.upload(rows)
            buf.consolidate()
            return buf.download()
        self.check(st)
        return rows[: n_out.value].copy()


class DeviceRows:
    """Library-owned device row buffer (mzgpu_buf)."""

    def __init__(self, ctx, row_bytes):
        self.ctx, self.row_bytes = ctx, row_bytes
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_buf_new(ctx.h, row_bytes, C.byref(h)))
        self.h = h

    def __len__(self):
        return F.lib.mzgpu_buf_len(self.h)

    def upload(self, rows):
        rows = np.ascontiguousarray(rows)
        assert rows.dtype.itemsize == self.row_bytes
        self.ctx.check(F.lib.mzgpu_buf_upload(self.h, _ptr(rows), len(rows), F.MEM_HOST))
        return self

    def append(self, rows):
        rows = np.ascontiguousarray(rows)
        assert rows.dtype.itemsize == self.row_bytes
        self.ctx.check(F.lib.mzgpu_buf_append(self.h, _ptr(rows), len(rows), F.MEM_HOST))
        return self

    def download(self):
        n = len(self)
        out = np.zeros(n, dtype=F.DTYPES[self.row_bytes])
        got = C.c_uint64(0)
        self.ctx.check(F.lib.mzgpu_buf_download(self.h, _ptr(out), n, F.MEM_HOST, C.byref(got)))
        return out

    def append_buf(self, other):
        """Append another device buffer's rows without reading its length back."""
        self.ctx.check(F.lib.mzgpu_buf_append_buf(self.h, other.h))
        return self

    def append_buf_at_most(self, other, max_rows):
        """append_buf where the caller bounds other's row count (checked on the device)."""
        self.ctx.check(F.lib.mzgpu_buf_append_buf_at_most(self.h, other.h, max_rows))
        return self

    def device_ptr(self):
        return F.lib.mzgpu_buf_device_ptr(self.h)

    def clear(self):
        self.ctx.check(F.lib.mzgpu_buf_clear(self.h))

    def consolidate(self):
        self.ctx.check(F.lib.mzgpu_buf_consolidate(self.h))
        return self

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_buf_free(self.h)
            self.h = None


def seal_many(batchers, upper):
    """Seal several batchers at one frontier (mzgpu_batcher_seal_many): the same batches as
    [b.seal_lazy(upper) for b in batchers]; update-batch-sized seals share one launch."""
    k = len(batchers)
    if k == 0:
        return []
    hs = (C.c_void_p * k)(*[b.h for b in batchers])
    outs = (C.c_void_p * k)()
    batchers[0].ctx.check(F.lib.mzgpu_batcher_seal_many(k, hs, upper, outs))
    return [Batch(b.ctx, C.c_void_p(outs[i]), b.row_bytes) for i, b in enumerate(batchers)]


class Batch:
    def __init__(self, ctx, h, row_bytes):
        self.ctx, self.h, self.row_bytes = ctx, h, row_bytes

    @staticmethod
    def build(ctx, rows, lower, upper, since=0):
        """Builder::seal on unsorted updates with an explicit description."""
        rows = np.ascontiguousarray(rows)
        h = C.c_void_p()
        ctx.check(
            F.lib.mzgpu_batch_build(
                ctx.h, rows.dtype.itemsize, _ptr(rows), len(rows), F.MEM_HOST, F.Desc(lower, upper, since), C.byref(h)
            )
        )
        return Batch(ctx, h, rows.dtype.itemsize)

    def __len__(self):
        return F.lib.mzgpu_batch_len(self.h)

    def keys(self):
        return F.lib.mzgpu_batch_keys(self.h)

    def desc(self):
        d = F.lib.mzgpu_batch_desc(self.h)
        return (d.lower, d.upper, d.since)

    def rows(self):
        n = len(self)
        out = np.zeros(n, dtype=F.DTYPES[self.row_bytes])
        got = C.c_uint64(0)
        self.ctx.check(F.lib.mzgpu_batch_export(self.h, _ptr(out), n, F.MEM_HOST, C.byref(got)))
        return out

    def merge(self, other, since):
        h = C.c_void_p()
        self.ctx.check(F.lib.mzgpu_batch_merge(self.h, other.h, since, C.byref(h)))
        return Batch(self.ctx, h, self.row_bytes)

    # -- a8: batched cursor calls
    def seek_keys(self, keys):
        """Cursor::seek_key for every key: array of (key found, first row, rows of that key);
        len == 0 where the cursor ran off the end."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        runs = np.zeros(len(keys), dtype=F.KEY_RUN)
        self.ctx.check(F.lib.mzgpu_batch_seek_keys(self.h, _ptr(keys), len(keys), F.MEM_HOST, _ptr(runs)))
        return runs

    def key_page(self, first_ordinal, max_keys):
        """step_key in pages: the distinct keys [first_ordinal, first_ordinal + max_keys) with their runs."""
        runs = np.zeros(max_keys, dtype=F.KEY_RUN)
        n = C.c_uint64(0)
        self.ctx.check(F.lib.mzgpu_batch_key_page(self.h, first_ordinal, max_keys, F.MEM_HOST, _ptr(runs), C.byref(n)))
        return runs[: n.value]

    def rows_range(self, first, length):
        """The update rows [first, first + length) in cursor order (get_val / step_val / map_times)."""
        out = np.zeros(length, dtype=F.DTYPES[self.row_bytes])
        self.ctx.check(F.lib.mzgpu_batch_rows(self.h, first, length, _ptr(out), F.MEM_HOST))
        return out

    def index(self):
        """The hash index, for tests and diagnostics: (slots as HASH_SLOT records, distinct keys,
        longest key run saturating at 1024)."""
        n_slots, n_keys, longest = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        st = F.lib.mzgpu_batch_index_export(self.h, None, 0, F.MEM_HOST, C.byref(n_slots), C.byref(n_keys), C.byref(longest))
        if st not in (F.OK, F.E_CAPACITY):
            self.ctx.check(st)
        slots = np.zeros(n_slots.value, dtype=F.HASH_SLOT)
        self.ctx.check(
            F.lib.mzgpu_batch_index_export(
                self.h, _ptr(slots), len(slots), F.MEM_HOST, C.byref(n_slots), C.byref(n_keys), C.byref(longest)
            )
        )
        return slots, n_keys.value, longest.value

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_batch_release(self.h)
            self.h = None


class Builder:
    """Builder::{push, done} (OrdValBuilder): chunks in, one batch out."""

    def __init__(self, ctx, row_bytes=32, capacity=0):
        self.ctx, self.row_bytes = ctx, row_bytes
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_builder_new(ctx.h, row_bytes, capacity, C.byref(h)))
        self.h = h

    def push(self, rows):
        rows = np.ascontiguousarray(rows)
        assert rows.dtype.itemsize == self.row_bytes
        self.ctx.check(F.lib.mzgpu_builder_push(self.h, _ptr(rows), len(rows), F.MEM_HOST))

    def push_buf(self, dev_rows):
        self.ctx.check(F.lib.mzgpu_builder_push_buf(self.h, dev_rows.h))

    def done(self, lower, upper, since=0):
        h = C.c_void_p()
        self.ctx.check(F.lib.mzgpu_builder_done(self.h, F.Desc(lower, upper, since), C.byref(h)))
        return Batch(self.ctx, h, self.row_bytes)

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_builder_free(self.h)
            self.h = None


class Batcher:
    def __init__(self, ctx, row_bytes=32):
        self.ctx, self.row_bytes = ctx, row_bytes
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_batcher_new(ctx.h, row_bytes, C.byref(h)))
        self.h = h

    def push_container(self, rows):
        rows = np.ascontiguousarray(rows)
        assert rows.dtype.itemsize == self.row_bytes
        self.ctx.check(F.lib.mzgpu_batcher_push(self.h, _ptr(rows), len(rows), F.MEM_HOST))

    def push_device(self, dev_rows):
        self.ctx.check(F.lib.mzgpu_batcher_push(self.h, dev_rows.device_ptr(), len(dev_rows), F.MEM_DEVICE))

    def push_buf(self, dev_rows):
        """push_container for rows in a device buffer; its length is not read back."""
        self.ctx.check(F.lib.mzgpu_batcher_push_buf(self.h, dev_rows.h))

    def seal_lazy(self, upper):
        """seal without asking for the new frontier: nothing returns to the host."""
        h = C.c_void_p()
        self.ctx.check(F.lib.mzgpu_batcher_seal(self.h, upper, C.byref(h), None))
        return Batch(self.ctx, h, self.row_bytes)

    def seal(self, upper):
        h = C.c_void_p()
        lower = C.c_uint64(0)
        self.ctx.check(F.lib.mzgpu_batcher_seal(self.h, upper, C.byref(h), C.byref(lower)))
        return Batch(self.ctx, h, self.row_bytes)

    def frontier(self):
        return F.lib.mzgpu_batcher_frontier(self.h)

    def __len__(self):
        return F.lib.mzgpu_batcher_len(self.h)

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_batcher_free(self.h)
            self.h = None


class Spine:
    """The trace behind an arrangement."""

    def __init__(self, ctx, row_bytes=32, effort=1, _borrowed=None):
        self.ctx, self.row_bytes = ctx, row_bytes
        self._owned = _borrowed is None
        if _borrowed is None:
            h = C.c_void_p()
            ctx.check(F.lib.mzgpu_spine_new(ctx.h, row_bytes, effort, C.byref(h)))
            self.h = h
        else:
            self.h = _borrowed

    def insert(self, batch):
        self.ctx.check(F.lib.mzgpu_spine_insert(self.h, batch.h))

    def exert(self, effort):
        did = C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_spine_exert(self.h, effort, C.byref(did)))
        return bool(did.value)

    def exert_logic(self, proportionality=16):
        return F.lib.mzgpu_spine_exert_logic(self.h, proportionality)

    def set_logical_compaction(self, frontier):
        self.ctx.check(F.lib.mzgpu_spine_set_logical_compaction(self.h, frontier))

    def set_physical_compaction(self, frontier):
        self.ctx.check(F.lib.mzgpu_spine_set_physical_compaction(self.h, frontier))

    def get_logical_compaction(self):
        return F.lib.mzgpu_spine_get_logical_compaction(self.h)

    def get_physical_compaction(self):
        return F.lib.mzgpu_spine_get_physical_compaction(self.h)

    def read_upper(self):
        return F.lib.mzgpu_spine_read_upper(self.h)

    def num_batches_through(self, upper):
        arr = (C.c_void_p * 128)()
        n = C.c_uint32(0)
        self.ctx.check(F.lib.mzgpu_spine_batches_through(self.h, upper, arr, 128, C.byref(n)))
        return n.value

    def layers(self):
        out = (C.c_uint64 * (4 * 64))()
        n = C.c_uint32(0)
        self.ctx.check(F.lib.mzgpu_spine_layers(self.h, out, 64, C.byref(n)))
        return [tuple(int(out[4 * i + j]) for j in range(4)) for i in range(n.value)]

    def size(self):
        """ArrangementSize: {size_bytes, capacity_bytes, allocations, batches, updates}."""
        out = np.zeros(1, dtype=F.ARRANGEMENT_SIZE)
        self.ctx.check(F.lib.mzgpu_spine_size(self.h, _ptr(out)))
        return {k: int(out[k][0]) for k in out.dtype.names}

    def export(self):
        """as_collection: consolidated contents, times advanced to `since`."""
        buf = DeviceRows(self.ctx, self.row_bytes)
        self.ctx.check(F.lib.mzgpu_spine_export(self.h, buf.h))
        return buf.download()

    def __del__(self):
        if getattr(self, "h", None) and self._owned and self.ctx.h:
            F.lib.mzgpu_spine_free(self.h)
            self.h = None


class JoinCore:
    """mz_join_core over two arrangements."""

    def __init__(self, ctx, trace1, trace2, closure=None):
        self.ctx, self.closure = ctx, closure
        self._keep = (trace1, trace2)
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_join_new(ctx.h, trace1.h, trace2.h, _clp(closure), C.byref(h)))
        self.h = h
        self.out = DeviceRows(ctx, 32 if closure is not None else 40)

    def push(self, side, batch, cap):
        self.ctx.check(F.lib.mzgpu_join_core_push(self.h, side, batch.h, cap))

    def work(self, fuel_rows=1 << 62):
        done = C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_join_core_work(self.h, fuel_rows, self.out.h, C.byref(done)))
        return bool(done.value)

    def work_until(self, fuel_rows, deadline_ns):
        """Work::process with the reference's yield function: stop after fuel_rows of results or at the
        first yield point after deadline_ns (time.monotonic_ns() clock; 0 = no deadline)."""
        done = C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_join_core_work_until(self.h, fuel_rows, deadline_ns, self.out.h, C.byref(done)))
        return bool(done.value)

    def results(self):
        return self.out.download()

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_join_free(self.h)
            self.h = None


class LinearJoin:
    """A LinearJoinPlan (src/compute-types/src/plan/join/linear_join.rs:26-62) rendered over the operators as
    src/compute/src/render/join/linear_join.rs:230-527 renders it.  stages: [(lookup Spine, stream_key closure,
    join closure)]; the source relation arrives as update rows, each lookup relation as the batch the caller has
    just inserted into its arrangement."""

    def __init__(self, ctx, stages, initial_closure=None, final_closure=None):
        self.ctx = ctx
        self._keep = [st[0] for st in stages]
        plan = F.LinearJoinPlan()
        plan.n_stages = len(stages)
        if initial_closure is not None:
            plan.has_initial_closure, plan.initial_closure = 1, initial_closure
        if final_closure is not None:
            plan.has_final_closure, plan.final_closure = 1, final_closure
        for i, (_, stream_key, closure) in enumerate(stages[: F.LINEAR_MAX_STAGES]):
            plan.stages[i].stream_key = stream_key
            plan.stages[i].closure = closure
        traces = (C.c_void_p * max(1, len(stages)))(*[st[0].h for st in stages])
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_linear_join_new(ctx.h, C.byref(plan), traces, C.byref(h)))
        self.h, self.n = h, len(stages)
        self.out = DeviceRows(ctx, 32)

    def step(self, source_rows, lookup_batches, upper):
        """One activation; returns the final collection's new updates (downloaded)."""
        src = DeviceRows(self.ctx, 32).upload(source_rows) if source_rows is not None and len(source_rows) else None
        lb = (C.c_void_p * self.n)(*[b.h if b is not None else None for b in lookup_batches])
        self.out.clear()
        self.ctx.check(F.lib.mzgpu_linear_join_step(self.h, src.h if src is not None else None, lb, upper, self.out.h))
        return self.out.download()

    def stage_trace_layers(self, stage):
        """Raw handle of the stage's "JoinStage" arrangement (owned by the operator)."""
        return F.lib.mzgpu_linear_join_stage_trace(self.h, stage)

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_linear_join_free(self.h)
            self.h = None


def half_join(ctx, stream, trace, cmp_mode, closure=None, consolidate_output=True):
    stream = np.ascontiguousarray(stream)
    out = DeviceRows(ctx, 32)
    ctx.check(
        F.lib.mzgpu_half_join(
            ctx.h, _ptr(stream), len(stream), F.MEM_HOST, trace.h, cmp_mode, _clp(closure), 1 if consolidate_output else 0, out.h
        )
    )
    return out.download()


def half_join_dev(ctx, dev_stream, trace, cmp_mode, closure=None, consolidate_output=False, out=None):
    """half_join over a device-resident stream; the result stays on the device (no read-back)."""
    out = out if out is not None else DeviceRows(ctx, 32)
    ctx.check(F.lib.mzgpu_half_join_buf(ctx.h, dev_stream.h, trace.h, cmp_mode, _clp(closure), 1 if consolidate_output else 0, out.h))
    return out


def half_join_many(ctx, requests):
    """Several half joins in one launch (mzgpu_half_join_many).  requests: (dev_stream, trace, cmp_mode,
    closure or None, out DeviceRows); requests naming the same `out` must be adjacent and append in order."""
    k = len(requests)
    if k == 0:
        return
    streams = (C.c_void_p * k)(*[r[0].h for r in requests])
    traces = (C.c_void_p * k)(*[r[1].h for r in requests])
    cmps = (C.c_int32 * k)(*[r[2] for r in requests])
    # a NULL entry means the identity closure (key, val2), as in mzgpu_half_join_buf
    cls = (C.c_void_p * k)(*[C.cast(C.pointer(r[3]), C.c_void_p) if r[3] is not None else None for r in requests])
    outs = (C.c_void_p * k)(*[r[4].h for r in requests])
    ctx.check(F.lib.mzgpu_half_join_many(ctx.h, k, streams, traces, cmps, cls, outs))


def delta_first_stage_many(ctx, requests):
    """build_update_stream + first half join of several delta paths in one launch
    (mzgpu_delta_first_stage_many).  requests: (batch, initial_closure or None, skip_time, trace, cmp_mode,
    closure or None, out DeviceRows)."""
    k = len(requests)
    if k == 0:
        return

    def ptrs(cls):
        return (C.c_void_p * k)(*[C.cast(C.pointer(c), C.c_void_p) if c is not None else None for c in cls])

    batches = (C.c_void_p * k)(*[r[0].h for r in requests])
    initial = ptrs([r[1] for r in requests])
    skips = (C.c_uint64 * k)(*[r[2] for r in requests])
    traces = (C.c_void_p * k)(*[r[3].h for r in requests])
    cmps = (C.c_int32 * k)(*[r[4] for r in requests])
    closures = ptrs([r[5] for r in requests])
    outs = (C.c_void_p * k)(*[r[6].h for r in requests])
    ctx.check(F.lib.mzgpu_delta_first_stage_many(ctx.h, k, batches, initial, skips, traces, cmps, closures, outs))


def update_stream_dev(ctx, batch, closure=None, skip_time=F.FRONTIER_EMPTY, out=None):
    out = out if out is not None else DeviceRows(ctx, 32)
    ctx.check(F.lib.mzgpu_update_stream(ctx.h, batch.h, _clp(closure), skip_time, out.h))
    return out


def update_stream(ctx, batch, closure=None, skip_time=F.FRONTIER_EMPTY):
    out = DeviceRows(ctx, 32)
    ctx.check(F.lib.mzgpu_update_stream(ctx.h, batch.h, _clp(closure), skip_time, out.h))
    return out.download()


def map_rows(ctx, rows, closure):
    rows = np.ascontiguousarray(rows)
    out = DeviceRows(ctx, 32)
    ctx.check(F.lib.mzgpu_map_rows(ctx.h, _ptr(rows), len(rows), F.MEM_HOST, _clp(closure), out.h))
    return out.download()


class ReduceAccumulable:
    def __init__(self, ctx, agg_kind=F.AGG_COUNT_SUM_I64):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_reduce_new(ctx.h, agg_kind, C.byref(h)))
        self.h = h

    def step(self, rows, upper):
        rows = np.ascontiguousarray(rows)
        out = DeviceRows(self.ctx, 64)
        self.ctx.check(F.lib.mzgpu_reduce_accumulable(self.h, _ptr(rows), len(rows), F.MEM_HOST, upper, out.h))
        return out.download()

    def step_dev(self, dev_rows, upper, out=None):
        """One activation over device-resident rows; corrections are appended to `out` on the device."""
        out = out if out is not None else DeviceRows(self.ctx, 64)
        self.ctx.check(F.lib.mzgpu_reduce_accumulable_buf(self.h, dev_rows.h, upper, out.h))
        return out

    def input_trace(self):
        return Spine(self.ctx, 80, _borrowed=F.lib.mzgpu_reduce_input_trace(self.h))


def accum_lane(kind, src=SRC_VAL1, shift=0, bits=64, sign_extend=False):
    """One lane of ReduceLanes: COUNT and SUM of the bit-field `bits` wide at `shift` of value word
    `src` (1 = val / val1, 2 = val2); an I64 field is sign-extended when `sign_extend`.  A kind of
    AGG_COUNT_SUM_I64 | ACCUM_DISTINCT makes the lane COUNT(DISTINCT col) / SUM(DISTINCT col)."""
    return (int(kind), int(src), int(shift), int(bits), bool(sign_extend))


class ReduceLanes:
    """COUNT / SUM of several value columns per key in one arrangement (mzgpu_reduce_lanes_new).
    `lanes` is a list of accum_lane(...) tuples; input rows are R32 (in_row_bytes=32) or R40 (40).
    Output rows have the dtype ROUT_LANES[class] (lane l in ["lanes"][:, l])."""

    def __init__(self, ctx, lanes, in_row_bytes=32):
        self.ctx = ctx
        self.n_lanes = len(lanes)
        self.in_row_bytes = in_row_bytes
        arr = (F.AccumLane * max(1, len(lanes)))()
        for i, (kind, src, shift, bits, sx) in enumerate(lanes):
            arr[i].kind = kind
            arr[i].sign_extend = 1 if sx else 0
            arr[i].field = F.Field(src, shift, bits, 0)
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_reduce_lanes_new(ctx.h, in_row_bytes, arr, len(lanes), C.byref(h)))
        self.h = h
        self.lane_class = F.lane_class(self.n_lanes)
        self.arr_row_bytes, self.out_row_bytes = F.LANE_ROW_BYTES[self.lane_class]

    def step(self, rows, upper):
        rows = np.ascontiguousarray(rows)
        out = DeviceRows(self.ctx, self.out_row_bytes)
        self.ctx.check(F.lib.mzgpu_reduce_lanes(self.h, _ptr(rows), len(rows), F.MEM_HOST, upper, out.h))
        return out.download().view(F.ROUT_LANES[self.lane_class])

    def step_dev(self, dev_rows, upper, out=None):
        """One activation over device-resident rows; corrections are appended to `out` on the device."""
        out = out if out is not None else DeviceRows(self.ctx, self.out_row_bytes)
        self.ctx.check(F.lib.mzgpu_reduce_lanes_buf(self.h, dev_rows.h, upper, out.h))
        return out

    def input_trace(self):
        return Spine(self.ctx, self.arr_row_bytes, _borrowed=F.lib.mzgpu_reduce_input_trace(self.h))

    def distinct_trace(self, lane):
        """The (key, value) pair arrangement (R32 rows) of distinct lane `lane`; None for any other lane."""
        h = F.lib.mzgpu_reduce_lanes_distinct_trace(self.h, lane)
        return Spine(self.ctx, 32, _borrowed=h) if h else None

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_reduce_free(self.h)
            self.h = None


class TopK(ReduceAccumulable):
    """TopK per key over (key, value) rows (BasicTopKPlan, src/compute/src/render/top_k.rs:215-248,
    521-673): `limit` < 0 or None = no limit; stepped like every other reduce kind."""

    def __init__(self, ctx, limit, offset=0, descending=False):
        self.ctx = ctx
        h = C.c_void_p()
        lim = -1 if limit is None else int(limit)
        ctx.check(F.lib.mzgpu_topk_new(ctx.h, lim, int(offset), 1 if descending else 0, C.byref(h)))
        self.h = h

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_reduce_free(self.h)
            self.h = None


def route(key, peers):
    return F.lib.mzgpu_route(key, peers)


def partition_many(ctx, bufs, peers):
    """The device half of an exchange round for `peers` workers (mzgpu_partition_many): returns
    [(rows grouped by destination, counts per destination)] for each DeviceRows in `bufs`."""
    k = len(bufs)
    outs = [DeviceRows(ctx, b.row_bytes) for b in bufs]
    ins_a = (C.c_void_p * k)(*[b.h for b in bufs])
    outs_a = (C.c_void_p * k)(*[o.h for o in outs])
    counts = (C.c_uint64 * (k * peers))()
    ctx.check(F.lib.mzgpu_partition_many(ctx.h, k, ins_a, peers, outs_a, counts))
    return [(outs[e].download(), [int(counts[e * peers + p]) for p in range(peers)]) for e in range(k)]


# -- exchange over peer memory (a13): setup helpers and the round itself
def p2p_export(ctx, landing_rows, region_row_bytes=32):
    """Allocate this worker's landing zone; returns the 64-byte IPC handle to all-gather."""
    h = (C.c_uint8 * F.P2P_HANDLE_BYTES)()
    ctx.check(F.lib.mzgpu_comm_p2p_export(ctx.h, landing_rows, region_row_bytes, h))
    return bytes(h)


def p2p_import(ctx, handles):
    """handles: list of every worker's handle (index = worker)."""
    raw = b"".join(handles)
    buf = (C.c_uint8 * len(raw)).from_buffer_copy(raw)
    ctx.check(F.lib.mzgpu_comm_p2p_import(ctx.h, buf))


def p2p_connect_local(ctxs, landing_rows, region_row_bytes=32):
    """All workers live in this process (tests: every worker on one GPU): map the zones directly."""
    for c in ctxs:
        c.check(F.lib.mzgpu_comm_p2p_export(c.h, landing_rows, region_row_bytes, None))
    zones = (C.c_void_p * len(ctxs))(*[F.lib.mzgpu_comm_p2p_zone(c.h) for c in ctxs])
    for c in ctxs:
        c.check(F.lib.mzgpu_comm_p2p_import_local(c.h, zones))


def exchange_p2p_send(ctx, bufs):
    a = (C.c_void_p * len(bufs))(*[b.h for b in bufs])
    ctx.check(F.lib.mzgpu_exchange_p2p_send(ctx.h, len(bufs), a))


def exchange_p2p_recv(ctx, outs, recv_ub=None):
    a = (C.c_void_p * len(outs))(*[b.h for b in outs])
    ub = (C.c_uint64 * len(outs))(*recv_ub) if recv_ub is not None else None
    ctx.check(F.lib.mzgpu_exchange_p2p_recv(ctx.h, len(outs), a, ub))


class Correction:
    """The MV sink's correction buffer on the device (CorrectionV2, src/compute/src/sink/correction_v2.rs)."""

    def __init__(self, ctx):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_correction_new(ctx.h, C.byref(h)))
        self.h = h

    def insert(self, rows, negate=False):
        rows = np.ascontiguousarray(rows)
        self.ctx.check(F.lib.mzgpu_correction_insert(self.h, _ptr(rows), len(rows), F.MEM_HOST, 1 if negate else 0))

    def insert_buf(self, dev_rows, negate=False):
        self.ctx.check(F.lib.mzgpu_correction_insert_buf(self.h, dev_rows.h, 1 if negate else 0))

    def updates_before(self, upper):
        out = DeviceRows(self.ctx, 32)
        self.ctx.check(F.lib.mzgpu_correction_updates_before(self.h, upper, out.h))
        return out.download()

    def advance_since(self, since):
        self.ctx.check(F.lib.mzgpu_correction_advance_since(self.h, since))

    def consolidate_at_since(self):
        self.ctx.check(F.lib.mzgpu_correction_consolidate_at_since(self.h))

    def __len__(self):
        return F.lib.mzgpu_correction_len(self.h)

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_correction_free(self.h)
            self.h = None


# ---- f4: the columnar wire format (Column<C>, src/timely-util/src/columnar.rs:54-222)
def column_decode(ctx, layout, words, out=None):
    """Column::borrow() + drain on the device: append the updates of one serialized container
    (numpy u64 words) to `out` (a DeviceRows; created if None) and return it."""
    words = np.ascontiguousarray(words, dtype="<u8")
    if out is None:
        out = DeviceRows(ctx, 16 if layout == F.COLUMN_U64X2 else 32)
    ctx.check(F.lib.mzgpu_column_decode(ctx.h, layout, _ptr(words), len(words), F.MEM_HOST, out.h))
    return out


def column_encode(dev_rows, layout, first=0, n=(1 << 64) - 1):
    """indexed::encode of rows [first, first + n) of a DeviceRows -> numpy u64 words."""
    ctx = dev_rows.ctx
    need = C.c_uint64(0)
    st = F.lib.mzgpu_column_encode(dev_rows.h, layout, first, n, None, 0, F.MEM_HOST, C.byref(need))
    if st not in (F.OK, F.E_CAPACITY):
        ctx.check(st)
    words = np.zeros(need.value, dtype="<u8")
    ctx.check(F.lib.mzgpu_column_encode(dev_rows.h, layout, first, n, _ptr(words), len(words), F.MEM_HOST, C.byref(need)))
    return words


def column_build(dev_rows, layout):
    """ColumnBuilder over a DeviceRows: the serialized containers it mints, in order."""
    ctx = dev_rows.ctx
    need, nch = C.c_uint64(0), C.c_uint32(0)
    st = F.lib.mzgpu_column_build(dev_rows.h, layout, None, 0, F.MEM_HOST, C.byref(need), None, 0, C.byref(nch))
    if st not in (F.OK, F.E_CAPACITY):
        ctx.check(st)
    words = np.zeros(need.value, dtype="<u8")
    sizes = np.zeros(max(1, nch.value), dtype="<u8")
    ctx.check(
        F.lib.mzgpu_column_build(
            dev_rows.h, layout, _ptr(words), len(words), F.MEM_HOST, C.byref(need),
            sizes.ctypes.data_as(C.POINTER(C.c_uint64)), len(sizes), C.byref(nch),
        )
    )
    out, at = [], 0
    for i in range(nch.value):
        out.append(words[at : at + int(sizes[i])])
        at += int(sizes[i])
    return out


def batch_walk_column(batch, layout, key=None, first=0, fuel=(1 << 64) - 1):
    """walk_cursor over one batch into a serialized container (src/compute/src/render/context.rs:1299-1355);
    returns (words, rows emitted)."""
    ctx = batch.ctx
    kp = C.byref(C.c_uint64(key)) if key is not None else None
    need, nrows = C.c_uint64(0), C.c_uint64(0)
    st = F.lib.mzgpu_batch_walk_column(batch.h, kp, first, fuel, layout, None, 0, F.MEM_HOST, C.byref(need), C.byref(nrows))
    if st not in (F.OK, F.E_CAPACITY):
        ctx.check(st)
    words = np.zeros(need.value, dtype="<u8")
    ctx.check(
        F.lib.mzgpu_batch_walk_column(batch.h, kp, first, fuel, layout, _ptr(words), len(words), F.MEM_HOST, C.byref(need), C.byref(nrows))
    )
    return words, nrows.value
