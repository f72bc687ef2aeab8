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
    MONO_F64,
    MONO_OUT,
    RMONO,
    ORDER_F64,
    RTOPK,
    TOPK_NO_LIMIT,
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
    ROUT_HAVING_ERR_SHIFT,
    HAVING_ERR_DIVISION_BY_ZERO,
    HAVING_ERR_NUMERIC_FIELD_OVERFLOW,
    HAVING_ERR_INT32_OUT_OF_RANGE,
    HAVING_ERR_INT64_OUT_OF_RANGE,
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
    """mz_join_core over two arrangements.  `closure` is a bit-field closure (F.Closure) or a JoinClosure; with a
    JoinClosure, work() and work_until() also append the error rows to self.errs (R32)."""

    def __init__(self, ctx, trace1, trace2, closure=None):
        self.ctx, self.closure = ctx, closure
        self._keep = (trace1, trace2, closure)
        h = C.c_void_p()
        self.errs = None
        if isinstance(closure, JoinClosure):
            ctx.check(F.lib.mzgpu_join_new_mfp(ctx.h, trace1.h, trace2.h, closure.h, C.byref(h)))
            self.out, self.errs = DeviceRows(ctx, closure.out_row_bytes), DeviceRows(ctx, 32)
        else:
            ctx.check(F.lib.mzgpu_join_new(ctx.h, trace1.h, trace2.h, _clp(closure), C.byref(h)))
            self.out = DeviceRows(ctx, 32 if closure is not None else 40)
        self.h = h

    def push(self, side, batch, cap):
        self.ctx.check(F.lib.mzgpu_join_core_push(self.h, side, batch.h, cap))

    def work(self, fuel_rows=1 << 62):
        if self.errs is not None:
            return self.work_until(fuel_rows, 0)
        done = C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_join_core_work(self.h, fuel_rows, self.out.h, C.byref(done)))
        return bool(done.value)

    def work_mfp(self, fuel_rows, deadline_ns=0, out=None, errs=None):
        """mzgpu_join_core_work_mfp into `out` / `errs` (default: self.out / self.errs); returns done."""
        done = C.c_int32(0)
        out = out if out is not None else self.out
        errs = errs if errs is not None else self.errs
        self.ctx.check(F.lib.mzgpu_join_core_work_mfp(self.h, fuel_rows, deadline_ns, out.h, errs.h if errs is not None
                                                      else None, C.byref(done)))
        return bool(done.value)

    def work_until(self, fuel_rows, deadline_ns):
        """Work::process with the reference's yield function: stop after fuel_rows of results or at the
        first yield point after deadline_ns (time.monotonic_ns() clock; 0 = no deadline)."""
        if self.errs is not None:
            return self.work_mfp(fuel_rows, deadline_ns)
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


def half_join_mfp(ctx, stream, trace, cmp_mode, jc, consolidate_output=True):
    """half_join with a JoinClosure: returns (rows, errors), the errors R32 (code, payload, time, diff)."""
    stream = np.ascontiguousarray(stream)
    out, errs = DeviceRows(ctx, jc.out_row_bytes), DeviceRows(ctx, 32)
    ctx.check(F.lib.mzgpu_half_join_mfp(ctx.h, _ptr(stream), len(stream), F.MEM_HOST, trace.h, cmp_mode, jc.h,
                                        1 if consolidate_output else 0, out.h, errs.h))
    return out.download(), errs.download()


def half_join_mfp_dev(ctx, dev_stream, trace, cmp_mode, jc, consolidate_output=False, out=None, errs=None):
    """half_join_mfp over a device-resident stream; (out, errs) stay on the device."""
    out = out if out is not None else DeviceRows(ctx, jc.out_row_bytes)
    errs = errs if errs is not None else DeviceRows(ctx, 32)
    ctx.check(F.lib.mzgpu_half_join_mfp_buf(ctx.h, dev_stream.h, trace.h, cmp_mode, jc.h,
                                            1 if consolidate_output else 0, out.h, errs.h))
    return out, errs


def half_join_many_mfp(ctx, requests, errs=None):
    """mzgpu_half_join_many_mfp.  requests: (dev_stream, trace, cmp_mode, JoinClosure, out DeviceRows); returns
    `errs` (a new DeviceRows unless given) with the errors of every request, consolidated."""
    errs = errs if errs is not None else DeviceRows(ctx, 32)
    k = len(requests)
    streams = (C.c_void_p * max(1, k))(*[r[0].h for r in requests])
    traces = (C.c_void_p * max(1, k))(*[r[1].h for r in requests])
    cmps = (C.c_int32 * max(1, k))(*[r[2] for r in requests])
    jcs = (C.c_void_p * max(1, k))(*[r[3].h for r in requests])
    outs = (C.c_void_p * max(1, k))(*[r[4].h for r in requests])
    ctx.check(F.lib.mzgpu_half_join_many_mfp(ctx.h, k, streams, traces, cmps, jcs, outs, errs.h))
    return errs


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


class _Reduce:
    """What every reduce operator shares.  A subclass sets step and step_dev with _steps(), and _out_rb and
    _arr_rb, the row bytes of its output and of its input arrangement.  The operator is freed with this object,
    and a Spine from input_trace() borrows the operator's arrangement: it must not outlive the operator."""

    def _create(self, ctx, new, *args):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(new(ctx.h, *args, C.byref(h)))
        self.h = h

    def input_trace(self):
        return Spine(self.ctx, self._arr_rb, _borrowed=F.lib.mzgpu_reduce_input_trace(self.h))

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_reduce_free(self.h)
            self.h = None


def _steps(host_fn, buf_fn, errs_rb=None):
    """step() and step_dev() of a reduce operator class: its host-form and buffer-form step functions, and the row
    bytes of its error rows (None: the operator has no error rows).  They call the class's own entry points
    whatever operator they are given, so the library refuses an operator of another kind."""
    host, buf = getattr(F.lib, host_fn), getattr(F.lib, buf_fn)

    def outs(self, out=None, errs=None):
        out = out if out is not None else DeviceRows(self.ctx, self._out_rb)
        if errs_rb is None:
            return (out,)
        return out, errs if errs is not None else DeviceRows(self.ctx, errs_rb)

    def step(self, rows, upper):
        """One activation over host rows: the output rows, or (output, errors) for an operator with error rows."""
        rows = np.ascontiguousarray(rows)
        o = outs(self)
        self.ctx.check(host(self.h, _ptr(rows), len(rows), F.MEM_HOST, upper, *(x.h for x in o)))
        got = tuple(x.download() for x in o)
        return got if errs_rb else got[0]

    def step_dev(self, dev_rows, upper, out=None, errs=None):
        """One activation over device-resident rows; its output (and errors, for an operator with error rows) are
        appended on the device."""
        o = outs(self, out, errs)
        self.ctx.check(buf(self.h, dev_rows.h, upper, *(x.h for x in o)))
        return o if errs_rb else o[0]

    return step, step_dev


def _accum_lanes(lanes):
    arr = (F.AccumLane * max(1, len(lanes)))()
    for i, (kind, src, shift, bits, sx) in enumerate(lanes):
        arr[i].kind = kind
        arr[i].sign_extend = 1 if sx else 0
        arr[i].field = F.Field(src, shift, bits, 0)
    return arr


def _order_lanes(order):
    arr = (F.OrderLane * max(1, len(order)))()
    for i, (src, shift, bits, sx, desc, f64) in enumerate(order):
        arr[i].sign_extend = 1 if sx else 0
        arr[i].descending = 1 if desc else 0
        arr[i].flags = F.ORDER_F64 if f64 else 0
        arr[i].field = F.Field(src, shift, bits, 0)
    return arr


class ReduceAccumulable(_Reduce):
    """One-column reduce (mzgpu_reduce_new)."""

    step, step_dev = _steps("mzgpu_reduce_accumulable", "mzgpu_reduce_accumulable_buf")
    _out_rb = 64
    # the input arrangement's rows: exploded accumulators (mzgpu_racc), or the (key, value) rows
    # themselves for MIN / MAX / TopK
    row_bytes = _arr_rb = 80

    def __init__(self, ctx, agg_kind=F.AGG_COUNT_SUM_I64):
        if agg_kind in (F.AGG_MIN, F.AGG_MAX):
            self.row_bytes = self._arr_rb = 32
        self._create(ctx, F.lib.mzgpu_reduce_new, agg_kind)


def accum_lane(kind, src=SRC_VAL1, shift=0, bits=64, sign_extend=False):
    """One lane of ReduceLanes: COUNT and SUM of the bit-field `bits` wide at `shift` of value word
    `src` (1 = val / val1, 2 = val2); an I64 field is sign-extended when `sign_extend`.  A kind of
    AGG_COUNT_SUM_I64 | ACCUM_DISTINCT makes the lane COUNT(DISTINCT col) / SUM(DISTINCT col).  For
    ReduceMonotonic the kind is AGG_MIN or AGG_MAX and `sign_extend` chooses signed order."""
    return (int(kind), int(src), int(shift), int(bits), bool(sign_extend))



def order_lane(src=SRC_VAL1, shift=0, bits=64, sign_extend=False, descending=False, f64=False):
    """One ColumnOrder of TopKMonotonic's order key: the bit-field `bits` wide at `shift` of value word `src`
    (1 = val / val1, 2 = val2), compared signed (sign-extended) when `sign_extend`, reversed when
    `descending`.  `f64` marks a float64 column, which the operator refuses (E_UNSUPPORTED)."""
    return (int(src), int(shift), int(bits), bool(sign_extend), bool(descending), bool(f64))

# HAVING ops (mzgpu_having_op): one constructor per opcode.  An op is (code, arg, shift, bits,
# sign_extend, constant value or None); having() builds the descriptor and its constant pool.
def h_key(shift=0, bits=64, sign_extend=False):
    """INT: bits [shift, shift + bits) of the output key, sign-extended when asked."""
    return (F.HOP_KEY, 0, int(shift), int(bits), 1 if sign_extend else 0, None)


def h_count(lane):
    """INT: COUNT of `lane`."""
    return (F.HOP_COUNT, int(lane), 0, 0, 0, None)


def h_sum(lane):
    """NUM (int64 lane) or FLOAT (float64 lane): SUM of `lane`; NULL when its NULL flag is set."""
    return (F.HOP_SUM, int(lane), 0, 0, 0, None)


def h_int(v):
    return (F.HOP_INT, 0, 0, 0, 0, int(v))


def h_num(v):
    return (F.HOP_NUM, 0, 0, 0, 0, int(v))


def h_float(x):
    return (F.HOP_FLOAT, 0, 0, 0, 0, float(x))


def h_add(width=64):
    return (F.HOP_ADD, int(width), 0, 0, 0, None)


def h_sub(width=64):
    return (F.HOP_SUB, int(width), 0, 0, 0, None)


def h_mul(width=64):
    return (F.HOP_MUL, int(width), 0, 0, 0, None)


def h_div(width=64):
    return (F.HOP_DIV, int(width), 0, 0, 0, None)


def h_cmp(op):
    """op: "eq", "ne", "lt", "le", "gt" or "ge" (signed, or OrderedFloat for FLOAT)."""
    return (F.HOP_CMP, _CMP[op], 0, 0, 0, None)


def h_and():
    return (F.HOP_AND, 0, 0, 0, 0, None)


def h_or():
    return (F.HOP_OR, 0, 0, 0, 0, None)


def h_not():
    return (F.HOP_NOT, 0, 0, 0, 0, None)


def having(*predicates):
    """The mzgpu_having of a list of predicates, each a list of h_*() ops in postfix order.  A program past the
    descriptor's limits (predicates, ops per predicate, distinct constants) raises MzGpuError(E_INVALID), as
    the library does for a descriptor it cannot hold."""
    if len(predicates) > F.HAVING_MAX_PREDICATES:
        raise MzGpuError(F.E_INVALID, f"having: {len(predicates)} predicates (at most {F.HAVING_MAX_PREDICATES})")
    for p, ops in enumerate(predicates):
        if len(ops) > F.HAVING_MAX_OPS:
            raise MzGpuError(F.E_INVALID, f"having: predicate {p} has {len(ops)} ops (at most {F.HAVING_MAX_OPS})")
    hv = F.Having()
    hv.n_predicates = len(predicates)
    pool = []
    for p, ops in enumerate(predicates):
        hv.n_ops[p] = len(ops)
        for i, (code, arg, shift, bits, sx, value) in enumerate(ops):
            o = hv.ops[p][i]
            o.code, o.arg, o.shift, o.bits, o.sign_extend = code, arg, shift, bits, sx
            if value is None:
                continue
            if code == F.HOP_FLOAT:
                words = (int(np.float64(value).view(np.uint64)), 0)
            else:
                words = (value & (2**64 - 1), (value >> 64) & (2**64 - 1))
            if words not in pool:
                if len(pool) == F.HAVING_MAX_CONSTS:
                    raise MzGpuError(F.E_INVALID, f"having: more than {F.HAVING_MAX_CONSTS} distinct constants")
                pool.append(words)
            o.konst = pool.index(words)
    hv.n_consts = len(pool)
    for k, (lo, hi) in enumerate(pool):
        hv.consts[k].lo, hv.consts[k].hi = lo, hi
    return hv


class ReduceLanes(_Reduce):
    """COUNT / SUM of several value columns per key in one arrangement (mzgpu_reduce_lanes_new).
    `lanes` is a list of accum_lane(...) tuples; input rows are R32 (in_row_bytes=32) or R40 (40).
    Output rows have the dtype ROUT_LANES[class] (lane l in ["lanes"][:, l]).  `having`: a HAVING
    filter, having(...) or an F.Having (mzgpu_reduce_lanes_new_having); its errors are in bits
    16-18 of "flags" (ROUT_HAVING_ERR_SHIFT)."""

    _step, step_dev = _steps("mzgpu_reduce_lanes", "mzgpu_reduce_lanes_buf")

    def __init__(self, ctx, lanes, in_row_bytes=32, having=None):
        self.n_lanes = len(lanes)
        self.in_row_bytes = in_row_bytes
        args = (in_row_bytes, _accum_lanes(lanes), len(lanes))
        if having is None:
            self._create(ctx, F.lib.mzgpu_reduce_lanes_new, *args)
        else:
            self._create(ctx, F.lib.mzgpu_reduce_lanes_new_having, *args, C.byref(having))
        self.lane_class = F.lane_class(self.n_lanes)
        self.arr_row_bytes, self.out_row_bytes = self._arr_rb, self._out_rb = F.LANE_ROW_BYTES[self.lane_class]

    def step(self, rows, upper):
        return ReduceLanes._step(self, rows, upper).view(F.ROUT_LANES[self.lane_class])

    def distinct_trace(self, lane):
        """The (key, value) pair arrangement (R32 rows) of distinct lane `lane`; None for any other lane."""
        h = F.lib.mzgpu_reduce_lanes_distinct_trace(self.h, lane)
        return Spine(self.ctx, 32, _borrowed=h) if h else None


class TopKMonotonic(_Reduce):
    """MonotonicTop1 / MonotonicTopK over append-only input (mzgpu_topk_monotonic_new): the first `limit`
    rows per key in the order of `order` (order_lane() tuples, at most 3; ties by val1, then val2), with only
    that window arranged.  Top1 is limit=1; LIMIT NULL is TOPK_NO_LIMIT.  Input rows are R32
    (in_row_bytes=32) or R40 (40).  step() returns (changes, errors): the window's changes as rows of the
    input width, and R16 error rows (key = time, diff = rows with diff <= 0 at that time).  input_trace() is the
    window arrangement (RTOPK rows)."""

    step, step_dev = _steps("mzgpu_topk_monotonic", "mzgpu_topk_monotonic_buf", 16)
    _arr_rb = 72

    def __init__(self, ctx, order, limit, in_row_bytes=32, must_consolidate=False):
        self.in_row_bytes = self._out_rb = in_row_bytes
        self._create(ctx, F.lib.mzgpu_topk_monotonic_new, in_row_bytes, _order_lanes(order), len(order), int(limit),
                     1 if must_consolidate else 0)


class TopKBasic(_Reduce):
    """BasicTopKPlan over input with retractions (mzgpu_topk_basic_new): per key the units in positions
    [offset, offset + limit) of its live rows in the order of `order` (order_lane() tuples, at most 3; ties by
    val1, then val2).  LIMIT NULL is TOPK_NO_LIMIT.  Input rows are R32 (in_row_bytes=32) or R40 (40), with any
    diffs.  step() returns (changes, errors): the window's changes as rows of the input width, and R32 error rows
    (key, 0, time, +1 entering / -1 leaving the negative-count state).  input_trace() is the whole live input
    (RTOPK rows)."""

    step, step_dev = _steps("mzgpu_topk_basic", "mzgpu_topk_basic_buf", 32)
    _arr_rb = 72

    def __init__(self, ctx, order, limit, offset=0, in_row_bytes=32):
        self.in_row_bytes = self._out_rb = in_row_bytes
        self._create(ctx, F.lib.mzgpu_topk_basic_new, in_row_bytes, _order_lanes(order), len(order), int(limit),
                     int(offset))

    def negatives_trace(self):
        """The negatives arrangement: R32 rows (key, 0, time, delta), summed per key its negative-count rows."""
        return Spine(self.ctx, 32, _borrowed=F.lib.mzgpu_topk_basic_negatives_trace(self.h))


def hop(code, arg=0, shift=0, bits=0, sign_extend=0, konst=0):
    """One op of a HAVING / MFP program (mzgpu_having_op) as a tuple."""
    return (code, arg, shift, bits, sign_extend, konst)


def col(src, shift=0, bits=64, signed=False, code=F.HOP_COL):
    """Push a bit-field of source word `src` (SRC_KEY / SRC_VAL1 / SRC_VAL2): INT, or with `code` an
    MZTS (HOP_COL_MZTS), TS (HOP_COL_TS) or DATE (HOP_COL_DATE) column."""
    return hop(code, src, shift, bits, 1 if signed else 0)


def map_ref(i):
    """Push the value of map expression `i` (HOP_MAP)."""
    return hop(F.HOP_MAP, i)


def field_map(i, shift=0, bits=64, dst_shift=0):
    """An output field taking bits [shift, shift + bits) of map expression `i`, placed at `dst_shift`."""
    return (F.SRC_MAP0 + i, shift, bits, dst_shift)


def interval_const(micros=0, days=0, months=0):
    """An interval constant for HOP_TS_ADD_IV: (lo, hi) with lo = microseconds, hi = days | months << 32."""
    return (micros & (2**64 - 1), (days & 0xFFFFFFFF) | ((months & 0xFFFFFFFF) << 32))


def _put_ops(dst, ops):
    for i, o in enumerate(ops[:F.MFP_MAX_OPS]):
        dst[i].code, dst[i].arg, dst[i].shift, dst[i].bits, dst[i].sign_extend, dst[i].konst = o


def _put_consts(dst, consts):
    for k, (lo, hi) in enumerate(consts[:F.MFP_MAX_CONSTS]):
        dst[k].lo, dst[k].hi = lo & (2**64 - 1), hi & (2**64 - 1)


def _mfp_structs(fields, predicates, temporal, consts, in_row_bytes, out_row_bytes, maps, map_consts):
    """The mzgpu_mfp and (None without expressions) mzgpu_mfp_map of a plan."""
    m = F.Mfp()
    m.in_row_bytes, m.out_row_bytes = in_row_bytes, out_row_bytes
    for w, fl in enumerate(fields):
        m.n_fields[w] = len(fl)
        for i, f in enumerate(fl[:6]):
            m.fields[w][i] = F.Field(*f)
    m.n_predicates, m.n_temporal, m.n_consts = len(predicates), len(temporal), len(consts)
    for p, ops in enumerate(predicates[:F.MFP_MAX_PREDICATES]):
        m.n_ops[p] = len(ops)
        _put_ops(m.ops[p], ops)
    for p, (cmp, ops) in enumerate(temporal[:F.MFP_MAX_TEMPORAL]):
        m.temporal_cmp[p] = cmp
        m.n_temporal_ops[p] = len(ops)
        _put_ops(m.temporal_ops[p], ops)
    _put_consts(m.consts, consts)
    if not maps:
        return m, None
    mp = F.MfpMap()
    mp.n_exprs, mp.n_consts = len(maps), len(map_consts)
    for e, ops in enumerate(maps[:F.MFP_MAX_MAPS]):
        mp.n_ops[e] = len(ops)
        _put_ops(mp.ops[e], ops)
    _put_consts(mp.consts, map_consts)
    return m, mp


class Mfp:
    """A temporal filter (mzgpu_mfp_new): the MfpPlan of a `WHERE mz_now() ...` query.  `fields` gives the
    output words (key, val1, val2) as lists of (src, shift, bits, dst_shift); `predicates` are op lists (hop());
    `temporal` is a list of (cmp, ops) for `mz_now() cmp expr`; `consts` are (lo, hi) pairs.  step() returns
    (updates, errors): the updates of time < upper, consolidated, and R32 error rows (code, payload, time, diff);
    future updates are held until an upper passes them.  `maps` are the map expressions (op lists over
    `map_consts`, mzgpu_mfp_new_map): predicates and temporal programs read them with map_ref(), output fields with
    field_map()."""

    def __init__(self, ctx, fields, predicates=(), temporal=(), consts=(), in_row_bytes=32, out_row_bytes=32,
                 until=F.FRONTIER_EMPTY, maps=(), map_consts=()):
        self.ctx, self.in_row_bytes, self.out_row_bytes = ctx, in_row_bytes, out_row_bytes
        m, mp = _mfp_structs(fields, predicates, temporal, consts, in_row_bytes, out_row_bytes, maps, map_consts)
        h = C.c_void_p()
        if mp is None:
            ctx.check(F.lib.mzgpu_mfp_new(ctx.h, C.byref(m), until, C.byref(h)))
        else:
            ctx.check(F.lib.mzgpu_mfp_new_map(ctx.h, C.byref(m), C.byref(mp), until, C.byref(h)))
        self.h = h

    def step(self, rows, upper):
        rows = np.ascontiguousarray(rows)
        out, errs = DeviceRows(self.ctx, self.out_row_bytes), DeviceRows(self.ctx, 32)
        self.ctx.check(F.lib.mzgpu_mfp_step(self.h, _ptr(rows), len(rows), F.MEM_HOST, upper, out.h, errs.h))
        return out.download(), errs.download()

    def step_dev(self, dev_rows, upper, out=None, errs=None):
        """One step over device-resident rows; updates and errors are appended on the device."""
        out = out if out is not None else DeviceRows(self.ctx, self.out_row_bytes)
        errs = errs if errs is not None else DeviceRows(self.ctx, 32)
        self.ctx.check(F.lib.mzgpu_mfp_step_buf(self.h, dev_rows.h, upper, out.h, errs.h))
        return out, errs

    def frontier(self):
        """The least held time, or FRONTIER_EMPTY."""
        t = C.c_uint64(0)
        self.ctx.check(F.lib.mzgpu_mfp_frontier(self.h, C.byref(t)))
        return t.value

    def stats(self):
        """(held rows, buckets, rows the store read and wrote in the last step)."""
        a = (C.c_uint64 * 3)()
        self.ctx.check(F.lib.mzgpu_mfp_stats(self.h, a))
        return tuple(int(x) for x in a)

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_mfp_free(self.h)
            self.h = None


def lower_equivalences(classes):
    """JoinClosure's ready_equivalences as leading predicates: a class [e0, e1, ..., en] of expressions (op lists)
    becomes CMP_EQ(e0, e1), ..., CMP_EQ(e0, en)."""
    return [list(c[0]) + list(e) + [hop(F.HOP_CMP, _CMP["eq"])] for c in classes for e in c[1:]]


class JoinClosure:
    """The closure of the probe operators as a device MfpPlan (mzgpu_join_closure_new): JoinClosure
    { ready_equivalences, before } over the words (key, stream value, lookup value) = SRC_KEY / SRC_VAL1 / SRC_VAL2.
    `equivalences` are lowered ahead of `predicates` (lower_equivalences); the other arguments are those of Mfp
    without temporal predicates.  Pass it to half_join_mfp*, half_join_many_mfp or JoinCore."""

    def __init__(self, ctx, fields, predicates=(), consts=(), out_row_bytes=32, maps=(), map_consts=(),
                 equivalences=(), in_row_bytes=40, temporal=()):
        self.ctx, self.out_row_bytes = ctx, out_row_bytes
        preds = lower_equivalences(equivalences) + list(predicates)
        m, mp = _mfp_structs(fields, preds, temporal, consts, in_row_bytes, out_row_bytes, maps, map_consts)
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_join_closure_new(ctx.h, C.byref(m), C.byref(mp) if mp is not None else None,
                                               C.byref(h)))
        self.h = h

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_join_closure_free(self.h)
            self.h = None


class PeekPlan:
    """The plan of an index peek (mzgpu_peek_plan_new): an MfpPlan without temporal predicates over the trace's
    (key, val) = SRC_KEY / SRC_VAL1 (the arguments of Mfp), and the finishing: `order` (order_lane() tuples over the
    plan's OUTPUT words, at most 3), `limit` (None = no limit), `offset`, and `project` (per output word a list of
    (src, shift, bits, dst_shift) fields over the output words; () = the identity).  Pass it to peek / peek_many."""

    def __init__(self, ctx, fields, predicates=(), consts=(), out_rb=32, maps=(), map_consts=(), order=(), limit=None,
                 offset=0, project=(), in_row_bytes=32, temporal=()):
        self.ctx, self.out_row_bytes = ctx, out_rb
        m, mp = _mfp_structs(fields, predicates, temporal, consts, in_row_bytes, out_rb, maps, map_consts)
        fin = F.Finishing()
        fin.n_order = len(order)
        for i, (src, shift, bits, sx, desc, f64) in enumerate(order[:F.MAX_ORDER_LANES]):
            fin.order[i].sign_extend, fin.order[i].descending = int(sx), int(desc)
            fin.order[i].flags = F.ORDER_F64 if f64 else 0
            fin.order[i].field = F.Field(src, shift, bits, 0)
        fin.limit = F.TOPK_NO_LIMIT if limit is None else int(limit)
        fin.offset = int(offset)
        for w, fl in enumerate(project):
            fin.n_project[w] = len(fl)
            for i, f in enumerate(fl[:6]):
                fin.project[w][i] = F.Field(*f)
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_peek_plan_new(ctx.h, C.byref(m), C.byref(mp) if mp is not None else None,
                                            C.byref(fin), C.byref(h)))
        self.h = h

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_peek_plan_free(self.h)
            self.h = None


_NO_KEYS = np.zeros(1, dtype=np.uint64)  # the address of an empty literal list


def _peek_req(req, plan, as_of, literals, max_rows, keep):
    """Fill an mzgpu_peek_req; host arrays the call reads are appended to `keep`."""
    req.plan, req.as_of, req.max_rows, req.literals_mem = plan.h, int(as_of), int(max_rows), F.MEM_HOST
    if literals is not None:
        arr = np.ascontiguousarray(np.asarray(literals, dtype=np.uint64).reshape(-1))
        keep.append(arr)
        req.literals = (arr if len(arr) else _NO_KEYS).ctypes.data
        req.n_literals = len(arr)


def _peek_result(res, out):
    if res.status == F.PEEK_ROWS:
        return ("rows", out.download())
    if res.status == F.PEEK_NOT_READY:
        return ("not_ready", None)
    return ("error", (int(res.err_kind), tuple(int(x) for x in res.detail)))


def peek_many(ctx, spine, requests, err_spine=None):
    """k index peeks in one call (mzgpu_peek_many).  `requests` are dicts with `plan` (PeekPlan), `as_of` and
    optionally `literals` (None = a full scan; a sequence of keys) and `max_rows` (0 = none).  Returns one result per
    request, as peek() does."""
    k = len(requests)
    reqs, res, keep = (F.PeekReq * k)(), (F.PeekResult * k)(), []
    outs = [DeviceRows(ctx, r["plan"].out_row_bytes) for r in requests]
    for i, r in enumerate(requests):
        _peek_req(reqs[i], r["plan"], r["as_of"], r.get("literals"), r.get("max_rows", 0), keep)
    out_arr = (C.c_void_p * k)(*[o.h.value for o in outs])
    ctx.check(F.lib.mzgpu_peek_many(ctx.h, spine.h, err_spine.h if err_spine is not None else None, k, reqs, out_arr,
                                    res))
    return [_peek_result(res[i], outs[i]) for i in range(k)]


def peek(ctx, plan, spine, as_of, literals=None, err_spine=None, max_rows=0):
    """One index peek (mzgpu_peek) of `spine` at `as_of`: ("rows", rows) -- (w0, w1[, w2], as_of, copies) in
    finishing order --, ("not_ready", None) or ("error", (PEEK_ERR_* kind, four detail words)).  `literals` None is a
    full scan, otherwise the keys to look up."""
    req, res, keep = F.PeekReq(), F.PeekResult(), []
    _peek_req(req, plan, as_of, literals, max_rows, keep)
    out = DeviceRows(ctx, plan.out_row_bytes)
    ctx.check(F.lib.mzgpu_peek(ctx.h, spine.h, err_spine.h if err_spine is not None else None, C.byref(req), out.h,
                               C.byref(res)))
    return _peek_result(res, out)


def field_fn(i, shift=0, bits=64, dst_shift=0):
    """An output field taking bits [shift, shift + bits) of FlatMap extension column `i`, placed at `dst_shift`."""
    return (F.SRC_FN0 + i, shift, bits, dst_shift)


class FlatMap:
    """FlatMap (mzgpu_flat_map_new): table function `kind` (TF_*) over each input row, its rows appended to the
    input and run through an MfpPlan (the arguments of Mfp).  `args` are the argument programs (op lists over
    `arg_consts`, reading the input row); `step_iv` the timestamp series step (interval_const()).  Extension column
    i is col(SRC_FN0 + i) in programs and field_fn(i) in the output.  step(rows, upper, fuel) starts an activation
    and expands its first `fuel` function rows, work(fuel) the next ones: each returns (updates, errors, done)."""

    def __init__(self, ctx, kind, args, fields, with_ordinality=False, arg_consts=(), step_iv=(0, 0), predicates=(),
                 temporal=(), consts=(), in_row_bytes=32, out_row_bytes=32, until=F.FRONTIER_EMPTY, maps=(),
                 map_consts=()):
        self.ctx, self.in_row_bytes, self.out_row_bytes = ctx, in_row_bytes, out_row_bytes
        tf = F.TableFunc()
        tf.kind, tf.with_ordinality, tf.n_consts = kind, 1 if with_ordinality else 0, len(arg_consts)
        for a, ops in enumerate(args[:3]):
            tf.n_ops[a] = len(ops)
            _put_ops(tf.ops[a], ops)
        _put_consts(tf.consts, arg_consts)
        tf.step_iv.lo, tf.step_iv.hi = step_iv[0] & (2**64 - 1), step_iv[1] & (2**64 - 1)
        m, mp = _mfp_structs(fields, predicates, temporal, consts, in_row_bytes, out_row_bytes, maps, map_consts)
        h = C.c_void_p()
        ctx.check(F.lib.mzgpu_flat_map_new(ctx.h, C.byref(tf), C.byref(m), C.byref(mp) if mp is not None else None,
                                           until, C.byref(h)))
        self.h = h

    def step(self, rows, upper, fuel=F.MFP_RESTORE_FUEL):
        rows = np.ascontiguousarray(rows)
        out, errs, done = DeviceRows(self.ctx, self.out_row_bytes), DeviceRows(self.ctx, 32), C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_flat_map_step(self.h, _ptr(rows), len(rows), F.MEM_HOST, upper, fuel, out.h,
                                                 errs.h, C.byref(done)))
        return out.download(), errs.download(), bool(done.value)

    def step_dev(self, dev_rows, upper, fuel=F.MFP_RESTORE_FUEL, out=None, errs=None):
        """step() over device-resident rows; updates and errors are appended on the device: (out, errs, done)."""
        out = out if out is not None else DeviceRows(self.ctx, self.out_row_bytes)
        errs = errs if errs is not None else DeviceRows(self.ctx, 32)
        done = C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_flat_map_step_buf(self.h, dev_rows.h, upper, fuel, out.h, errs.h, C.byref(done)))
        return out, errs, bool(done.value)

    def work(self, fuel=F.MFP_RESTORE_FUEL, out=None, errs=None):
        """The next `fuel` function rows of the activation: (updates, errors, done); with `out` / `errs`
        (DeviceRows) they are appended there and returned as they are."""
        dev = out is not None
        out = out if out is not None else DeviceRows(self.ctx, self.out_row_bytes)
        errs = errs if errs is not None else DeviceRows(self.ctx, 32)
        done = C.c_int32(0)
        self.ctx.check(F.lib.mzgpu_flat_map_work(self.h, fuel, out.h, errs.h, C.byref(done)))
        if dev:
            return out, errs, bool(done.value)
        return out.download(), errs.download(), bool(done.value)

    def frontier(self):
        """The least held time or, during an activation, unexpanded input time; FRONTIER_EMPTY if none."""
        t = C.c_uint64(0)
        self.ctx.check(F.lib.mzgpu_flat_map_frontier(self.h, C.byref(t)))
        return t.value

    def stats(self):
        """(held rows, buckets, rows the store touched in the last page, function rows still to expand)."""
        a = (C.c_uint64 * 4)()
        self.ctx.check(F.lib.mzgpu_flat_map_stats(self.h, a))
        return tuple(int(x) for x in a)

    def __del__(self):
        if getattr(self, "h", None) and self.ctx.h:
            F.lib.mzgpu_flat_map_free(self.h)
            self.h = None


class ReduceMonotonic(_Reduce):
    """MIN / MAX of several value columns per key over append-only input (mzgpu_reduce_monotonic_new,
    build_monotonic).  `lanes` are accum_lane(AGG_MIN | AGG_MAX, ...) tuples; sign_extend=True makes a lane
    an int64 aggregate (signed order), False an unsigned one.  Input rows are R32 (in_row_bytes=32) or R40
    (40).  step() returns (corrections, errors): corrections of dtype MONO_OUT[class] (lane l in
    ["vals"][:, l]), errors R16 rows (key = time, diff = rows with diff <= 0 at that time)."""

    step, step_dev = _steps("mzgpu_reduce_monotonic", "mzgpu_reduce_monotonic_buf", 16)

    def __init__(self, ctx, lanes, in_row_bytes=32, must_consolidate=False):
        self.n_lanes = len(lanes)
        self.in_row_bytes = in_row_bytes
        self._create(ctx, F.lib.mzgpu_reduce_monotonic_new, in_row_bytes, _accum_lanes(lanes), len(lanes),
                     1 if must_consolidate else 0)
        self.lane_class = F.mono_class(self.n_lanes)
        self.arr_row_bytes, self.out_row_bytes = self._arr_rb, self._out_rb = F.MONO_ROW_BYTES[self.lane_class]


class ReduceHierarchical(_Reduce):
    """MIN / MAX of several value columns per key over input with retractions (mzgpu_reduce_hierarchical_new,
    build_bucketed).  `lanes` are accum_lane(AGG_MIN | AGG_MAX, ...) tuples, as for ReduceMonotonic.  Input rows
    are R32 (in_row_bytes=32) or R40 (40).  step() returns (corrections, errors): corrections of dtype
    MONO_OUT[class] (lane l in ["vals"][:, l]), errors R32 rows (key, 0, time, +1 entering / -1 leaving the
    non-positive-accumulation state).  The arrangement (input_trace) holds the masked input rows."""

    step, step_dev = _steps("mzgpu_reduce_hierarchical", "mzgpu_reduce_hierarchical_buf", 32)

    def __init__(self, ctx, lanes, in_row_bytes=32):
        self.n_lanes = len(lanes)
        self.in_row_bytes = self._arr_rb = in_row_bytes
        self._create(ctx, F.lib.mzgpu_reduce_hierarchical_new, in_row_bytes, _accum_lanes(lanes), len(lanes))
        self.lane_class = F.mono_class(self.n_lanes)
        self.out_row_bytes = self._out_rb = F.MONO_ROW_BYTES[self.lane_class][1]


class TopK(ReduceAccumulable):
    """TopK per key over (key, value) rows (BasicTopKPlan, src/compute/src/render/top_k.rs:215-248,
    521-673): `limit` < 0 or None = no limit; stepped like every other reduce kind."""

    row_bytes = _arr_rb = 32

    def __init__(self, ctx, limit, offset=0, descending=False):
        lim = -1 if limit is None else int(limit)
        self._create(ctx, F.lib.mzgpu_topk_new, lim, int(offset), 1 if descending else 0)


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
