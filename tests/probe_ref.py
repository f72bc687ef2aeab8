"""Plain reference of the join probes (test infrastructure): half_join, the update stream, the probe
chains of half_join_many / delta_first_stage_many, and one join_core push.

Written from the definitions, not from the kernels:

  closure     include/mzgpu.h `mzgpu_closure`: out.key = OR of field(src) << dst_shift, out.val the
              same or a * (c - b) wrapping at 64 bits; the row is dropped unless every filter (an
              unsigned compare of a field with `rhs`) holds.  A field is bits [shift, shift + bits)
              of the key, the stream value (val1) or the lookup value (val2).
  probe       DESIGN.md sections 1-3: every stream row meets the rows of its key in every batch of
              the trace.  Half joins keep lookup rows with t2 <= t1 (LE) or t2 < t1 (LT) and emit at
              t1 (delta_join.rs: the stream's time never moves); join_core keeps every row and
              emits at max(t1, t2, meet) (mz_join_core.rs: both times joined with the capability).
              The diff is d1 * d2 wrapping at 64 bits.  Rows come out in stream order, then trace
              batch order, then lookup row order (the order DESIGN.md section 3 promises).
  update      build_update_stream (delta_join.rs): rows at `skip_time` are dropped, the initial
              closure maps (key, val) with val2 = 0.

Rows are (n, 4) u64 word matrices (key, val, time, diff) -- R40 join output is (n, 5): key, val1,
val2, time, diff.  Everything is vectorised with NumPy.
"""
import numpy as np

import arrangement_ref as aref

M64 = (1 << 64) - 1
FRONTIER_EMPTY = M64
LE, LT, JOIN = 0, 1, 2  # half join `le`, half join `lt`, join_core
CMP = {"eq": 0, "ne": 1, "lt": 2, "le": 3, "gt": 4, "ge": 5}
IDENTITY = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(2, 0, 64, 0)])  # a half join without a closure: (key, val2)


def _u(x, n):
    return np.broadcast_to(np.asarray(x, dtype=np.uint64), (n,))


def field(f, key, v1, v2):
    src, shift, bits = f[0], f[1], f[2]
    w = (key, v1, v2)[src] >> np.uint64(shift)
    if bits < 64:
        w = w & np.uint64((1 << bits) - 1)
    return w


def closure(c, key, v1, v2):
    """(keep, key', val') of a closure over arrays of (key, val1, val2).  `c` holds the closure's fields
    in make_closure's keyword form: key_fields / val_fields (src, shift, bits, dst_shift), filters
    (src, shift, bits, op, rhs), expr ((src, shift, bits) of a, the same of b, c)."""
    n = len(key)
    key, v1, v2 = _u(key, n), _u(v1, n), _u(v2, n)
    keep = np.ones(n, dtype=bool)
    for src, shift, bits, op, rhs in c.get("filters", ()):
        x = field((src, shift, bits), key, v1, v2)
        r = np.uint64(rhs)
        op = CMP[op] if isinstance(op, str) else op
        keep &= [x == r, x != r, x < r, x <= r, x > r, x >= r][op]
    k = np.zeros(n, dtype=np.uint64)
    for f in c.get("key_fields", ()):
        k |= field(f, key, v1, v2) << np.uint64(f[3])
    v = np.zeros(n, dtype=np.uint64)
    if c.get("expr") is not None:
        a, b, const = c["expr"]
        with np.errstate(over="ignore"):
            v = field(a, key, v1, v2) * (np.uint64(const) - field(b, key, v1, v2))
    else:
        for f in c.get("val_fields", ()):
            v |= field(f, key, v1, v2) << np.uint64(f[3])
    return keep, k, v


def _w(rows, nw=4):
    if rows is None:
        return np.zeros((0, nw), dtype=np.uint64)
    a = np.ascontiguousarray(rows)
    if a.dtype.names:
        return a.view(np.uint64).reshape(-1, a.dtype.itemsize // 8)
    return a.astype(np.uint64, copy=False).reshape(-1, nw)


def matches(stream, batches):
    """(stream row, batch, lookup row) of every key match, in stream x batch x row order."""
    s = _w(stream)
    n = len(s)
    parts = []
    for bi, b in enumerate(batches):
        b = _w(b)
        if n == 0 or len(b) == 0:
            continue
        lo = np.searchsorted(b[:, 0], s[:, 0], "left")
        cnt = np.searchsorted(b[:, 0], s[:, 0], "right") - lo
        tot = int(cnt.sum())
        if tot == 0:
            continue
        si = np.repeat(np.arange(n), cnt)
        start = np.cumsum(cnt) - cnt
        ri = lo[si] + (np.arange(tot) - np.repeat(start, cnt))
        parts.append((si, np.full(tot, bi), ri))
    if not parts:
        z = np.zeros(0, dtype=np.int64)
        return z, z, z
    si = np.concatenate([p[0] for p in parts])
    bi = np.concatenate([p[1] for p in parts])
    ri = np.concatenate([p[2] for p in parts])
    order = np.lexsort((ri, bi, si))
    return si[order], bi[order], ri[order]


def probe(stream, batches, mode, meet=0, closure_=None, swap_vals=False):
    """The probe of `stream` against a trace whose batches (each sorted by key) are `batches`, in
    trace order.  Half joins (LE / LT) without a closure emit (key, val2); JOIN without a closure
    emits R40 (key, val1, val2, time, diff); with `swap_vals` (join_core side 1) the stream value is
    val2 and the lookup value val1."""
    s = _w(stream)
    bs = [_w(b) for b in batches]
    si, bi, ri = matches(s, bs)
    allb = np.concatenate(bs) if bs else np.zeros((0, 4), dtype=np.uint64)
    off = np.cumsum([0] + [len(b) for b in bs])[:-1]
    lk = allb[off[bi] + ri] if len(si) else np.zeros((0, 4), dtype=np.uint64)
    st = s[si]
    t1, t2 = st[:, 2], lk[:, 2]
    if mode == LE:
        keep = t2 <= t1
    elif mode == LT:
        keep = t2 < t1
    else:
        keep = np.ones(len(si), dtype=bool)
    st, lk, t1, t2 = st[keep], lk[keep], t1[keep], t2[keep]
    if mode == JOIN:
        t = np.maximum(np.maximum(t1, t2), np.uint64(meet))
    else:
        t = t1
    with np.errstate(over="ignore"):
        d = st[:, 3] * lk[:, 3]
    key = st[:, 0]
    va, vb = (lk[:, 1], st[:, 1]) if swap_vals else (st[:, 1], lk[:, 1])
    if closure_ is None and mode == JOIN:
        return np.stack([key, va, vb, t, d], axis=1) if len(key) else np.zeros((0, 5), dtype=np.uint64)
    c = IDENTITY if closure_ is None else closure_
    ok, k, v = closure(c, key, va, vb)
    out = np.stack([k, v, t, d], axis=1)[ok] if len(key) else np.zeros((0, 4), dtype=np.uint64)
    return out


def half_join(stream, batches, mode, closure_=None):
    return probe(stream, batches, mode, 0, closure_)


def update_stream(batch_rows, closure_=None, skip_time=FRONTIER_EMPTY):
    """build_update_stream over a sealed batch's rows (in the batch's order)."""
    w = _w(batch_rows)
    keep = np.ones(len(w), dtype=bool) if skip_time == FRONTIER_EMPTY else w[:, 2] != np.uint64(skip_time)
    w = w[keep]
    if closure_ is None or len(w) == 0:
        return w.copy()
    ok, k, v = closure(closure_, w[:, 0], w[:, 1], 0)
    out = w[ok].copy()
    out[:, 0], out[:, 1] = k[ok], v[ok]
    return out


def half_join_chain(requests, outputs):
    """The probe chains of half_join_many / delta_first_stage_many.  requests: dicts with `batches`,
    `mode`, `closure`, `out` (an index into `outputs`) and either `stream` rows or `batch` rows plus
    `initial` / `skip_time` (the update stream formed in front of the probe).  Every output is what
    it held, then the outputs of the requests naming it, in request order."""
    outs = [_w(o).copy() for o in outputs]
    for r in requests:
        if "batch" in r:
            stream = update_stream(r["batch"], r.get("initial"), r.get("skip_time", FRONTIER_EMPTY))
        else:
            stream = r["stream"]
        got = half_join(stream, r["batches"], r["mode"], r.get("closure"))
        outs[r["out"]] = np.concatenate([outs[r["out"]], got])
    return outs


def join_core_push(batch_rows, other_batches, side, cap, closure_=None):
    """One join_core work item, consolidated (Work::process): the pushed batch against the other
    side's batches acknowledged before it, with meet = cap.  Side 1's batch probes as val2."""
    got = probe(batch_rows, other_batches, JOIN, cap, closure_, swap_vals=side == 1)
    return aref.consolidate(got)
