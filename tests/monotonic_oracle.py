"""CPU restatement of the monotonic MIN / MAX reduce (test infrastructure).

build_monotonic (src/compute/src/render/reduce.rs:1138-1253), which the planner uses for append-only
inputs instead of the bucket tree (HierarchicalPlan::Monotonic, src/compute-types/src/plan/reduce.rs:160-250):

  1. consolidate_named_if(must_consolidate): the (key, aggregate inputs) rows are consolidated by
     (data, time) first (reduce.rs:1152-1167), so a +1 / -1 pair at one time cancels.
  2. ensure_monotonic (src/timely-util/src/operator.rs:425-456): a row is kept iff diff > 0; every other
     row is one error (t, +1) in the error collection, whatever its diff.
  3. explode: the kept row's values move into the diff as one Min / Max monoid per aggregate
     (reduce.rs:1182-1190, get_monoid :2297-2332); multiplying by a positive diff is the identity.
  4. arrange with plus_equals = per-aggregate min / max (:2193-2233); IsZero is always false (:2235-2244).
  5. reduce_abelian emits (key, values) per key: (-old, +new) on every change, +new for a key's first row.

Everything here is Python ints, written from those rules and not from the library.  Rows come back in
the byte layouts of include/mzgpu.h: output (key, C values, time, diff), arrangement (key, time, C lane
words [, 4 pad words]) with lane word = value ^ 2^63 (signed lanes), complemented for MIN.
"""
import numpy as np

M64 = (1 << 64) - 1
AGG_MIN, AGG_MAX = 4, 5
ROW_BYTES = {4: (48, 56), 8: (112, 88)}  # class -> (arrangement, output)


def mono_class(n_lanes):
    return 4 if n_lanes <= 4 else 8


def dtypes(c):
    arr_b, out_b = ROW_BYTES[c]
    pad = (arr_b - 16 - 8 * c) // 8
    arr = [("key", "<u8"), ("time", "<u8"), ("lanes", "<u8", (c,))] + ([("_pad", "<u8", (pad,))] if pad else [])
    out = [("key", "<u8"), ("vals", "<u8", (c,)), ("time", "<u8"), ("diff", "<i8")]
    return np.dtype(arr), np.dtype(out)


def lane_value(lane, words):
    """(value as an unsigned 64-bit int, the order key as a Python int) of one lane of one row."""
    kind, src, shift, bits, sx = lane
    v = (words[src] >> shift) & ((1 << bits) - 1)
    if sx and bits < 64 and (v >> (bits - 1)) & 1:
        v |= M64 ^ ((1 << bits) - 1)
    return v


def order_key(lane, v):
    """the value's place in the lane's order: signed lanes compare as i64, unsigned as u64"""
    return v - (1 << 64) if lane[4] and v >> 63 else v


class ReduceMonotonic:
    """`lanes`: (kind, src, shift, bits, sign_extend) tuples with kind AGG_MIN / AGG_MAX (src 1 = val / val1,
    2 = val2).  step(rows, upper) returns (corrections, errors), export(since) the arrangement's contents
    with times advanced to `since`."""

    def __init__(self, lanes, in_row_bytes=32, must_consolidate=False):
        self.lanes = list(lanes)
        self.iw = in_row_bytes // 8
        self.must_consolidate = must_consolidate
        self.cls = mono_class(len(self.lanes))
        self.arr_dtype, self.out_dtype = dtypes(self.cls)
        self.pending = []  # input rows (words) not yet sealed
        self.arranged = {}  # (key, time) -> accumulated values (natural values, one per lane)
        self.acc = {}  # key -> accumulated values over every sealed batch
        self.output = {}  # key -> the key's current output values

    def _plus(self, a, b):
        if a is None:
            return list(b)
        out = []
        for lane, x, y in zip(self.lanes, a, b):
            kx, ky = order_key(lane, x), order_key(lane, y)
            pick_y = ky < kx if lane[0] == AGG_MIN else ky > kx
            out.append(y if pick_y else x)
        return out

    def _data(self, w):
        """consolidate_named_if's data: the key and the lanes' inputs"""
        return (w[0],) + tuple(lane_value(l, w) for l in self.lanes)

    def step(self, rows, upper):
        w = np.ascontiguousarray(rows).view(np.uint64).reshape(len(rows), self.iw)
        self.pending += [[int(x) for x in r] for r in w]
        now = [r for r in self.pending if r[self.iw - 2] < upper]
        self.pending = [r for r in self.pending if r[self.iw - 2] >= upper]
        # 1. (data, time, diff) updates, consolidated if asked
        upd = [(self._data(r), r[self.iw - 2], s64(r[self.iw - 1])) for r in now]
        if self.must_consolidate:
            acc = {}
            for d, t, x in upd:
                acc[(d, t)] = acc.get((d, t), 0) + x
            upd = [(d, t, x) for (d, t), x in acc.items() if x != 0]
        # 2. ensure_monotonic
        errs = {}
        batch = {}
        for d, t, x in upd:
            if x <= 0:
                errs[t] = errs.get(t, 0) + 1
                continue
            # 3-4. explode and arrange
            batch[(d[0], t)] = self._plus(batch.get((d[0], t)), d[1:])
        # 5. reduce_abelian
        corr = {}
        for key, t in sorted(batch):
            v = batch[(key, t)]
            self.arranged[(key, t)] = self._plus(self.arranged.get((key, t)), v)
            old = self.acc.get(key)
            new = self._plus(old, v)
            self.acc[key] = new
            if old == new:
                continue
            if old is not None:
                corr[(key, *old, t)] = corr.get((key, *old, t), 0) - 1
            corr[(key, *new, t)] = corr.get((key, *new, t), 0) + 1
            self.output[key] = new
        pad = [0] * (self.cls - len(self.lanes))
        out = [(k[0], *k[1:-1], *pad, k[-1], d & M64) for k, d in corr.items() if d != 0]
        out.sort(key=lambda r: r[:-1])
        out = np.array(out, dtype=np.uint64).reshape(-1, self.cls + 3).view(self.out_dtype).reshape(-1)
        err = np.array(sorted(errs.items()), dtype=np.uint64).reshape(-1, 2)
        err = err.view(np.dtype([("key", "<u8"), ("diff", "<i8")])).reshape(-1)
        return out, err

    def encode(self, vals):
        words = []
        for lane, v in zip(self.lanes, vals):
            x = v ^ (1 << 63) if lane[4] else v
            words.append(x ^ M64 if lane[0] == AGG_MIN else x)
        return words + [0] * (self.cls - len(self.lanes))

    def export(self, since=0):
        acc = {}
        for (key, t), v in self.arranged.items():
            k = (key, max(t, since))
            acc[k] = self._plus(acc.get(k), v)
        aw = self.arr_dtype.itemsize // 8
        rows = [[key, t] + self.encode(v) for (key, t), v in sorted(acc.items())]
        rows = [r + [0] * (aw - len(r)) for r in rows]
        return np.array(rows, dtype=np.uint64).reshape(-1, aw).view(self.arr_dtype).reshape(-1)

    def collection(self):
        """the accumulated output: key -> values"""
        return {k: tuple(v) for k, v in self.output.items()}


def s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x
