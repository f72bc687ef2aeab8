"""CPU restatement of the hierarchical MIN / MAX reduce (test infrastructure).

build_bucketed / build_bucketed_negated_output (src/compute/src/render/reduce.rs:796-1135), the plan the
reference picks for MIN / MAX over a collection that can retract (HierarchicalPlan::Bucketed), as
include/mzgpu.h states it for mzgpu_reduce_hierarchical_new:

  1. every input row is masked to the value bits some lane reads, and the rows are consolidated by
     (key, masked val1, masked val2): the reference arranges (key, row of the aggregates' inputs);
  2. per key and time, over the live rows (times <= t, non-zero accumulated count):
       every count positive -> one output row, each lane the MIN / MAX of its field;
       some count negative  -> no output row, and the key is in the error state;
       no live row          -> no output row;
  3. output rows (key, C values, time, diff): (-old, +new) whenever the row changes; error rows
     (key, 0, time, +1 entering / -1 leaving the error state).  Both consolidated and sorted.

Everything here is Python ints, written from those rules and not from the library.
"""
import numpy as np

from monotonic_oracle import AGG_MIN, M64, dtypes, lane_value, mono_class, order_key, s64

R32 = np.dtype([("key", "<u8"), ("val", "<u8"), ("time", "<u8"), ("diff", "<i8")])


def masks(lanes):
    """the value bits the lanes read, per source word (1 = val / val1, 2 = val2)"""
    m = {1: 0, 2: 0}
    for _, src, shift, bits, _ in lanes:
        m[src] |= ((1 << bits) - 1) << shift
    return m


def key_value(lanes, live, key):
    """The per-key function over live {masked value words: count}: ("row", values), ("err", None) or None."""
    live = {v: c for v, c in live.items() if c != 0}
    if not live:
        return None
    if any(c < 0 for c in live.values()):
        return ("err", None)
    vals = []
    for lane in lanes:
        vs = [lane_value(lane, (key,) + v) for v in live]
        pick = min if lane[0] == AGG_MIN else max
        vals.append(pick(vs, key=lambda x: order_key(lane, x)))
    return ("row", tuple(vals))


class ReduceHierarchical:
    """`lanes`: (kind, src, shift, bits, sign_extend) tuples with kind AGG_MIN / AGG_MAX.  step(rows, upper)
    returns (corrections, errors); export(since) the arrangement's contents with times advanced to `since`."""

    def __init__(self, lanes, in_row_bytes=32):
        self.lanes = list(lanes)
        self.iw = in_row_bytes // 8
        self.cls = mono_class(len(self.lanes))
        _, self.out_dtype = dtypes(self.cls)
        m = masks(self.lanes)
        self.mask = (m[1], m[2]) if self.iw == 5 else (m[1],)
        self.pending = []  # input rows (words) not yet sealed
        self.arranged = {}  # (key, masked value words, time) -> count
        self.live = {}  # key -> {masked value words: count}
        self.state = {}  # key -> the per-key function's current result

    def step(self, rows, upper):
        w = np.ascontiguousarray(rows).view(np.uint64).reshape(len(rows), self.iw)
        self.pending += [[int(x) for x in r] for r in w]
        now = [r for r in self.pending if r[self.iw - 2] < upper]
        self.pending = [r for r in self.pending if r[self.iw - 2] >= upper]
        by_key = {}
        for r in now:
            v = tuple(x & m for x, m in zip(r[1 : self.iw - 2], self.mask))
            t, d = r[self.iw - 2], s64(r[self.iw - 1])
            self.arranged[(r[0], v, t)] = self.arranged.get((r[0], v, t), 0) + d
            by_key.setdefault(r[0], {}).setdefault(t, []).append((v, d))
        corr, errs = {}, {}
        for key in sorted(by_key):
            live = self.live.setdefault(key, {})
            old = self.state.get(key)
            for t in sorted(by_key[key]):
                for v, d in by_key[key][t]:
                    live[v] = live.get(v, 0) + d
                new = key_value(self.lanes, live, key)
                if old != new:
                    for res, d in ((old, -1), (new, 1)):
                        if res is not None and res[0] == "row":
                            k = (key, res[1], t)
                            corr[k] = corr.get(k, 0) + d
                    if (old is not None and old[0] == "err") != (new is not None and new[0] == "err"):
                        errs[(key, t)] = errs.get((key, t), 0) + (1 if new is not None and new[0] == "err" else -1)
                old = new
            self.state[key] = old
        pad = [0] * (self.cls - len(self.lanes))
        out = sorted((k, *v, *pad, t, d & M64) for (k, v, t), d in corr.items() if d != 0)
        out = np.array(out, dtype=np.uint64).reshape(-1, self.cls + 3).view(self.out_dtype).reshape(-1)
        err = sorted((k, 0, t, d & M64) for (k, t), d in errs.items() if d != 0)
        err = np.array(err, dtype=np.uint64).reshape(-1, 4).view(R32).reshape(-1)
        return out, err

    def export(self, since=0):
        """the arrangement: masked input rows (key, val1[, val2], time, diff), consolidated, times advanced"""
        acc = {}
        for (key, v, t), d in self.arranged.items():
            k = (key, v, max(t, since))
            acc[k] = acc.get(k, 0) + d
        rows = [[key, *v, t, d & M64] for (key, v, t), d in sorted(acc.items()) if d != 0]
        return np.array(rows, dtype=np.uint64).reshape(-1, self.iw)

    def collection(self):
        """the accumulated output: key -> values (keys in the error state or empty have none)"""
        return {k: s[1] for k, s in self.state.items() if s is not None and s[0] == "row"}

    def errors(self):
        """the keys currently in the error state"""
        return {k for k, s in self.state.items() if s is not None and s[0] == "err"}
