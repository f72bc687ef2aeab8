"""CPU restatement of the distinct lanes of the multi-column accumulable reduce (test infrastructure).

build_accumulable's distinct_aggrs (src/compute/src/render/reduce.rs:1338-1373): for a distinct
aggregate over datum i the input is mapped to ((key, value_i), ()), arranged ("Arranged Accumulable
Distinct"), and reduce_abelian with logic `t.push(((), Diff::ONE))` emits the pair while its accumulated
multiplicity is non-zero (negative included).  Each such output update is explode_one'd into a diff
vector whose Diff is the update's +-1 and whose only non-zero Accum is this aggregate's, from
datum_to_accumulator(value); those vectors are concatenated with the simple_aggrs explode (:1310-1336),
which exists only when there is at least one plain aggregate, before the one ArrangeAccumulable
arrangement.  So a key's total is [a plain lane exists] * (sum of its input diffs) + the number of
present pairs over all distinct lanes.

ReduceLanesDistinct extends lanes_oracle.ReduceLanes: a lane whose kind carries ACCUM_DISTINCT (0x100)
keeps a (key, value) -> multiplicity map; each step replays the lane's new pair updates in time order and
turns presence changes into diff vectors.  The arrangement, the reduce_abelian walk and finalize are the
base class's, unchanged.
"""
import numpy as np
from lanes_oracle import M64, ReduceLanes, s64

ACCUM_DISTINCT = 0x100


class ReduceLanesDistinct(ReduceLanes):
    """`lanes` as for ReduceLanes, a kind may carry ACCUM_DISTINCT.  pair_export(l) returns the consolidated
    contents of distinct lane l's pair arrangement as R32 rows."""

    def __init__(self, oracle, lanes, in_row_bytes=32):
        lanes = list(lanes)
        self.distinct = [bool(l[0] & ACCUM_DISTINCT) for l in lanes]
        super().__init__(oracle, [(l[0] & ~ACCUM_DISTINCT, *l[1:]) for l in lanes], in_row_bytes)
        self.plain = not all(self.distinct)
        self.pair_pending = []  # (lane, key, value, time, diff) not sealed yet
        self.pair_mult = {l: {} for l, d in enumerate(self.distinct) if d}  # (key, value) -> multiplicity
        self.pair_arranged = {l: {} for l in self.pair_mult}  # (key, value, time) -> accumulated diff
        self._upper = 0

    def step(self, rows, upper):
        self._upper = upper
        return super().step(rows, upper)

    def _values(self, rows, lane):
        kind, src, shift, bits, sx = self.lanes[lane]
        w = np.ascontiguousarray(rows).view(np.uint64).reshape(len(rows), self.in_words)
        v = w[:, src] >> np.uint64(shift)
        if bits < 64:
            v = v & np.uint64((1 << bits) - 1)
            if sx:
                neg = (v >> np.uint64(bits - 1)) & np.uint64(1) == np.uint64(1)
                v = np.where(neg, v | np.uint64(M64 ^ ((1 << bits) - 1)), v)
        return w, v

    def _explode(self, rows):
        out = super()._explode(rows) if self.plain else []
        for _, _, vec in out:
            for l, d in enumerate(self.distinct):
                if d:
                    vec[1 + l] = [0, 0, 0, 0, 0]
        return out + self._presence(rows)

    def _presence(self, rows):
        """The new pair updates of every distinct lane, sealed at the current upper: their presence changes
        as exploded (key, time, diff vector) entries."""
        for l in self.pair_mult:
            w, v = self._values(rows, l)
            t, d = w[:, self.in_words - 2], w[:, self.in_words - 1]
            self.pair_pending += [(l, int(w[i, 0]), int(v[i]), int(t[i]), s64(int(d[i]))) for i in range(len(rows))]
        batch, keep = {}, []
        for l, key, val, t, d in self.pair_pending:
            if t < self._upper:
                batch[(l, key, val, t)] = s64(batch.get((l, key, val, t), 0) + d)
            else:
                keep.append((l, key, val, t, d))
        self.pair_pending = keep
        changes = []  # (lane, key, value, time, +-1)
        for (l, key, val, t), d in sorted(batch.items()):
            if d == 0:
                continue
            arr = self.pair_arranged[l]
            arr[(key, val, t)] = s64(arr.get((key, val, t), 0) + d)
            m = self.pair_mult[l].get((key, val), 0)
            m2 = s64(m + d)
            self.pair_mult[l][(key, val)] = m2
            if (m != 0) != (m2 != 0):
                changes.append((l, key, val, t, 1 if m2 != 0 else -1))
        out = []
        for l, key, val, t, s in changes:
            r32 = np.zeros(1, dtype=self.o.R32)
            r32["key"], r32["val"], r32["time"], r32["diff"] = key, val, t, s
            (e,) = self.o.explode(r32, self.lanes[l][0])
            vec = self._zero_vec()
            vec[0] = s
            acc = ((int(e["acc_hi"]) & M64) << 64) | int(e["acc_lo"])
            vec[1 + l] = [int(e["non_nulls"]), acc, int(e["pos_infs"]), int(e["neg_infs"]), int(e["nans"])]
            out.append((key, t, vec))
        return out

    def pair_export(self, lane):
        rows = [(k, v, t, d & M64) for (k, v, t), d in sorted(self.pair_arranged[lane].items()) if d != 0]
        return np.array(rows, dtype=np.uint64).reshape(-1, 4).view(self.o.R32).reshape(-1)
