"""CPU restatement of the multi-column accumulable reduce (test infrastructure).

build_accumulable over several aggregates (src/compute/src/render/reduce.rs:1261-1471; the plan's
AccumulablePlan, src/compute-types/src/plan/reduce.rs:146-158): explode_one turns every input row
into (Vec<Accum>, Diff) with one Accum per aggregate (reduce.rs:1313-1334), the arrangement holds that
vector per (key, time), and reduce_abelian finalizes every aggregate of a key into ONE output row
(finalize_accum, reduce.rs:1671-1835) with the AccumulableErrorCheck per aggregate (reduce.rs:1410-1466).
An aggregate here is a "lane": COUNT and SUM of one bit-field of the input row (mzgpu_accum_lane).

The per-value arithmetic is the oracle's own: each lane's Accum comes from the oracle's explode of
the one-column kind (datum_to_accumulator and Multiply<Diff>, including the saturating 2^24 fixed
point of floats), and each lane's finalized value and flags from the oracle's finalize.  What this
module adds is the vector of Accums: the component-wise Semigroup (reduce.rs:1940-2041), IsZero of the
whole vector (reduce.rs:1905-1938) and the reduce_abelian walk over a key's times, which emits the
retraction of the key's previous row and its new row whenever the accumulated vector changes
(extensions/reduce.rs:52-107).  Rows are returned in the byte layout of include/mzgpu.h.
"""
import numpy as np

M64, M128 = (1 << 64) - 1, (1 << 128) - 1
ROW_BYTES = {1: (80, 64), 2: (128, 96), 4: (224, 144), 8: (416, 240)}  # class -> (arrangement, output)


def s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def lane_dtypes(c):
    """(arrangement, output) row dtypes of lane class c; the pad words are fields, so copies keep every byte."""
    arr_b, out_b = ROW_BYTES[c]
    lane = np.dtype([(f, "<i8") for f in ("non_nulls", "acc_lo", "acc_hi", "pos_infs", "neg_infs", "nans")])
    out_lane = np.dtype([("count", "<i8"), ("sum_lo", "<u8"), ("sum_hi", "<i8")])
    arr = np.dtype({"names": ["key", "time", "total", "lanes", "_pad"],
                    "formats": ["<u8", "<u8", "<i8", (lane, (c,)), "<i8"],
                    "offsets": [0, 8, 16, 24, 24 + 48 * c], "itemsize": arr_b})
    out = np.dtype({"names": ["key", "lanes", "flags", "time", "diff", "_pad"],
                    "formats": ["<u8", (out_lane, (c,)), "<u8", "<u8", "<i8", ("<i8", (out_b - 32 - 24 * c) // 8)],
                    "offsets": [0, 8, 8 + 24 * c, 16 + 24 * c, 24 + 24 * c, 32 + 24 * c], "itemsize": out_b})
    return arr, out


class ReduceLanes:
    """`lanes`: (kind, src, shift, bits, sign_extend) tuples (kind 0 = i64, 1 = f64; src 1 = val / val1,
    2 = val2); input rows are R32 (in_row_bytes 32) or R40 (40).  step() returns the output
    corrections, consolidated; export() the consolidated contents of the arrangement."""

    def __init__(self, oracle, lanes, in_row_bytes=32):
        self.o = oracle
        self.lanes = list(lanes)
        self.in_words = in_row_bytes // 8
        self.cls = next(c for c in (1, 2, 4, 8) if c >= len(self.lanes))
        self.arr_dtype, self.out_dtype = lane_dtypes(self.cls)
        self.pending = []  # exploded updates not yet sealed (time >= the last upper)
        self.arranged = {}  # (key, time) -> accumulated diff vector: the arrangement's contents
        self.acc = {}  # key -> accumulated diff vector over every sealed batch
        self.output = {}  # key -> finalized values of the key's current output row

    # ---- the diff vector: [total, (non_nulls, acc i128, pos_infs, neg_infs, nans) per lane]
    def _zero_vec(self):
        return [0] + [[0, 0, 0, 0, 0] for _ in self.lanes]

    @staticmethod
    def _add(a, b):
        a[0] = s64(a[0] + b[0])
        for x, y in zip(a[1:], b[1:]):
            x[0], x[1] = s64(x[0] + y[0]), (x[1] + y[1]) & M128
            x[2], x[3], x[4] = s64(x[2] + y[2]), s64(x[3] + y[3]), s64(x[4] + y[4])

    @staticmethod
    def _is_zero(v):
        return v[0] == 0 and all(not any(x) for x in v[1:])

    def _explode(self, rows):
        w = np.ascontiguousarray(rows).view(np.uint64).reshape(len(rows), self.in_words)
        key, time, diff = w[:, 0], w[:, self.in_words - 2], w[:, self.in_words - 1]
        per_lane = []
        for kind, src, shift, bits, sx in self.lanes:
            v = w[:, src] >> np.uint64(shift)
            if bits < 64:
                v = v & np.uint64((1 << bits) - 1)
                if kind == 0 and sx:
                    neg = (v >> np.uint64(bits - 1)) & np.uint64(1) == np.uint64(1)
                    v = np.where(neg, v | np.uint64(M64 ^ ((1 << bits) - 1)), v)
            r32 = np.zeros(len(rows), dtype=self.o.R32)
            r32["key"], r32["val"], r32["time"], r32["diff"] = key, v, time, diff.view(np.int64)
            per_lane.append(self.o.explode(r32, kind))
        out = []
        for i in range(len(rows)):
            vec = [int(diff[i].view(np.int64))]
            for e in per_lane:
                r = e[i]
                acc = ((int(r["acc_hi"]) & M64) << 64) | int(r["acc_lo"])
                vec.append([int(r["non_nulls"]), acc, int(r["pos_infs"]), int(r["neg_infs"]), int(r["nans"])])
            out.append((int(key[i]), int(time[i]), vec))
        return out

    def _finalize(self, key, v):
        vals, flags = [], 0
        for l, ((kind, *_), x) in enumerate(zip(self.lanes, v[1:])):
            racc = np.zeros(1, dtype=self.o.RACC)
            racc["key"], racc["total"], racc["non_nulls"] = key, v[0], x[0]
            racc["acc_lo"], racc["acc_hi"] = x[1] & M64, s64(x[1] >> 64)
            racc["pos_infs"], racc["neg_infs"], racc["nans"] = x[2], x[3], x[4]
            (f,) = self.o.finalize(racc, kind)
            vals += [int(f["count"]) & M64, int(f["sum_lo"]), int(f["sum_hi"]) & M64]
            flags |= int(f["flags"]) << (2 * l)
        return tuple(vals + [0, 0, 0] * (self.cls - len(self.lanes)) + [flags])

    def step(self, rows, upper):
        self.pending += self._explode(rows)
        batch, keep = {}, []
        for key, t, vec in self.pending:
            if t < upper:
                self._add(batch.setdefault((key, t), self._zero_vec()), vec)
            else:
                keep.append((key, t, vec))
        self.pending = keep
        corrections = {}
        for key, t in sorted(batch):
            d = batch[(key, t)]
            if self._is_zero(d):
                continue
            s = self.acc.setdefault(key, self._zero_vec())
            self._add(s, d)
            self._add(self.arranged.setdefault((key, t), self._zero_vec()), d)
            old = self.output.get(key)
            new = None if self._is_zero(s) else self._finalize(key, s)
            if old == new:
                continue
            if old is not None:
                corrections[(key, *old, t)] = corrections.get((key, *old, t), 0) - 1
            if new is not None:
                corrections[(key, *new, t)] = corrections.get((key, *new, t), 0) + 1
                self.output[key] = new
            else:
                del self.output[key]
        ow = self.out_dtype.itemsize // 8
        rows_out = [k + (d & M64,) + (0,) * (ow - len(k) - 1) for k, d in sorted(corrections.items()) if d != 0]
        return np.array(rows_out, dtype=np.uint64).reshape(-1, ow).view(self.out_dtype).reshape(-1)

    def export(self):
        aw = self.arr_dtype.itemsize // 8
        rows = []
        for (key, t), v in sorted(self.arranged.items()):
            if self._is_zero(v):
                continue
            words = [key, t, v[0] & M64]
            for x in v[1:]:
                words += [x[0] & M64, x[1] & M64, x[1] >> 64, x[2] & M64, x[3] & M64, x[4] & M64]
            rows.append(words + [0] * (aw - len(words)))
        return np.array(rows, dtype=np.uint64).reshape(-1, aw).view(self.arr_dtype).reshape(-1)
