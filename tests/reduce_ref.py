"""Plain reference of the one-column reduce operator (mzgpu_reduce_new / mzgpu_topk_new: agg kinds 0-6),
written from the header's definitions (include/mzgpu.h, mzgpu_racc / mzgpu_rout and the MZGPU_AGG_*
comments) in Python ints, for the tests.

One class per operator: `step(rows, upper)` takes (key, val, time, diff) R32 updates and returns the
activation's mzgpu_rout rows as an (n, 8) u64 matrix, consolidated and ordered as consolidate() orders
them (the first six words compared as unsigned, in order); `export(since)` returns the arrangement's
contents with times advanced to `since` (as Spine.export does).

Arithmetic:
  * diffs, totals, counts and the float counters wrap at 64 bits; the SUM accumulator wraps at 128.
  * f64 values: the accumulator of x is `x * 2.0**24` (an IEEE double product) converted as Rust's
    `as i128` converts: NaN -> 0, truncation toward zero, saturation at -2^127 / 2^127 - 1.  +-inf and
    NaN are counted in their own counters instead.  The SUM is float(accumulator) (round to nearest,
    ties to even) divided by 2^24.
  * the batcher holds updates at times >= upper until a later activation ships them.

Outputs: corrections are emitted at every distinct time of a changed key, in time order, as
(-old, +new) whenever the finalized row changes."""
import struct

import numpy as np

import arrangement_ref as aref

M64 = (1 << 64) - 1
M128 = (1 << 128) - 1
FE = aref.FRONTIER_EMPTY
SCALE = 2.0**24
I128_MAX, I128_MIN = (1 << 127) - 1, -(1 << 127)
NAN_BITS, PINF_BITS, NINF_BITS = 0x7FF8000000000000, 0x7FF0000000000000, 0xFFF0000000000000
I64, F64, DISTINCT, THRESHOLD, MIN, MAX, TOPK = range(7)


def s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def s128(x):
    x &= M128
    return x - (1 << 128) if x >> 127 else x


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits & M64))[0]


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def as_i128(x):
    """Rust `x as i128` for a double."""
    if x != x:
        return 0
    if x >= 2.0**127:
        return I128_MAX
    if x <= -(2.0**127):
        return I128_MIN
    return int(x)  # truncates toward zero


def accum_f64(x):
    """The SUM accumulator of one float64 value (before the diff multiplies it)."""
    return as_i128(x * SCALE)


def sum_f64(acc):
    """The finite SUM of a float64 accumulator: float(i128), round to nearest even, / 2^24."""
    return float(s128(acc)) / SCALE


def rows_of(rows):
    """(key, val, time, diff) tuples of Python ints (diff signed) from an R32 array or (n, 4) words."""
    if isinstance(rows, list):
        return [(int(k), int(v), int(t), s64(int(d))) for k, v, t, d in rows]
    return [(k, v, t, s64(d)) for k, v, t, d in aref.words(rows, 32).tolist()]


def out_words(rows):
    """(key, count, sum_lo, sum_hi, flags, time, diff) tuples -> consolidated (n, 8) u64 rows."""
    w = np.zeros((len(rows), 8), dtype=np.uint64)
    if rows:
        w[:, :7] = np.array([[x & M64 for x in r] for r in rows], dtype=np.uint64)
    return aref.consolidate(w)


class _Op:
    """The batcher and the arrangement's history, shared by every kind."""

    def __init__(self):
        self.stash = []
        self.hist = {}  # arrangement key (key, time) or (key, val, time) -> summed update

    def _ship(self, rows, upper):
        self.stash.extend(rows_of(rows))
        if upper == FE:
            ship, self.stash = self.stash, []
        else:
            ship = [r for r in self.stash if r[2] < upper]
            self.stash = [r for r in self.stash if r[2] >= upper]
        return ship


# ------------------------------------------------------------------ kinds 0-3
def explode(kind, val, diff):
    """The diff vector (total, non_nulls, acc, pos_infs, neg_infs, nans) of one update."""
    if kind in (DISTINCT, THRESHOLD):
        return (diff, 0, 0, 0, 0, 0)
    if kind == I64:
        return (diff, diff, s64(val) * diff, 0, 0, 0)
    x = f64(val)
    if x != x:
        return (diff, diff, 0, 0, 0, diff)
    if x == float("inf"):
        return (diff, diff, 0, diff, 0, 0)
    if x == float("-inf"):
        return (diff, diff, 0, 0, diff, 0)
    return (diff, diff, accum_f64(x) * diff, 0, 0, 0)


def vadd(a, b):
    return (s64(a[0] + b[0]), s64(a[1] + b[1]), s128(a[2] + b[2]), s64(a[3] + b[3]), s64(a[4] + b[4]), s64(a[5] + b[5]))


ZERO = (0, 0, 0, 0, 0, 0)


def finalize(kind, S):
    """(count, sum_lo, sum_hi, flags) of a non-zero accumulation (mzgpu_rout)."""
    total, nn, acc, pinf, ninf, nans = S
    if kind == DISTINCT:
        return (1, 0, 0, 2 if total < 0 else 0)
    accum_zero = S[1:] == ZERO[1:]
    flags = (1 if total > 0 and accum_zero else 0) | (2 if total == 0 and not accum_zero else 0)
    if kind == F64:
        if nans > 0 or (pinf > 0 and ninf > 0):
            lo = NAN_BITS
        elif pinf > 0:
            lo = PINF_BITS
        elif ninf > 0:
            lo = NINF_BITS
        else:
            lo = bits(sum_f64(acc))
        hi = 0
    else:
        lo, hi = acc & M64, s64(acc >> 64)
    if flags & 1:
        lo = hi = 0
    return (nn, lo, hi, flags)


class Reduce(_Op):
    """mzgpu_reduce_new(kind) for kinds 0-3 (COUNT/SUM i64, COUNT/SUM f64, DISTINCT, threshold)."""

    def __init__(self, kind):
        super().__init__()
        assert kind in (I64, F64, DISTINCT, THRESHOLD)
        self.kind = kind
        self.acc = {}  # key -> accumulated diff vector over every shipped update

    def step(self, rows, upper):
        new = {}
        for k, v, t, d in self._ship(rows, upper):
            kt = new.setdefault(k, {})
            kt[t] = vadd(kt.get(t, ZERO), explode(self.kind, v, d))
        out = []
        for k in sorted(new):
            S = self.acc.get(k, ZERO)
            for t in sorted(new[k]):
                S2 = vadd(S, new[k][t])
                self.hist[(k, t)] = vadd(self.hist.get((k, t), ZERO), new[k][t])
                if self.kind == THRESHOLD:
                    m1, m2 = max(S[0], 0), max(S2[0], 0)
                    if m1 != m2:
                        out.append((k, 0, 0, 0, 0, t, m2 - m1))
                else:
                    old = finalize(self.kind, S) if S != ZERO else None
                    fresh = finalize(self.kind, S2) if S2 != ZERO else None
                    if old != fresh:
                        if old is not None:
                            out.append((k, *old, t, -1))
                        if fresh is not None:
                            out.append((k, *fresh, t, 1))
                S = S2
            self.acc[k] = S
        return out_words(out)

    def export(self, since=0):
        """The arrangement's mzgpu_racc rows: (key, time, total, non_nulls, acc_lo, acc_hi, pos_infs,
        neg_infs, nans, pad), consolidated at `since`."""
        acc = {}
        for (k, t), d in self.hist.items():
            t = t if since == FE else max(t, since)
            acc[(k, t)] = vadd(acc.get((k, t), ZERO), d)
        rows = [(k, t, d[0], d[1], d[2] & M64, d[2] >> 64, d[3], d[4], d[5], 0) for (k, t), d in sorted(acc.items()) if d != ZERO]
        w = np.zeros((len(rows), 10), dtype=np.uint64)
        if rows:
            w[:] = np.array([[x & M64 for x in r] for r in rows], dtype=np.uint64)
        return w


# ------------------------------------------------------------------ kinds 4-6
class _Values(_Op):
    """MIN / MAX / TopK: the arrangement holds the (key, value) updates themselves."""

    def __init__(self):
        super().__init__()
        self.counts = {}  # key -> {value: accumulated count}

    def evaluate(self, counts):
        raise NotImplementedError

    def changes(self, k, old, fresh, t):
        raise NotImplementedError

    def step(self, rows, upper):
        new = {}
        for k, v, t, d in self._ship(rows, upper):
            new.setdefault(k, {}).setdefault(t, []).append((v, d))
            self.hist[(k, v, t)] = s64(self.hist.get((k, v, t), 0) + d)
        out = []
        for k in sorted(new):
            c = self.counts.setdefault(k, {})
            old = self.evaluate(c)
            for t in sorted(new[k]):
                for v, d in new[k][t]:
                    c[v] = s64(c.get(v, 0) + d)
                fresh = self.evaluate(c)
                out.extend(self.changes(k, old, fresh, t))
                old = fresh
        return out_words(out)

    def live(self, k):
        """The key's values with a non-zero accumulated count."""
        return {v: n for v, n in self.counts.get(k, {}).items() if n != 0}

    def export(self, since=0):
        """The arrangement's R32 rows (key, val, time, diff), consolidated at `since`."""
        acc = {}
        for (k, v, t), d in self.hist.items():
            t = t if since == FE else max(t, since)
            acc[(k, v, t)] = s64(acc.get((k, v, t), 0) + d)
        rows = [(k, v, t, d & M64) for (k, v, t), d in sorted(acc.items()) if d != 0]
        return np.array(rows, dtype=np.uint64).reshape(-1, 4)


class MinMax(_Values):
    """mzgpu_reduce_new(MZGPU_AGG_MIN / MZGPU_AGG_MAX): values compare as u64; any negative count of a
    live value is the error row (flags bit 1, aggregate 0)."""

    def __init__(self, kind):
        super().__init__()
        assert kind in (MIN, MAX)
        self.kind = kind

    def evaluate(self, counts):
        live = {v: n for v, n in counts.items() if n != 0}
        if not live:
            return None
        if any(n < 0 for n in live.values()):
            return (0, 0, 0, 2)
        return (0, min(live) if self.kind == MIN else max(live), 0, 0)

    def changes(self, k, old, fresh, t):
        if old == fresh:
            return []
        return ([(k, *old, t, -1)] if old is not None else []) + ([(k, *fresh, t, 1)] if fresh is not None else [])


class TopK(_Values):
    """mzgpu_topk_new(limit, offset, descending): the live values in order, `offset` copies skipped and
    at most `limit` copies kept (None: no limit); any negative count is the error row (diff +-1).  Rows
    carry the value in sum_lo and the change of its multiplicity inside the window as the diff."""

    def __init__(self, limit, offset=0, descending=False):
        super().__init__()
        self.limit, self.offset, self.desc = (None if limit is None or limit < 0 else limit), offset, descending

    def window(self, counts):
        """(error, {value: multiplicity inside the window})."""
        live = {v: n for v, n in counts.items() if n != 0}
        if any(n < 0 for n in live.values()):
            return True, {}
        skip, left, win = self.offset, self.limit, {}
        for v in sorted(live, reverse=self.desc):
            n = live[v]
            s = min(skip, n)
            skip, n = skip - s, n - s
            if left is not None:
                n = min(n, left)
                left -= n
            if n > 0:
                win[v] = n
            if left == 0:
                break
        return False, win

    evaluate = window

    def changes(self, k, old, fresh, t):
        out = []
        if old[0] != fresh[0]:
            out.append((k, 0, 0, 0, 2, t, 1 if fresh[0] else -1))
        for v in set(old[1]) | set(fresh[1]):
            d = fresh[1].get(v, 0) - old[1].get(v, 0)
            if d:
                out.append((k, 0, v, 0, 0, t, d))
        return out


def make(kind, limit=None, offset=0, descending=False):
    if kind == TOPK:
        return TopK(limit, offset, descending)
    if kind in (MIN, MAX):
        return MinMax(kind)
    return Reduce(kind)
