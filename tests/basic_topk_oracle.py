"""CPU restatement of the basic TopK plan (BasicTopKPlan, build_topk_negated_stage,
src/compute/src/render/top_k.rs:521-673) and the direct definition mzgpu_topk_basic_new is checked against.

Rows are (key, val1, val2, time, diff) tuples; R32 input has val2 = 0.  Order lanes are those of
tests/monotonic_topk_oracle.py: within a key rows compare by the encoded lane words in sequence, then by
(val1, val2) as unsigned words.

* `NegatedStage`: the reference's stage one group at a time -- `must_shrink`, negate every row, sort by
  compare_columns, skip `offset` units, take `limit` units back -- and the dataflow's input.concat(negated
  output).  Its validating branch ("Negative multiplicities in TopK") maps to the header's stand-in: the key
  has no window and one error row (key, 0, t, +1) when it enters that state, (key, 0, t, -1) when it leaves.
* `BasicTopKDefinition`: the live units of a key sorted and sliced [offset, offset + limit).

Both emit, per new time in ascending order, the change of every row's multiplicity in the window, and keep the
input arrangement (RTOPK rows) and the per-key count of rows with a negative accumulated count.
"""
from collections import Counter, defaultdict

from monotonic_topk_oracle import M64, NO_LIMIT, order_words

__all__ = ["M64", "NO_LIMIT", "NegatedStage", "BasicTopKDefinition", "negated_stage", "sliced_window"]


def negated_stage(source, limit, offset):
    """build_topk_negated_stage over one group: source {sort_key: count} (consolidated, non-zero) ->
    (negated output [(sort_key, diff)], error).  The window is source + negated output."""
    if any(c < 0 for c in source.values()):
        return [], True
    total = sum(source.values())
    must_shrink = offset > 0 or (limit != NO_LIMIT and limit < total)
    if not must_shrink:
        return [], False
    out = [(sk, -c) for sk, c in source.items()]  # negate all
    skip, left = offset, limit
    for sk in sorted(source):  # compare_columns, then the row
        c = source[sk]
        if skip > 0:  # skip `offset` units: they stay negated
            s = min(skip, c)
            skip -= s
            c -= s
        if c > 0 and left > 0:  # take `limit` units: they come back
            take = c if limit == NO_LIMIT else min(c, left)
            out.append((sk, take))
            if limit != NO_LIMIT:
                left -= take
    return out, False


def sliced_window(counts, limit, offset):
    """the definition: None when some live count is negative, else {sort_key: units in [offset, offset + limit)}
    of the key's live units in order"""
    if any(c < 0 for c in counts.values()):
        return None
    end = offset + limit
    out, pos = {}, 0
    for sk in sorted(counts):
        c = counts[sk]
        if c <= 0:
            continue
        lo, hi = max(pos, offset), min(pos + c, end)
        if hi > lo:
            out[sk] = hi - lo
        pos += c
    return out


class _Base:
    def __init__(self, lanes, limit, offset=0, in_row_bytes=32):
        self.lanes, self.limit, self.offset = list(lanes), limit, offset
        self.r40 = in_row_bytes == 40
        self.acc = defaultdict(Counter)  # key -> {sort_key: count}
        self.rows = []  # every input row as (key, o0, o1, o2, v1, v2, time, diff)

    def sk(self, v1, v2):
        return order_words(v1, v2, self.lanes) + (v1, v2)

    def window(self, key):
        raise NotImplementedError

    def step(self, rows):
        """-> (out rows (key, v1, v2, time, diff) sorted, error rows (key, 0, time, +-1) sorted)"""
        by_time = defaultdict(list)
        for r in rows:
            by_time[r[3]].append(r)
            self.rows.append((r[0],) + self.sk(r[1], r[2]) + (r[3], r[4]))
        out, errs = [], []
        for t in sorted(by_time):
            touched = {r[0] for r in by_time[t]}
            old = {k: self.window(k) for k in touched}
            for k, v1, v2, _, d in by_time[t]:
                a = self.acc[k]
                sk = self.sk(v1, v2)
                a[sk] += d
                if a[sk] == 0:
                    del a[sk]
            for k in touched:
                new = self.window(k)
                if (old[k] is None) != (new is None):
                    errs.append((k, 0, t, 1 if new is None else -1))
                a, b = old[k] or {}, new or {}
                for sk in set(a) | set(b):
                    d = b.get(sk, 0) - a.get(sk, 0)
                    if d:
                        out.append((k, sk[3], sk[4], t, d))
        return sorted(out), sorted(errs)

    def input_rows(self, since=0):
        """the input arrangement's RTOPK rows (key, o0, o1, o2, v1, v2, time, diff), times advanced to `since`,
        consolidated and sorted"""
        acc = Counter()
        for r in self.rows:
            acc[r[:6] + (max(r[6], since),)] += r[7]
        return sorted(k + (d,) for k, d in acc.items() if d != 0)

    def negatives(self):
        """{key: number of its rows with a negative accumulated count}, keys with none left out"""
        out = {}
        for k, a in self.acc.items():
            n = sum(1 for c in a.values() if c < 0)
            if n:
                out[k] = n
        return out


class NegatedStage(_Base):
    """the reference's stage: window = input + negated output; the validating branch is the error state"""

    def window(self, key):
        src = self.acc.get(key, {})
        neg, error = negated_stage(src, self.limit, self.offset)
        if error:
            return None
        w = Counter(src)
        for sk, d in neg:
            w[sk] += d
        return {sk: c for sk, c in w.items() if c != 0}


class BasicTopKDefinition(_Base):
    """the live units sorted and sliced [offset, offset + limit)"""

    def window(self, key):
        return sliced_window(self.acc.get(key, {}), self.limit, self.offset)
