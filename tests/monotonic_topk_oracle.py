"""CPU restatement of the monotonic TopK plans (MonotonicTop1 / MonotonicTopK,
src/compute/src/render/top_k.rs:102-214), and the direct definition the operator is checked against.

Rows are (key, val1, val2, time, diff) tuples; R32 input has val2 = 0.  An order lane is
(src, shift, bits, sign_extend, descending) with src 1 = val1, 2 = val2.  Within a key rows compare by the
encoded lane words in sequence, then by (val1, val2) as unsigned words (the fixed-width stand-in for
compare_columns(order_key, l, r, || l.cmp(r))).

* `TopKDefinition`: the window at every time is the first `limit` units per key of the accumulated kept
  input; each activation emits, per new time in ascending order, the change of every row's multiplicity in
  the window.  Its `window()` is what the operator's arrangement holds after compaction.
* `TopKRestatement`: the reference's steps one by one -- consolidate_named_if, ensure_monotonic
  (operator.rs:425-456), intra-timestamp thinning (render_intra_ts_thinning / TopKBatch, top_k.rs:675-850,
  with its compaction and its cut inside the last record), the topk stage with offset 0 over the thinned
  input plus the feedback, and the delayed feedback that retracts the input rows that fell out of the
  window (top_k.rs:171-213).
"""
from collections import Counter, defaultdict

M64 = (1 << 64) - 1
NO_LIMIT = (1 << 63) - 1


def field(v1, v2, lane):
    src, shift, bits = lane[0], lane[1], lane[2]
    w = v1 if src == 1 else v2
    w >>= shift
    if bits < 64:
        w &= (1 << bits) - 1
    return w


def order_words(v1, v2, lanes):
    """the window row's o0..o2: field (sign-extended when signed) ^ 2^63 if signed, complemented if
    descending; unused words 0"""
    o = []
    for lane in lanes:
        v = field(v1, v2, lane)
        bits, sx, desc = lane[2], lane[3], lane[4]
        if sx and bits < 64 and (v >> (bits - 1)) & 1:
            v |= (M64 << bits) & M64
        if sx:
            v ^= 1 << 63
        if desc:
            v ^= M64
        o.append(v)
    return tuple(o + [0] * (3 - len(o)))


def consolidate(rows):
    acc = Counter()
    for k, v1, v2, t, d in rows:
        acc[(k, v1, v2, t)] += d
    return [(k, v1, v2, t, d) for (k, v1, v2, t), d in sorted(acc.items()) if d != 0]


def ensure_monotonic(rows):
    """(kept rows, errors): a row is kept iff diff > 0; every other row is one error at its time"""
    kept, errs = [], Counter()
    for r in rows:
        if r[4] > 0:
            kept.append(r)
        else:
            errs[r[3]] += 1
    return kept, sorted(errs.items())


def top_units(pairs, limit):
    """pairs: {sort_key: count} of one key -> {sort_key: count in the first `limit` units}"""
    out, used = {}, 0
    for sk in sorted(pairs):
        if used >= limit:
            break
        c = pairs[sk]
        if c <= 0:
            continue
        take = min(c, limit - used)
        out[sk] = take
        used += take
    return out


def _window(acc, limit):
    return {k: top_units(p, limit) for k, p in acc.items()}


def _diff(old, new):
    """(key, sort_key, change) for every row whose window multiplicity changed"""
    out = []
    for k in set(old) | set(new):
        a, b = old.get(k, {}), new.get(k, {})
        for sk in set(a) | set(b):
            d = b.get(sk, 0) - a.get(sk, 0)
            if d:
                out.append((k, sk, d))
    return out


class TopKDefinition:
    def __init__(self, lanes, limit, in_row_bytes=32, must_consolidate=False):
        self.lanes, self.limit, self.r40, self.must = list(lanes), limit, in_row_bytes == 40, must_consolidate
        self.acc = defaultdict(Counter)  # key -> {(o0, o1, o2, v1, v2): units}
        self.changes = []  # (key, o0, o1, o2, v1, v2, time, diff): what the window arrangement receives

    def sk(self, v1, v2):
        return order_words(v1, v2, self.lanes) + (v1, v2)

    def step(self, rows):
        """-> (out rows (key, v1, v2, time, diff) sorted, errors [(time, count)] sorted)"""
        rows = consolidate(rows) if self.must else list(rows)
        kept, errs = ensure_monotonic(rows)
        out = []
        by_time = defaultdict(list)
        for r in kept:
            by_time[r[3]].append(r)
        for t in sorted(by_time):
            touched = {r[0] for r in by_time[t]}
            old = _window({k: self.acc[k] for k in touched}, self.limit)
            for k, v1, v2, _, d in by_time[t]:
                self.acc[k][self.sk(v1, v2)] += d
            new = _window({k: self.acc[k] for k in touched}, self.limit)
            for k, sk, d in _diff(old, new):
                out.append((k, sk[3], sk[4], t, d))
                self.changes.append((k,) + sk + (t, d))
        return sorted(out), errs

    def window(self, since=None):
        """the window arrangement's rows, times advanced to `since` and consolidated (since=None: the live
        window itself, one row per window row at time 0 -- what compaction to any frontier leaves when every
        time is below it)"""
        acc = Counter()
        for c in self.changes:
            t = c[6] if since is None or c[6] >= since else since
            acc[c[:6] + (0 if since is None else t,)] += c[7]
        return sorted(k + (d,) for k, d in acc.items() if d != 0)


class TopKRestatement:
    """the reference's dataflow, one time at a time"""

    def __init__(self, lanes, limit, in_row_bytes=32, must_consolidate=False):
        self.lanes, self.limit, self.must = list(lanes), limit, must_consolidate
        self.arranged = defaultdict(Counter)  # the topk stage's input: thinned input + feedback
        self.output = {}  # the topk stage's output collection
        self.pending_feedback = []  # retractions produced at the previous time, applied at the next one

    def sk(self, v1, v2):
        return order_words(v1, v2, self.lanes) + (v1, v2)

    def thin(self, rows):
        """TopKBatch per key at one time: records sorted by the order, compacted, and cut at `limit` units;
        the last record kept loses the units past the limit"""
        per_key = defaultdict(list)
        for k, v1, v2, _, d in rows:
            per_key[k].append((self.sk(v1, v2), d))
        out = []
        for k, recs in per_key.items():
            recs.sort()
            merged = []
            for sk, d in recs:  # compaction: equal records fold
                if merged and merged[-1][0] == sk:
                    merged[-1] = (sk, merged[-1][1] + d)
                else:
                    merged.append((sk, d))
            used = 0
            for sk, d in merged:
                if used >= self.limit:
                    break
                take = min(d, self.limit - used)
                out.append((k, sk, take))
                used += take
        return out

    def step(self, rows):
        rows = consolidate(rows) if self.must else list(rows)
        kept, errs = ensure_monotonic(rows)
        by_time = defaultdict(list)
        for r in kept:
            by_time[r[3]].append(r)
        out = []
        for t in sorted(by_time):
            for k, sk, d in self.pending_feedback:  # the delayed feedback lands at a later time
                self.arranged[k][sk] += d
            self.pending_feedback = []
            touched = set()
            for k, sk, d in self.thin(by_time[t]):
                self.arranged[k][sk] += d
                touched.add(k)
            new = {k: top_units(self.arranged[k], self.limit) for k in touched}
            old = {k: self.output.get(k, {}) for k in touched}
            for k, sk, d in _diff(old, new):
                out.append((k, sk[3], sk[4], t, d))
            for k in touched:
                self.output[k] = new[k]
                # feedback: retract every arranged unit outside the window
                for sk, c in self.arranged[k].items():
                    extra = c - new[k].get(sk, 0)
                    if extra:
                        self.pending_feedback.append((k, sk, -extra))
        return sorted(out), errs
