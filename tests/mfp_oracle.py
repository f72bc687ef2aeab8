"""Plain-Python restatement of the temporal filter (mzgpu_mfp_new, include/mzgpu.h).

- `bounds(temporal)`: MfpPlan::create_from's lower / upper bound lists (src/expr/src/linear.rs:1772-1804).
- `evaluate(plan, row, time, diff, until)`: MfpPlan::evaluate (linear.rs:1865-1971), quirks included.
- `BucketChain`: insert / peel / restore of src/timely-util/src/temporal.rs:59-211, over lists of rows.
- `Operator`: the step contract (what is released at each upper, what is held).
- `direct(...)`: the definition: at a valid time t, the input rows accumulated to t that pass the
  predicates with lower <= t < upper.
"""
from collections import defaultdict

U64 = 2**64
MAX = U64 - 1
EMPTY = MAX
HOP_COL, HOP_INT, HOP_ADD, HOP_SUB, HOP_MUL, HOP_DIV, HOP_CMP, HOP_AND, HOP_OR, HOP_NOT = 1, 4, 7, 8, 9, 10, 11, 12, 13, 14
HOP_COL_MZTS, HOP_INT_TO_MZTS, HOP_COL_TS, HOP_COL_DATE = 15, 16, 17, 18
HOP_TS_ADD_IV, HOP_TS_TO_MZTS, HOP_DATE_TO_MZTS = 19, 20, 21
EQ, NE, LT, LE, GT, GE = 0, 1, 2, 3, 4, 5
E_DIV0, E_OVF, E_I32, E_I64, E_MZTS_RANGE, E_STEP, E_TS_RANGE = 1, 2, 3, 4, 5, 6, 7
TS_LOW_US, TS_HIGH_US = -210863692800000000, 8210266876799999999


def s64(x):
    x &= U64 - 1
    return x - U64 if x >= 2**63 else x


def run(ops, consts, w):
    """Returns (err, payload, value)."""
    st = []
    for (code, arg, shift, bits, sx, k) in ops:
        if code in (HOP_COL, HOP_COL_TS, HOP_COL_DATE):
            a = (w[arg] >> shift) & ((1 << bits) - 1)
            if sx and (a >> (bits - 1)) & 1:
                a -= 1 << bits
            st.append([0, 0, s64(a) if code != HOP_COL or sx or bits == 64 else a])
        elif code == HOP_COL_MZTS:
            st.append([0, 0, (w[arg] >> shift) & ((1 << bits) - 1)])
        elif code == HOP_INT:
            st.append([0, 0, s64(consts[k][0])])
        elif code == HOP_NOT:
            if st[-1][0] == 0:
                st[-1][2] ^= 1
        elif code in (HOP_INT_TO_MZTS, HOP_TS_TO_MZTS, HOP_DATE_TO_MZTS, HOP_TS_ADD_IV):
            e, p, a = st[-1]
            if e:
                continue
            if code == HOP_TS_ADD_IV:
                lo, hi = consts[k]
                days = (hi & 0xFFFFFFFF) - (1 << 32) if hi & 0x80000000 else hi & 0xFFFFFFFF
                r = a + days * 86400000000 + s64(lo)
                st[-1] = [E_TS_RANGE, 0, a] if not (TS_LOW_US <= r <= TS_HIGH_US) else [0, 0, r]
            else:
                r = a if code == HOP_INT_TO_MZTS else (a // 1000 if code == HOP_TS_TO_MZTS else a * 86400000)
                st[-1] = [E_MZTS_RANGE, a % U64, a] if r < 0 else [0, 0, r]
        else:
            y = st.pop()
            x = st[-1]
            if code in (HOP_AND, HOP_OR):
                dom = 0 if code == HOP_AND else 1
                if (x[0] == 0 and x[2] == dom) or (y[0] == 0 and y[2] == dom):
                    st[-1] = [0, 0, dom]
                elif y[0] > x[0]:
                    st[-1] = [y[0], y[1], x[2]]
                continue
            if x[0] or y[0]:
                if not x[0]:
                    st[-1] = [y[0], y[1], x[2]]
                continue
            a, b = x[2], y[2]
            if code == HOP_CMP:
                r = {EQ: a == b, NE: a != b, LT: a < b, LE: a <= b, GT: a > b, GE: a >= b}[arg]
                st[-1] = [0, 0, 1 if r else 0]
                continue
            if code == HOP_DIV:
                if b == 0:
                    st[-1] = [E_DIV0, 0, 0]
                    continue
                lo = -(2**31) if arg == 32 else -(2**63)
                if b == -1 and a == lo:
                    st[-1] = [E_I32 if arg == 32 else E_I64, 0, 0]
                    continue
                q = abs(a) // abs(b)
                r = q if (a >= 0) == (b >= 0) else -q
            else:
                r = a + b if code == HOP_ADD else (a - b if code == HOP_SUB else a * b)
            lim = 2**31 if arg == 32 else 2**63
            st[-1] = [E_OVF, 0, 0] if not (-lim <= r < lim) else [0, 0, r]
    return st[0][0], st[0][1], st[0][2]


def bounds(temporal):
    """MfpPlan::create_from: (lower, upper) lists of (program index, step)."""
    lower, upper = [], []
    for i, (cmp, _ops) in enumerate(temporal):
        if cmp == EQ:
            lower.append((i, False))
            upper.append((i, True))
        elif cmp == LT:
            upper.append((i, False))
        elif cmp == LE:
            upper.append((i, True))
        elif cmp == GT:
            lower.append((i, True))
        elif cmp == GE:
            lower.append((i, False))
        else:
            raise ValueError("unsupported temporal comparison")
    return lower, upper


def _bound(temporal, consts, w, b):
    e, p, v = run(temporal[b[0]][1], consts, w)
    if e:
        return e, p, 0
    if b[1]:
        if v == MAX:
            return E_STEP, 0, 0
        v += 1
    return 0, 0, v


def valid(t, until):
    """!until.less_equal(t); until = EMPTY (the empty antichain) makes every time valid, u64::MAX included."""
    return until == EMPTY or t < until


def evaluate(plan, w, time, diff, until):
    """MfpPlan::evaluate: ([(time, diff)], [(code, payload, time, diff)])."""
    preds, temporal, consts = plan["predicates"], plan["temporal"], plan["consts"]
    for ops in preds:
        e, p, v = run(ops, consts, w)
        if e:
            return [], [(e, p, time, diff)]
        if v == 0:
            return [], []
    lower_b, upper_b = bounds(temporal)
    lower = time
    for b in lower_b:
        e, p, v = _bound(temporal, consts, w, b)
        if e:
            return [], [(e, p, time, diff)]
        lower = max(lower, v)
    if not valid(lower, until):
        return [], []
    upper = None
    for b in upper_b:
        if upper == lower:
            break
        e, p, v = _bound(temporal, consts, w, b)
        if e:
            return [], [(e, p, time, diff)]
        upper = v if upper is None else min(upper, v)
        if upper < lower:
            upper = lower
    if upper is not None and not valid(upper, until):
        upper = None
    if upper == lower:
        return [], []
    out = [(lower, diff)]
    if upper is not None:
        out.append((upper, -diff))
    return out, []


def project(plan, w):
    words = []
    for fl in plan["fields"]:
        acc = 0
        for (src, shift, bits, dst) in fl:
            acc |= (((w[src] >> shift) & ((1 << bits) - 1)) << dst) & (U64 - 1)
        words.append(acc)
    return words


def consolidate(rows):
    """rows: (words tuple, time, diff) -> sorted by (words, time), diffs summed (wrapping), zeros dropped."""
    acc = defaultdict(int)
    for wds, t, d in rows:
        acc[(tuple(wds), t)] += d
    out = []
    for (wds, t), d in sorted(acc.items()):
        d = s64(d)
        if d:
            out.append((wds, t, d))
    return out


class BucketChain:
    """BucketChain over lists of (time, payload) with fuel counted in rows."""

    def __init__(self):
        self.content = {0: (64, [])}

    @staticmethod
    def end(start, bits):
        e = start + (1 << bits)
        return None if e >= U64 else e

    def range_of(self, t):
        s = max(k for k in self.content if k <= t)
        return s, self.content[s][0]

    def insert(self, rows):
        for r in rows:
            s, _ = self.range_of(r[0])
            self.content[s][1].append(r)

    def _split(self, start, bits, rows, fuel):
        bits -= 1
        mid = start + (1 << bits)
        lo = [r for r in rows if r[0] < mid]
        hi = [r for r in rows if r[0] >= mid]
        fuel[0] -= len(lo)
        self.content[start] = (bits, lo)
        self.content[mid] = (bits, hi)

    def peel(self, upper):
        out = []
        while self.content:
            start = min(self.content)
            if upper != EMPTY and upper <= start:
                break
            bits, rows = self.content.pop(start)
            e = self.end(start, bits)
            if upper != EMPTY and (e is None or upper < e):
                self._split(start, bits, rows, [0])
            else:
                out.extend(rows)
        return out

    def restore(self, fuel):
        fuel = [fuel]
        new = {}
        last = -2
        while fuel[0] > 0 and self.content:
            t = min(self.content)
            bits, rows = self.content.pop(t)
            if bits <= last + 2:
                new[t] = (bits, rows)
                last = bits
            else:
                self._split(t, bits, rows, fuel)
        new.update(self.content)
        self.content = dict(sorted(new.items()))
        return fuel[0]

    def held(self):
        return sum(len(r) for _, r in self.content.values())


class Operator:
    """The step contract: (out, errs) per step, plus frontier() and held()."""

    def __init__(self, plan, until=EMPTY, in_words=4):
        self.plan, self.until, self.nw = plan, until, in_words
        self.chain = BucketChain()

    def step(self, rows, upper):
        ready, errs = [], []
        for r in rows:
            w = [int(r[0]), int(r[1]), int(r[2]) if self.nw == 5 else 0]
            time, diff = int(r[self.nw - 2]), s64(int(r[self.nw - 1]))
            upd, err = evaluate(self.plan, w, time, diff, self.until)
            errs.extend(((c, p), t, d) for c, p, t, d in err)
            proj = tuple(project(self.plan, w))
            for t, d in upd:
                if upper == EMPTY or t < upper:
                    ready.append((proj, t, d))
                else:
                    self.chain.insert([(t, (proj, d))])
        for t, (proj, d) in self.chain.peel(upper):
            ready.append((proj, t, d))
        self.chain.restore(10**6)
        return consolidate(ready), consolidate(errs)

    def frontier(self):
        ts = [r[0] for _, rows in self.chain.content.values() for r in rows]
        return min(ts) if ts else EMPTY

    def held(self):
        return self.chain.held()


def direct(plan, history, t, until=EMPTY, in_words=4):
    """The filtered collection at valid time t: rows accumulated to t that pass with lower <= t < upper."""
    acc = []
    for r in history:
        w = [int(r[0]), int(r[1]), int(r[2]) if in_words == 5 else 0]
        time, diff = int(r[in_words - 2]), s64(int(r[in_words - 1]))
        upd, _ = evaluate(plan, w, time, diff, until)
        for ut, d in upd:
            if ut <= t:
                acc.append((tuple(project(plan, w)), 0, d))
    return consolidate(acc)


# ----------------------------------------------------------------- golden answers (tests/golden/temporal_filters.json)
CMP_NAMES = {"EQ": EQ, "LT": LT, "LE": LE, "GT": GT, "GE": GE}
ERR_NAMES = {"MzTimestampOutOfRange": E_MZTS_RANGE, "MzTimestampStepOverflow": E_STEP,
             "TimestampOutOfRange": E_TS_RANGE}


def golden_plan(case):
    """A golden case's plan: the rows' two columns projected as they are, its temporal predicates as programs."""
    temporal, consts = [], []
    for cmp, e in case["temporal"]:
        if "plus" in e:
            consts.append((e["plus"], 0))
            ops = [(HOP_COL, e["col"], 0, 32, 1, 0), (HOP_INT, 0, 0, 0, 0, len(consts) - 1),
                   (HOP_ADD, 32, 0, 0, 0, 0), (HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)]
        else:
            ops = [(HOP_COL_MZTS, e["col"], 0, 64, 0, 0)]
        temporal.append((CMP_NAMES[cmp], ops))
    return {"fields": [[(0, 0, 64, 0)], [(1, 0, 64, 0)]], "predicates": [], "temporal": temporal, "consts": consts}


def golden_check(case, step):
    """Drive `step(rows, upper) -> (out, errs)` (tuples as Operator.step returns them) through a golden case:
    the rows at time 0, then one step per AS OF time t with upper = t + 1 (FRONTIER_EMPTY past u64::MAX - 1).
    Returns [] when every AS OF answer and the expected error match, else a list of mismatches."""
    released, errs, bad = [], [], []
    rows = [[a, b, 0, 1] for a, b in case["rows"]]
    for t in sorted(int(k) for k in case["as_of"]):
        upper = t + 1 if t + 1 < EMPTY else EMPTY
        out, err = step(rows, upper)
        rows = []
        released.extend(out)
        errs.extend(err)
        acc = defaultdict(int)
        for w, ut, d in released:
            if ut <= t:
                acc[tuple(w)] += d
        got = sorted(w for w, d in acc.items() for _ in range(d) if d > 0)
        want = sorted(tuple(r) for r in case["as_of"][str(t)])
        if got != want or any(d < 0 for d in acc.values()):
            bad.append((t, got, want))
    if "error" in case:
        e = case["error"]
        seen = [c for c, t, d in errs if c[0] == ERR_NAMES[e["code"]] and t <= e["as_of"] and d > 0]
        if not seen:
            bad.append(("error", errs, e))
    elif errs:
        bad.append(("errors", errs))
    return bad
