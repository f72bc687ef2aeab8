"""Plain-Python restatement of the MfpPlan with map expressions (mzgpu_mfp_new_map, include/mzgpu.h), built on
tests/mfp_oracle.py.

- `run(ops, consts, w, mv)`: one program of the interpreter with the map opcodes (MAP, NEG, ABS, MOD,
  INT64_TO_INT32, IF); `mv` holds the expression values a MAP may read.
- `support(ops)`: 1 + the highest MAP index a program reads.
- `evaluate(plan, w, time, diff, until)`: SafeMfpPlan::evaluate_inner (src/expr/src/linear.rs:1680-1700) followed
  by MfpPlan::evaluate's temporal bounds (linear.rs:1865-1971): (updates, errors, expression values).
- `project(plan, w, mv)`: the output words over the input words and the expression values.
- `Operator`: mfp_oracle.Operator's step contract over this evaluation.

A plan is mfp_oracle's dict plus "maps" (op lists) and "map_consts".
"""
import mfp_oracle as O

HOP_MAP, HOP_NEG, HOP_ABS, HOP_MOD, HOP_INT64_TO_INT32, HOP_IF = 23, 24, 25, 26, 27, 28
SRC_MAP0 = 16
U64, s64 = O.U64, O.s64


def _lo(width):
    return -(2**31) if width == 32 else -(2**63)


def run(ops, consts, w, mv):
    """Returns (err, payload, value); an INT is a Python int, a BOOL 0 / 1, an MZTS its unsigned value."""
    st = []
    for (code, arg, shift, bits, sx, k) in ops:
        if code in (O.HOP_COL, O.HOP_COL_TS, O.HOP_COL_DATE):
            a = (w[arg] >> shift) & ((1 << bits) - 1)
            if sx and (a >> (bits - 1)) & 1:
                a -= 1 << bits
            st.append([0, 0, s64(a) if code != O.HOP_COL or sx or bits == 64 else a])
        elif code == O.HOP_COL_MZTS:
            st.append([0, 0, (w[arg] >> shift) & ((1 << bits) - 1)])
        elif code == O.HOP_INT:
            st.append([0, 0, s64(consts[k][0])])
        elif code == HOP_MAP:
            st.append([0, 0, mv[arg]])
        elif code == O.HOP_NOT:
            if st[-1][0] == 0:
                st[-1][2] ^= 1
        elif code == HOP_IF:
            e, t = st.pop(), st.pop()
            if st[-1][0] == 0:
                st[-1] = list(t if st[-1][2] == 1 else e)
        elif code in (O.HOP_INT_TO_MZTS, O.HOP_TS_TO_MZTS, O.HOP_DATE_TO_MZTS, O.HOP_TS_ADD_IV):
            e, p, a = st[-1]
            if e:
                continue
            if code == O.HOP_TS_ADD_IV:
                lo, hi = consts[k]
                days = (hi & 0xFFFFFFFF) - (1 << 32) if hi & 0x80000000 else hi & 0xFFFFFFFF
                r = a + days * 86400000000 + s64(lo)
                st[-1] = [O.E_TS_RANGE, 0, a] if not (O.TS_LOW_US <= r <= O.TS_HIGH_US) else [0, 0, r]
            else:
                r = a if code == O.HOP_INT_TO_MZTS else (a // 1000 if code == O.HOP_TS_TO_MZTS else a * 86400000)
                st[-1] = [O.E_MZTS_RANGE, a % U64, a] if r < 0 else [0, 0, r]
        elif code in (HOP_NEG, HOP_ABS, HOP_INT64_TO_INT32):
            e, p, a = st[-1]
            if e:
                continue
            if code == HOP_INT64_TO_INT32:
                st[-1] = [0, 0, a] if -(2**31) <= a < 2**31 else [O.E_I32, a % U64, a]
            elif a == _lo(arg):  # checked_neg / checked_abs
                st[-1] = [O.E_I32 if arg == 32 else O.E_I64, a % U64, a]
            else:
                st[-1] = [0, 0, -a if code == HOP_NEG else abs(a)]
        else:
            y = st.pop()
            x = st[-1]
            if code in (O.HOP_AND, O.HOP_OR):
                dom = 0 if code == O.HOP_AND else 1
                if (x[0] == 0 and x[2] == dom) or (y[0] == 0 and y[2] == dom):
                    st[-1] = [0, 0, dom]
                elif y[0] > x[0] or (y[0] and y[0] == x[0] and y[1] == 0):
                    # std::cmp::max of the errors: of one code, the division's "a / b" message (payload 0)
                    # orders after NEG / ABS's operand
                    st[-1] = [y[0], y[1], x[2]]
                continue
            if x[0] or y[0]:
                if not x[0]:
                    st[-1] = [y[0], y[1], x[2]]
                continue
            a, b = x[2], y[2]
            if code == O.HOP_CMP:
                r = {O.EQ: a == b, O.NE: a != b, O.LT: a < b, O.LE: a <= b, O.GT: a > b, O.GE: a >= b}[arg]
                st[-1] = [0, 0, 1 if r else 0]
                continue
            if code in (O.HOP_DIV, HOP_MOD):
                if b == 0:
                    st[-1] = [O.E_DIV0, 0, 0]
                    continue
                if code == HOP_MOD:  # checked_rem(b).unwrap_or(0); the remainder takes the dividend's sign
                    r = 0 if b == -1 else (abs(a) % abs(b)) * (1 if a >= 0 else -1)
                    st[-1] = [0, 0, r]
                    continue
                if b == -1 and a == _lo(arg):
                    st[-1] = [O.E_I32 if arg == 32 else O.E_I64, 0, 0]
                    continue
                q = abs(a) // abs(b)
                r = q if (a >= 0) == (b >= 0) else -q
            else:
                r = a + b if code == O.HOP_ADD else (a - b if code == O.HOP_SUB else a * b)
            lim = 2**31 if arg == 32 else 2**63
            st[-1] = [O.E_OVF, 0, 0] if not (-lim <= r < lim) else [0, 0, r]
    return st[0][0], st[0][1], st[0][2]


def support(ops):
    return max([o[1] + 1 for o in ops if o[0] == HOP_MAP], default=0)


def _bound(plan, w, mv, b):
    e, p, v = run(plan["temporal"][b[0]][1], plan["consts"], w, mv)
    if e:
        return e, p, 0
    if b[1]:
        if v == O.MAX:
            return O.E_STEP, 0, 0
        v += 1
    return 0, 0, v


def evaluate(plan, w, time, diff, until):
    """([(time, diff)], [(code, payload, time, diff)], expression values)."""
    maps, mconsts = plan.get("maps", []), plan.get("map_consts", [])
    mv = []

    def eval_to(n):  # evaluate_inner's `while input_arity + expression < support`
        while len(mv) < n:
            e, p, v = run(maps[len(mv)], mconsts, w, mv)
            if e:
                return e, p
            mv.append(v)
        return None

    for ops in plan["predicates"]:
        err = eval_to(support(ops))
        if err:
            return [], [(err[0], err[1], time, diff)], mv
        e, p, v = run(ops, plan["consts"], w, mv)
        if e:
            return [], [(e, p, time, diff)], mv
        if v != 1:
            return [], [], mv
    err = eval_to(len(maps))
    if err:
        return [], [(err[0], err[1], time, diff)], mv
    lower_b, upper_b = O.bounds(plan["temporal"])
    lower = time
    for b in lower_b:
        e, p, v = _bound(plan, w, mv, b)
        if e:
            return [], [(e, p, time, diff)], mv
        lower = max(lower, v)
    if not O.valid(lower, until):
        return [], [], mv
    upper = None
    for b in upper_b:
        if upper == lower:
            break
        e, p, v = _bound(plan, w, mv, b)
        if e:
            return [], [(e, p, time, diff)], mv
        upper = v if upper is None else min(upper, v)
        if upper < lower:
            upper = lower
    if upper is not None and not O.valid(upper, until):
        upper = None
    if upper == lower:
        return [], [], mv
    out = [(lower, diff)]
    if upper is not None:
        out.append((upper, -diff))
    return out, [], mv


def project(plan, w, mv):
    words = []
    for fl in plan["fields"]:
        acc = 0
        for (src, shift, bits, dst) in fl:
            v = mv[src - SRC_MAP0] % U64 if src >= SRC_MAP0 else w[src]
            acc |= (((v >> shift) & ((1 << bits) - 1)) << dst) & (U64 - 1)
        words.append(acc)
    return words


class Operator(O.Operator):
    """mfp_oracle.Operator with map expressions: (out, errs) per step."""

    def step(self, rows, upper):
        ready, errs = [], []
        for r in rows:
            w = [int(r[0]), int(r[1]), int(r[2]) if self.nw == 5 else 0]
            time, diff = int(r[self.nw - 2]), s64(int(r[self.nw - 1]))
            upd, err, mv = evaluate(self.plan, w, time, diff, self.until)
            errs.extend(((c, p), t, d) for c, p, t, d in err)
            if not upd:
                continue
            proj = tuple(project(self.plan, w, mv))
            for t, d in upd:
                if upper == O.EMPTY or t < upper:
                    ready.append((proj, t, d))
                else:
                    self.chain.insert([(t, (proj, d))])
        for t, (proj, d) in self.chain.peel(upper):
            ready.append((proj, t, d))
        self.chain.restore(10**6)
        return O.consolidate(ready), O.consolidate(errs)


# ----------------------------------------------------------------- golden answers (tests/golden/mfp_map_arithmetic.json)
GOLDEN_OPS = {"MOD": HOP_MOD, "DIV": O.HOP_DIV, "NEG": HOP_NEG, "ABS": HOP_ABS}
GOLDEN_ERRS = {"DivisionByZero": O.E_DIV0, "Int32OutOfRange": O.E_I32, "Int64OutOfRange": O.E_I64}


def golden_program(case):
    """A golden case as one expression over constants: (ops, consts)."""
    consts = [(a % U64, U64 - 1 if a < 0 else 0) for a in case["args"]]
    ops = [(O.HOP_INT, 0, 0, 0, 0, k) for k in range(len(consts))]
    ops.append((GOLDEN_OPS[case["op"]], case["width"], 0, 0, 0, 0))
    return ops, consts


def golden_expect(case):
    """(err, payload or None when checked by code only, value)."""
    if "error" in case:
        pay = int(case["payload"]) % U64 if "payload" in case else None
        return GOLDEN_ERRS[case["error"]], pay, None
    return 0, 0, case["result"]


# ----------------------------------------------------------------- random plans the host accepts
CONST_POOL = [0, 1, -1, 10, 16, 2**31 - 1, -(2**31), -(2**63)]  # MZGPU_MFP_MAX_CONSTS


def _consts(vals):
    return [(v % U64, U64 - 1 if v < 0 else 0) for v in vals]


def depth_of(ops):
    d = m = 0
    for o in ops:
        c = o[0]
        if c in (O.HOP_COL, O.HOP_COL_MZTS, O.HOP_COL_TS, O.HOP_COL_DATE, O.HOP_INT, HOP_MAP):
            d += 1
        elif c == HOP_IF:
            d -= 2
        elif c not in (O.HOP_NOT, HOP_NEG, HOP_ABS, HOP_INT64_TO_INT32, O.HOP_INT_TO_MZTS, O.HOP_TS_TO_MZTS,
                       O.HOP_DATE_TO_MZTS, O.HOP_TS_ADD_IV):
            d -= 1
        m = max(m, d)
    return m


class PlanGen:
    """Random typed programs over `in_words` input words: 'i32' (int32 on the host), 'i64' (any INT), 'bool'.
    Tracks whether a program may carry an INT64_TO_INT32 error (kept out of AND / OR)."""

    def __init__(self, rng, in_words, consts, map_ty, new_ops=True):
        self.rng, self.nw, self.consts, self.map_ty, self.new_ops = rng, in_words, consts, map_ty, new_ops

    def _konst(self, want32):
        ks = [k for k, v in enumerate(self.consts) if not want32 or -(2**31) <= v < 2**31]
        return [(O.HOP_INT, 0, 0, 0, 0, self.rng.choice(ks))]

    def leaf(self, t):
        r, w = self.rng, self.rng.randrange(self.nw - 2)
        maps = [j for j, mt in enumerate(self.map_ty) if mt == t or (t == "i64" and mt == "i32")]
        if maps and r.random() < 0.35:
            return [(HOP_MAP, r.choice(maps), 0, 0, 0, 0)], False
        if t == "bool":
            (a, va), (b, vb) = self.leaf("i64"), self.leaf("i64")
            return a + b + [(O.HOP_CMP, r.randrange(6), 0, 0, 0, 0)], va or vb
        if r.random() < 0.3:
            return self._konst(t == "i32"), False
        if t == "i32":
            return [r.choice([(O.HOP_COL, w, 0, 32, 1, 0), (O.HOP_COL, w, 8, 8, 0, 0), (O.HOP_COL, w, 0, 31, 0, 0)])], False
        return [r.choice([(O.HOP_COL, w, 0, 64, 0, 0), (O.HOP_COL, w, 0, 32, 1, 0), (O.HOP_COL, w, 4, 60, 1, 0)])], False

    def gen(self, t, depth):
        r = self.rng
        if depth == 0 or r.random() < 0.25:
            return self.leaf(t)
        width = 32 if t == "i32" else 64
        k = r.randrange(4) if self.new_ops else r.choice([0, 1, 3])
        if t == "bool":
            if k == 0:
                (a, va) = self.gen("bool", depth - 1)
                return a + [(O.HOP_NOT, 0, 0, 0, 0, 0)], va
            if k == 1:
                (a, va), (b, vb) = self.gen("bool", depth - 1), self.gen("bool", depth - 1)
                if not (va or vb):
                    return a + b + [(r.choice([O.HOP_AND, O.HOP_OR]), 0, 0, 0, 0, 0)], False
            if k == 2:
                return self._if(t, depth)
            (a, va), (b, vb) = self.gen("i64", depth - 1), self.gen("i64", depth - 1)
            return a + b + [(O.HOP_CMP, r.randrange(6), 0, 0, 0, 0)], va or vb
        if k == 0:
            (a, va), (b, vb) = self.gen(t, depth - 1), self.gen(t, depth - 1)
            code = r.choice([O.HOP_ADD, O.HOP_SUB, O.HOP_MUL, O.HOP_DIV] + [HOP_MOD, HOP_MOD] * self.new_ops)
            return a + b + [(code, width, 0, 0, 0, 0)], va or vb
        if k == 1 and self.new_ops:
            (a, va) = self.gen(t, depth - 1)
            return a + [(r.choice([HOP_NEG, HOP_ABS]), width, 0, 0, 0, 0)], va
        if k == 2:
            return self._if(t, depth)
        if t == "i32" and self.new_ops:
            (a, va) = self.gen("i64", depth - 1)
            return a + [(HOP_INT64_TO_INT32, 0, 0, 0, 0, 0)], True
        return self.leaf(t)

    def _if(self, t, depth):
        (c, vc), (a, va), (b, vb) = self.gen("bool", depth - 1), self.gen(t, depth - 1), self.gen(t, depth - 1)
        return c + a + b + [(HOP_IF, 0, 0, 0, 0, 0)], vc or va or vb

    def program(self, t, depth=3):
        while True:
            ops, v = self.gen(t, depth)
            if len(ops) <= 16 and depth_of(ops) <= 8:
                return ops, v


def random_plan(rng, in_words=4, out_words=4, n_maps=None, n_preds=None, temporal=None, new_ops=True):
    """A plan with 0-4 map expressions (one may be an mz_timestamp for a temporal bound), 0-2 predicates and the
    projection of input words and expressions; every program is one the host accepts.  new_ops=False keeps the
    predicates to the opcodes of mzgpu_mfp_new before expressions."""
    consts = CONST_POOL
    mconsts = list(reversed(CONST_POOL))
    map_ty = []
    g = PlanGen(rng, in_words, mconsts, map_ty)
    maps = []
    n_maps = rng.randrange(5) if n_maps is None else n_maps
    for _ in range(n_maps):
        t = rng.choice(["i32", "i64", "bool", "mzts"])
        if t == "mzts":  # ABS(col % 16 * 10)::mz_timestamp, a time in [0, 150)
            ops = [(O.HOP_COL, rng.randrange(in_words - 2), 0, 32, 1, 0), (O.HOP_INT, 0, 0, 0, 0, mconsts.index(16)),
                   (HOP_MOD, 32, 0, 0, 0, 0), (O.HOP_INT, 0, 0, 0, 0, mconsts.index(10)),
                   (O.HOP_MUL, 32, 0, 0, 0, 0), (HOP_ABS, 32, 0, 0, 0, 0), (O.HOP_INT_TO_MZTS, 0, 0, 0, 0, 0)]
        else:
            ops, _ = g.program(t)
        maps.append(ops)
        map_ty.append(t)
    pg = PlanGen(rng, in_words, consts, map_ty, new_ops)
    preds = [pg.program("bool")[0] for _ in range(rng.randrange(3) if n_preds is None else n_preds)]
    mz = [j for j, t in enumerate(map_ty) if t == "mzts"]
    if temporal is None:
        temporal = []
        if mz and rng.random() < 0.7:
            temporal.append((rng.choice([O.GE, O.LT, O.LE, O.GT, O.EQ]), [(HOP_MAP, rng.choice(mz), 0, 0, 0, 0)]))
    fields = [[(0, 0, 64, 0)]]
    for _w in range(1, out_words - 2):
        fl = []
        if n_maps and rng.random() < 0.8:
            fl.append((SRC_MAP0 + rng.randrange(n_maps), 0, rng.choice([64, 32, 16]), 0))
        if not fl or rng.random() < 0.3:
            fl.append((rng.randrange(in_words - 2), 0, 16, 48))
        fields.append(fl)
    return {"fields": fields, "predicates": preds, "temporal": temporal, "consts": _consts(consts), "maps": maps,
            "map_consts": _consts(mconsts)}
