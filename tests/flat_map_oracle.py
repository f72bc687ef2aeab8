"""Plain-Python restatement of FlatMap (mzgpu_flat_map_new, include/mzgpu.h), built on tests/mfp_map_oracle.py.

- `series_count(start, stop, step)`: the number of values of range_step_inclusive, by formula.
- `range_step_inclusive(start, stop, step, bits)`: the values, by literal iteration with the checked-add stop.
- `evaluate_func(tf, w)`: the argument programs and TableFunc::eval (func.rs:3520-3620, WithOrdinality::eval
  :3912-3960): an error (code, payload), or (count, start, step, mult) -- function row j has the columns
  (start + j * step, j + 1) and diff mult.
- `Operator`: the step / work contract, page by page over the activation's function rows, each through
  mfp_map_oracle's MfpPlan evaluation and mfp_oracle's bucket chain.

A table function is a dict: kind (TF_*), with_ordinality, args (op lists), consts, step_us (timestamp series).
"""
import mfp_map_oracle as M
import mfp_oracle as O

TF_GENERATE_SERIES_INT32, TF_GENERATE_SERIES_INT64, TF_GENERATE_SERIES_TIMESTAMP = 1, 2, 3
TF_REPEAT_ROW, TF_REPEAT_ROW_NON_NEGATIVE, TF_GUARD_SUBQUERY_SIZE = 4, 5, 6
SRC_FN0 = 8
E_INVALID_PARAMETER_VALUE, E_MULTIPLE_ROWS, E_NEGATIVE_ROWS, E_INTERNAL = 8, 9, 10, 11
U64, s64 = O.U64, O.s64


def series_count(start, stop, step):
    if step > 0 and start <= stop:
        return (stop - start) // step + 1
    if step < 0 and start >= stop:
        return (start - stop) // -step + 1
    return 0


def range_step_inclusive(start, stop, step, bits=64):
    """num::range_step_inclusive over i<bits>, as TimestampRangeStepInclusive restates it: a generator."""
    lo, hi = -(2 ** (bits - 1)), 2 ** (bits - 1) - 1
    state, rev, done = start, step < 0, False
    while not done and ((rev and state >= stop) or (not rev and state <= stop)):
        yield state
        nxt = state + step
        if nxt < lo or nxt > hi:  # checked_add overflow
            done = True
        else:
            state = nxt


def n_columns(tf):
    series = tf["kind"] <= TF_GENERATE_SERIES_TIMESTAMP
    return (1 if series else 0) + (1 if tf.get("with_ordinality") else 0)


def evaluate_func(tf, w):
    """(code, payload) on an error, else (count, start, step, mult)."""
    args = []
    for ops in tf["args"]:
        e, p, v = M.run(ops, tf.get("consts", []), w, [])
        if e:
            return (e, p)
        args.append(v)
    kind = tf["kind"]
    if kind <= TF_GENERATE_SERIES_TIMESTAMP:
        step = tf["step_us"] if kind == TF_GENERATE_SERIES_TIMESTAMP else args[2]
        if step == 0:
            return (E_INVALID_PARAMETER_VALUE, 0)
        return (series_count(args[0], args[1], step), args[0], step, 1)
    n = args[0]
    if kind == TF_REPEAT_ROW:
        return (1 if n != 0 else 0, 0, 0, n)
    if kind == TF_REPEAT_ROW_NON_NEGATIVE:
        if n < 0:
            return (E_INVALID_PARAMETER_VALUE, n % U64)
        if n == 0:
            return (0, 0, 0, 1)
        if tf.get("with_ordinality"):
            return (n, 1, 1, 1)  # n unit rows, the ordinal 1 + j as column 0
        return (1, 0, 0, n)
    if n == 1:
        return (0, 0, 0, 1)
    return (E_MULTIPLE_ROWS if n > 1 else E_NEGATIVE_ROWS if n < 0 else E_INTERNAL, 0)


def function_rows(tf, w):
    """The function rows of one input row: (columns, diff) pairs (small counts only), or an error."""
    r = evaluate_func(tf, w)
    if len(r) == 2:
        return r
    count, start, step, mult = r
    cols = []
    for j in range(count):
        c = [start + j * step, j + 1][: max(n_columns(tf), 0)]
        cols.append((c, mult))
    return cols


class Operator(O.Operator):
    """step(rows, upper, fuel) / work(fuel) -> (out, errs, done), pages of `fuel` function rows."""

    def __init__(self, tf, plan, until=O.EMPTY, in_words=4):
        super().__init__(plan, until, in_words)
        self.tf = tf
        self.pending = None  # (rows' words / time / diff / record, next ordinal, total)
        self.upper = 0

    def step(self, rows, upper, fuel=10**6):
        assert self.pending is None, "an activation is unfinished"
        recs, errs, total = [], [], 0
        for r in rows:
            w = [int(r[0]), int(r[1]), int(r[2]) if self.nw == 5 else 0] + [0] * 7
            time, diff = int(r[self.nw - 2]), s64(int(r[self.nw - 1]))
            f = evaluate_func(self.tf, w)
            if len(f) == 2:
                errs.append((f, time, diff))
                continue
            if f[0]:
                recs.append((total, w, time, diff, f))
                total += f[0]
        self.pending, self.upper, self.first_errs = (recs, 0, total), upper, errs
        return self.work(fuel)

    def work(self, fuel=10**6):
        if self.pending is None:
            return [], [], True
        recs, g, total = self.pending
        page = min(fuel, total - g)
        ready, errs = [], list(self.first_errs)
        self.first_errs = []
        import bisect
        starts = [r[0] for r in recs]
        o = g
        while o < g + page:
            k = bisect.bisect_right(starts, o) - 1
            base, w0, time, diff, (count, start, step, mult) = recs[k]
            for j in range(o - base, min(count, g + page - base)):
                w = list(w0)
                w[SRC_FN0], w[SRC_FN0 + 1] = (start + j * step) % U64, j + 1
                d = s64(mult * diff)
                upd, err, mv = M.evaluate(self.plan, w, time, d, self.until)
                errs.extend(((c, p), t, dd) for c, p, t, dd in err)
                if upd:
                    proj = tuple(M.project(self.plan, w, mv))
                    for t, dd in upd:
                        if self.upper == O.EMPTY or t < self.upper:
                            ready.append((proj, t, dd))
                        else:
                            self.chain.insert([(t, (proj, dd))])
            o = base + count if base + count < g + page else g + page
        for t, (proj, d) in self.chain.peel(self.upper):
            ready.append((proj, t, d))
        self.chain.restore(10**6)
        g += page
        self.pending = None if g == total else (recs, g, total)
        return O.consolidate(ready), O.consolidate(errs), self.pending is None


# ----------------------------------------------------------------- golden answers (tests/golden/table_func.json)
# Columns are 32-bit values, column c in bits [32 * (c % 2), +32) of word c // 2 (sign-extended when read);
# an output row holds the input columns and then the function's columns in the same layout.
TF_KINDS = {"generate_series_int32": TF_GENERATE_SERIES_INT32, "generate_series_int64": TF_GENERATE_SERIES_INT64,
            "repeat_row": TF_REPEAT_ROW, "repeat_row_non_negative": TF_REPEAT_ROW_NON_NEGATIVE}


def col_op(c):
    return (O.HOP_COL, c // 2, 32 * (c % 2), 32, 1, 0)


def golden_stage(stage, n_in):
    """(tf, plan) of one FlatMap of a golden case over n_in input columns."""
    consts, args = [], []
    for a in stage["args"]:
        if a[0] == "col":
            args.append([col_op(a[1])])
        else:
            consts.append((a[1] % U64, U64 - 1 if a[1] < 0 else 0))
            args.append([(O.HOP_INT, 0, 0, 0, 0, len(consts) - 1)])
    tf = {"kind": TF_KINDS[stage["func"]], "with_ordinality": stage.get("ordinality", False), "args": args,
          "consts": consts}
    n_out = n_in + n_columns(tf)
    fields = [[], [], []]
    for c in range(n_out):
        src = (c // 2, 32 * (c % 2), 32) if c < n_in else (SRC_FN0 + c - n_in, 0, 32)
        fields[c // 2].append((src[0], src[1], src[2], 32 * (c % 2)))
    preds = []
    for (x, y) in stage.get("filter_eq", []):
        def op(ref):
            return col_op(ref) if ref < n_in else (O.HOP_COL, SRC_FN0 + ref - n_in, 0, 64, 0, 0)
        preds.append([op(x), op(y), (O.HOP_CMP, O.EQ, 0, 0, 0, 0)])
    plan = {"fields": fields, "predicates": preds, "temporal": [], "consts": [], "maps": [], "map_consts": []}
    return tf, plan, n_out


def encode_columns(vals):
    w = [0, 0, 0]
    for c, v in enumerate(vals):
        w[c // 2] |= (v % 2**32) << (32 * (c % 2))
    return w


def decode_columns(words, n):
    out = []
    for c in range(n):
        v = (words[c // 2] >> (32 * (c % 2))) & 0xFFFFFFFF
        out.append(v - 2**32 if v >= 2**31 else v)
    return out


def golden_rows(case, rows):
    """The case's answer from final consolidated rows ((words, time, diff), n_out): a sorted list with each row
    repeated diff times, after the case's projection."""
    got = []
    for (wds, t, d), n in rows:
        cols = decode_columns(list(wds), n)
        if "project" in case:
            cols = [cols[i] for i in case["project"]]
        got.extend([cols] * d)
    return sorted(got)
