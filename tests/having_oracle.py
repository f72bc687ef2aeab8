"""CPU restatement of the HAVING filter of the multi-column accumulable reduce (test infrastructure).

render_reduce hands every reduce its fused mfp_after (src/compute/src/render/reduce.rs:64-78), and
build_accumulable evaluates it on (key, finalized aggregates) inside the ReduceAccumulable closure
(:1384-1409, evaluate_mfp_after :1474-1499): the key's output row exists only while the predicates hold.
AccumulableErrorCheck reports the predicates' errors whatever the filter does (:1452-1464); this project
carries errors as row flags, so an error row is kept, with the error in flag bits 16-18.

The evaluator works on Python values -- ints with explicit i32 / i64 range checks, floats, bools, None for
NULL and Err for an error -- and restates the reference's rules:
  predicates in order, the first that is not TRUE drops the row, an error stops evaluation
      (SafeMfpPlan::evaluate_inner, src/expr/src/linear.rs:1680-1700);
  add / sub / mul_int32 / 64: checked at their width, NumericFieldOverflow
      (src/expr/src/scalar/func.rs:107, 117, 690, 700, 904, 914);
  div_int32 / 64: DivisionByZero, truncation, MIN / -1 Int32OutOfRange / Int64OutOfRange (func.rs:1037-1059);
  both operands evaluated, the first one's error wins, then the second's, then NULL propagates
      (the eager argument unpacking, src/repr/src/scalar.rs:2126-2160);
  comparisons of Datum::Float64 are OrderedFloat's (src/repr/src/scalar.rs:99);
  variadic And / Or: FALSE (TRUE) wins over an error, else the larger error, else NULL
      (src/expr/src/scalar/func/variadic.rs:74-99, 1147-1170);
  errors ordered as the EvalError variants (src/expr/src/scalar.rs:1724-1740).

ReduceLanesHaving reuses ReduceLanesDistinct (and through it ReduceLanes) unchanged except _finalize,
which returns None for a row the filter hides and adds the error bits to the flags.  Ops are the tuples
of materialize_b200's h_*() constructors: (code, arg, shift, bits, sign_extend, constant value or None).
"""
import math
import struct

from distinct_lanes_oracle import ReduceLanesDistinct
from lanes_oracle import M64

KEY, COUNT, SUM, INT, NUM, FLOAT = 1, 2, 3, 4, 5, 6
ADD, SUB, MUL, DIV, CMP, AND, OR, NOT = 7, 8, 9, 10, 11, 12, 13, 14
CMPS = {"eq": 0, "ne": 1, "lt": 2, "le": 3, "gt": 4, "ge": 5}
DIVISION_BY_ZERO, NUMERIC_FIELD_OVERFLOW, INT32_OUT_OF_RANGE, INT64_OUT_OF_RANGE = 1, 2, 3, 4
ERR_SHIFT = 16


def key(shift=0, bits=64, sign_extend=False):
    return (KEY, 0, shift, bits, 1 if sign_extend else 0, None)


def count(lane):
    return (COUNT, lane, 0, 0, 0, None)


def sum_(lane):
    return (SUM, lane, 0, 0, 0, None)


def int_(v):
    return (INT, 0, 0, 0, 0, v)


def num(v):
    return (NUM, 0, 0, 0, 0, v)


def float_(x):
    return (FLOAT, 0, 0, 0, 0, float(x))


def add(w=64):
    return (ADD, w, 0, 0, 0, None)


def sub(w=64):
    return (SUB, w, 0, 0, 0, None)


def mul(w=64):
    return (MUL, w, 0, 0, 0, None)


def div(w=64):
    return (DIV, w, 0, 0, 0, None)


def cmp(op):
    return (CMP, CMPS[op], 0, 0, 0, None)


def and_():
    return (AND, 0, 0, 0, 0, None)


def or_():
    return (OR, 0, 0, 0, 0, None)


def not_():
    return (NOT, 0, 0, 0, 0, None)


class Err:
    def __init__(self, code):
        self.code = code

    def __repr__(self):
        return f"Err({self.code})"


def f64_of_bits(b):
    return struct.unpack("<d", struct.pack("<Q", b & M64))[0]


def _in_width(x, w):
    return -(1 << (w - 1)) <= x < (1 << (w - 1))


def _arith(code, w, a, b):
    if code == DIV:
        if b == 0:
            return Err(DIVISION_BY_ZERO)
        q = abs(a) // abs(b)
        q = q if (a < 0) == (b < 0) else -q  # truncation toward zero
        if not _in_width(q, w):  # only MIN / -1
            return Err(INT32_OUT_OF_RANGE if w == 32 else INT64_OUT_OF_RANGE)
        return q
    r = {ADD: a + b, SUB: a - b, MUL: a * b}[code]
    return r if _in_width(r, w) else Err(NUMERIC_FIELD_OVERFLOW)


def _order_key(x):
    if isinstance(x, float):
        return (1, 0.0) if math.isnan(x) else (0, x)  # NaN above everything, equal to NaN; -0.0 == 0.0
    return (0, x)


def _compare(op, a, b):
    ka, kb = _order_key(a), _order_key(b)
    return [ka == kb, ka != kb, ka < kb, ka <= kb, ka > kb, ka >= kb][op]


def _logic(dominant, a, b):
    if a is dominant or b is dominant:
        return dominant
    errs = [x for x in (a, b) if isinstance(x, Err)]
    if errs:
        return max(errs, key=lambda e: e.code)
    if a is None or b is None:
        return None
    return not dominant


def evaluate(predicates, key_word, lane_kinds, vals, flags):
    """The filter on one finalized row: vals = C x (count, sum_lo, sum_hi) words.  Returns ("err", code),
    "drop" or "pass"."""
    for ops in predicates:
        st = []
        for code, arg, shift, bits, sx, value in ops:
            if code == KEY:
                v = (key_word >> shift) & ((1 << bits) - 1)
                if (sx or bits == 64) and v >> (bits - 1):  # (a 64-bit field is the i64 itself)
                    v -= 1 << bits
                st.append(v)
            elif code == COUNT:
                c = vals[3 * arg]
                st.append(c - (1 << 64) if c >> 63 else c)
            elif code == SUM:
                if (flags >> (2 * arg)) & 1:
                    st.append(None)
                elif lane_kinds[arg] == 1:
                    st.append(f64_of_bits(vals[3 * arg + 1]))
                else:
                    s = vals[3 * arg + 1] | (vals[3 * arg + 2] << 64)
                    st.append(s - (1 << 128) if s >> 127 else s)
            elif code in (INT, NUM, FLOAT):
                st.append(value)
            elif code == NOT:
                a = st.pop()
                st.append(a if a is None or isinstance(a, Err) else not a)
            else:
                b, a = st.pop(), st.pop()
                if code in (AND, OR):
                    st.append(_logic(code == OR, a, b))
                elif isinstance(a, Err):
                    st.append(a)
                elif isinstance(b, Err):
                    st.append(b)
                elif a is None or b is None:
                    st.append(None)
                elif code == CMP:
                    st.append(_compare(arg, a, b))
                else:
                    st.append(_arith(code, arg, a, b))
        (r,) = st
        if isinstance(r, Err):
            return ("err", r.code)
        if r is not True:
            return "drop"
    return "pass"


def filter_row(predicates, lane_kinds, row):
    """A finalized row tuple (key, C x (count, sum_lo, sum_hi), flags) -> the visible row with the error
    bits added, or None."""
    key_word, vals, flags = row[0], row[1:-1], row[-1]
    r = evaluate(predicates, key_word, lane_kinds, vals, flags)
    if isinstance(r, tuple):
        flags |= r[1] << ERR_SHIFT
    if isinstance(r, tuple) or r == "pass" or flags & 0xAAAA:
        return (key_word, *vals, flags)
    return None


class ReduceLanesHaving(ReduceLanesDistinct):
    """ReduceLanesDistinct whose output rows pass through `predicates` (a list of op lists)."""

    def __init__(self, oracle, lanes, in_row_bytes=32, predicates=()):
        super().__init__(oracle, lanes, in_row_bytes)
        self.predicates = [list(p) for p in predicates]

    def _finalize(self, key, v):
        row = super()._finalize(key, v)
        if not self.predicates:
            return row
        out = filter_row(self.predicates, [l[0] for l in self.lanes], (key, *row))
        return None if out is None else out[1:]
