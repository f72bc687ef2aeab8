"""The one-column reduce reference (tests/reduce_ref.py) pinned against the CPU oracle on random
activation sequences, by hand at the f64 fixed point's edges and the 64-bit wrap of a multiplicity,
and against the reference-held SQL answers in tests/golden/."""
import json
import os

import numpy as np
import pytest

import arrangement_ref as aref
import reduce_ref as ref
import sql_golden as sg

M64 = ref.M64
HERE = os.path.dirname(os.path.abspath(__file__))
TOPK_SHAPES = [(1, 0, False), (3, 0, True), (2, 1, False), (None, 2, True), (0, 0, False), (40, 0, False)]


def r32(rows):
    a = np.zeros((len(rows), 4), dtype=np.uint64)
    for i, (k, v, t, d) in enumerate(rows):
        a[i] = (k & M64, v & M64, t, d & M64)
    return a


def as_r32(oracle, w):
    return np.ascontiguousarray(w, dtype=np.uint64).view(oracle.R32).reshape(-1)


def words(a):
    return aref.words(a, a.dtype.itemsize)


def f64_values(rng, n):
    """Floats across the fixed point's branches: small ones, x * 2^24 near 2^63, in [2^116, 2^127),
    saturating, specials, signed zeros and subnormals."""
    v = rng.integers(-(10**6), 10**6, size=n).astype(np.float64) / 7.0
    pick = rng.integers(0, 12, size=n)
    big = np.ldexp(rng.random(n) + 1.0, rng.integers(30, 104, size=n)) * rng.choice([-1.0, 1.0], size=n)
    v = np.where(pick < 4, big, v)
    specials = np.array([np.nan, np.inf, -np.inf, 1e300, -1e300, 0.0, -0.0, 5e-324, 2.0**103, -(2.0**103)])
    v = np.where(pick == 4, specials[rng.integers(0, len(specials), size=n)], v)
    return v.view(np.uint64)


def activations(rng, kind, steps, keys, t0=0):
    """Random activations: values of the kind's domain, diffs of both signs (counts go negative and
    recover), retractions of earlier rows, times spread over three per activation."""
    t, live = t0, []
    for step in range(steps):
        n = int(rng.integers(0, 2500))
        w = np.zeros((n, 4), dtype=np.uint64)
        w[:, 0] = rng.zipf(1.4, size=n).astype(np.uint64) % np.uint64(keys)
        if kind == ref.F64:
            w[:, 1] = f64_values(rng, n)
        elif kind == ref.I64:
            w[:, 1] = rng.integers(-(2**63), 2**63, size=n, dtype=np.int64).view(np.uint64)
            w[::5, 1] = rng.integers(-50, 50, size=len(w[::5])).astype(np.int64).view(np.uint64)
        else:
            w[:, 1] = rng.integers(0, 40, size=n, dtype=np.uint64) * np.uint64(0x0123456789ABCDEF)
        w[:, 2] = rng.integers(t, t + 3, size=n, dtype=np.uint64)
        w[:, 3] = rng.integers(-1, 3, size=n).astype(np.int64).view(np.uint64)
        if live and step % 3 == 2:
            old = np.concatenate(live)
            back = old[rng.random(len(old)) < 0.4].copy()
            back[:, 3] = (-back[:, 3].view(np.int64)).view(np.uint64)
            back[:, 2] = rng.integers(t, t + 3, size=len(back), dtype=np.uint64)
            w = np.concatenate([w, back])
            live = []
        else:
            live.append(w.copy())
        t += 3
        yield w, t


# ------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("kind", [0, 1, 2, 3, 4, 5])
def test_reduce_matches_oracle(oracle, kind):
    rng = np.random.default_rng(31 + kind)
    r, o = ref.make(kind), oracle.Reduce(kind)
    n_out = 0
    for w, upper in activations(rng, kind, 14, 300):
        got, want = r.step(w, upper), words(o.step(as_r32(oracle, w), upper))
        assert got.tobytes() == want.tobytes(), (kind, upper, len(got), len(want))
        n_out += len(got)
    assert n_out > 500


@pytest.mark.parametrize("limit,offset,desc", TOPK_SHAPES)
def test_topk_matches_oracle(oracle, limit, offset, desc):
    rng = np.random.default_rng(41 + (limit or 0) + offset)
    r, o = ref.make(ref.TOPK, limit, offset, desc), oracle.TopK(-1 if limit is None else limit, offset, desc)
    for w, upper in activations(rng, ref.TOPK, 12, 200):
        got, want = r.step(w, upper), words(o.step(as_r32(oracle, w), upper))
        assert got.tobytes() == want.tobytes(), (limit, offset, desc, upper)


def test_rows_at_or_past_upper_wait_in_the_batcher(oracle):
    """Updates at times >= upper ship with a later activation, in both."""
    for kind in (0, 4):
        r, o = ref.make(kind), oracle.Reduce(kind)
        a = r32([(1, 5, 0, 1), (1, 7, 4, 1), (2, 9, 9, 2), (1, 3, M64 - 1, 1)])
        for rows, upper in ((a, 3), (a[:0], 5), (a[:0], ref.FE)):
            assert r.step(rows, upper).tobytes() == words(o.step(as_r32(oracle, rows), upper)).tobytes()


# ------------------------------------------------------------------ by hand
def test_f64_fixed_point_constants():
    assert ref.accum_f64(1e300) == ref.I128_MAX
    assert ref.accum_f64(-(2.0**103)) == ref.I128_MIN
    assert ref.accum_f64(-1.5 * 2.0**-24) == -1
    assert ref.accum_f64(2.0**39 + 2.0**-13) == (1 << 63) + (1 << 11)  # x * 2^24 just past 2^63
    assert ref.accum_f64(-(2.0**100)) == -(1 << 124)
    assert ref.accum_f64(5e-324) == 0 and ref.accum_f64(-0.0) == 0
    # i128 -> f64: a tie rounds to even, the sticky bit breaks it, -2^127 is exact
    assert ref.sum_f64((1 << 117) + (1 << 64)) == 2.0**93
    assert ref.sum_f64((1 << 117) + (1 << 64) + 1) == (2.0**117 + 2.0**65) / 2.0**24
    assert ref.sum_f64(ref.I128_MIN) == -(2.0**103)
    assert ref.sum_f64((1 << 53) + 1) == 2.0**29  # a tie below 2^64 (lo only)
    assert ref.sum_f64((1 << 53) + 3) == (2.0**53 + 4) / 2.0**24


def test_f64_sums_and_flags_by_hand():
    """Sums landing on the tie and the sticky bit, a saturated sum, and a net-zero total whose only
    non-zero accumulator word is pos_infs (flag bit 1)."""
    b = ref.bits
    r = ref.Reduce(ref.F64)
    rows = [(1, b(2.0**93), 0, 1), (1, b(2.0**40), 0, 1),
            (2, b(2.0**93), 0, 1), (2, b(2.0**40), 0, 1), (2, b(2.0**-24), 0, 1),
            (3, b(-1e300), 0, 1),
            (4, b(float("inf")), 0, 1), (4, b(0.0), 0, -1),
            (5, b(float("nan")), 0, 2), (5, b(float("inf")), 0, 1)]
    out = r.step(r32(rows), 1)
    got = {int(k): (int(c), int(lo), int(hi), int(f)) for k, c, lo, hi, f, _, _, _ in out.tolist()}
    assert got[1] == (2, b(2.0**93), 0, 0)
    assert got[2] == (3, b((2.0**117 + 2.0**65) / 2.0**24), 0, 0)
    assert got[3] == (1, b(-(2.0**103)), 0, 0)
    assert got[4] == (0, ref.PINF_BITS, 0, 2)
    assert got[5] == (3, ref.NAN_BITS, 0, 0)


def test_i64_sums_wrap_at_128_bits():
    r = ref.Reduce(ref.I64)
    big = (1 << 63) - 1
    out = r.step(r32([(1, big, 0, big), (1, big, 0, big), (1, big, 1, big), (1, -(1 << 63), 1, -(1 << 63))]), 2)
    final = [row for row in out.tolist() if row[6] == 1 and row[5] == 1][0]
    want = ref.s128(3 * big * big + (1 << 126))
    assert (final[2], ref.s64(final[3])) == (want & M64, want >> 64)


def test_multiplicity_wraps_past_i64_max(oracle):
    """DISTINCT and threshold over a multiplicity that wraps past i64::MAX to a negative total."""
    big = (1 << 63) - 1
    rows = [r32([(7, 0, 0, big)]), r32([(7, 0, 1, 2)]), r32([(7, 0, 2, -3)])]
    for kind in (ref.DISTINCT, ref.THRESHOLD):
        r, o = ref.make(kind), oracle.Reduce(kind)
        outs = []
        for i, w in enumerate(rows):
            got = r.step(w, i + 1)
            assert got.tobytes() == words(o.step(as_r32(oracle, w), i + 1)).tobytes()
            outs.append([(row[4], ref.s64(row[6])) for row in got.tolist()])
        if kind == ref.DISTINCT:
            assert outs == [[(0, 1)], [(0, -1), (2, 1)], [(0, 1), (2, -1)]]
        else:
            assert outs == [[(0, big)], [(0, -big)], [(0, big - 1)]]


def test_topk_offset_past_a_value_and_limit_inside_copies():
    r = ref.TopK(2, 3)
    out = r.step(r32([(1, 10, 0, 2), (1, 20, 0, 2), (1, 30, 0, 5)]), 1)
    assert [(row[2], row[6]) for row in out.tolist()] == [(20, 1), (30, 1)]
    r = ref.TopK(None, 0, True)
    out = r.step(r32([(1, 10, 0, 1), (1, 20, 0, -1)]), 1)
    assert [(row[2], row[4], row[6]) for row in out.tolist()] == [(0, 2, 1)]


# ------------------------------------------------------------------ reference-held answers
class RefOps(sg.OracleOps):
    """sql_golden's adapter with the reduce taken from the reference."""

    name = "reduce_ref"

    def reduce(self, kind, rows):
        return ref.make(kind).step(rows, 1).view(self.o.ROUT).reshape(-1)


def test_reference_reproduces_sqllogictest_answers(oracle):
    fx = sg.load()
    ops = RefOps(oracle)
    ran = 0
    for case in fx["cases"]:
        if case["shape"] == "sum_of_nulls":
            continue
        got = sg.norm(sg.evaluate(ops, case, fx["tables"]))
        assert got == sg.norm([tuple(r) for r in case["expect"]]), (case["name"], case["cite"])
        ran += 1
    assert ran >= 12


def test_reference_topk_reproduces_sqllogictest_answers():
    with open(os.path.join(HERE, "golden", "sqllogictest_topk.json")) as f:
        fx = json.load(f)
    rows = fx["cities"]["rows"]
    states = sorted({r[1] for r in rows})
    names = [r[0] for r in rows]
    for case in fx["per_group"]:
        w = []
        for name, state, pop in rows:
            if pop is None:
                pop = (1 << 40) - 1 if case["nulls_first"] else 0
            w.append((states.index(state), (pop << 8) | names.index(name), 0, 1))
        out = ref.TopK(case["limit"], 0, case["descending"]).step(r32(w), 1).tolist()
        assert all(row[4] == 0 and row[6] == 1 for row in out)
        assert {(states[row[0]], names[row[2] & 0xFF]) for row in out} == {tuple(x) for x in case["answer"]}
        assert len(out) == len(case["answer"])
    for case in fx["global"]:
        cur = [(0, v, 0, 1) for v in case["t"]]
        for st in case["stages"]:
            out = ref.TopK(st["limit"], st["offset"]).step(r32(cur), 1).tolist()
            cur = [(0, row[2], 0, ref.s64(row[6])) for row in out]
        assert sorted(v for _, v, _, _ in cur) == case["answer"], case["name"]
        assert all(d == 1 for *_, d in cur)
