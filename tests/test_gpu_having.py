"""HAVING filters of the lanes operator (mzgpu_reduce_lanes_new_having) on the GPU: byte for byte against
the CPU restatement (output, main arrangement, pair arrangements), an always-TRUE filter against the
unfiltered operator, reference-held answers, rejections, and a full-size run against numpy."""
import ctypes as C

import numpy as np
import pytest

import lanes_paths_ref as R
from having_oracle import ERR_SHIFT, ReduceLanesHaving, cmp, count, div, int_, key, num, sum_
from test_oracle_distinct_lanes import D, distinct_activations
from test_oracle_having import (
    CROSSING,
    DIVISION_RETRACTED,
    FIXTURE_PLANS,
    NULL_SUM_LANES,
    NULL_SUM_PREDS,
    NULL_SUM_ROWS,
    SCENARIOS,
    evaluator_case_op_rows,
    evaluator_cases,
    fixture_expect,
    having_sum_cases,
    load_fixture,
    run_fixture_case,
    run_having_sum,
    run_steps,
)
from test_gpu_reduce_paths import _key_rows

pytestmark = pytest.mark.gpu

I64, F64, VAL1, VAL2 = 0, 1, 1, 2


@pytest.fixture(scope="module")
def mz():
    import materialize_b200 as m

    return m


@pytest.fixture(scope="module")
def ctx(mz):
    # the full-size run takes several GB of device memory: hand it back when the module ends
    c = mz.Context(0)
    yield c
    c.sync()
    c.close()


def same_bytes(a, b):
    assert a.dtype.itemsize == b.dtype.itemsize
    assert len(a) == len(b), (len(a), len(b))
    assert a.tobytes() == b.tobytes()


def gpu_op(mz, ctx, in_rb, lanes, preds):
    return mz.ReduceLanes(ctx, [mz.accum_lane(*l) for l in lanes], in_rb, having=mz.having(*preds))


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_having_matches_restatement(mz, ctx, oracle, name):
    in_rb, lanes, preds = SCENARIOS[name]
    o = ReduceLanesHaving(oracle, lanes, in_rb, preds)
    g = gpu_op(mz, ctx, in_rb, lanes, preds)
    rng = np.random.default_rng(7 + len(name))
    for a, upper in distinct_activations(rng, in_rb // 8, steps=10, keys=300):
        same_bytes(g.step(a, upper), o.step(a, upper))
        same_bytes(g.input_trace().export(), o.export())
        for l, lane in enumerate(lanes):
            if lane[0] & D:
                same_bytes(g.distinct_trace(l).export(), o.pair_export(l))


def test_small_scenarios_match_restatement(mz, ctx, oracle):
    """Threshold crossings, a division by zero that appears and is retracted, and NULL SUMs through the distinct
    total rule: every activation byte for byte against the restatement."""
    for lanes, preds, steps in (CROSSING, DIVISION_RETRACTED):
        for g, o in zip(run_steps(gpu_op(mz, ctx, 32, lanes, preds), steps),
                        run_steps(ReduceLanesHaving(oracle, lanes, 32, preds), steps)):
            same_bytes(g, o)
    for preds, visible in NULL_SUM_PREDS:
        (g,) = run_steps(gpu_op(mz, ctx, 32, NULL_SUM_LANES, preds), [(NULL_SUM_ROWS, 1)])
        (o,) = run_steps(ReduceLanesHaving(oracle, NULL_SUM_LANES, 32, preds), [(NULL_SUM_ROWS, 1)])
        same_bytes(g, o)
        assert len(g) == (1 if visible else 0)


def test_evaluator_cases_on_one_key_gpu_operators(mz, ctx, oracle):
    """Every evaluator case (comparisons on INT / NUM / FLOAT with NaN, +-inf and -0.0, overflow at both widths,
    MIN / -1, division by zero, error precedence, AND / OR with NULL and errors, predicate order, key fields)
    through a one-key GPU operator: the same bytes as the restatement, visible exactly when the reference's
    answer says so, with its error in flag bits 16-18."""
    for preds, key_word, null, want in evaluator_cases():
        steps = [(evaluator_case_op_rows(key_word, null), 1)]
        (g,) = run_steps(gpu_op(mz, ctx, 32, NULL_SUM_LANES, preds), steps)
        (o,) = run_steps(ReduceLanesHaving(oracle, NULL_SUM_LANES, 32, preds), steps)
        same_bytes(g, o)
        assert len(g) == (0 if want == "drop" else 1), (preds, want)
        if isinstance(want, tuple):
            assert (int(g[0]["flags"]) >> ERR_SHIFT) & 7 == want[1], (preds, want)


@pytest.mark.parametrize("n_lanes", [1, 2, 4, 8])
def test_two_pass_path_past_the_single_pass_bound(mz, n_lanes):
    """Batches of 26 M distinct keys: at two output rows per new (key, time) that is past the single-pass bound
    (48 Mi output rows), so the corrections run in the two-pass form, k_corrections<C, false / true> without a
    filter and k_corrections_having<C, false / true> with one; the profile report shows which kernels ran.
    The unfiltered output is compared row for row with the NumPy expectation of tests/lanes_paths_ref.py (in
    key-rank slices, to bound host memory), and its arrangement on 2000 sampled keys.  One time per key and
    activation, so the filtered corrections are exactly the unfiltered operator's corrections that the filter
    lets through, with the error bits added: the predicates are COUNT / (key & 255) >= 0 (a division by zero
    on every 256th key) and SUM(lane 0) < 0.  The second activation retracts half of the keys and adds a row
    to the other half (the prior batch is read back through the hash index).  val2 holds float64 bits
    (NaN, +-inf, -0.0 among them) for the float64 lane."""
    lanes = R.LANES8[:n_lanes]  # bit-fields of val1 and val2 and, from 4 lanes on, the float64 lane of val2
    preds = [[count(0), key(0, 8), div(64), int_(0), cmp("ge")], [sum_(0), num(0), cmp("lt")]]
    rng = np.random.default_rng(50 + n_lanes)
    n = 26_000_000
    keys = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(2**40 - 1)  # distinct
    first = np.zeros(n, dtype=mz.R40)
    first["key"] = keys
    first["val1"] = rng.integers(0, 2**64, size=n, dtype=np.uint64)
    first["val2"] = R.f64_words(rng, n)
    first["diff"] = 1
    second = first.copy()
    second["time"] = 1
    back = rng.random(n) < 0.5
    second["diff"] = np.where(back, -1, 1)
    second["val1"] = np.where(back, first["val1"], rng.integers(0, 2**64, size=n, dtype=np.uint64))
    second["val2"] = np.where(back, first["val2"], R.f64_words(rng, n))
    batches = [(first, 1), (second, 2)]
    w1, w2 = (np.ascontiguousarray(b).view(np.uint64).reshape(n, 5) for b in (first, second))

    def run(having):
        c = mz.Context(0)
        op = mz.ReduceLanes(c, [mz.accum_lane(*l) for l in lanes], 40, having=having)
        c.profile(True)
        c.profile_report()
        outs = [op.step(b, upper) for b, upper in batches]
        kernels = set(c.profile_report())
        if having is None:
            pick = np.sort(rng.choice(n, size=2000, replace=False))
            got = _key_rows(mz, c, op, w1[pick, 0])
            assert got.tobytes() == R.two_pass_arrangement("lanes", lanes, w1, w2, pick).tobytes()
        print(f"having two-pass, {n_lanes} lanes{'' if having is None else ', filtered'}: device_bytes_peak",
              c.stats()["device_bytes_peak"])
        del op
        c.close()
        return outs, kernels

    plain, plain_kernels = run(None)
    # the unfiltered output, row for row, in key-rank slices of the expectation
    keys = np.sort(first["key"])
    width = 1 << 22
    for lo in range(0, n, width):
        hi = min(n, lo + width)
        want = R.two_pass_expect("lanes", lanes, w1, w2, lo, hi)[:2]
        for got, w in zip(plain, want):
            a, b = np.searchsorted(got["key"], keys[lo]), np.searchsorted(got["key"], keys[hi - 1], side="right")
            g = np.ascontiguousarray(got[a:b]).view(np.uint64).reshape(b - a, -1)
            assert g.shape == w.shape and g.tobytes() == w.tobytes(), (lo, g.shape, w.shape)
    filtered, kernels = run(mz.having(*preds))
    def ran(names, kernel):  # the profile report writes the launch's kernel expression with "_" for " "
        return any(kernel.replace(" ", "_") in k for k in names)

    assert ran(plain_kernels, "(k_corrections<C, false>)") and ran(plain_kernels, "(k_corrections<C, true>)"), plain_kernels
    assert not ran(plain_kernels, "k_corrections_lb"), plain_kernels
    assert ran(kernels, "(k_corrections_having<C, false>)"), kernels
    assert ran(kernels, "(k_corrections_having<C, true>)"), kernels
    assert not ran(kernels, "k_corrections_lb"), kernels
    n_err = 0
    for u, f in zip(plain, filtered):
        err = (u["key"] & np.uint64(255)) == 0
        visible = err | (u["lanes"][:, 0]["sum_hi"] < 0)
        want = u[visible].copy()
        want["flags"] |= np.where(err[visible], np.uint64(1 << ERR_SHIFT), np.uint64(0))
        assert 0 < len(want) < len(u)
        same_bytes(f, want)
        n_err += int(err[visible].sum())
    assert n_err > 0


def test_always_true_filter_is_the_unfiltered_operator(mz, ctx):
    """count(0) >= 0 OR ... holds for every row: output and arrangement are byte-identical to no filter."""
    in_rb, lanes, _ = SCENARIOS["c8_r40_eight_lanes"]
    true_preds = [[count(0), count(0), cmp("eq")], [key(), key(), cmp("ge")]]
    f = gpu_op(mz, ctx, in_rb, lanes, true_preds)
    u = mz.ReduceLanes(ctx, [mz.accum_lane(*l) for l in lanes], in_rb)
    z = mz.ReduceLanes(ctx, [mz.accum_lane(*l) for l in lanes], in_rb, having=mz.having())  # no predicates
    rng = np.random.default_rng(11)
    for a, upper in distinct_activations(rng, in_rb // 8, steps=8, keys=500):
        want = u.step(a, upper)
        same_bytes(f.step(a, upper), want)
        same_bytes(z.step(a, upper), want)
    same_bytes(f.input_trace().export(), u.input_trace().export())


def test_fixture_cases_through_one_gpu_operator(mz, ctx):
    for case in load_fixture()["cases"]:
        assert case["name"] in FIXTURE_PLANS
        got = run_fixture_case(lambda i, l, p: gpu_op(mz, ctx, i, l, p), case)
        assert got == fixture_expect(case), case["name"]
    for case, pairs in having_sum_cases():
        assert run_having_sum(lambda i, l, p: gpu_op(mz, ctx, i, l, p), pairs) == sorted(case["expect"]), case["name"]


def _raw(mz, preds_raw, consts=()):
    """An F.Having from raw (code, arg, shift, bits, sign_extend, konst) ops: malformed programs included."""
    F = mz._ffi
    hv = F.Having()
    hv.n_predicates = len(preds_raw)
    for p, ops in enumerate(preds_raw):
        hv.n_ops[p] = len(ops)
        for i, (code, arg, shift, bits, sx, k) in enumerate(ops):
            o = hv.ops[p][i]
            o.code, o.arg, o.shift, o.bits, o.sign_extend, o.konst = code, arg, shift, bits, sx, k
    hv.n_consts = len(consts)
    for k, (lo, hi) in enumerate(consts):
        hv.consts[k].lo, hv.consts[k].hi = lo, hi
    return hv


def test_rejections_leave_the_context_usable(mz, ctx):
    F = mz._ffi
    E_INVALID, E_UNSUPPORTED = -1, -4
    lanes = [mz.accum_lane(I64, VAL1), mz.accum_lane(F64, VAL1)]
    c0 = [(1, 0)]  # constant 0: the INT / NUM 1
    cnt, one, gt = (F.HOP_COUNT, 0, 0, 0, 0, 0), (F.HOP_INT, 0, 0, 0, 0, 0), (F.HOP_CMP, 4, 0, 0, 0, 0)
    good = [cnt, one, gt]
    cases = [
        ([[(15, 0, 0, 0, 0, 0)] + good[1:]], c0, E_INVALID),  # unknown opcode
        ([[(0, 0, 0, 0, 0, 0)] + good[1:]], c0, E_INVALID),
        ([[one, gt]], c0, E_INVALID),  # stack underflow
        ([[one] * 9 + [gt] * 7], c0, E_INVALID),  # depth 9
        ([[(F.HOP_COUNT, 2, 0, 0, 0, 0), one, gt]], c0, E_INVALID),  # lane >= n_lanes
        ([[(F.HOP_KEY, 0, 60, 8, 0, 0), one, gt]], c0, E_INVALID),  # key field past bit 63
        ([[(F.HOP_KEY, 0, 0, 0, 0, 0), one, gt]], c0, E_INVALID),  # empty key field
        ([[cnt, (F.HOP_INT, 0, 0, 0, 0, 1), gt]], c0, E_INVALID),  # constant index out of range
        ([[cnt, one]], c0, E_INVALID),  # two values left
        ([[cnt, one, (F.HOP_ADD, 64, 0, 0, 0, 0)]], c0, E_INVALID),  # an INT left, not a BOOL
        ([[cnt, one, (F.HOP_CMP, 6, 0, 0, 0, 0)]], c0, E_INVALID),  # compare op
        ([[cnt, one, (F.HOP_ADD, 16, 0, 0, 0, 0), one, gt]], c0, E_INVALID),  # width
        ([[cnt, one, (F.HOP_ADD, 32, 0, 0, 0, 0), one, gt]], c0, E_INVALID),  # 32-bit op on a bigint COUNT
        ([[cnt, (F.HOP_NOT, 0, 0, 0, 0, 0), one, gt]], c0, E_INVALID),  # NOT of an INT
        ([[cnt, one, (F.HOP_INT, 0, 0, 0, 0, 1), gt]], [(1, 0), (0, 1)], E_INVALID),  # INT constant past i64
        ([good] * 5, c0, E_INVALID),  # five predicates
        ([[]], c0, E_INVALID),  # an empty predicate
        # well-formed, outside the subset
        ([[(F.HOP_SUM, 0, 0, 0, 0, 0), (F.HOP_NUM, 0, 0, 0, 0, 0), (F.HOP_ADD, 64, 0, 0, 0, 0), one, gt]], c0, E_UNSUPPORTED),
        ([[(F.HOP_SUM, 1, 0, 0, 0, 0), one, gt]], c0, E_UNSUPPORTED),  # FLOAT against INT
        ([[(F.HOP_SUM, 1, 0, 0, 0, 0), (F.HOP_FLOAT, 0, 0, 0, 0, 0), (F.HOP_MUL, 64, 0, 0, 0, 0), one, gt]], c0, E_UNSUPPORTED),
        ([good + good + [(F.HOP_CMP, 0, 0, 0, 0, 0)]], c0, E_UNSUPPORTED),  # BOOL = BOOL
    ]
    for preds, consts, status in cases:
        hv = _raw(mz, preds[:4], consts)
        if len(preds) > 4:
            hv.n_predicates = len(preds)
        h = C.c_void_p()
        st = F.lib.mzgpu_reduce_lanes_new_having(ctx.h, 32, (F.AccumLane * 2)(*[F.AccumLane(k, sx, F.Field(s, sh, b, 0)) for k, s, sh, b, sx in lanes]),
                                                 2, C.byref(hv), C.byref(h))
        assert st == status, (preds, st, F.lib.mzgpu_last_error(ctx.h))
        assert not h
    # lane errors are reported before the filter is looked at
    with pytest.raises(mz.MzGpuError) as e:
        mz.ReduceLanes(ctx, [mz.accum_lane(2, VAL1)], 32, having=mz.having([count(0), int_(0), cmp("gt")]))
    assert e.value.status == E_INVALID
    # the context still works, and a valid filter runs
    r = gpu_op(mz, ctx, 32, [(I64, VAL1, 0, 64, False)], [[count(0), key(), div(64), int_(0), cmp("ge")]])
    a = np.zeros(3, dtype=mz.R32)
    a["key"], a["val"], a["diff"] = [0, 2, 2], [4, 4, 6], 1
    o = r.step(a, 1)
    assert [int(k) for k in o["key"]] == [0, 2] and int(o["flags"][0]) == 1 << ERR_SHIFT and int(o["flags"][1]) == 0
    assert len(ctx.consolidate(np.zeros(4, dtype=mz.R32))) == 0


def test_having_full_size_against_numpy(mz, ctx):
    """About 20 M R40 rows over 1 M keys, 4 lanes, and a selective two-predicate filter (COUNT > 22 and
    SUM(val2 lane) < 0), then incremental batches with half retractions; after every step the operator's
    visible rows equal per-key COUNT / SUM from numpy, filtered the same way."""
    rng = np.random.default_rng(41)
    nk, n = 1_000_000, 20_000_000
    lanes = [(I64, VAL1, 0, 32, True), (I64, VAL1, 32, 32, True), (I64, VAL2, 0, 64, False), (I64, VAL2, 0, 16, False)]
    preds = [[count(0), int_(22), cmp("gt")], [sum_(2), int_(0), cmp("lt")]]
    r = gpu_op(mz, ctx, 40, lanes, preds)

    def batch(m, t):
        a = np.zeros(m, dtype=mz.R40)
        a["key"] = rng.integers(0, nk, size=m, dtype=np.uint64)
        a["val1"] = rng.integers(0, 2**64, size=m, dtype=np.uint64)
        a["val2"] = rng.integers(-(2**40), 2**40, size=m, dtype=np.int64).view(np.uint64)
        a["time"], a["diff"] = t, 1
        return a

    live = batch(n, 0)
    outs = [r.step(live, 1)]
    check_state(outs, live, nk)
    for step in range(1, 3):
        fresh = batch(500_000, step)
        back_idx = np.unique(rng.integers(0, len(live), size=500_000))
        back = live[back_idx].copy()
        back["time"], back["diff"] = step, -1
        outs.append(r.step(np.concatenate([fresh, back]), step + 1))
        keep = np.ones(len(live), dtype=bool)
        keep[back_idx] = False
        live = np.concatenate([live[keep], fresh])
        check_state(outs, live, nk)
    print("having full size: device_bytes_peak", ctx.stats()["device_bytes_peak"])


def check_state(outs, live, nk):
    out = np.concatenate(outs)
    step = np.concatenate([np.full(len(o), i) for i, o in enumerate(outs)])
    order = np.lexsort((out["diff"], step, out["key"]))
    out, step = out[order], step[order]
    last = np.r_[out["key"][1:] != out["key"][:-1], True]
    cur = out[last & (out["diff"] == 1)]
    keys = live["key"].astype(np.int64)
    cnt = np.bincount(keys, minlength=nk)
    v2 = live["val2"].view(np.int64)
    s2 = np.bincount(keys, weights=v2.astype(np.float64), minlength=nk)
    assert np.abs(s2).max() < 2.0**53
    s2 = s2.astype(np.int64)
    w = np.nonzero((cnt > 22) & (s2 < 0))[0]
    assert 0 < len(w) < nk // 4
    assert np.array_equal(cur["key"].astype(np.int64), w)
    assert np.all(cur["flags"] == 0)
    assert np.array_equal(cur["lanes"][:, 0]["count"], cnt[w])
    assert np.array_equal(cur["lanes"][:, 2]["sum_lo"].view(np.int64), s2[w])
    lo1 = (live["val1"] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    lo1 = np.where(lo1 >= 2**31, lo1 - 2**32, lo1)
    s0 = np.bincount(keys, weights=lo1.astype(np.float64), minlength=nk).astype(np.int64)
    assert np.array_equal(cur["lanes"][:, 0]["sum_lo"].view(np.int64), s0[w])
