"""The reference of the probes with an MfpPlan closure (join_mfp_ref), pinned on the CPU: a plan equivalent to
a bit-field closure gives probe_ref's output, the equivalence lowering matches JoinClosure::apply, and the golden
answers of Materialize's joins.slt are reproduced."""
import json
import os

import numpy as np

import join_mfp_ref as jref
import mfp_map_oracle as M
import probe_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
COL, INT, CMP, DIV = M.O.HOP_COL, M.O.HOP_INT, M.O.HOP_CMP, M.O.HOP_DIV


def col(src, bits=20):
    return (COL, src, 0, bits, 0, 0)


def gen(rng, n, keys, times=(0, 4)):
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = rng.integers(0, keys, size=n, dtype=np.uint64)
    w[:, 1] = rng.integers(0, 1 << 20, size=n, dtype=np.uint64)
    w[:, 2] = rng.integers(times[0], times[1], size=n, dtype=np.uint64)
    w[:, 3] = rng.integers(1, 3, size=n).astype(np.uint64)
    return w


def test_bit_field_equivalent_plan():
    rng = np.random.default_rng(1)
    batches = [ref.aref.consolidate(gen(rng, 400, 60)) for _ in range(2)]
    stream = gen(rng, 300, 60)
    cl = dict(key_fields=[(0, 0, 64, 0)], val_fields=[(1, 0, 20, 0), (2, 0, 20, 20)],
              filters=[(2, 0, 20, "lt", 1 << 19)])
    plan = {"fields": [[(0, 0, 64, 0)], [(1, 0, 20, 0), (2, 0, 20, 20)]],
            "predicates": [[col(2), (INT, 0, 0, 0, 0, 0), (CMP, 2, 0, 0, 0, 0)]], "temporal": [],
            "consts": [(1 << 19, 0)], "maps": [], "map_consts": []}
    for mode in (ref.LE, ref.LT):
        want = ref.half_join(stream, batches, mode, cl)
        got, errs = jref.probe_mfp(stream, batches, mode, plan)
        assert got.tobytes() == want.tobytes() and len(errs) == 0


def test_equivalence_lowering_matches_join_closure_apply():
    consts = [(0, 0), (3, 0)]
    zero, three = (INT, 0, 0, 0, 0, 0), (INT, 0, 0, 0, 0, 1)
    e_div = [col(1), col(2), (DIV, 64, 0, 0, 0, 0)]  # an error when v2 = 0
    cases = [
        [[[col(0)], [col(1)]]],                                   # 2 expressions
        [[[col(0)], [col(1)], [col(2)]]],                         # 3 expressions
        [[e_div, [col(1)]]],                                      # error in e0
        [[[col(1)], e_div]],                                      # error in a later expression
        [[[col(0)], [col(1)], e_div]],                            # error after a mismatch
        [[[col(0)], [three], e_div], [[col(1)], [zero]]],         # two classes
    ]
    words = [[a, b, c] for a in (0, 3, 5) for b in (0, 3, 5) for c in (0, 3)]
    for classes in cases:
        plan = {"fields": [[(0, 0, 64, 0)], [(1, 0, 64, 0)]], "predicates": jref.lower_equivalences(classes),
                "temporal": [], "consts": consts, "maps": [], "map_consts": []}
        for w in words:
            err, ok = jref.join_closure_apply(classes, dict(plan, predicates=[]), w)
            upd, errs, _ = M.evaluate(plan, w, 0, 1, jref.M64)
            assert (errs[0][0], errs[0][1]) == err if errs else err is None, (classes, w)
            assert bool(upd) == ok, (classes, w)


def test_golden_join_closures():
    for case in json.load(open(os.path.join(HERE, "golden", "join_closures.json"))):
        lw = np.zeros((len(case["left"]), 4), np.uint64)
        lw[:, 1], lw[:, 2], lw[:, 3] = np.array(case["left"], np.int64).view(np.uint64), 1, 1
        rw = np.zeros((len(case["right"]), 4), np.uint64)
        rw[:, 1], rw[:, 3] = np.array(case["right"], np.int64).view(np.uint64), 1
        plan = {"fields": [[(1, 0, 64, 0)], [(M.SRC_MAP0, 0, 64, 0)]],
                "predicates": [[tuple(o) for o in p] for p in case["predicates"]], "temporal": [],
                "consts": [tuple(c) for c in case["consts"]], "maps": [[tuple(o) for o in m] for m in case["maps"]],
                "map_consts": [tuple(c) for c in case["map_consts"]]}
        out, errs = jref.probe_mfp(lw, [ref.aref.consolidate(rw)], ref.LE, plan)
        got = sorted((int(np.int64(x.view(np.int64))), int(np.int64(y.view(np.int64)))) for x, y in out[:, :2])
        assert got == sorted(tuple(x) for x in case["expect_rows"])
        assert [int(e[0]) for e in errs] == case["expect_error_codes"]
