"""`peek_ref` against known answers from Materialize's sqllogictests (tests/golden/index_peeks.json) and against an
independent transcription of the reference's index peek: PeekResultIterator (the MfpPlan before the diffs are
summed, literal keys by a forward-only seek), collect_ok_finished_data (the thinning at twice offset + limit) and
RowSetFinishing::finish (order_by over the columns' values, signed or not, reversed for DESC, then the whole row;
offset and limit in units; the projection).  The random traces keep clear of the stand-ins include/mzgpu.h lists: every pair has a positive count
at as_of (nothing in the future, nothing cancelled), whole rows tie-break as unsigned words, and a LIMIT always comes
with an ORDER BY.  Results are compared as the finished sequence of units (row, as_of) repeated by copies."""
import functools
import json
import os
import random

import numpy as np

import arrangement_ref as aref
import mfp_map_oracle as M
import peek_ref as P

M64 = (1 << 64) - 1
HERE = os.path.dirname(os.path.abspath(__file__))
O = M.O


def signed(x, bits=64):
    x &= (1 << bits) - 1
    return x - (1 << bits) if x >> (bits - 1) else x


def column(row, src, shift, bits):
    return (row[src] >> shift) & ((1 << bits) - 1)


def compare_rows(order, l, r):
    """compare_columns(order_by, l, r, || l.cmp(r)) over fixed-width rows: each lane's column as the integer it is
    (two's complement for a signed lane), reversed for DESC; then the whole row, word by word."""
    for (src, shift, bits, sx, desc, _f64) in order:
        a, b = column(l, src, shift, bits), column(r, src, shift, bits)
        if sx:
            a, b = signed(a, bits), signed(b, bits)
        if a != b:
            c = -1 if a < b else 1
            return -c if desc else c
    return (l > r) - (l < r)


def transcription(rows, plan, as_of, out_words, order, limit, offset, project, literals):
    by_key = {}
    for key, val, t, d in aref.words(rows, 32).tolist():
        by_key.setdefault(key, {}).setdefault(val, []).append((t, signed(d)))
    keys = sorted(by_key)
    if literals is not None:  # seek each literal in sorted order, never backwards
        keys = [k for k in sorted(set(literals)) if k in by_key]
    results = []
    need = None if limit is None else offset + limit
    for key in keys:
        for val in sorted(by_key[key]):
            w = [key, val, 0]
            upd, err, mv = M.evaluate(dict(plan, temporal=[]), w, 0, 1, M64)
            if err:
                return ("error", (P.ERR_MFP, (err[0][0], err[0][1] & M64, key, val)))
            if not upd:
                continue
            copies = sum(d for t, d in by_key[key][val] if t <= as_of)
            if copies < 0:
                return ("error", (P.ERR_RETRACTION, (key, val, copies & M64, 0)))
            if copies == 0:
                continue
            row = tuple([x & M64 for x in M.project(plan, w, mv)] + [0] * (3 - out_words))[:3]
            results.append((row, copies))
            if need is not None and len(results) >= 2 * need:
                results.sort(key=functools.cmp_to_key(lambda x, y: compare_rows(order, x[0], y[0])))
                del results[need:]
    results.sort(key=functools.cmp_to_key(lambda x, y: compare_rows(order, x[0], y[0])))
    units = [row for row, c in results for _ in range(c)]
    units = units[offset:] if limit is None else units[offset:offset + limit]
    out = []
    for row in units:
        pw = list(row[:out_words])
        if any(project):
            pw = [sum((column(row, f[0], f[1], f[2]) << f[3]) & M64 for f in fl) for fl in project] + [0] * out_words
            pw = pw[:out_words]
        out.append(tuple(pw + [as_of]))
    return ("rows", out)


def expand(res):
    if res[0] != "rows":
        return res
    return ("rows", [tuple(int(x) for x in r[:-1]) for r in res[1] for _ in range(int(r[-1]))])


def test_reference_against_transcription():
    r = random.Random(7)
    rng = np.random.default_rng(7)
    import materialize_b200._ffi as F

    for case in range(150):
        out_words = 2 + case % 2
        n = r.choice([0, 5, 60, 400])
        w = np.zeros((n, 4), dtype=np.uint64)
        w[:, 0] = rng.integers(0, 40, n)
        w[:, 1] = rng.integers(0, 6, n)
        w[:, 2] = rng.integers(0, 10, n)
        w[:, 3] = rng.integers(1, 4, n)
        rows = aref.as_rows(w, F.R32)
        plan = M.random_plan(r, in_words=4, out_words=out_words + 2, temporal=[])
        order = [(r.randrange(out_words), r.choice([0, 4]), r.choice([8, 16, 60]), r.random() < 0.5, r.random() < 0.5,
                  False) for _ in range(r.randrange(1, 4))]
        limit = r.choice([None, 0, 1, 3, 10])
        offset = r.choice([0, 2, 7])
        project = [] if r.random() < 0.5 else [[(r.randrange(out_words), 0, 16, 0)] for _ in range(out_words)]
        literals = None if r.random() < 0.5 else [r.randrange(45) for _ in range(r.randrange(8))] * 2
        got = P.peek(rows, plan, 9, out_words, order, limit, offset, project, literals)
        want = transcription(rows, plan, 9, out_words, order, limit, offset, project, literals)
        assert expand(got) == want, case


# ---- the golden cases.  Lowering, as the header's stand-in 5 and INTEGRATION.md describe it: int columns are 20-bit
# fields (every value in these tables is below 2^19); the index key is its columns packed a << 40 | b << 20 | c, the
# value the remaining columns packed the same way; order lanes are signed 32-bit reads of the int column.
FIELD = 20


def pack(vals):
    x = 0
    for v in vals:
        x = (x << FIELD) | v
    return x


def golden():
    with open(os.path.join(HERE, "golden", "index_peeks.json")) as f:
        return json.load(f)


def golden_lowering(case, tables):
    """(R32 rows of the index, plan, finishing, literal keys or None, as_of, decode(out words) -> selected values)."""
    t = tables[case["table"]]
    cols = t["columns"]
    kcols = case.get("index_columns", cols[:1])
    vcols = [c for c in cols if c not in kcols]
    rows = [(pack([r[cols.index(c)] for c in kcols]), pack([r[cols.index(c)] for c in vcols]), 0, 1) for r in t["rows"]]
    d = t.get("delete")
    if d is not None and case.get("after_delete"):
        rows += [(k, v, 1, M64) for (k, v, _, _), r in zip(list(rows), t["rows"]) if r[cols.index(d["column"])] == d["value"]]

    def where(c):  # (output word, shift) of column c: word 0 the key, word 1 the value
        ws = (kcols, vcols)
        w = 0 if c in kcols else 1
        return w, FIELD * (len(ws[w]) - 1 - ws[w].index(c))

    order = []
    for c, dirn in case.get("order_by", []):
        w, sh = where(c)
        order.append((w, sh, FIELD, True, dirn == "desc", False))
    preds, maps, consts = [], [], []
    if case.get("filter"):  # ((a = 1) AND (b = 4 * a)) OR ((a = 2) AND (b = 5 * a)) OR ((a = 3) AND (b = a + 20))
        def col(c):
            w, sh = where(c)
            return (O.HOP_COL, w, sh, FIELD, 1, 0)

        def k(v):
            if (v, 0) not in consts:
                consts.append((v, 0))
            return (O.HOP_INT, 0, 0, 0, 0, consts.index((v, 0)))

        eq, land, lor = (O.HOP_CMP, 0, 0, 0, 0, 0), (O.HOP_AND, 0, 0, 0, 0, 0), (O.HOP_OR, 0, 0, 0, 0, 0)
        mul, add = (O.HOP_MUL, 64, 0, 0, 0, 0), (O.HOP_ADD, 64, 0, 0, 0, 0)
        # one map expression per OR branch (a program holds at most MZGPU_MFP_MAX_OPS ops), the predicate ORs them
        maps = [[col("a"), k(1), eq, col("b"), k(4), col("a"), mul, eq, land],
                [col("a"), k(2), eq, col("b"), k(5), col("a"), mul, eq, land],
                [col("a"), k(3), eq, col("b"), col("a"), k(20), add, eq, land]]
        preds = [[(M.HOP_MAP, 0, 0, 0, 0, 0), (M.HOP_MAP, 1, 0, 0, 0, 0), lor, (M.HOP_MAP, 2, 0, 0, 0, 0), lor]]
    plan = {"fields": [[(0, 0, 64, 0)], [(1, 0, 64, 0)]], "predicates": preds, "temporal": [], "consts": [],
            "maps": maps, "map_consts": consts}
    fin = {"order": order, "limit": case.get("limit"), "offset": case.get("offset", 0)}
    lits = [pack(v) for v in case["lookup"]] if "lookup" in case else None
    as_of = 1 if case.get("after_delete") else 0

    def decode(words):
        out = []
        for c in case["select"]:
            w, sh = where(c)
            out.append((int(words[w]) >> sh) & ((1 << FIELD) - 1))
        return out

    return np.array(rows, dtype=np.uint64).reshape(-1, 4), plan, fin, lits, as_of, decode


def golden_answer(case, decode, out):
    """The selected values of output rows (w0, w1, as_of, copies), each row repeated by its copies; sorted when the
    query is rowsort."""
    got = [decode(r) for r in out.tolist() for _ in range(int(r[-1]))]
    return sorted(got) if case["rowsort"] else got


def test_reference_against_sqllogictest_answers():
    import materialize_b200._ffi as F

    g = golden()
    assert len(g["cases"]) == 9
    for case in g["cases"]:
        w, plan, fin, lits, as_of, decode = golden_lowering(case, g["tables"])
        got = P.peek(aref.as_rows(w, F.R32), plan, as_of, 2, literals=lits, **fin)
        assert got[0] == "rows", case
        assert golden_answer(case, decode, got[1]) == case["expect"], (case["file"], case["line"])
