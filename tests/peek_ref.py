"""Plain reference of the index peeks (mzgpu_peek_many; test infrastructure).

It composes `arrangement_ref` (the trace's rows consolidated) with `mfp_map_oracle` (the plan without temporal
bounds, then projected), and applies the rules include/mzgpu.h states: the frontier checks, the error trace first,
the first failing pair in (key, val) order, then ORDER BY (ties by the output words) / OFFSET / LIMIT over copies,
the projection and max_rows.
"""
import numpy as np

import arrangement_ref as aref
import mfp_map_oracle as M

M64 = (1 << 64) - 1
EMPTY = M64
ERR_SINCE, ERR_ERRS_ROW, ERR_ERRS_RETRACTION, ERR_MFP, ERR_RETRACTION, ERR_TOO_LARGE = 1, 2, 3, 4, 5, 6


def _s64(x):
    x = int(x)
    return x - (1 << 64) if x >> 63 else x


def _field(f, w):
    src, shift, bits = f[0], f[1], f[2]
    return (w[src] >> shift) & ((1 << bits) - 1)


def encode(order, w):
    """The order lanes of output words w, as unsigned words (order_lane() tuples)."""
    out = []
    for (src, shift, bits, sx, desc, _f64) in order:
        v = _field((src, shift, bits), w)
        if sx and bits < 64 and (v >> (bits - 1)) & 1:
            v |= (M64 << bits) & M64
        v ^= ((1 << 63) if sx else 0) ^ (M64 if desc else 0)
        out.append(v)
    return out + [0] * (3 - len(out))


def accumulate(rows, as_of, keys=None):
    """{(w0, w1): count at as_of} of R32 rows (sorted by the pair), optionally only keys in `keys`."""
    w = aref.words(rows, 32) if len(rows) else np.zeros((0, 4), np.uint64)
    acc = {}
    for r in w:
        if int(r[2]) <= as_of and (keys is None or int(r[0]) in keys):
            p = (int(r[0]), int(r[1]))
            acc[p] = (acc.get(p, 0) + _s64(r[3]))
    return sorted((p, c) for p, c in acc.items() if c != 0)


def pairs_to_rows(plan, pairs):
    """(kept rows [(output words (3), copies)] or None, failure or None) of the plan over the accumulated pairs."""
    out = []
    for (key, val), c in pairs:
        w = [key, val, 0]
        upd, err, mv = M.evaluate(dict(plan, temporal=[]), w, 0, c, M64)
        if err:
            code, pay = err[0][0], err[0][1]
            return None, (ERR_MFP, (code, pay & M64, key, val))
        if not upd:
            continue
        if c < 0:
            return None, (ERR_RETRACTION, (key, val, c & M64, 0))
        ow = [x & M64 for x in M.project(plan, w, mv)]
        out.append((ow + [0] * (3 - len(ow)), c))
    return out, None


def finish(rows, out_words, as_of, order=(), limit=None, offset=0, project=()):
    """The finishing: rows equal before the projection merged, ordered, cut in units, projected."""
    merged = {}
    for w, c in rows:
        merged[tuple(w)] = merged.get(tuple(w), 0) + c
    ordered = sorted(merged.items(), key=lambda wc: encode(order, list(wc[0])) + list(wc[0]))
    end = None if limit is None else offset + limit
    out, at = [], 0
    for w, c in ordered:
        s, e = at, at + c
        at = e
        a, b = max(s, offset), e if end is None else min(e, end)
        if b > a:
            pw = list(w[:out_words])
            if any(project):
                pw = [0] * out_words
                for k, fl in enumerate(project):
                    for f in fl:
                        pw[k] |= (_field(f, list(w)) << f[3]) & M64
            out.append(pw + [as_of, b - a])
        if end is not None and at >= end:
            break
    return np.array(out, dtype=np.uint64).reshape(-1, out_words + 2)


def peek(ok_rows, plan, as_of, out_words=2, order=(), limit=None, offset=0, project=(), literals=None, err_rows=None,
         max_rows=0, ok_upper=EMPTY, err_upper=EMPTY, since=0):
    """("rows", array of (w0, w1[, w2], as_of, copies)), ("not_ready", None) or ("error", (kind, 4 detail words))."""
    if (ok_upper != EMPTY and ok_upper <= as_of) or (err_rows is not None and err_upper != EMPTY and
                                                     err_upper <= as_of):
        return ("not_ready", None)
    if since > as_of:
        return ("error", (ERR_SINCE, (since, as_of, 0, 0)))
    if err_rows is not None:
        for (code, pay), c in accumulate(err_rows, as_of):
            if c > 0:
                return ("error", (ERR_ERRS_ROW, (code, pay, 0, 0)))
            return ("error", (ERR_ERRS_RETRACTION, (code, pay, c & M64, 0)))
    keys = None if literals is None else set(int(x) for x in literals)
    rows, fail = pairs_to_rows(plan, accumulate(ok_rows, as_of, keys))
    if fail:
        return ("error", fail)
    out = finish(rows, out_words, as_of, order, limit, offset, project)
    if max_rows and len(out) > max_rows:
        return ("error", (ERR_TOO_LARGE, (len(out), 0, 0, 0)))
    return ("rows", out)
