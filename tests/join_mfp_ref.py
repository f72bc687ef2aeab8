"""Plain reference of the probes with an MfpPlan closure (mzgpu_join_closure; test infrastructure).

It composes `probe_ref` (the matches in probe order, their times and diffs) with `mfp_map_oracle` (the plan
evaluated without temporal bounds, then projected): per match (key, va, vb) at (t, d) one output row, or one
error row (code, payload, t, d).  Output rows keep probe order; error rows are consolidated.
"""
import numpy as np

import arrangement_ref as aref
import mfp_map_oracle as M
import probe_ref as P

M64 = (1 << 64) - 1


def _s64(x):
    x = int(x)
    return x - (1 << 64) if x >> 63 else x


def probe_mfp(stream, batches, mode, plan, meet=0, swap_vals=False):
    """(out rows (n, out words), consolidated error rows (m, 4)) of the probe with `plan` as the closure."""
    s = P._w(stream)
    bs = [P._w(b) for b in batches]
    si, bi, ri = P.matches(s, bs)
    allb = np.concatenate(bs) if bs else np.zeros((0, 4), dtype=np.uint64)
    off = np.cumsum([0] + [len(b) for b in bs])[:-1]
    nw = 2 + len(plan["fields"])
    out, errs = [], []
    for a, b, r in zip(si, bi, ri):
        st, lk = s[a], allb[off[b] + r]
        t1, t2 = int(st[2]), int(lk[2])
        if (mode == P.LE and not t2 <= t1) or (mode == P.LT and not t2 < t1):
            continue
        t = max(t1, t2, meet) if mode == P.JOIN else t1
        d = (int(st[3]) * int(lk[3])) & M64
        va, vb = (int(lk[1]), int(st[1])) if swap_vals else (int(st[1]), int(lk[1]))
        w = [int(st[0]), va, vb]
        upd, err, mv = M.evaluate(dict(plan, temporal=[]), w, t, _s64(d), M64)
        if err:
            c, p, _, _ = err[0]
            errs.append((c, p & M64, t, d))
        elif upd:
            out.append([x & M64 for x in M.project(plan, w, mv)] + [t, d])
    o = np.array(out, dtype=np.uint64).reshape(-1, nw)
    e = aref.consolidate(np.array(errs, dtype=np.uint64).reshape(-1, 4)) if errs else np.zeros((0, 4), np.uint64)
    return o, e


def join_core_push(batch_rows, other_batches, side, cap, plan):
    """One join_core work item with an MfpPlan closure: (consolidated rows, consolidated errors)."""
    o, e = probe_mfp(batch_rows, other_batches, P.JOIN, plan, cap, swap_vals=side == 1)
    return aref.consolidate(o) if len(o) else o, e


def lower_equivalences(classes):
    """ready_equivalences as leading predicates: [e0, e1, ..., en] -> CMP_EQ(e0, e1), ..., CMP_EQ(e0, en)."""
    return [list(c[0]) + list(e) + [(M.O.HOP_CMP, 0, 0, 0, 0, 0)] for c in classes for e in c[1:]]


def join_closure_apply(classes, plan, w):
    """JoinClosure::apply transcribed: each class's expressions are evaluated in order and compared with the first;
    the first error or mismatch ends the row; then the plan.  (error, passed)."""
    for c in classes:
        e, p, v0 = M.run(c[0], plan["consts"], w, [])
        if e:
            return (e, p), False
        for x in c[1:]:
            e, p, v = M.run(x, plan["consts"], w, [])
            if e:
                return (e, p), False
            if v != v0:
                return None, False
    upd, err, _ = M.evaluate(dict(plan, temporal=[]), w, 0, 1, M64)
    if err:
        return (err[0][0], err[0][1]), False
    return None, bool(upd)
