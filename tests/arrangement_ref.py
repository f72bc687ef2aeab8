"""Plain reference of the arrangement kernels' arithmetic at every row width (test infrastructure).

Consolidation, seal and merge of update rows, and the invariants of a batch's hash index, restated
on raw u64 words with NumPy and Python ints.  The layout of every width comes from one table that
restates `RowT` (materialize_b200/csrc/common.cuh): NW words per row, the first NK of them the sort
key, then ND diff words; TW is the time word (-1: none).  The diff arithmetic is `diff_add` /
`diff_is_zero` of the same file:

  ND = 1, 2   word 0 is the diff and wraps at 64 bits (ND = 2: word 1 is a pad word, left alone)
  ND >= 8     word 0 is the total (wraps at 64 bits), then (ND - 1) // 6 lanes of
              (non_nulls, acc_lo, acc_hi, pos_infs, neg_infs, nans): (acc_lo, acc_hi) is an i128
              that wraps at 128 bits, every other word wraps at 64 bits; the last word is a pad

A diff vector is zero when word 0 is (ND <= 2), when words 0..6 are (ND = 8: the pad is ignored),
or when every word is (ND > 8).  Inputs keep their pad words at 0.
"""
import numpy as np

FRONTIER_EMPTY = (1 << 64) - 1
M32 = np.uint64(0xFFFFFFFF)

# row bytes -> (NW, NK, ND, TW), as RowT<RB>
LAYOUT = {
    16: (2, 1, 1, -1),
    32: (4, 3, 1, 2),
    40: (5, 4, 1, 3),
    64: (8, 6, 2, 5),
    80: (10, 2, 8, 1),
    128: (16, 2, 14, 1),
    224: (28, 2, 26, 1),
    416: (52, 2, 50, 1),
}
RUN_SAT = 1024  # the longest key run a batch reports saturates here
SLOT_ROW_MASK = (1 << 44) - 1


def words(rows, row_bytes=None):
    """(n, NW) u64 view of a row array (structured rows or a u64 matrix)."""
    a = np.ascontiguousarray(rows)
    rb = row_bytes or (a.dtype.itemsize if a.dtype.names else a.shape[-1] * 8)
    return a.view(np.uint64).reshape(-1, LAYOUT[rb][0])


def as_rows(w, dtype):
    return np.ascontiguousarray(w, dtype=np.uint64).view(dtype).reshape(-1)


def lanes(nd):
    return (nd - 1) // 6 if nd >= 8 else 0


def sort_rows(w):
    """Rows ordered by their key words, compared as unsigned and in order (stable)."""
    nk = LAYOUT[w.shape[1] * 8][1]
    if len(w) == 0:
        return w.copy()
    order = np.lexsort([w[:, k] for k in reversed(range(nk))])
    return w[order]


def _seg_sum(col, starts):
    return np.add.reduceat(col, starts) if len(col) else col[:0]


def _seg_sum_i128(lo, hi, starts):
    """Segment sums of the i128 (lo, hi) mod 2^128, vectorised over 32-bit halves of lo."""
    a = _seg_sum(lo & M32, starts)  # < 2^32 per row: exact for up to 2^32 rows
    b = _seg_sum(lo >> np.uint64(32), starts)
    c = (a >> np.uint64(32)) + b
    out_lo = (a & M32) | ((c & M32) << np.uint64(32))
    out_hi = _seg_sum(hi, starts) + (c >> np.uint64(32))
    return out_lo, out_hi


def is_zero(w):
    """diff_is_zero of every row of `w`."""
    _, nk, nd, _ = LAYOUT[w.shape[1] * 8]
    d = w[:, nk:]
    if nd <= 2:
        return d[:, 0] == 0
    if nd == 8:
        return ~np.any(d[:, :7], axis=1)
    return ~np.any(d, axis=1)


def consolidate(rows):
    """Sort by the key words, sum the diffs of equal keys, drop zeros: (m, NW) u64."""
    w = sort_rows(words(rows))
    nw, nk, nd, _ = LAYOUT[w.shape[1] * 8]
    if len(w) == 0:
        return w
    head = np.ones(len(w), dtype=bool)
    head[1:] = np.any(w[1:, :nk] != w[:-1, :nk], axis=1)
    starts = np.flatnonzero(head)
    out = w[starts].copy()
    with np.errstate(over="ignore"):
        out[:, nk] = _seg_sum(w[:, nk], starts)
        for l in range(lanes(nd)):
            b = nk + 1 + 6 * l
            for j in (0, 3, 4, 5):
                out[:, b + j] = _seg_sum(w[:, b + j], starts)
            out[:, b + 1], out[:, b + 2] = _seg_sum_i128(w[:, b + 1], w[:, b + 2], starts)
    return out[~is_zero(out)]


def advance(rows, since):
    """Times advanced to max(time, since); FRONTIER_EMPTY (the empty antichain) changes nothing."""
    w = words(rows).copy()
    tw = LAYOUT[w.shape[1] * 8][3]
    if tw >= 0 and since != FRONTIER_EMPTY:
        np.maximum(w[:, tw], np.uint64(since), out=w[:, tw])
    return w


def merge(a, b, since):
    """Batch::Merger: consolidate(advance(a ++ b, since))."""
    return consolidate(advance(np.concatenate([words(a), words(b)]), since))


def seal(stash, upper):
    """Batcher::seal: (shipped rows, kept rows, frontier).  Rows with time < upper ship, the rest
    stay; the frontier is the smallest kept time, or FRONTIER_EMPTY when nothing stays."""
    w = consolidate(stash)
    tw = LAYOUT[w.shape[1] * 8][3]
    if upper == FRONTIER_EMPTY or tw < 0:
        return w, w[:0], FRONTIER_EMPTY
    ship = w[:, tw] < np.uint64(upper)
    kept = w[~ship]
    return w[ship], kept, int(kept[:, tw].min()) if len(kept) else FRONTIER_EMPTY


# ------------------------------------------------------------------ hash index
def mix64(k):
    """The index's hash (murmur3 finalizer, mix64 in common.cuh), on a u64 array."""
    k = np.asarray(k, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xFF51AFD7ED558CCD)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xC4CEB9FE1A85EC53)
        k ^= k >> np.uint64(33)
    return k


def key_runs(rows):
    """(distinct keys, first row of each, run length of each) of sorted rows (key = word 0)."""
    keys = words(rows)[:, 0]
    if len(keys) == 0:
        z = np.zeros(0, dtype=np.uint64)
        return z, z.astype(np.int64), z.astype(np.int64)
    head = np.ones(len(keys), dtype=bool)
    head[1:] = keys[1:] != keys[:-1]
    first = np.flatnonzero(head)
    run = np.diff(np.append(first, len(keys)))
    return keys[first], first, run


def build_index(rows, run_limit, mask=None):
    """An index as a builder would leave it: slots (S, 2) u64 {key, meta}, keys inserted in order by
    linear probing.  A run shorter than `run_limit` is stored in meta, a longer one as 0."""
    keys, first, run = key_runs(rows)
    if mask is None:
        s = 2
        while s < 2 * len(words(rows)):
            s <<= 1
        mask = s - 1
    slots = np.zeros((mask + 1, 2), dtype=np.uint64)
    for k, f, r, h in zip(keys.tolist(), first.tolist(), run.tolist(), (mix64(keys) & np.uint64(mask)).tolist()):
        while slots[h, 1] != 0:
            h = (h + 1) & mask
        slots[h] = (k, (f + 1) | ((r if r < run_limit else 0) << 44))
    return slots


def check_index(rows, slots, mask, n_keys, longest):
    """Assert the invariants of a batch's hash index over its sorted rows; returns the table's
    longest probe distance.  Run lengths may be encoded by any builder: meta >> 44 is 0 or the run."""
    slots = np.ascontiguousarray(slots).view(np.uint64).reshape(-1, 2)
    size = mask + 1
    keys, first, run = key_runs(rows)
    n_rows = len(words(rows))
    assert size & mask == 0 and size >= 2, f"table size {size} is not a power of two"
    assert len(slots) == size, (len(slots), size)
    assert size >= 2 * len(keys), f"{size} slots for {len(keys)} keys: load factor above 1/2"
    assert n_keys == len(keys), f"distinct keys {n_keys}, rows have {len(keys)}"
    want_longest = min(int(run.max()), RUN_SAT) if len(run) else 0
    assert longest == want_longest, f"longest run {longest}, rows have {want_longest}"
    occ = slots[:, 1] != 0
    assert int(occ.sum()) == len(keys), f"{int(occ.sum())} occupied slots for {len(keys)} keys"
    if len(keys) == 0:
        return 0
    pos = np.flatnonzero(occ)
    skeys, meta = slots[pos, 0], slots[pos, 1]
    order = np.argsort(skeys, kind="stable")
    skeys, meta, pos = skeys[order], meta[order], pos[order]
    assert np.array_equal(skeys, keys), "the occupied slots do not hold exactly the distinct keys"
    row = (meta & np.uint64(SLOT_ROW_MASK)).astype(np.int64) - 1
    bad = np.flatnonzero(row != first)
    assert len(bad) == 0, f"key {int(keys[bad[0]])}: slot says first row {int(row[bad[0]])}, rows say {int(first[bad[0]])}"
    rl = (meta >> np.uint64(44)).astype(np.int64)
    bad = np.flatnonzero((rl != 0) & (rl != run))
    assert len(bad) == 0, f"key {int(keys[bad[0]])}: slot says run {int(rl[bad[0]])}, rows say {int(run[bad[0]])}"
    assert int(first.max()) < n_rows
    # linear probing from mix64(key) & mask must reach the key's slot over occupied slots only:
    # the probe distance is below the length of the occupied stretch that ends at the slot
    empty0 = int(np.flatnonzero(~occ)[0])
    rot = np.roll(occ, -empty0)
    idx = np.arange(size)
    last_empty = np.maximum.accumulate(np.where(rot, 0, idx))
    stretch = np.roll(idx - last_empty, empty0)  # occupied slots ending at each slot
    home = (mix64(keys) & np.uint64(mask)).astype(np.int64)
    dist = (pos - home) & mask
    bad = np.flatnonzero(dist >= stretch[pos])
    assert len(bad) == 0, f"key {int(keys[bad[0]])}: an empty slot breaks its probe chain"
    return int(dist.max())
