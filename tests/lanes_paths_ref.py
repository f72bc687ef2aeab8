"""Vectorised NumPy expectations of the multi-column reduces for batches too large for the Python
restatements (tests/lanes_oracle.py, tests/monotonic_oracle.py): the two-pass cases, where every
activation has at most one row per key.  Written from the definitions in include/mzgpu.h and pinned
to the restatements by tests/test_ref_lanes_paths.py.

Lanes (mzgpu_reduce_lanes_*): a row's diff vector is (total, C x (non_nulls, acc_lo, acc_hi, pos_infs,
neg_infs, nans)); an I64 lane accumulates diff x the (sign-extended) field as an i128, an F64 lane
diff x trunc(x * 2^24) (the values used here stay below 2^62 after scaling, so the saturating cast never
saturates) or its infinity / NaN count.  The output row of a key is (key, C x (count, sum_lo, sum_hi),
flags, time, diff): bit 2l is set when total > 0 and lane l's accumulation is zero (its SUM is NULL,
sum words 0), bit 2l+1 when total == 0 and the lane's accumulation is not.

Monotonic MIN / MAX (mzgpu_reduce_monotonic_*): lane word = field (sign-extended when asked) ^ 2^63 for
a signed lane, complemented for MIN; a key's accumulation is the per-word max, and its output row is
(key, C decoded values, time, diff).

An activation emits, per key of its batch, the retraction of the key's previous row and its new row when
they differ (both at the batch's time), so a key's corrections are at most two rows; they are ordered as
the kernels leave them: keys ascending, a key's rows by their words after the key."""
import numpy as np

M64 = (1 << 64) - 1
I64, F64 = 0, 1
AGG_MIN, AGG_MAX = 4, 5
LANE_ROW_BYTES = {1: (80, 64), 2: (128, 96), 4: (224, 144), 8: (416, 240)}  # class -> (arrangement, output)
MONO_ROW_BYTES = {4: (48, 56), 8: (112, 88)}
QNAN, PINF, NINF = 0x7FF8000000000000, 0x7FF0000000000000, 0xFFF0000000000000
U = np.uint64


def lane_class(n_lanes):
    return next(c for c in (1, 2, 4, 8) if c >= n_lanes)


def mono_class(n_lanes):
    return 4 if n_lanes <= 4 else 8


def field(w, lane, extend):
    """The lane's bit-field of every row of w ((n, in_words) u64), sign-extended when `extend` and asked."""
    _, src, shift, bits, sx = lane
    v = w[:, src] >> U(shift)
    if bits < 64:
        v = v & U((1 << bits) - 1)
        if sx and extend:
            neg = ((v >> U(bits - 1)) & U(1)) == U(1)
            v = np.where(neg, v | U(M64 ^ ((1 << bits) - 1)), v)
    return v


# ------------------------------------------------------------------ lanes
def _i128(x, neg):
    """(lo, hi) of an i128 whose low word is x and which is negative where `neg`."""
    return x, np.where(neg, U(M64), U(0))


def lane_vectors(w, lanes):
    """The exploded diff vector of every row ((n, 1 + 6 C) u64, C the lanes' class); diffs must be +-1."""
    n, iw = w.shape
    cls = lane_class(len(lanes))
    d = w[:, iw - 1].view(np.int64)
    assert np.all(np.abs(d) == 1)
    neg_d = d < 0
    out = np.zeros((n, 1 + 6 * cls), dtype=np.uint64)
    out[:, 0] = w[:, iw - 1]
    for l, lane in enumerate(lanes):
        v = field(w, lane, lane[0] == I64)
        o = out[:, 1 + 6 * l : 7 + 6 * l]
        o[:, 0] = w[:, iw - 1]
        if lane[0] == I64:
            sv = v.view(np.int64)
            x = np.where(neg_d, U(0) - v, v)  # diff x value mod 2^64
            o[:, 1], o[:, 2] = _i128(x, np.where(neg_d, sv > 0, sv < 0))
        else:
            f = v.view(np.float64)
            nan, pinf, ninf = np.isnan(f), f == np.inf, f == -np.inf
            fin = ~(nan | pinf | ninf)
            y = np.where(fin, f, 0.0) * 16777216.0
            assert np.all(np.abs(y) < 2.0**62), "outside the non-saturating range of this reference"
            fx = np.trunc(y).astype(np.int64) * d
            o[:, 1], o[:, 2] = _i128(fx.view(np.uint64), fx < 0)
            for k, m in ((3, pinf), (4, ninf), (5, nan)):
                o[:, k] = np.where(m, w[:, iw - 1], U(0))
    return out


def vec_add(a, b):
    """Component-wise sum of diff vectors: i64 words wrap, each lane's (acc_lo, acc_hi) adds as an i128."""
    s = a + b
    for l in range((a.shape[1] - 1) // 6):
        lo = 2 + 6 * l
        s[:, lo + 1] += (s[:, lo] < a[:, lo]).astype(np.uint64)
    return s


def lane_finalize(vec, lanes):
    """(n, 3 C + 1) u64: C x (count, sum_lo, sum_hi) and the flags of each vector (rows that exist)."""
    n = len(vec)
    cls = lane_class(len(lanes))
    total = vec[:, 0].view(np.int64)
    out = np.zeros((n, 3 * cls + 1), dtype=np.uint64)
    flags = np.zeros(n, dtype=np.uint64)
    for l, lane in enumerate(lanes):
        nn, lo, hi, p, ng, nan = (vec[:, 1 + 6 * l + k] for k in range(6))
        zero = (nn | lo | hi | p | ng | nan) == U(0)
        null = (total > 0) & zero
        err = (total == 0) & ~zero
        if lane[0] == I64:
            s_lo, s_hi = lo, hi
        else:
            assert np.all(hi == np.where(lo.view(np.int64) < 0, U(M64), U(0))), "sum past i64 in this reference"
            fin = (lo.view(np.int64).astype(np.float64) / 16777216.0).view(np.uint64)
            p, ng, nan = p.view(np.int64), ng.view(np.int64), nan.view(np.int64)
            s_lo = np.where((nan > 0) | ((p > 0) & (ng > 0)), U(QNAN),
                            np.where(p > 0, U(PINF), np.where(ng > 0, U(NINF), fin)))
            s_hi = np.zeros(n, dtype=np.uint64)
        out[:, 3 * l] = nn
        out[:, 3 * l + 1] = np.where(null, U(0), s_lo)
        out[:, 3 * l + 2] = np.where(null, U(0), s_hi)
        flags |= (null.astype(np.uint64) | (err.astype(np.uint64) << U(1))) << U(2 * l)
    out[:, 3 * cls] = flags
    return out


def _corrections(keys, old, had, new, has, t, out_words):
    """Per key (ascending): -old where had, +new where has, unless both exist and are equal; a key's two
    rows ordered by their value words (they share the time).  old / new: (n, V) value words."""
    nv = old.shape[1]
    same = had & has & np.all(old == new, axis=1)
    ret, add = had & ~same, has & ~same
    diff = old != new
    first = np.argmax(diff, axis=1)
    rows_ = np.arange(len(keys))
    new_first = diff[rows_, first] & (new[rows_, first] < old[rows_, first])

    def block(vals, d):
        b = np.zeros((len(keys), out_words), dtype=np.uint64)
        b[:, 0] = keys
        b[:, 1 : 1 + nv] = vals
        b[:, 1 + nv] = t
        b[:, 2 + nv] = U(d & M64)
        return b

    r_b, a_b = block(old, -1), block(new, 1)
    # slot 0 / slot 1 of each key, then drop the rows that are not emitted
    lo = np.where(new_first[:, None], a_b, r_b)
    hi = np.where(new_first[:, None], r_b, a_b)
    keep_lo = np.where(new_first, add, ret)
    keep_hi = np.where(new_first, ret, add)
    both = np.stack([lo, hi], axis=1).reshape(-1, out_words)
    keep = np.stack([keep_lo, keep_hi], axis=1).reshape(-1)
    return both[keep]


def lanes_activation(keys, prior, had, delta, t, lanes):
    """Output rows of one activation whose batch holds one (key, t) row per key, keys ascending:
    prior = the keys' accumulated vectors before it (had: the key had any), delta = the batch's vectors.
    Returns (rows, the accumulated vectors after it)."""
    cls = lane_class(len(lanes))
    after = vec_add(prior, delta)
    has = np.any(after != 0, axis=1)
    had = had & np.any(prior != 0, axis=1)
    old, new = lane_finalize(prior, lanes), lane_finalize(after, lanes)
    return _corrections(keys, old, had, new, has, t, LANE_ROW_BYTES[cls][1] // 8), after


def lanes_arrangement(keys, times, vecs):
    """Arrangement rows (key, time, vector, zero padding) of (key, time) rows, one per entry, sorted."""
    cls = (vecs.shape[1] - 1) // 6
    w = np.zeros((len(keys), LANE_ROW_BYTES[cls][0] // 8), dtype=np.uint64)
    w[:, 0], w[:, 1], w[:, 2 : 2 + vecs.shape[1]] = keys, times, vecs
    return w[np.lexsort([w[:, 1], w[:, 0]])]


# ------------------------------------------------------------------ monotonic MIN / MAX
def mono_xor(lanes):
    cls = mono_class(len(lanes))
    xm = np.zeros(cls, dtype=np.uint64)
    for l, (kind, _, _, _, sx) in enumerate(lanes):
        xm[l] = U(((1 << 63) if sx else 0) ^ (M64 if kind == AGG_MIN else 0))
    return xm


def mono_words(w, lanes):
    """The arrangement lane words of every row ((n, C) u64; unused lanes zero)."""
    cls = mono_class(len(lanes))
    xm = mono_xor(lanes)
    out = np.zeros((len(w), cls), dtype=np.uint64)
    for l, lane in enumerate(lanes):
        out[:, l] = field(w, lane, True) ^ xm[l]
    return out


def mono_activation(keys, prior, had, words, t, lanes):
    """Output rows of one activation whose batch holds one (key, t) row per key (all diffs positive), keys
    ascending: prior = the keys' accumulated lane words (had: the key is arranged), words = the batch's.
    Returns (rows, the accumulated words after it)."""
    cls = mono_class(len(lanes))
    after = np.where(had[:, None], np.maximum(prior, words), words)
    xm = mono_xor(lanes)
    xm[len(lanes):] = 0
    dec = lambda x: np.where(np.arange(cls) < len(lanes), x ^ xm, U(0))  # noqa: E731
    rows_ = _corrections(keys, dec(prior), had, dec(after), np.ones(len(keys), dtype=bool), t,
                         MONO_ROW_BYTES[cls][1] // 8)
    return rows_, after


def mono_arrangement(keys, times, words):
    cls = words.shape[1]
    w = np.zeros((len(keys), MONO_ROW_BYTES[cls][0] // 8), dtype=np.uint64)
    w[:, 0], w[:, 1], w[:, 2 : 2 + cls] = keys, times, words
    return w[np.lexsort([w[:, 1], w[:, 0]])]


# ------------------------------------------------------------------ the two-pass cases
# R40 lanes: bit-fields of val1 and val2 (signed and unsigned, at both ends of the word) and the float64
# lane of val2; the first n of them for n lanes.  two_pass_lanes maps them onto R32 input.
LANES8 = [(I64, 1, 0, 32, True), (I64, 2, 0, 64, False), (I64, 1, 32, 32, True), (F64, 2, 0, 64, False),
          (I64, 1, 63, 1, True), (I64, 2, 52, 12, False), (I64, 1, 0, 64, False), (I64, 2, 40, 9, True)]
MONO8 = [(AGG_MAX, 1, 0, 64, False), (AGG_MIN, 2, 0, 64, True), (AGG_MIN, 1, 8, 8, True), (AGG_MAX, 2, 63, 1, False),
         (AGG_MIN, 1, 0, 63, False), (AGG_MAX, 2, 0, 32, True), (AGG_MAX, 1, 40, 24, True), (AGG_MIN, 2, 3, 17, False)]


def two_pass_lanes(n_lanes, iw, mono=False):
    """The first n_lanes of MONO8 / LANES8, reading val1 only on R32 input (iw = 4)."""
    lanes = (MONO8 if mono else LANES8)[:n_lanes]
    return lanes if iw == 5 else [(k, 1, s, b, sx) for k, _, s, b, sx in lanes]


def spread_keys(n):
    """n distinct keys below 2^40 (an odd multiplier is a bijection), in no particular order."""
    return (np.arange(n, dtype=np.uint64) * U(0x9E3779B1)) & U(2**40 - 1)


def f64_words(rng, n):
    """float64 bits: multiples of 2^-24 below 2^36 in magnitude, -0.0, 1 in 64 of each of NaN, +inf, -inf."""
    x = rng.integers(-(2**60), 2**60, size=n, dtype=np.int64).astype(np.float64) / 2.0**24
    x[rng.random(n) < 1 / 64] = np.nan
    x[rng.random(n) < 1 / 64] = np.inf
    x[rng.random(n) < 1 / 64] = -np.inf
    x[rng.random(n) < 1 / 64] = -0.0
    return x.view(np.uint64)


def lanes_input(rng, n, iw):
    """Two activations over n distinct keys: one row per key at time 0 (diff 1), then at time 1 either its
    retraction (about half of the keys) or a row of fresh values.  The last value word is float64 bits
    (f64_words), the others any 64 bits.  Returns (first, second, back) as (n, iw) word arrays."""
    w1 = np.zeros((n, iw), dtype=np.uint64)
    w1[:, 0] = spread_keys(n)
    w1[:, 1 : iw - 3] = rng.integers(0, 2**64, size=(n, iw - 4), dtype=np.uint64)
    w1[:, iw - 3] = f64_words(rng, n)
    w1[:, iw - 1] = 1
    back = rng.random(n) < 0.5
    w2 = w1.copy()
    w2[:, iw - 2] = 1
    w2[:, iw - 1] = np.where(back, U(M64), U(1))
    w2[~back, 1 : iw - 3] = rng.integers(0, 2**64, size=(int((~back).sum()), iw - 4), dtype=np.uint64)
    w2[~back, iw - 3] = f64_words(rng, int((~back).sum()))
    return w1, w2, back


def mono_input(rng, n, iw):
    """Two activations over n distinct keys, all diffs positive: one row per key at time 0, then one at
    time 1 that repeats the key's values (no change) for about half of the keys and has fresh values for
    the others.  Returns (first, second, fresh)."""
    w1 = np.zeros((n, iw), dtype=np.uint64)
    w1[:, 0] = spread_keys(n)
    w1[:, 1 : iw - 2] = rng.integers(0, 2**64, size=(n, iw - 3), dtype=np.uint64)
    w1[:, iw - 1] = rng.integers(1, 3, size=n).astype(np.uint64)
    fresh = rng.random(n) < 0.5
    w2 = w1.copy()
    w2[:, iw - 2] = 1
    w2[fresh, 1 : iw - 2] = rng.integers(0, 2**64, size=(int(fresh.sum()), iw - 3), dtype=np.uint64)
    return w1, w2, fresh


def two_pass_expect(kind, lanes, w1, w2, lo=0, hi=None):
    """The outputs of the two activations of lanes_input / mono_input (kind "lanes" / "mono") for the keys of
    rank [lo, hi) in key order.  Returns (first, second, order): order[lo:hi] indexes those keys' rows."""
    order = np.argsort(w1[:, 0], kind="stable")[lo:hi]
    a, b = w1[order], w2[order]
    keys = a[:, 0]
    none = np.zeros(len(keys), dtype=bool)
    if kind == "lanes":
        d1, d2 = lane_vectors(a, lanes), lane_vectors(b, lanes)
        first, acc = lanes_activation(keys, np.zeros_like(d1), none, d1, 0, lanes)
        second, _ = lanes_activation(keys, acc, ~none, d2, 1, lanes)
    else:
        m1, m2 = mono_words(a, lanes), mono_words(b, lanes)
        first, acc = mono_activation(keys, np.zeros_like(m1), none, m1, 0, lanes)
        second, _ = mono_activation(keys, acc, ~none, m2, 1, lanes)
    return first, second, order


def two_pass_arrangement(kind, lanes, w1, w2, idx):
    """The arrangement rows of the keys of rows idx of the two activations (times 0 and 1)."""
    a, b = w1[idx], w2[idx]
    t = np.r_[np.zeros(len(idx), np.uint64), np.ones(len(idx), np.uint64)]
    keys = np.r_[a[:, 0], b[:, 0]]
    if kind == "lanes":
        return lanes_arrangement(keys, t, np.concatenate([lane_vectors(a, lanes), lane_vectors(b, lanes)]))
    return mono_arrangement(keys, t, np.concatenate([mono_words(a, lanes), mono_words(b, lanes)]))
