"""Pin tests/arrangement_ref.py before the GPU suite compares the kernels with it: consolidate, seal
and merge equal the CPU oracle's byte for byte at the widths the oracle has, the wide diff vectors
sum as the lanes restatement sums them (i128 carries and wrap-around included), and check_index
accepts both run-length encodings of a batch's index and rejects every broken one."""
import json
import os

import numpy as np
import pytest

import arrangement_ref as ref
from lanes_oracle import ReduceLanes

HERE = os.path.dirname(os.path.abspath(__file__))
M64 = (1 << 64) - 1
DT = {16: "R16", 32: "R32", 40: "R40", 64: "ROUT", 80: "RACC"}


def random_words(rng, rb, n, key_range=40, time_range=6, big_diffs=False):
    """Rows of width rb with clumped keys (so that sums happen); diffs small or near +-2^63."""
    nw, nk, nd, tw = ref.LAYOUT[rb]
    w = np.zeros((n, nw), dtype=np.uint64)
    for k in range(nk):
        w[:, k] = rng.integers(0, key_range if k != tw else time_range, size=n, dtype=np.uint64)
    if big_diffs:
        d = rng.choice(np.array([1, -1, (1 << 62), -(1 << 62), (1 << 63) - 1, -(1 << 63)], dtype=np.int64), size=n)
    else:
        d = rng.integers(-3, 4, size=n, dtype=np.int64)
    w[:, nk] = d.view(np.uint64)
    if nd >= 8:
        for l in range(ref.lanes(nd)):
            b = nk + 1 + 6 * l
            w[:, b] = rng.integers(-2, 3, size=n, dtype=np.int64).view(np.uint64)
            w[:, b + 1] = rng.integers(0, 1 << 64, size=n, dtype=np.uint64) if big_diffs else rng.integers(0, 5, size=n, dtype=np.uint64)
            w[:, b + 2] = rng.integers(-2, 2, size=n, dtype=np.int64).view(np.uint64)
            for j in (3, 4, 5):
                w[:, b + j] = rng.integers(0, 2, size=n, dtype=np.uint64)
    return w


def oracle_rows(oracle, w, rb):
    return ref.as_rows(w, getattr(oracle, DT[rb]))


@pytest.mark.parametrize("rb", [16, 32, 40, 64, 80])
@pytest.mark.parametrize("big", [False, True])
def test_consolidate_matches_oracle(oracle, rb, big):
    rng = np.random.default_rng(rb + big)
    for n in (0, 1, 2, 7, 100, 5000):
        w = random_words(rng, rb, n, key_range=3 if n < 100 else 40, big_diffs=big)
        got = ref.consolidate(w)
        want = oracle.consolidate(oracle_rows(oracle, w, rb))
        assert got.tobytes() == want.tobytes(), (rb, n)


def test_consolidate_drops_sums_that_wrap_to_zero(oracle):
    w = np.zeros((3, 4), dtype=np.uint64)
    w[:, 3] = np.array([(1 << 63) - 1, (1 << 63) - 1, 2], dtype=np.uint64)  # 2^64 = 0
    assert len(ref.consolidate(w)) == 0
    assert len(oracle.consolidate(oracle_rows(oracle, w, 32))) == 0


@pytest.mark.parametrize("rb", [32, 80])
def test_seal_matches_oracle_batcher(oracle, rb):
    rng = np.random.default_rng(3 + rb)
    ob = oracle.Batcher(rb)
    stash = np.zeros((0, ref.LAYOUT[rb][0]), dtype=np.uint64)
    for step, upper in enumerate([2, 2, 5, 9, ref.FRONTIER_EMPTY]):
        w = random_words(rng, rb, 400, time_range=10, big_diffs=step % 2 == 1)
        ob.push(oracle_rows(oracle, w, rb))
        stash = np.concatenate([stash, w])
        shipped, kept, frontier = ref.seal(stash, upper)
        got = ob.seal(upper)
        assert shipped.tobytes() == got.rows().tobytes(), (rb, upper)
        assert frontier == ob.frontier()
        stash = kept


@pytest.mark.parametrize("rb", [32, 80])
def test_merge_matches_oracle_batches(oracle, rb):
    rng = np.random.default_rng(5 + rb)
    tw = ref.LAYOUT[rb][3]
    for since in (0, 3, 7, 100, ref.FRONTIER_EMPTY):
        a = ref.consolidate(random_words(rng, rb, 300, time_range=8))
        b = ref.consolidate(random_words(rng, rb, 200, time_range=8, big_diffs=True))
        b[:, tw] += np.uint64(4)
        oa = oracle.Batch.build(oracle_rows(oracle, a, rb), 0, 12)
        obb = oracle.Batch.build(oracle_rows(oracle, b, rb), 12, 20)
        want = oa.merge(obb, since).rows()
        assert ref.merge(a, b, since).tobytes() == want.tobytes(), (rb, since)


def test_golden_merger_vectors():
    fx = json.load(open(os.path.join(HERE, "golden", "consolidate_vectors.json")))
    for case in fx["merger_keyval"]["cases"]:
        chains = [np.array([r for chunk in case[c] for r in chunk], dtype=np.int64).reshape(-1, 4) for c in ("chain1", "chain2")]
        got = ref.merge(chains[0].view(np.uint64), chains[1].view(np.uint64), 0)
        want = np.array(case["expected"], dtype=np.int64).reshape(-1, 4).view(np.uint64)
        assert got.tobytes() == want.tobytes(), case["name"]


def _vec(words_row, c):
    v = [ref_s64(int(words_row[2]))]
    for l in range(c):
        x = [int(t) for t in words_row[3 + 6 * l : 9 + 6 * l]]
        v.append([ref_s64(x[0]), x[1] | (x[2] << 64), ref_s64(x[3]), ref_s64(x[4]), ref_s64(x[5])])
    return v


def ref_s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


@pytest.mark.parametrize("rb", [80, 128, 224, 416])
def test_wide_diff_sums_match_lanes_restatement(rb):
    """Per (key, time), the summed diff vector and its zero test equal ReduceLanes._add / _is_zero:
    carries out of acc_lo, acc_hi wrapping past 2^127 and 2^128, vectors that cancel exactly."""
    c = {80: 1, 128: 2, 224: 4, 416: 8}[rb]
    nw = ref.LAYOUT[rb][0]
    rng = np.random.default_rng(rb)
    w = random_words(rng, rb, 3000, key_range=30, time_range=3, big_diffs=True)
    # a group whose acc_lo carries many times and whose acc_hi wraps
    extra = np.zeros((6, nw), dtype=np.uint64)
    extra[:, 0], extra[:, 1], extra[:, 2] = 1000, 1, 1
    for l in range(c):
        extra[:, 4 + 6 * l] = M64
        extra[:, 5 + 6 * l] = np.uint64((1 << 63) - 1)
    # a group that cancels to exactly zero (every lane word included)
    cancel = random_words(rng, rb, 5, big_diffs=True)
    cancel[:, 0], cancel[:, 1] = 1001, 0
    neg = cancel.copy()
    neg[:, 2:] = (-(neg[:, 2:].view(np.int64))).view(np.uint64)  # componentwise two's complement
    for l in range(c):  # the i128 negation borrows across the words
        lo, hi = cancel[:, 4 + 6 * l], cancel[:, 5 + 6 * l]
        neg[:, 4 + 6 * l] = (-lo.view(np.int64)).view(np.uint64)
        neg[:, 5 + 6 * l] = (~hi) + (lo == 0).astype(np.uint64)
    w = np.concatenate([w, extra, cancel, neg])
    got = {(int(r[0]), int(r[1])): r for r in ref.consolidate(w)}
    sums = {}
    for r in w:
        ReduceLanes._add(sums.setdefault((int(r[0]), int(r[1])), [0] + [[0] * 5 for _ in range(c)]), _vec(r, c))
    assert (1001, 0) not in got and ReduceLanes._is_zero(sums[(1001, 0)])
    assert sums[(1000, 1)][1][1] >> 64 != 0  # the carry case did carry
    for k, v in sums.items():
        if ReduceLanes._is_zero(v):
            assert k not in got, k
        else:
            assert _vec(got[k], c) == v, k


def _sorted_rows(rng, n, keys):
    w = np.zeros((n, 4), dtype=np.uint64)
    w[:, 0] = rng.choice(keys, size=n)
    w[:, 1] = np.arange(n, dtype=np.uint64)
    w[:, 3] = 1
    return ref.sort_rows(w)


@pytest.mark.parametrize("run_limit", [65, ref.RUN_SAT])
def test_check_index_accepts_both_run_encodings(run_limit):
    rng = np.random.default_rng(9)
    keys = np.concatenate([rng.integers(0, 1 << 64, size=300, dtype=np.uint64), np.array([0, M64], dtype=np.uint64)])
    w = _sorted_rows(rng, 6000, keys)
    w = np.concatenate([w, np.tile(np.array([[M64 - 1, 0, 0, 1]], dtype=np.uint64), (1500, 1))])  # a run past 1024
    w = ref.sort_rows(w)
    slots = ref.build_index(w, run_limit)
    _, first, run = ref.key_runs(w)
    ref.check_index(w, slots, len(slots) - 1, len(first), min(int(run.max()), 1024))


def test_check_index_rejects_broken_tables():
    rng = np.random.default_rng(10)
    w = _sorted_rows(rng, 500, rng.integers(0, 1 << 64, size=400, dtype=np.uint64))
    slots = ref.build_index(w, ref.RUN_SAT)
    mask = len(slots) - 1
    _, first, run = ref.key_runs(w)
    nk, longest = len(first), int(run.max())
    occ = np.flatnonzero(slots[:, 1])

    def broken(f):
        s = slots.copy()
        f(s)
        with pytest.raises(AssertionError):
            ref.check_index(w, s, mask, nk, longest)

    broken(lambda s: s.__setitem__((occ[0], 1), s[occ[0], 1] + np.uint64(1)))  # first row off by one
    broken(lambda s: s.__setitem__((occ[1], 1), (s[occ[1], 1] & np.uint64(ref.SLOT_ROW_MASK)) | np.uint64(999 << 44)))
    broken(lambda s: s.__setitem__(occ[2], 0))  # a key is missing
    # a probe chain broken by an empty slot: move a displaced key one slot further out
    home = (ref.mix64(slots[occ, 0]) & np.uint64(mask)).astype(np.int64)
    disp = occ[np.flatnonzero(home != occ)]
    assert len(disp), "400 keys in 1024 slots collide"
    p = int(disp[0])
    q = (p + 1) & mask
    while slots[q, 1] != 0:
        q = (q + 1) & mask

    def move(s):
        s[q], s[p] = s[p].copy(), 0

    broken(move)
    with pytest.raises(AssertionError):
        ref.check_index(w, slots, mask, nk + 1, longest)
    with pytest.raises(AssertionError):
        ref.check_index(w, slots, mask, nk, longest + 1)
    ref.check_index(w, slots, mask, nk, longest)
