"""The vectorised expectations of tests/lanes_paths_ref.py, which check the two-pass cases of the
multi-column reduces on the GPU, pinned to the restatements they abbreviate (tests/lanes_oracle.py,
tests/monotonic_oracle.py): at a few thousand keys, with the same input shapes, every lane class and both
input widths, the outputs of both activations and the arrangement are equal byte for byte."""
import numpy as np
import pytest

import lanes_paths_ref as R
from lanes_oracle import ReduceLanes
from monotonic_oracle import ReduceMonotonic

N = 3000


def words(a):
    return np.ascontiguousarray(a).view(np.uint64).reshape(len(a), -1)


def same(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    if got.tobytes() != want.tobytes():
        bad = int(np.flatnonzero(np.any(got != want, axis=1))[0])
        raise AssertionError(f"row {bad} of {len(want)}: got {got[bad].tolist()}, want {want[bad].tolist()}")


@pytest.mark.parametrize("n_lanes", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("iw", [4, 5])
def test_lanes_expectation_equals_restatement(oracle, n_lanes, iw):
    lanes = R.two_pass_lanes(n_lanes, iw)
    w1, w2, back = R.lanes_input(np.random.default_rng(10 * n_lanes + iw), N, iw)
    o = ReduceLanes(oracle, lanes, 8 * iw)
    first, second, order = R.two_pass_expect("lanes", lanes, w1, w2)
    same(first, words(o.step(w1, 1)))
    same(second, words(o.step(w2, 2)))
    same(R.two_pass_arrangement("lanes", lanes, w1, w2, np.arange(N)), words(o.export()))
    # the shapes the expectation has to get right are there
    f = w1[:, iw - 3].view(np.float64)
    assert np.isnan(f).any() and np.isinf(f).any() and (np.signbit(f) & (f == 0)).any()
    assert back.any() and (~back).any()
    if n_lanes >= 4:  # the NaN / infinity results of the float64 lane
        assert len(np.unique(second[:, 11])) > 10


@pytest.mark.parametrize("n_lanes", [3, 4, 5, 8])
@pytest.mark.parametrize("iw", [4, 5])
def test_mono_expectation_equals_restatement(n_lanes, iw):
    lanes = R.two_pass_lanes(n_lanes, iw, mono=True)
    w1, w2, fresh = R.mono_input(np.random.default_rng(20 * n_lanes + iw), N, iw)
    o = ReduceMonotonic(lanes, 8 * iw)
    first, second, order = R.two_pass_expect("mono", lanes, w1, w2)
    for w, upper, want in ((w1, 1, first), (w2, 2, second)):
        out, errs = o.step(w, upper)
        assert len(errs) == 0
        same(want, words(out))
    same(R.two_pass_arrangement("mono", lanes, w1, w2, np.arange(N)), words(o.export()))
    # keys with fresh values change (unless every lane keeps its extremum), repeated values never do
    changed = np.unique(second[:, 0])
    assert 0 < len(changed) <= fresh.sum()
    assert not np.isin(w1[~fresh, 0], changed).any()


def test_sampled_arrangement_rows_and_key_slices(oracle):
    """The arrangement of a sample of keys, and the outputs in key-rank slices, are the matching parts of
    the whole."""
    lanes = R.two_pass_lanes(8, 5)
    w1, w2, _ = R.lanes_input(np.random.default_rng(7), N, 5)
    o = ReduceLanes(oracle, lanes, 40)
    want1, want2 = words(o.step(w1, 1)), words(o.step(w2, 2))
    got1, got2 = [], []
    for lo in range(0, N, 700):
        a, b, _ = R.two_pass_expect("lanes", lanes, w1, w2, lo, lo + 700)
        got1.append(a)
        got2.append(b)
    same(np.concatenate(got1), want1)
    same(np.concatenate(got2), want2)
    pick = np.sort(np.random.default_rng(8).choice(N, size=200, replace=False))
    arr = words(o.export())
    same(R.two_pass_arrangement("lanes", lanes, w1, w2, pick), arr[np.isin(arr[:, 0], w1[pick, 0])])
