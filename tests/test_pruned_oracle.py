"""CPU: the numpy restatement of rnnt_loss_pruned (tests/pruned_oracle.py) against brute-force enumeration of every
monotone path, over the kinds of windows the loss accepts, and against oracle.from_logits for a window that covers
the whole lattice."""
import numpy as np
import pytest

from oracle import oracle
from tests import pruned_oracle as po


def make(N, T, S, U, V, seed, blank=0):
    rng = np.random.RandomState(seed)
    x = rng.randn(N, T, S, V) * 2.0
    ys = rng.randint(0, V - 1, (N, U - 1))
    ys = np.where(ys >= blank, ys + 1, ys).astype(np.int32)
    return x, ys


def monotone(N, T, S, U, xn, yn, seed):
    """k2-like windows: non-decreasing starts that keep the window inside [0, Un - S] where the lattice allows."""
    rng = np.random.RandomState(seed)
    r = np.zeros((N, T), np.int32)
    for n in range(N):
        Un = int(yn[n]) + 1
        hi = max(Un - S, 0)
        r[n] = np.sort(rng.randint(0, hi + 1, T))
        r[n, 0] = 0
    return r


# name -> (N, T, S, U, V, blank, xn, yn, ranges (N, T))
CASES = {
    "monotone": (2, 5, 2, 4, 5, 0, [5, 4], [3, 2], None),
    "non_monotone": (2, 4, 2, 4, 4, 1, [4, 4], [3, 3], [[0, 2, 1, 2], [1, 0, 2, 1]]),
    "r_negative": (2, 4, 3, 4, 4, 0, [4, 3], [3, 2], [[-1, 0, -2, 1], [-1, 0, 0, 0]]),
    "r_past_end": (2, 4, 3, 4, 5, 2, [4, 4], [3, 2], [[0, 1, 2, 3], [0, 1, 1, 2]]),
    "s_above_u": (2, 4, 6, 3, 4, 0, [4, 3], [2, 1], [[0, -1, 0, -2], [-3, 0, 0, 0]]),
    "cuts_every_path": (2, 4, 2, 4, 4, 0, [4, 4], [3, 3], [[0, 0, 0, 0], [0, 1, 2, 2]]),   # lattice 0 never reaches u = 3
    # lattice 0 (one frame) misses u = 2, lattice 2 (no labels) misses u = 0 at frame 1
    "one_frame_and_no_labels": (3, 3, 2, 3, 4, 0, [1, 3, 3], [2, 0, 0], [[0, 0, 0], [0, 0, 0], [0, 1, 0]]),
}


def inputs(name):
    N, T, S, U, V, blank, xn, yn, r = CASES[name]
    x, ys = make(N, T, S, U, V, seed=len(name), blank=blank)
    xn, yn = np.asarray(xn, np.int32), np.asarray(yn, np.int32)
    r = monotone(N, T, S, U, xn, yn, seed=3) if r is None else np.asarray(r, np.int32)
    return x, ys, xn, yn, r, blank


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_equals_brute_force(name):
    x, ys, xn, yn, r, blank = inputs(name)
    c0, g0 = po.pruned(x, ys, xn, yn, r, blank)
    c1, g1 = po.brute_force(x, ys, xn, yn, r, blank)
    np.testing.assert_allclose(c0, c1, rtol=1e-12)
    live = np.isfinite(c1)
    np.testing.assert_allclose(g0[live], g1[live], atol=1e-12)
    # a lattice without a path: cost +inf, NaN on its cells' rows
    for n in np.flatnonzero(~live):
        rows = [(t, s) for (m, t, s, u) in po.cells(r, xn, yn, x.shape[2]) if m == n]
        assert rows and all(np.isnan(g0[n, t, s]).all() for t, s in rows)
    if name == "cuts_every_path":
        assert list(live) == [False, True]
    if name == "one_frame_and_no_labels":
        assert list(live) == [False, True, False]


def test_whole_lattice_window_equals_from_logits():
    """S = U and ranges = 0: the windows are the lattice, and the loss is rnnt_loss_from_logits's."""
    N, T, U, V, blank = 3, 5, 4, 6, 2
    x, ys = make(N, T, U, U, V, seed=9, blank=blank)
    xn, yn = np.array([5, 3, 4], np.int32), np.array([3, 2, 0], np.int32)
    r = np.zeros((N, T), np.int32)
    go = np.array([0.5, 1.0, 2.0])
    c0, g0 = po.pruned(x, ys, xn, yn, r, blank, 0.3, grad_output=go)
    c1, g1 = oracle.from_logits(x, ys, xn, yn, blank, 0.3, grad_output=go)
    # oracle.dense takes its log-probs as float32
    np.testing.assert_allclose(c0, c1, rtol=1e-6)
    np.testing.assert_allclose(g0, g1, atol=1e-6)
