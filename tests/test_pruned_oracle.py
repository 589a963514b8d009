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


# ------------------------------------------------------------------------------------------ pruned_oracle.lattice
def same_dead_classes(c0, g0, c1, g1):
    """Equal cost classes (+inf where the other is), NaN on exactly the same gradient elements."""
    assert np.array_equal(np.isinf(c0), np.isinf(c1)) and np.isfinite(c0[~np.isinf(c0)]).all()
    assert np.array_equal(np.isnan(g0), np.isnan(g1))


@pytest.mark.parametrize("name", sorted(CASES))
def test_lattice_restatement_equals_the_full_tensor_one(name):
    x, ys, xn, yn, r, blank = inputs(name)
    go = np.linspace(0.5, 2.0, len(xn))
    c0, g0 = po.lattice(x, ys, xn, yn, r, blank, 0.25, grad_output=go)
    c1, g1 = po.pruned(x, ys, xn, yn, r, blank, 0.25, grad_output=go)
    same_dead_classes(c0, g0, c1, g1)
    live = np.isfinite(c1)
    np.testing.assert_allclose(c0[live], c1[live], rtol=1e-12)
    np.testing.assert_allclose(g0[live], g1[live], rtol=0, atol=1e-12)
    c2, g2 = po.brute_force(x, ys, xn, yn, r, blank)
    c0, g0 = po.lattice(x, ys, xn, yn, r, blank)
    np.testing.assert_allclose(c0, c2, rtol=1e-12)
    np.testing.assert_allclose(g0[live], g2[live], rtol=0, atol=1e-12)


def random_case(seed, N, T, S, U, V, cut=()):
    """Ragged lattices with live_windows, lattice k cut by cut[k] (None: left live)."""
    rng = np.random.RandomState(seed)
    blank = int(rng.randint(0, V))
    x, ys = make(N, T, S, U, V, seed=seed + 1000, blank=blank)
    xn = rng.randint(max(1, (U - 1 + 1) // 2), T + 1, N).astype(np.int32)
    yn = np.minimum(rng.randint(0, U, N), 2 * xn).astype(np.int32)
    xn[0], yn[0] = T, min(U - 1, 2 * T)
    for k, kind in enumerate(cut):
        if kind == "one_frame":
            xn[k] = 1
            yn[k] = min(yn[k], 1)
        elif kind == "no_labels":
            yn[k] = 0
        elif kind in ("gap",):
            xn[k], yn[k] = T, U - 1
    r = po.live_windows(rng, xn, yn, T, S)
    for k, kind in enumerate(cut):
        if kind is not None:
            r = po.cut_windows(rng, r, xn, yn, S, k, kind)
    return x, ys, xn, yn, r, blank


@pytest.mark.parametrize("seed", range(6))
def test_lattice_restatement_on_random_windows_against_brute_force(seed):
    """Arbitrary live windows (non-monotone, gaps, clipping on both sides), small enough to enumerate every path."""
    x, ys, xn, yn, r, blank = random_case(seed, 3, 5, 3, 4, 5)
    c0, g0 = po.lattice(x, ys, xn, yn, r, blank)
    c1, g1 = po.brute_force(x, ys, xn, yn, r, blank)
    assert np.isfinite(c1).all()
    np.testing.assert_allclose(c0, c1, rtol=1e-12)
    np.testing.assert_allclose(g0, g1, rtol=0, atol=1e-12)


CUTS = [("gap", None, "last"), (None, "int32_max", "int32_min"), (None, "one_frame", "no_labels")]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("cut", CUTS, ids=["-".join(map(str, c)) for c in CUTS])
def test_lattice_restatement_on_random_windows_against_the_full_tensor(seed, cut):
    """Larger lattices with FastEmit and grad_output: live windows, and windows that cut every path of a lattice
    (+inf cost and NaN rows in both restatements, brute force agreeing where it can enumerate)."""
    x, ys, xn, yn, r, blank = random_case(seed + 10, 3, 12, 4, 9, 7, cut)
    go = np.array([0.5, 1.0, 2.0])
    c0, g0 = po.lattice(x, ys, xn, yn, r, blank, 0.3, grad_output=go)
    c1, g1 = po.pruned(x, ys, xn, yn, r, blank, 0.3, grad_output=go)
    dead = [kind is not None for kind in cut]
    assert list(np.isinf(c1)) == dead, (c1, cut)
    same_dead_classes(c0, g0, c1, g1)
    live = ~np.array(dead)
    np.testing.assert_allclose(c0[live], c1[live], rtol=1e-12)
    np.testing.assert_allclose(g0[live], g1[live], rtol=0, atol=1e-12)
    for k in np.flatnonzero(~live):               # NaN on every row of the dead lattice's cells, nothing else
        n, t, s, _ = po.window_rows(r[k:k + 1], xn[k:k + 1], yn[k:k + 1], x.shape[2])
        rows = np.zeros(x.shape[1:3], bool)
        rows[t, s] = True
        assert np.isnan(g0[k][rows]).all() and not np.isnan(g0[k][~rows]).any() and (g0[k][~rows] == 0).all()


def test_live_windows_clip_on_both_sides_and_are_not_monotone():
    """The generator's promise: one path stays alive, and a batch has live frames clipped left (r < 0) and right
    (r + S > Un), non-monotone steps, and INT32_MIN / INT32_MAX in padding frames."""
    rng = np.random.RandomState(5)
    N, T, S, U = 6, 40, 5, 30
    xn = rng.randint(20, T + 1, N).astype(np.int32)
    yn = rng.randint(10, U, N).astype(np.int32)
    xn[0] = T
    r = po.live_windows(rng, xn, yn, T, S)
    left, right = po.clipping_frames(r, xn, yn, S)
    assert left > 0 and right > 0, (left, right)
    assert any((np.diff(r[n, :xn[n]].astype(np.int64)) < 0).any() for n in range(N))
    pad = np.concatenate([r[n, xn[n]:] for n in range(N)])
    assert (pad == po.INT32_MIN).any() and (pad == po.INT32_MAX).any()
    x, ys = make(N, T, S, U, 6, seed=1)
    c, _ = po.lattice(x, ys, xn, yn, r)
    assert np.isfinite(c).all()
