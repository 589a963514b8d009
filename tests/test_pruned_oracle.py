"""CPU: the numpy restatement of rnnt_loss_pruned (tests/pruned_oracle.py) against brute-force enumeration of every
monotone path, over the kinds of windows the loss accepts, and against oracle.from_logits for a window that covers
the whole lattice."""
import numpy as np
import pytest

from oracle import oracle
from tests import path_oracle as pa
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


# ------------------------------------------------------------------------------------------ every type (path_oracle)
def test_pruned_every_type_is_the_regular_lattice():
    """path_oracle.pruned with rnnt_type regular, no penalty, is pruned_oracle.lattice: costs and window-logit
    gradients to 1e-10, FastEmit and a non-uniform grad_output included."""
    rng = np.random.RandomState(17)
    N, T, S, U, V = 5, 9, 3, 7, 6
    x = rng.randn(N, T, S, V) * 2
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    xn = np.array([9, 7, 5, 9, 3], np.int32)
    yn = np.array([6, 4, 2, 5, 1], np.int32)
    r = po.live_windows(rng, xn, yn, T, S)
    go = np.linspace(0.5, 1.5, N)
    for lam in (0.0, 0.3):
        c0, g0 = po.lattice(x, ys, xn, yn, r, 0, lam, grad_output=go)
        c1, g1 = pa.pruned(x, ys, xn, yn, r, 0, "regular", 0.0, lam, grad_output=go)
        assert np.isfinite(c0).all()
        np.testing.assert_allclose(c1, c0, rtol=1e-10, atol=0)
        np.testing.assert_allclose(g1, g0, rtol=0, atol=1e-10)


@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_pruned_every_type_against_brute_force(kind):
    """path_oracle.pruned on tiny modified / constrained lattices with a penalty: the costs are path enumeration's
    (path_oracle.brute_force on the windowed, penalised pairs), the window-logit gradient the central differences of
    its own costs; windows that cut every path give +inf and zero rows."""
    rng = np.random.RandomState(5 if kind == "modified" else 6)
    N, T, S, U, V = 4, 5, 2, 4, 5
    x = rng.randn(N, T, S, V)
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    xn = np.array([5, 4, 5, 3], np.int32)
    yn = np.array([3, 2, 3, 1], np.int32)
    r = np.zeros((N, T), np.int32)
    for n in range(N):                                           # windows that move by at most 1 around a path
        r[n, 1:] = np.minimum(np.cumsum(rng.randint(0, 2, T - 1)), max(int(yn[n]) + 1 - S, 0))
    r[2, 2:] = 3                                                 # a gap: lattice 2 has no path
    lam, go = 0.2, np.array([0.5, 1.0, 1.5, 0.7])
    c, g = pa.pruned(x, ys, xn, yn, r, 0, kind, lam, grad_output=go)
    lp = po.log_softmax(x)
    lab = np.concatenate([ys, np.zeros((N, 1), np.int32)], axis=1)
    P = np.full((N, T, U, 2), -np.inf)
    n, t, s, u = po.window_rows(r, xn, yn, S)
    P[n, t, u, 0] = lp[n, t, s, 0]
    P[n, t, u, 1] = lp[n, t, s, lab[n, u]]
    for k in range(N):
        P[k, :xn[k], :yn[k], 1] += lam * ((xn[k] - 1) / 2.0 - np.arange(xn[k]))[:, None]
    cb, _ = pa.brute_force(P, xn, yn, kind)
    assert c[2] == np.inf and cb[2] == np.inf and not g[2].any()
    live = np.isfinite(cb)
    assert live.sum() >= 2
    np.testing.assert_allclose(c[live], cb[live], rtol=1e-12)
    h = 1e-6
    num = np.zeros_like(x)
    for idx in np.ndindex(x.shape):
        if not live[idx[0]]:
            continue
        xp, xm = x.copy(), x.copy()
        xp[idx] += h
        xm[idx] -= h
        k = idx[0]
        num[idx] = go[k] * (pa.pruned(xp, ys, xn, yn, r, 0, kind, lam)[0][k] -
                            pa.pruned(xm, ys, xn, yn, r, 0, kind, lam)[0][k]) / (2 * h)
    np.testing.assert_allclose(g[live], num[live], rtol=0, atol=1e-7)
