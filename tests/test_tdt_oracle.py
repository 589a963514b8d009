"""CPU: the fp64 TDT restatement (tests/tdt_oracle.py) against brute force over every path and against central finite
differences, on tiny lattices.  This is the definition the GPU tests of rnnt_loss_tdt check against."""
import numpy as np
import pytest

from tests.tdt_oracle import random_case, tdt, tdt_brute

DURATION_SETS = [(0, 1, 2, 3, 4), (1,), (0, 2, 5), (2, 3)]


def _agree(a, b, tol=1e-12):
    assert np.array_equal(np.isnan(a), np.isnan(b))
    assert np.array_equal(np.isinf(a), np.isinf(b))
    fin = np.isfinite(a)
    np.testing.assert_allclose(a[fin], b[fin], rtol=tol, atol=tol)


@pytest.mark.parametrize("durations", DURATION_SETS)
@pytest.mark.parametrize("sigma", [0.0, 0.05])
def test_restatement_equals_brute_force(durations, sigma):
    rng = np.random.RandomState(len(durations) * 7 + int(sigma * 100))
    for blank in (0, 2):
        x, labels, xn, yn = random_case(rng, 4, 6, 4, 5, durations)
        c0, g0, post, _ = tdt(x, labels, xn, yn, durations, sigma, blank)
        c1, g1 = tdt_brute(x, labels, xn, yn, durations, sigma, blank)
        _agree(c0, c1)
        _agree(g0, g1)
        # occupation = Pb + Pl = sum of Pd
        np.testing.assert_allclose(post[..., 0] + post[..., 1], post[..., 2:].sum(-1), atol=1e-12)


def test_long_duration_short_lattice():
    """durations [0, 16] with T <= 6: only label edges (d = 0) and no blank can end a path -> no path (+inf)"""
    rng = np.random.RandomState(3)
    x, labels, xn, yn = random_case(rng, 3, 6, 3, 4, (0, 16))
    c0, g0, _, _ = tdt(x, labels, xn, yn, (0, 16))
    c1, g1 = tdt_brute(x, labels, xn, yn, (0, 16))
    assert np.isposinf(c0).all() and np.isposinf(c1).all()
    assert (g0 == 0).all() and (g1 == 0).all()


def test_max_duration_exactly_reaches_the_end():
    """durations [0, 16] with T = 16: the one blank of duration 16 from (0, Un-1) ends the path"""
    rng = np.random.RandomState(4)
    x, labels, xn, yn = random_case(rng, 2, 16, 2, 3, (0, 16))
    xn[:] = 16
    c0, g0, _, _ = tdt(x, labels, xn, yn, (0, 16))
    c1, g1 = tdt_brute(x, labels, xn, yn, (0, 16))
    _agree(c0, c1)
    _agree(g0, g1)
    assert np.isfinite(c0).all()


def test_label_equal_to_blank():
    rng = np.random.RandomState(5)
    x, labels, xn, yn = random_case(rng, 3, 5, 4, 4, (0, 1, 2))
    labels[:, 1] = 0
    c0, g0, _, _ = tdt(x, labels, xn, yn, (0, 1, 2), 0.0, 0)
    c1, g1 = tdt_brute(x, labels, xn, yn, (0, 1, 2), 0.0, 0)
    _agree(c0, c1)
    _agree(g0, g1)


@pytest.mark.parametrize("where", ["tokens", "durations"])
def test_minus_inf_masks(where):
    rng = np.random.RandomState(6)
    durations = (0, 1, 2)
    x, labels, xn, yn = random_case(rng, 4, 6, 4, 5, durations)
    sl = slice(0, 5) if where == "tokens" else slice(5, 8)
    part = x[..., sl]
    part[rng.rand(*part.shape) < 0.3] = -np.inf
    # never a whole row -inf here (that is the NaN class)
    part[..., 0] = np.where(np.isinf(part).all(-1), 0.0, part[..., 0])
    c0, g0, _, _ = tdt(x, labels, xn, yn, durations)
    c1, g1 = tdt_brute(x, labels, xn, yn, durations)
    _agree(c0, c1)
    _agree(g0, g1)


def test_dead_lattice_classes():
    rng = np.random.RandomState(7)
    durations = (1, 2)
    x, labels, xn, yn = random_case(rng, 6, 5, 3, 4, durations)
    xn[:] = 5
    yn[:] = 2
    x[0, :, :, 0] = -np.inf                # no blank anywhere: no path -> +inf
    x[1, :, :, 4:] = [0.0, -np.inf]        # every duration 1 ... still a path (d = 1 only): finite
    xn[2] = 0                              # invalid lengths: NaN, zero gradient
    labels[3, 0] = 9                       # live label outside [0, V): NaN, zero gradient
    x[4, 1, 1, 2] = np.nan                 # NaN in a live row: NaN on the live rows
    x[5, 4, 2, 1] = np.nan                 # NaN in a padding row... live here (xn = 5, yn = 2): NaN too
    yn[5] = 1                              # ... now u = 2 is padding: no effect
    c0, g0, _, _ = tdt(x, labels, xn, yn, durations)
    c1, g1 = tdt_brute(x, labels, xn, yn, durations)
    _agree(c0, c1)
    _agree(g0, g1)
    assert np.isposinf(c0[0]) and (g0[0] == 0).all()
    assert np.isfinite(c0[1])
    assert np.isnan(c0[2]) and (g0[2] == 0).all()
    assert np.isnan(c0[3]) and (g0[3] == 0).all()
    assert np.isnan(c0[4]) and np.isnan(g0[4, :5, :3]).all() and (g0[4, :, 3:] == 0).all()
    assert np.isfinite(c0[5]) and (g0[5, :, 2] == 0).all()
    # structurally dead: Tn < min(d > 0)
    x2, l2, xn2, yn2 = random_case(rng, 1, 3, 2, 4, (2, 3))
    xn2[:] = 1
    c2, g2, _, _ = tdt(x2, l2, xn2, yn2, (2, 3))
    assert np.isposinf(c2).all() and (g2 == 0).all()


@pytest.mark.parametrize("durations", [(0, 1, 2), (2, 3)])
def test_gradient_matches_finite_differences(durations):
    rng = np.random.RandomState(8)
    x, labels, xn, yn = random_case(rng, 2, 5, 3, 4, durations)
    sigma, blank = 0.05, 1
    labels[labels == blank] = 2
    c, g, _, _ = tdt(x, labels, xn, yn, durations, sigma, blank)
    h = 1e-6
    idx = [tuple(rng.randint(0, s) for s in x.shape) for _ in range(40)]
    for i in idx:
        xp, xm = x.copy(), x.copy()
        xp[i] += h
        xm[i] -= h
        cp = tdt(xp, labels, xn, yn, durations, sigma, blank)[0][i[0]]
        cm = tdt(xm, labels, xn, yn, durations, sigma, blank)[0][i[0]]
        if not np.isfinite(c[i[0]]):
            continue
        assert abs((cp - cm) / (2 * h) - g[i]) < 1e-6, (i, (cp - cm) / (2 * h), g[i])
