"""CPU: the fp64 multi-blank restatement (tests/multiblank_oracle.py) against brute force over every path, central
finite differences, a time-major formulation and the regular transducer lattice, on tiny lattices.  This is the
definition the GPU tests of rnnt_loss_multiblank check against."""
import numpy as np
import pytest

from tests.multiblank_oracle import multiblank, multiblank_brute, multiblank_time_major, random_case
from tests.path_oracle import lattice

DURATION_SETS = [(2,), (2, 4), (2, 4, 8), (2, 3, 5), (3,)]


def _agree(a, b, tol=1e-12):
    assert np.array_equal(np.isnan(a), np.isnan(b))
    assert np.array_equal(np.isinf(a), np.isinf(b))
    fin = np.isfinite(a)
    np.testing.assert_allclose(a[fin], b[fin], rtol=tol, atol=tol)


@pytest.mark.parametrize("durations", DURATION_SETS)
@pytest.mark.parametrize("sigma", [0.0, 0.05])
def test_restatement_equals_brute_force(durations, sigma):
    rng = np.random.RandomState(len(durations) * 7 + int(sigma * 100) + durations[-1])
    B = len(durations)
    for blank in (None, B):
        x, labels, xn, yn = random_case(rng, 4, 7, 4, B + 4, B)
        if blank is not None:
            labels = labels + B + 1                          # tokens above the blanks
        c0, g0, post, _ = multiblank(x, labels, xn, yn, durations, sigma, blank)
        c1, g1 = multiblank_brute(x, labels, xn, yn, durations, sigma, blank)
        _agree(c0, c1)
        _agree(g0, g1)
        assert np.isfinite(c0).all()                         # the standard blank always gives a path


def test_masked_minus_inf():
    rng = np.random.RandomState(3)
    durations = (2, 4)
    x, labels, xn, yn = random_case(rng, 4, 8, 4, 7, len(durations), mask=0.3)
    x[..., -1] = np.where(np.isinf(x).all(-1), 0.0, x[..., -1])     # never a whole row -inf (the NaN class)
    c0, g0, _, _ = multiblank(x, labels, xn, yn, durations, 0.05)
    c1, g1 = multiblank_brute(x, labels, xn, yn, durations, 0.05)
    _agree(c0, c1)
    _agree(g0, g1)


def test_label_equal_to_a_blank_column():
    rng = np.random.RandomState(5)
    durations = (2, 3)
    x, labels, xn, yn = random_case(rng, 3, 6, 4, 6, 2)
    labels[:, 0] = 5                                         # the standard blank
    labels[:, 1] = 4                                         # big blank 0
    c0, g0, _, _ = multiblank(x, labels, xn, yn, durations)
    c1, g1 = multiblank_brute(x, labels, xn, yn, durations)
    _agree(c0, c1)
    _agree(g0, g1)


@pytest.mark.parametrize("durations", [(2, 4), (2, 3, 5, 9, 16)])
def test_time_major_formulation(durations):
    rng = np.random.RandomState(17)
    x, labels, xn, yn = random_case(rng, 5, 20, 6, len(durations) + 5, len(durations))
    c0, _, _, _ = multiblank(x, labels, xn, yn, durations, 0.05)
    c1 = multiblank_time_major(x, labels, xn, yn, durations, 0.05)
    np.testing.assert_allclose(c0, c1, rtol=1e-12)


def test_big_blanks_masked_is_the_regular_transducer():
    """sigma = 0 and every big-blank logit at -inf: the regular transducer on log_softmax with blank = V - 1"""
    rng = np.random.RandomState(6)
    durations = (2, 4, 8)
    V = 9
    x, labels, xn, yn = random_case(rng, 4, 10, 5, V, 3)
    x[..., V - 4:V - 1] = -np.inf
    c0, g0, post, _ = multiblank(x, labels, xn, yn, durations)
    lp = x - np.log(np.exp(x).sum(-1, keepdims=True))
    lab = np.concatenate([labels, np.zeros((4, 1), np.int32)], 1)
    idx = np.broadcast_to(lab[:, None, :, None], lp.shape[:3] + (1,))
    pairs = np.stack([lp[..., V - 1], np.take_along_axis(lp, idx, -1)[..., 0]], -1)
    c1, _, _ = lattice(pairs, xn, yn)
    np.testing.assert_allclose(c0, c1, rtol=1e-12)
    assert (post[..., 2:] == 0).all() and (g0[..., V - 4:V - 1] == 0).all()


def test_degenerate_classes():
    rng = np.random.RandomState(7)
    durations = (2, 3)
    V = 6
    x, labels, xn, yn = random_case(rng, 7, 5, 3, V, 2)
    xn[:] = 5
    yn[:] = 2
    x[0, :, :, :V - 1] = -np.inf                 # only the standard blank: no label edge -> no path (+inf)
    x[1, :, :, V - 3:V - 1] = -np.inf            # big blanks masked: a path remains
    xn[2] = 0                                    # invalid lengths: NaN, zero gradient
    labels[3, 0] = 9                             # live label outside [0, V): NaN, zero gradient
    x[4, 1, 1, 2] = np.nan                       # NaN in a live row: NaN on the live rows
    x[5, 4, 2, 1] = np.nan                       # NaN in a padding row (yn = 1): no effect
    yn[5] = 1
    x[6, 2, 0] = -np.inf                         # a live row all -inf: NaN
    c0, g0, _, _ = multiblank(x, labels, xn, yn, durations)
    c1, g1 = multiblank_brute(x, labels, xn, yn, durations)
    _agree(c0, c1)
    _agree(g0, g1)
    assert np.isposinf(c0[0]) and (g0[0] == 0).all()
    assert np.isfinite(c0[1])
    assert np.isnan(c0[2]) and (g0[2] == 0).all()
    assert np.isnan(c0[3]) and (g0[3] == 0).all()
    assert np.isnan(c0[4]) and np.isnan(g0[4, :5, :3]).all()
    assert np.isfinite(c0[5]) and (g0[5, :, 2] == 0).all()
    assert np.isnan(c0[6]) and np.isnan(g0[6, :5, :3]).all()
    # one frame, no labels: only the standard blank ends the path (every big blank is longer than the lattice)
    x2, l2, xn2, yn2 = random_case(rng, 1, 3, 1, V, 2)
    xn2[:] = 1
    c2, g2, post2, _ = multiblank(x2, l2, xn2, yn2, durations)
    np.testing.assert_allclose(c2, -(x2[0, 0, 0, V - 1] - np.log(np.exp(x2[0, 0, 0]).sum())), rtol=1e-12)
    assert (post2[0, 0, 0] == [1.0, 0.0, 0.0, 0.0]).all()


@pytest.mark.parametrize("durations", [(2,), (2, 3)])
def test_gradient_matches_finite_differences(durations):
    rng = np.random.RandomState(8)
    B = len(durations)
    x, labels, xn, yn = random_case(rng, 2, 6, 3, B + 4, B)
    sigma, blank = 0.05, B
    labels = labels + B + 1
    c, g, _, _ = multiblank(x, labels, xn, yn, durations, sigma, blank)
    h = 1e-6
    for _ in range(40):
        i = tuple(rng.randint(0, s) for s in x.shape)
        xp, xm = x.copy(), x.copy()
        xp[i] += h
        xm[i] -= h
        cp = multiblank(xp, labels, xn, yn, durations, sigma, blank)[0][i[0]]
        cm = multiblank(xm, labels, xn, yn, durations, sigma, blank)[0][i[0]]
        assert abs((cp - cm) / (2 * h) - g[i]) < 1e-6, (i, (cp - cm) / (2 * h), g[i])
