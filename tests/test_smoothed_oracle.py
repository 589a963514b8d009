"""CPU checks of the fp64 restatement of the smoothed simple loss (tests/smoothed_oracle.py), which the GPU tests take
as the truth: it is the plain simple loss at zero scales, its autograd gradients are the central differences of its
costs (padding lm rows and an invalid lattice included), its costs do not move when a row of am or lm is shifted by a
constant, and a padding row of lm reaches another lattice's cost exactly when am_only_scale > 0."""
import numpy as np
import pytest

from tests import simple_oracle as so
from tests import smoothed_oracle as sm


def make(N, T, U, V, seed, blank=0):
    rng = np.random.RandomState(seed)
    am = rng.randn(N, T, V) * 1.5
    lm = rng.randn(N, U, V) * 1.5
    ys = rng.randint(0, V - 1, (N, U - 1))
    ys = np.where(ys >= blank, ys + 1, ys).astype(np.int32)
    xn = rng.randint(max(T // 2, 1), T + 1, (N,)).astype(np.int32)
    yn = rng.randint(0, U, (N,)).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    return am, lm, ys, xn, yn


def test_zero_scales_is_the_simple_loss():
    am, lm, ys, xn, yn = make(3, 6, 4, 7, seed=1, blank=2)
    go = np.array([0.5, 1.0, 1.5])
    c0, da0, dl0 = so.simple(am, lm, ys, xn, yn, blank=2, grad_output=go)
    # simple_oracle runs its recurrence on float32-rounded log-probs: so does this comparison
    c1, da1, dl1 = sm.smoothed(am, lm, ys, xn, yn, blank=2, grad_output=go, round_pairs=True)
    np.testing.assert_allclose(c1, c0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(da1, da0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(dl1, dl0, rtol=0, atol=1e-12)


@pytest.mark.parametrize("scales", [(0.25, 0.0), (0.0, 0.3), (0.1, 0.1)])
def test_gradients_are_central_differences(scales):
    """Lattice 1 has padding lm rows (yn < U-1), lattice 2 invalid lengths (xn > T): its cost is NaN and out of the
    objective, yet with sa > 0 its lm rows move the others' costs through the unigram."""
    sl, sa = scales
    N, T, U, V = 3, 4, 4, 5
    am, lm, ys, xn, yn = make(N, T, U, V, seed=7)
    yn[1], xn[2] = 1, T + 1
    go = np.array([1.0, 0.7, 1.3])
    c, dam, dlm = sm.smoothed(am, lm, ys, xn, yn, 0, sl, sa, grad_output=go)
    assert np.isnan(c[2]) and np.isfinite(c[:2]).all()

    def obj(a, l):
        cc = sm.smoothed(a, l, ys, xn, yn, 0, sl, sa)[0]
        return float(np.nansum(cc * go))

    h = 1e-6
    for x, g in ((am, dam), (lm, dlm)):
        num = np.zeros_like(x)
        for idx in np.ndindex(x.shape):
            xp, xm = x.copy(), x.copy()
            xp[idx] += h
            xm[idx] -= h
            num[idx] = (obj(xp, lm) - obj(xm, lm) if x is am else obj(am, xp) - obj(am, xm)) / (2 * h)
        np.testing.assert_allclose(g, num, rtol=0, atol=2e-6)
    pad = dlm[1, int(yn[1]) + 1:]            # lattice 1's padding rows, and every row of the invalid lattice 2
    if sa > 0:
        assert np.abs(pad).max() > 1e-4 and np.abs(dlm[2]).max() > 1e-4
    else:
        assert (pad == 0).all() and (dlm[2] == 0).all()


@pytest.mark.parametrize("scales", [(0.25, 0.0), (0.0, 0.3), (0.1, 0.1), (0.5, 0.45)])
def test_row_shift_invariance(scales):
    sl, sa = scales
    am, lm, ys, xn, yn = make(3, 5, 4, 6, seed=3)
    c0 = sm.smoothed(am, lm, ys, xn, yn, 0, sl, sa)[0]
    for which, n, r in (("am", 0, 2), ("am", 2, 0), ("lm", 1, 1), ("lm", 0, 3)):
        a, l = am.copy(), lm.copy()
        (a if which == "am" else l)[n, r] += 3.7
        c1 = sm.smoothed(a, l, ys, xn, yn, 0, sl, sa)[0]
        np.testing.assert_allclose(c1, c0, rtol=0, atol=1e-12)


@pytest.mark.parametrize("scales", [(0.0, 0.0), (0.25, 0.0), (0.0, 0.3), (0.1, 0.1)])
def test_padding_row_couples_the_batch_iff_am_only_scale(scales):
    sl, sa = scales
    am, lm, ys, xn, yn = make(2, 5, 5, 6, seed=4)
    yn[1] = 2                                   # lm rows 3 and 4 of lattice 1 are padding
    c0 = sm.smoothed(am, lm, ys, xn, yn, 0, sl, sa)[0]
    l = lm.copy()
    l[1, 4] = np.random.RandomState(0).randn(6) * 3
    c1 = sm.smoothed(am, l, ys, xn, yn, 0, sl, sa)[0]
    assert (abs(c1[0] - c0[0]) > 1e-6) == (sa > 0)
    assert (abs(c1[1] - c0[1]) > 1e-6) == (sa > 0)
