"""CPU checks of the fp64 restatement of the smoothed simple loss (tests/smoothed_oracle.py), which the GPU tests take
as the truth: it is the plain simple loss at zero scales, its autograd gradients are the central differences of its
costs (padding lm rows and an invalid lattice included), its costs do not move when a row of am or lm is shifted by a
constant, and a padding row of lm reaches another lattice's cost exactly when am_only_scale > 0."""
import numpy as np
import pytest
import torch

from tests import path_oracle as pa
from tests import pruned_oracle as po
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


# ------------------------------------------------------------------------------------------ factorised
SCALES = [(0.25, 0.0), (0.0, 0.3), (0.1, 0.1), (0.5, 0.45)]
FACTORISED = [  # N, T, U, V, blank
    (3, 6, 4, 7, 0),
    (4, 9, 6, 5, 2),
    (2, 70, 66, 4, 1),                # more than one 64-row / 64-column tile of the kernels' contractions
]


def edge_inputs(N, T, U, V, blank, seed):
    """make()'s inputs with padding rows in lattice 1, invalid lengths in lattice 2 (N >= 3) and about a quarter of
    the labels equal to blank."""
    am, lm, ys, xn, yn = make(N, T, U, V, seed=seed, blank=blank)
    rng = np.random.RandomState(seed + 1)
    ys[rng.rand(*ys.shape) < 0.25] = blank
    yn[1] = min(int(yn[1]), U - 2)
    if N >= 3:
        xn[2] = T + 1
    return am, lm, ys, xn, yn


@pytest.mark.parametrize("scales", [(0.0, 0.0)] + SCALES)
@pytest.mark.parametrize("shape", FACTORISED)
def test_factorised_is_smoothed(shape, scales):
    """The factorised restatement gives smoothed()'s costs, d am, d lm and pair gradients, labels equal to blank,
    padding rows and an invalid lattice included; with detach_unigram the same d lm as smoothed()'s."""
    N, T, U, V, blank = shape
    sl, sa = scales
    am, lm, ys, xn, yn = edge_inputs(N, T, U, V, blank, seed=T + U)
    assert (ys[:, :int(yn[0])] == blank).any()
    go = np.linspace(0.5, 1.5, N)
    want = sm.smoothed(am, lm, ys, xn, yn, blank, sl, sa, grad_output=go, want_pairs=True)
    got = sm.factorised(am, lm, ys, xn, yn, blank, sl, sa, grad_output=go)
    if N >= 3:
        assert np.isnan(got[0][2]) and not got[1][2].any() and not got[3][2].any()
        assert np.isfinite(np.delete(got[0], 2)).all()
    for name, x, y in zip(("costs", "d am", "d lm", "pair grads"), got, want):
        np.testing.assert_allclose(x, y, rtol=0, atol=1e-10, err_msg=name)
    if sa > 0:
        d0 = sm.smoothed(am, lm, ys, xn, yn, blank, sl, sa, grad_output=go, detach_unigram=True)[2]
        d1 = sm.factorised(am, lm, ys, xn, yn, blank, sl, sa, grad_output=go, detach_unigram=True)[2]
        np.testing.assert_allclose(d1, d0, rtol=0, atol=1e-10)
        assert np.abs(d1 - got[2]).max() > 1e-4


def test_factorised_zero_scales_is_the_simple_oracle():
    """At zero scales, with its pairs rounded to float32 as simple_oracle's log-probs are, the factorised restatement
    is simple_oracle.simple (the full joint through oracle.from_logits), over several tiles."""
    N, T, U, V, blank = 3, 70, 66, 6, 2
    am, lm, ys, xn, yn = make(N, T, U, V, seed=5, blank=blank)
    go = np.array([0.5, 1.0, 1.5])
    c0, da0, dl0 = so.simple(am, lm, ys, xn, yn, blank=blank, grad_output=go)
    c1, da1, dl1, _ = sm.factorised(am, lm, ys, xn, yn, blank, grad_output=go, round_pairs=True)
    np.testing.assert_allclose(c1, c0, rtol=1e-12)
    np.testing.assert_allclose(da1, da0, rtol=0, atol=1e-10)
    np.testing.assert_allclose(dl1, dl0, rtol=0, atol=1e-10)


def test_vectorised_recurrences_are_the_per_lattice_ones():
    """alphas() / betas() over a ragged batch equal pruned_oracle._alphas / _betas lattice by lattice, and are -inf
    outside every lattice; lattice_grads' costs are -beta[0,0]."""
    rng = np.random.RandomState(3)
    N, T, U = 5, 13, 9
    B, L = np.log(rng.rand(N, T, U)), np.log(rng.rand(N, T, U))
    Tn = np.array([13, 1, 7, 13, 0])
    Un = np.array([9, 4, 1, 5, 0])
    a, b = sm.alphas(B, L, Tn, Un), sm.betas(B, L, Tn, Un)
    costs, gb, gl = sm.lattice_grads(B, L, Tn, Un)
    for n in range(N - 1):
        t, u = Tn[n], Un[n]
        np.testing.assert_allclose(a[n, :t, :u], po._alphas(B[n, :t, :u], L[n, :t, :u]), rtol=1e-14, atol=0)
        np.testing.assert_allclose(b[n, :t, :u], po._betas(B[n, :t, :u], L[n, :t, :u]), rtol=1e-14, atol=0)
        outside = np.ones((T, U), bool)
        outside[:t, :u] = False
        assert (a[n][outside] == -np.inf).all() and (b[n][outside] == -np.inf).all()
        assert not gb[n][outside].any() and not gl[n][outside].any()
        assert costs[n] == -b[n, 0, 0]
        assert gb[n, t - 1, u - 1] == pytest.approx(-1.0, abs=1e-12)
    assert (a[N - 1] == -np.inf).all() and np.isnan(costs[N - 1]) and not gb[N - 1].any()


# ------------------------------------------------------------------------------------------ rnnt_type, delay_penalty
def test_factorised_regular_without_penalty_is_unchanged():
    am, lm, ys, xn, yn = edge_inputs(3, 9, 6, 5, 2, seed=12)
    go = np.linspace(0.5, 1.5, 3)
    for scales in [(0.0, 0.0), (0.1, 0.1)]:
        a = sm.factorised(am, lm, ys, xn, yn, 2, *scales, grad_output=go)
        b = sm.factorised(am, lm, ys, xn, yn, 2, *scales, grad_output=go, rnnt_type="regular", delay_penalty=0.0)
        for x, y in zip(a, b):
            assert np.array_equal(x, y, equal_nan=True)


@pytest.mark.parametrize("kind", ["regular", "modified", "constrained"])
@pytest.mark.parametrize("scales", [(0.0, 0.0), (0.25, 0.0), (0.1, 0.1)])
def test_factorised_types_are_the_path_oracle_on_its_pairs(kind, scales):
    """The costs and pair gradients factorised() returns are path_oracle.lattice's on its own pairs (pairs() with the
    penalty added in fp64), lattices with invalid lengths and more labels than frames included."""
    N, T, U, V = 4, 8, 6, 5
    am, lm, ys, xn, yn = make(N, T, U, V, seed=31)
    xn[:] = [8, 5, 9, 3]                                     # lattice 2: invalid lengths
    yn[:] = [5, 4, 2, 5]                                     # lattice 3: Un - 1 = 5 > Tn = 3
    lam = 0.05
    c, _, _, pg = sm.factorised(am, lm, ys, xn, yn, 0, *scales, rnnt_type=kind, delay_penalty=lam)
    a, l = torch.tensor(am), torch.tensor(lm)
    norm = torch.logsumexp(a[:, :, None, :] + l[:, None, :, :], dim=-1)
    pb, pl = sm.pairs(a, l, norm, ys, yn, 0, *scales)
    P = np.stack([pb.numpy(), pl.numpy()], -1)
    for n in range(N):
        if 1 <= xn[n] <= T:
            P[n, :xn[n], :yn[n], 1] += lam * ((xn[n] - 1) / 2.0 - np.arange(xn[n]))[:, None]
    c0, g0, _ = pa.lattice(P, xn, yn, kind)
    assert np.isnan(c[2]) and np.isnan(c0[2])
    assert (c[3] == np.inf) == (kind != "regular")
    np.testing.assert_allclose(c, c0, rtol=1e-12)
    np.testing.assert_allclose(pg, g0, rtol=0, atol=1e-12)


@pytest.mark.parametrize("kind", ["regular", "modified", "constrained"])
def test_factorised_types_gradients_are_central_differences(kind):
    """d am and d lm of factorised() with a penalty and smoothing are the central differences of its costs."""
    N, T, U, V = 2, 5, 4, 4
    am, lm, ys, xn, yn = make(N, T, U, V, seed=9)
    xn[:], yn[:] = [5, 4], [3, 2]
    go = np.array([0.7, 1.3])
    sl, sa, lam = 0.1, 0.1, 0.2
    c, dam, dlm, _ = sm.factorised(am, lm, ys, xn, yn, 0, sl, sa, grad_output=go, rnnt_type=kind, delay_penalty=lam)
    assert np.isfinite(c).all()

    def obj(a, l):
        return float((sm.factorised(a, l, ys, xn, yn, 0, sl, sa, rnnt_type=kind, delay_penalty=lam)[0] * go).sum())

    h = 1e-6
    for x, g in ((am, dam), (lm, dlm)):
        num = np.zeros_like(x)
        for idx in np.ndindex(x.shape):
            xp, xm = x.copy(), x.copy()
            xp[idx] += h
            xm[idx] -= h
            num[idx] = (obj(xp, lm) - obj(xm, lm) if x is am else obj(am, xp) - obj(am, xm)) / (2 * h)
        np.testing.assert_allclose(g, num, rtol=0, atol=2e-6)
