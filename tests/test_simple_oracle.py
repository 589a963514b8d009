"""CPU: the restatements of tests/simple_oracle.py that the GPU tests of rnnt_loss_simple compare against.

  1. simple(): the loss of the simple joint and its am / lm gradients, checked against central differences;
  2. prune_ranges(): equal to the literal per-frame loop, on random and adversarial occupations (NaN, ties, Un <= S,
     Un = S+1, Tn = 1, padding frames, invalid lengths), and the ranges have every promised property;
  3. on tiny lattices, brute-force enumeration of every path under the pruned loss (tests/pruned_oracle.py) with these
     ranges finds a path of non-zero probability in every lattice the windows can reach."""
import numpy as np
import pytest

from tests import pruned_oracle as po
from tests import simple_oracle as so


def make(N, T, U, V, seed, blank=0):
    rng = np.random.RandomState(seed)
    am = rng.randn(N, T, V) * 2
    lm = rng.randn(N, U, V) * 2
    ys = rng.randint(0, V - 1, (N, U - 1)).astype(np.int32)
    ys = np.where(ys >= blank, ys + 1, ys).astype(np.int32)
    xn = rng.randint(max(T // 2, 1), T + 1, (N,)).astype(np.int32)
    yn = rng.randint(0, U, (N,)).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    return am, lm, ys, xn, yn


@pytest.mark.parametrize("blank", [0, 2])
def test_simple_gradient_is_the_derivative(blank):
    N, T, U, V = 2, 4, 3, 5
    am, lm, ys, xn, yn = make(N, T, U, V, seed=1 + blank, blank=blank)
    go = np.array([1.0, -0.5])
    costs, dam, dlm = so.simple(am, lm, ys, xn, yn, blank, grad_output=go)
    assert np.isfinite(costs).all()
    h = 1e-2                                  # the oracle takes its log-probs in float32: a step well above their rounding

    def f(a, l):
        return float((so.simple(a, l, ys, xn, yn, blank)[0] * go).sum())

    for which, x, d in (("am", am, dam), ("lm", lm, dlm)):
        num = np.zeros_like(x)
        for idx in np.ndindex(x.shape):
            xp, xm = x.copy(), x.copy()
            xp[idx] += h
            xm[idx] -= h
            num[idx] = (f(xp, lm) - f(xm, lm)) / (2 * h) if which == "am" else (f(am, xp) - f(am, xm)) / (2 * h)
        np.testing.assert_allclose(d, num, atol=2e-3, err_msg=which)


def random_pg(rng, N, T, U):
    return -rng.rand(N, T, U, 2).astype(np.float32)


def adversarial_pg(rng, N, T, U):
    """Integer-valued occupations (ties everywhere), NaN cells and whole NaN frames, -0.0 and +-inf."""
    pg = -rng.randint(0, 3, (N, T, U, 2)).astype(np.float32)
    pg[rng.rand(N, T, U, 2) < 0.05] = np.nan
    pg[rng.rand(N, T, U, 2) < 0.05] = -0.0
    pg[rng.rand(N, T, U, 2) < 0.02] = -np.inf
    pg[0, 0] = np.nan
    return pg


LENGTHS = [  # T, U, S, xn, yn (one lattice each)
    (6, 4, 5, [6], [3]),           # Un <= S
    (6, 6, 5, [6], [5]),           # Un = S + 1
    (6, 9, 4, [1], [8]),           # Tn = 1, unreachable
    (1, 3, 4, [1], [2]),           # Tn = 1, Un <= S
    (9, 7, 3, [5], [6]),           # padding frames
    (7, 12, 2, [7], [11]),         # S = 2
    (5, 20, 3, [5], [19]),         # unreachable: r climbs by S-1 a frame
    (8, 5, 3, [0], [2]),           # invalid: xn = 0
    (8, 5, 3, [9], [2]),           # invalid: xn > T
    (8, 5, 3, [4], [5]),           # invalid: yn + 1 > U
    (8, 5, 3, [4], [-1]),          # invalid: yn < 0
    (12, 10, 4, [12], [9]),
]


@pytest.mark.parametrize("kind", ["random", "adversarial"])
@pytest.mark.parametrize("case", range(len(LENGTHS)))
def test_ranges_rule_and_properties(case, kind):
    T, U, S, xn, yn = LENGTHS[case]
    xn, yn = np.array(xn, np.int32), np.array(yn, np.int32)
    rng = np.random.RandomState(case)
    pg = (random_pg if kind == "random" else adversarial_pg)(rng, 1, T, U)
    r = so.prune_ranges(pg, xn, yn, S)
    np.testing.assert_array_equal(r, so.prune_ranges_scalar(pg, xn, yn, S))
    so.check_ranges(r, xn, yn, S, U)


def test_ranges_ties_take_the_first_window():
    # every score equal: r0 = 0 on every live frame, then the ranges climb only as the last frame requires
    T, U, S = 6, 8, 3
    pg = np.zeros((1, T, U, 2), np.float32)
    r = so.prune_ranges(pg, np.array([T], np.int32), np.array([U - 1], np.int32), S)
    np.testing.assert_array_equal(r[0], [0, 0, 0, 1, 3, 5])
    # a frame whose every score is NaN takes 0 too
    pg[0, 2] = np.nan
    np.testing.assert_array_equal(so.prune_ranges(pg, np.array([T], np.int32), np.array([U - 1], np.int32), S)[0],
                                  [0, 0, 0, 1, 3, 5])


def test_ranges_follow_the_occupation():
    # occupation concentrated on the diagonal u = t: each frame's window starts where the mass is
    T, U, S = 8, 8, 3
    pg = np.zeros((1, T, U, 2), np.float32)
    for t in range(T):
        pg[0, t, t, 0] = -1.0
        pg[0, t, t, 1] = -1.0
    r = so.prune_ranges(pg, np.array([T], np.int32), np.array([U - 1], np.int32), S)[0]
    so.check_ranges(r[None], [T], [U - 1], S, U)
    assert all(r[t] <= t <= r[t] + S - 1 for t in range(T)), r


@pytest.mark.parametrize("seed", range(6))
def test_real_occupations(seed):
    rng = np.random.RandomState(seed)
    N, T, U, V, S = 3, 9, 7, 6, [2, 3, 4, 5, 8, 3][seed]
    lp = np.log(rng.dirichlet(np.ones(V), (N, T, U)))
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    xn = np.array([T, rng.randint(1, T + 1), rng.randint(1, T + 1)], np.int32)
    yn = np.array([U - 1, rng.randint(0, U), rng.randint(0, U)], np.int32)
    pg = so.pair_grads_of(lp, ys, xn, yn)
    r = so.prune_ranges(pg, xn, yn, S)
    np.testing.assert_array_equal(r, so.prune_ranges_scalar(pg, xn, yn, S))
    so.check_ranges(r, xn, yn, S, U)


@pytest.mark.parametrize("seed", range(8))
def test_every_reachable_lattice_keeps_a_path(seed):
    rng = np.random.RandomState(100 + seed)
    S = int(rng.randint(2, 4))
    T, U, V = int(rng.randint(1, 5)), int(rng.randint(1, 6)), 4
    N = 3
    xn = rng.randint(1, T + 1, (N,)).astype(np.int32)
    yn = rng.randint(0, U, (N,)).astype(np.int32)
    pg = (random_pg if seed % 2 else adversarial_pg)(rng, N, T, U)
    r = so.prune_ranges(pg, xn, yn, S)
    so.check_ranges(r, xn, yn, S, U)
    x = rng.randn(N, T, S, V)
    ys = rng.randint(1, V, (N, max(U - 1, 0))).astype(np.int32).reshape(N, U - 1)
    costs, _ = po.brute_force(x, ys, xn, yn, r)
    for n in range(N):
        if so.reachable(int(xn[n]), int(yn[n]) + 1, S):
            assert np.isfinite(costs[n]), (n, xn[n], yn[n], r[n])
