"""CPU: the TDT alignment oracle (tests/tdt_align_oracle.py) against brute-force path enumeration on tiny lattices --
the best float32 fold bit for bit, the returned path's fold equal to its score, the tie rule where exact ties are
planted -- and its classes against the loss oracle's (tests/tdt_oracle.py)."""
import numpy as np
import pytest

from tests.tdt_align_oracle import align_np, brute, fold, logprobs, lse_np
from tests.tdt_oracle import random_case, tdt

DURATIONS = [(1,), (0, 1, 2, 3, 4), (0, 1, 2, 3, 4, 5), (0, 1, 16), (0, 2, 3), (1, 2)]


def lattice(x, V, sigma=0.0):
    return logprobs(x, lse_np(x, V), V, sigma)


def key(edges):
    """the tie rule as an order on paths: compared from the terminal edge backwards, blank before label, then the
    shorter duration"""
    return [(0 if k == "b" else 1, d) for _, _, k, d in reversed(edges)]


@pytest.mark.parametrize("durations", DURATIONS)
@pytest.mark.parametrize("sigma", [0.0, 0.05])
def test_best_fold_against_brute_force(durations, sigma):
    rng = np.random.RandomState(3 + len(durations))
    V = 4
    x, labels, xn, yn = random_case(rng, 6, 7, 4, V, durations)
    lp = lattice(x, V, sigma)
    scores, frames, fdur, paths = align_np(lp, labels, xn, yn, durations, 0)
    for n in range(6):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        every = brute(lp, labels, n, Tn, Un, 0, durations)
        if not every or max(p[0] for p in every) <= np.float32(-5e29):
            assert scores[n] == -np.inf and (frames[n] == -1).all() and paths[n] == []
            continue
        best = max(p[0] for p in every)
        assert scores[n].tobytes() == np.float32(best).tobytes(), (n, scores[n], best)
        assert fold(paths[n], lp, labels, n, 0, list(durations)).tobytes() == scores[n].tobytes()
        assert any(e == paths[n] for _, e in every)
        labs = [(t, u, d) for t, u, k, d in paths[n] if k == "l"]
        assert [u for _, u, _ in labs] == list(range(Un - 1))
        assert list(frames[n, :Un - 1]) == [t for t, _, _ in labs]
        assert list(fdur[n, :Un - 1]) == [d for _, _, d in labs]
        assert (frames[n, Un - 1:] == -1).all() and (fdur[n, Un - 1:] == -1).all()


@pytest.mark.parametrize("durations", DURATIONS)
def test_planted_ties_follow_the_rule(durations):
    """log-probs on a coarse dyadic grid: every fold is exact, so many paths tie for the best score; the chosen one is
    the first under the tie rule"""
    rng = np.random.RandomState(17 + len(durations))
    N, T, U, D = 16, 7, 4, len(durations)
    W = 3 + D
    lp = -(rng.rand(N, T, U, W) < 0.25).astype(np.float32)          # values 0 and -1
    labels = rng.randint(1, 3, (N, U - 1)).astype(np.int32)
    xn = rng.randint(1, T + 1, N).astype(np.int32)
    yn = rng.randint(0, U, N).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    scores, _, _, paths = align_np(lp, labels, xn, yn, durations, 0)
    ties = 0
    for n in range(N):
        every = brute(lp, labels, n, int(xn[n]), int(yn[n]) + 1, 0, durations)
        if not every:
            assert scores[n] == -np.inf
            continue
        best = max(p[0] for p in every)
        top = [e for s, e in every if s == best]
        ties += len(top) > 1
        assert scores[n] == best
        assert paths[n] == min(top, key=key)
    assert ties >= 3


def test_blank_equal_to_a_label_and_blank_last():
    rng = np.random.RandomState(5)
    durations = (0, 1, 2)
    V = 5
    x, labels, xn, yn = random_case(rng, 4, 6, 4, V, durations)
    labels[1, 0] = V - 1
    lp = lattice(x, V)
    scores, _, _, paths = align_np(lp, labels, xn, yn, durations, V - 1)
    for n in range(4):
        every = brute(lp, labels, n, int(xn[n]), int(yn[n]) + 1, V - 1, durations)
        best = max(p[0] for p in every)
        assert scores[n].tobytes() == np.float32(best).tobytes()
        assert fold(paths[n], lp, labels, n, V - 1, list(durations)) == scores[n]


def test_float64_sweep_matches_brute_force_in_float64():
    rng = np.random.RandomState(9)
    durations = (0, 1, 3)
    V = 4
    x, labels, xn, yn = random_case(rng, 3, 6, 3, V, durations)
    lp = lattice(x, V)
    s64 = align_np(lp, labels, xn, yn, durations, 0, dtype=np.float64)[0]
    for n in range(3):
        every = brute(lp, labels, n, int(xn[n]), int(yn[n]) + 1, 0, durations)
        best = max(fold(e, lp, labels, n, 0, list(durations), np.float64) for _, e in every)
        assert s64[n] == best


@pytest.mark.parametrize("durations", [(0, 1, 2, 3, 4), (1,), (0, 2, 5)])
def test_classes_match_the_loss_oracle(durations):
    """NaN cost <-> NaN score, +inf cost <-> -inf score, finite <-> finite, on every degenerate class"""
    rng = np.random.RandomState(23)
    V, T, U = 5, 6, 4
    x, labels, xn, yn = random_case(rng, 12, T, U, V, durations, mask=0.15)
    D = len(durations)
    xn[1] = 0                                        # invalid lengths
    yn[2] = U
    labels[3, 0], yn[3] = V, max(int(yn[3]), 1)      # a live label outside [0, V)
    x[4, 0, 0, 2] = np.nan                           # a NaN in a live row
    x[5, int(xn[5]) - 1, int(yn[5]), 1] = np.inf     # +inf in a live row
    x[6, 0, 0, V:] = -np.inf                         # all-(-inf) duration logits in a live row
    x[7, 0, 0, :V] = -np.inf                         # all-(-inf) token logits
    xn[8] = min(d for d in durations if d > 0) - 1  # Tn < min(d > 0): dead, or invalid when that is 0
    x[9:11] = rng.randn(2, T, U, V + D)              # (unmasked)
    x[9, :, :, 0] = -np.inf                          # every blank masked: no path
    x[10, T - 1, U - 1] = np.nan                     # padding NaN when the lattice is shorter
    xn[10], yn[10] = T - 1, U - 2
    lp = lattice(x, V)
    scores = align_np(lp, labels, xn, yn, durations, 0)[0]
    costs = tdt(x, labels, xn, yn, durations)[0]
    assert np.array_equal(np.isnan(scores), np.isnan(costs)), (scores, costs)
    assert np.array_equal(scores == -np.inf, costs == np.inf), (scores, costs)
    assert np.isnan(scores[[1, 2, 3, 4, 5, 6, 7]]).all()
    assert scores[9] == -np.inf and np.isfinite(scores[10])
    fin = np.isfinite(costs)
    assert (scores[fin] <= -costs[fin] + 1e-4 * (1 + np.abs(costs[fin]))).all()
