"""CPU: the multi-blank alignment oracle (tests/multiblank_align_oracle.py) against brute-force path enumeration on tiny
lattices -- the best float32 fold bit for bit, the returned path's fold equal to its score, the tie rule where exact
ties are planted, the blank-count invariant -- its classes against the loss oracle's (tests/multiblank_oracle.py), and
with every big blank masked, the regular alignment oracle (tests/align_oracle.py)."""
import numpy as np
import pytest

from tests import align_oracle
from tests.multiblank_align_oracle import align_np, brute, fold, logprobs, lse_np
from tests.multiblank_oracle import multiblank, random_case

DURATIONS = [(2,), (2, 4), (2, 3), (2, 4, 8), (3, 5)]


def lattice(x, sigma=0.0):
    return logprobs(x, lse_np(x), sigma)


def key(edges, B):
    """the tie rule as an order on paths: compared from the terminal edge backwards, the standard blank first, then
    the big blanks by increasing duration, then the label"""
    rank = lambda k: 0 if k == 0 else B + 1 if k == 1 else k - 1
    return [rank(k) for _, _, k in reversed(edges)]


def check_path(n, edges, frames, counts, Tn, Un, durations):
    """label frames and counts read off the edge list; the counts cover the frames"""
    labs = [(t, u) for t, u, k in edges if k == 1]
    assert [u for _, u in labs] == list(range(Un - 1))
    assert list(frames[n, :Un - 1]) == [t for t, _ in labs]
    assert (frames[n, Un - 1:] == -1).all()
    assert counts[n, 0] == sum(k == 0 for _, _, k in edges)
    for i in range(len(durations)):
        assert counts[n, 1 + i] == sum(k == 2 + i for _, _, k in edges)
    assert counts[n, 0] + sum(d * counts[n, 1 + i] for i, d in enumerate(durations)) == Tn


@pytest.mark.parametrize("durations", DURATIONS)
@pytest.mark.parametrize("sigma", [0.0, 0.05])
def test_best_fold_against_brute_force(durations, sigma):
    B = len(durations)
    rng = np.random.RandomState(3 + B + durations[-1])
    V = B + 4
    x, labels, xn, yn = random_case(rng, 6, 9, 4, V, B)
    lp = lattice(x, sigma)
    scores, frames, counts, paths = align_np(lp, labels, xn, yn, durations, V - 1)
    for n in range(6):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        every = brute(lp, labels, n, Tn, Un, V - 1, durations)
        best = max(p[0] for p in every)
        assert scores[n].tobytes() == np.float32(best).tobytes(), (n, scores[n], best)
        assert fold(paths[n], lp, labels, n, V - 1).tobytes() == scores[n].tobytes()
        assert any(e == paths[n] for _, e in every)
        check_path(n, paths[n], frames, counts, Tn, Un, durations)


@pytest.mark.parametrize("durations", DURATIONS)
def test_planted_ties_follow_the_rule(durations):
    """log-probs on a coarse dyadic grid: every fold is exact, so many paths tie for the best score; the chosen one is
    the first under the tie rule"""
    B = len(durations)
    rng = np.random.RandomState(17 + B + durations[-1])
    N, T, U, V = 24, 9, 4, B + 3
    lp = -(rng.rand(N, T, U, V) < 0.3).astype(np.float32)          # values 0 and -1
    labels = rng.randint(0, 2, (N, U - 1)).astype(np.int32)
    xn = rng.randint(1, T + 1, N).astype(np.int32)
    yn = rng.randint(0, U, N).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    scores, frames, counts, paths = align_np(lp, labels, xn, yn, durations, V - 1)
    ties = {"any": 0, "blanks": 0}
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        every = brute(lp, labels, n, Tn, Un, V - 1, durations)
        best = max(p[0] for p in every)
        top = [e for s, e in every if s == best]
        assert scores[n] == best
        assert paths[n] == min(top, key=lambda e: key(e, B))
        check_path(n, paths[n], frames, counts, Tn, Un, durations)
        ties["any"] += len(top) > 1
        ties["blanks"] += len({tuple(k for _, _, k in e if k != 1) for e in top}) > 1   # different blank edges
    assert ties["any"] >= 5 and ties["blanks"] >= 3, ties


def test_terminal_tie_prefers_the_standard_blank_then_the_shorter_big_blank():
    """every log-prob 0: every path scores 0; walking back from the end the rule prefers the standard blank at every
    cell, so the path is both labels at frame 0 and then standard blanks only"""
    durations = (2, 4)
    T, U, V = 8, 3, 6
    lp = np.zeros((1, T, U, V), np.float32)
    labels = np.zeros((1, U - 1), np.int32)
    s, f, c, p = align_np(lp, labels, np.array([T]), np.array([U - 1]), durations, V - 1)
    assert s[0] == 0 and list(c[0]) == [T, 0, 0]
    assert list(f[0]) == [0, 0]
    lp[0, :, :, V - 1] = -1                                # standard blank -1: the big blanks take over
    s, f, c, p = align_np(lp, labels, np.array([T]), np.array([U - 1]), durations, V - 1)
    assert s[0] == 0 and list(c[0]) == [0, 4, 0]           # d = 2 four times, the shorter big blank wins the tie


def test_float64_sweep_matches_brute_force_in_float64():
    rng = np.random.RandomState(9)
    durations = (2, 3)
    x, labels, xn, yn = random_case(rng, 3, 8, 3, 6, 2)
    lp = lattice(x)
    s64 = align_np(lp, labels, xn, yn, durations, 5, dtype=np.float64)[0]
    for n in range(3):
        every = brute(lp, labels, n, int(xn[n]), int(yn[n]) + 1, 5, durations)
        best = max(fold(e, lp, labels, n, 5, np.float64) for _, e in every)
        assert s64[n] == best


@pytest.mark.parametrize("durations", [(2,), (2, 4, 8), (3, 5)])
def test_classes_match_the_loss_oracle(durations):
    """NaN cost <-> NaN score, +inf cost <-> -inf score, finite <-> finite, on every degenerate class"""
    B = len(durations)
    rng = np.random.RandomState(23)
    V, T, U = B + 5, 9, 4
    x, labels, xn, yn = random_case(rng, 12, T, U, V, B, mask=0.1)
    xn[1] = 0                                        # invalid lengths
    yn[2] = U
    labels[3, 0], yn[3] = V, max(int(yn[3]), 1)      # a live label outside [0, V)
    x[4, 0, 0, 2] = np.nan                           # a NaN in a live row
    x[5, int(xn[5]) - 1, int(yn[5]), 1] = np.inf     # +inf in a live row
    x[6, 0, 0, :] = -np.inf                          # an all -inf live row
    x[7:10] = rng.randn(3, T, U, V)                  # (unmasked)
    x[7, :, :, V - 1 - B:] = -np.inf                 # every blank masked: no path
    x[8, T - 1, U - 1] = np.nan                      # padding NaN when the lattice is shorter
    xn[8], yn[8] = T - 1, U - 2
    x[9, 0, 0, V - 1] = np.nan                       # NaN in the standard blank's column
    lp = lattice(x)
    scores, frames, counts, _ = align_np(lp, labels, xn, yn, durations, V - 1)
    costs = multiblank(x, labels, xn, yn, durations)[0]
    assert np.array_equal(np.isnan(scores), np.isnan(costs)), (scores, costs)
    assert np.array_equal(scores == -np.inf, costs == np.inf), (scores, costs)
    assert np.isnan(scores[[1, 2, 3, 4, 5, 6, 9]]).all()
    assert scores[7] == -np.inf and np.isfinite(scores[8])
    bad = ~np.isfinite(scores)
    assert (frames[bad] == -1).all() and (counts[bad] == -1).all()
    fin = np.isfinite(costs)
    assert (scores[fin] <= -costs[fin] + 1e-4 * (1 + np.abs(costs[fin]))).all()
    for n in np.flatnonzero(fin):
        assert counts[n, 0] + sum(d * counts[n, 1 + i] for i, d in enumerate(durations)) == xn[n]


@pytest.mark.parametrize("durations", [(2,), (2, 4, 8)])
def test_masked_big_blanks_are_the_regular_alignment(durations):
    """every big blank at -inf (clamped to -1e30): scores and frames are align_oracle.align_np's on the standard-blank
    and label log-probs, and the path takes only standard blanks"""
    B = len(durations)
    rng = np.random.RandomState(31 + B)
    V = B + 6
    x, labels, xn, yn = random_case(rng, 8, 12, 6, V, B)
    x[..., V - 1 - B:V - 1] = -np.inf
    lp = lattice(x)
    s, f, c, _ = align_np(lp, labels, xn, yn, durations, V - 1)
    s0, f0 = align_oracle.align_np(lp, labels, xn, yn, blank=V - 1)
    assert s.tobytes() == s0.tobytes()
    assert np.array_equal(f, f0)
    assert np.array_equal(c[:, 0], xn) and (c[:, 1:] == 0).all()
