"""CPU: the alignment oracle (tests/align_oracle.py, the numpy restatement of rnnt_align) against brute force -- every
alignment of small lattices enumerated, its score the float32 left-fold of its edges, the best one the largest score
with NaN below every number -- and its scores against the fp64 log-likelihood of oracle.ref_transduce_np."""
import itertools
import math

import numpy as np
import pytest

from oracle import oracle
from tests import align_oracle
from tests.common import make_inputs


def brute_force(B, L):
    """-> (best score, frames of the best paths (list), all paths' scores) of one lattice."""
    Tn, Un = B.shape
    best, arg = None, []
    for labels_at in itertools.combinations(range(Tn + Un - 2), Un - 1):   # move indices that are label edges
        s, t, u, fr = np.float32(0), 0, 0, []
        lab = set(labels_at)
        for m in range(Tn + Un - 2):
            if m in lab:
                s = np.float32(s + L[t, u])
                fr.append(t)
                u += 1
            else:
                s = np.float32(s + B[t, u])
                t += 1
        s = np.float32(s + B[Tn - 1, Un - 1])
        if np.isnan(s):
            if best is None:
                best, arg = s, []
            continue
        if best is None or np.isnan(best) or s > best:
            best, arg = s, [fr]
        elif s == best:
            arg.append(fr)
    return best, arg


def lattice(lp, ys, n, Tn, Un, blank):
    B = lp[n, :Tn, :Un, blank]
    L = np.stack([lp[n, :Tn, u, ys[n, u]] for u in range(Un - 1)], axis=1) if Un > 1 else np.zeros((Tn, 0), np.float32)
    return B, L


SHAPES = [(1, 1), (1, 5), (5, 1), (2, 2), (3, 4), (6, 6), (6, 3), (4, 6)]


def masked(lp, ys, n, Tn, Un, blank, rng, kind):
    if kind == "ninf" and Un > 1:                           # -inf on a random half of the label edges of one column
        k = rng.randint(Un - 1)
        rows = rng.rand(Tn) < 0.5
        lp[n, :Tn, k, ys[n, k]] = np.where(rows, -np.inf, lp[n, :Tn, k, ys[n, k]])
    elif kind == "blank_ninf":
        lp[n, rng.randint(Tn), rng.randint(Un), blank] = -np.inf
    elif kind == "nan":
        t, u = rng.randint(Tn), rng.randint(Un)
        lp[n, t, u, blank if (Un == 1 or rng.rand() < 0.5) else ys[n, min(u, Un - 2)]] = np.nan
    elif kind == "dead" and Un > 1:
        lp[n, :Tn, 0, ys[n, 0]] = -np.inf                   # label 0 can never be emitted
    elif kind == "all_nan":
        lp[n, Tn - 1, Un - 1, blank] = np.nan               # the last edge of every path


@pytest.mark.parametrize("kind", ["clean", "ninf", "blank_ninf", "nan", "dead", "all_nan"])
@pytest.mark.parametrize("Tn,Un", SHAPES)
def test_align_np_is_brute_force(Tn, Un, kind):
    blank = 2
    rng = np.random.RandomState(Tn * 31 + Un * 7 + len(kind))
    N = 3
    lp, ys, _, _ = make_inputs(N, Tn, Un, 6, seed=Tn * 10 + Un, blank=blank)
    xn, yn = np.full(N, Tn, np.int32), np.full(N, Un - 1, np.int32)
    for n in range(N):
        masked(lp, ys, n, Tn, Un, blank, rng, kind)
    scores, frames = align_oracle.align_np(lp, ys, xn, yn, blank)
    assert scores.dtype == np.float32 and frames.dtype == np.int32 and frames.shape == (N, Un - 1)
    for n in range(N):
        B, L = lattice(lp, ys, n, Tn, Un, blank)
        best, arg = brute_force(B, L)
        np.testing.assert_array_equal(scores[n], best)
        if not best > -np.inf:
            assert (frames[n] == -1).all()
            continue
        if len(arg) == 1:
            assert list(frames[n]) == arg[0], (n, frames[n], arg)
        else:
            assert list(frames[n]) in arg
        f = frames[n]
        assert (np.diff(f) >= 0).all() and (f >= 0).all() and (f <= Tn - 1).all()
        assert align_oracle.path_score_np(B, L, f) == scores[n]


@pytest.mark.parametrize("Tn,Un", [(6, 6), (5, 4), (2, 6)])
def test_brute_force_unique_optimum_frames(Tn, Un):
    """Continuous random inputs: one best path, and the oracle's frames are that path's."""
    lp, ys, xn, yn = make_inputs(8, Tn, Un, 5, seed=Tn + 100 * Un)
    scores, frames = align_oracle.align_np(lp, ys, xn, yn, 0)
    for n in range(8):
        B, L = lattice(lp, ys, n, Tn, Un, 0)
        best, arg = brute_force(B, L)
        assert len(arg) == 1
        assert scores[n] == best and list(frames[n]) == arg[0]


@pytest.mark.parametrize("T,U", [(1, 1), (6, 6), (12, 9), (30, 17), (3, 25)])
def test_scores_between_loglik_bounds(T, U):
    """max <= log-sum-exp <= max + log(number of paths), up to float32 rounding of the max."""
    lp, ys, xn, yn = make_inputs(4, T, U, 7, seed=T * U, random_lengths=True)
    scores, _ = align_oracle.align_np(lp, ys, xn, yn, 0)
    for n in range(4):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        cost, _, _, _ = oracle.ref_transduce_np(lp[n, :Tn, :Un], ys[n, :Un - 1], 0)
        ll = -cost
        slack = 1e-5 * (1.0 + abs(ll))
        assert scores[n] <= ll + slack
        assert scores[n] >= ll - math.log(math.comb(Tn + Un - 2, Un - 1)) - slack


def test_ties_emit_early():
    lp = np.full((2, 5, 4, 3), -1.0, np.float32)
    ys = np.array([[1, 2, 1], [2, 2, 1]], np.int32)
    scores, frames = align_oracle.align_np(lp, ys, np.array([5, 3], np.int32), np.array([3, 2], np.int32), 0)
    assert (frames[0] == 0).all() and list(frames[1]) == [0, 0, -1]
    assert scores[0] == np.float32(-8.0) and scores[1] == np.float32(-5.0)


def test_invalid_lengths():
    lp, ys, _, _ = make_inputs(4, 4, 3, 5, seed=1)
    scores, frames = align_oracle.align_np(lp, ys, np.array([0, 5, 4, 4], np.int32), np.array([1, 1, 3, -1], np.int32), 0)
    assert np.isnan(scores).all() and (frames == -1).all()
