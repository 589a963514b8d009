"""CPU: the numpy restatement of rnnt_align_from_logits on k2's lattices (tests/frames_align_oracle.py) against brute
force over every path, its tie rule, its frames and its classes; type 0 is align_oracle's."""
import numpy as np
import pytest

from tests import align_oracle
from tests import frames_align_oracle as fo

TYPES = (1, 2)


def weights(rng, Tn, Un, integer=False):
    if integer:
        return (-rng.randint(1, 3, (Tn, Un))).astype(np.float32), (-rng.randint(1, 3, (Tn, Un - 1))).astype(np.float32)
    return (rng.randn(Tn, Un) * 2 - 1).astype(np.float32), (rng.randn(Tn, Un - 1) * 2 - 1).astype(np.float32)


def penalised(B, L, lam):
    """B, L of a one-lattice batch after fo.delay_pairs"""
    Tn, Un = B.shape
    p = np.zeros((1, Tn, Un, 2), np.float32)
    p[0, :, :, 0] = B
    p[0, :, :Un - 1, 1] = L
    p = fo.delay_pairs(p, [Tn], [Un - 1], lam)
    return fo.lattice(p, 0, Tn, Un)


@pytest.mark.parametrize("lam", [0.0, 0.05])
@pytest.mark.parametrize("rnnt_type", TYPES)
def test_best_fold_is_brute_force_best(rnnt_type, lam):
    rng = np.random.RandomState(rnnt_type * 10 + int(lam * 100))
    for Tn in range(1, 8):
        for Un in range(1, min(Tn + 1, 5) + 1):
            for _ in range(3):
                B, L = penalised(*weights(rng, Tn, Un), lam)
                s, fr = fo.align_lattice_np(B, L, rnnt_type)
                paths = fo.brute(B, L, rnnt_type)
                best = max(p for p, _ in paths)
                assert s.tobytes() == best.tobytes(), (Tn, Un)
                assert fo.fold(B, L, fr, rnnt_type).tobytes() == s.tobytes()
                assert (np.diff(fr) > 0).all() and (fr >= 0).all() and (fr <= Tn - 1).all()


@pytest.mark.parametrize("rnnt_type", TYPES)
def test_planted_ties_follow_the_tie_rule(rnnt_type):
    """integer weights: folds are exact, many paths tie, and the kernel's rule picks the least backwards sequence"""
    rng = np.random.RandomState(7 + rnnt_type)
    for Tn in range(1, 8):
        for Un in range(1, min(Tn + 1, 5) + 1):
            for _ in range(4):
                B, L = weights(rng, Tn, Un, integer=True)
                s, fr = fo.align_lattice_np(B, L, rnnt_type)
                best, want = fo.tie_winner(fo.brute(B, L, rnnt_type), Tn)
                assert s == best and np.array_equal(fr, want), (Tn, Un, fr, want)


@pytest.mark.parametrize("rnnt_type", TYPES)
def test_all_equal_weights_emit_as_early_as_possible(rnnt_type):
    Tn, Un = 9, 5
    B = np.full((Tn, Un), -1.0, np.float32)
    L = np.full((Tn, Un - 1), -1.0, np.float32)
    s, fr = fo.align_lattice_np(B, L, rnnt_type)
    assert list(fr) == [0, 1, 2, 3]
    assert s == (-9.0 if rnnt_type == 1 else -13.0)


@pytest.mark.parametrize("rnnt_type", TYPES)
def test_classes(rnnt_type):
    rng = np.random.RandomState(3)
    # Un-1 = Tn: the one path emits every frame
    B, L = weights(rng, 6, 7)
    s, fr = fo.align_lattice_np(B, L, rnnt_type)
    assert list(fr) == list(range(6)) and s.tobytes() == fo.fold(B, L, fr, rnnt_type).tobytes()
    # Un-1 = Tn+1: no path, also with a NaN in the lattice
    B, L = weights(rng, 6, 8)
    B[2, 3] = np.nan
    s, fr = fo.align_lattice_np(B, L, rnnt_type)
    assert s == -np.inf and (fr == -1).all()
    # a label column that is -inf: no path above -inf
    B, L = weights(rng, 6, 4)
    L[:, 1] = -np.inf
    s, fr = fo.align_lattice_np(B, L, rnnt_type)
    assert s == -np.inf and (fr == -1).all()
    # every path NaN: both edges into (Tn, Un-1) are NaN
    B, L = weights(rng, 6, 4)
    B[5, 3] = np.nan
    L[5, 2] = np.nan
    s, fr = fo.align_lattice_np(B, L, rnnt_type)
    assert np.isnan(s) and (fr == -1).all()
    # one NaN edge: the best path avoids it, and NaN loses to -inf
    B, L = weights(rng, 6, 4)
    B[0, 0] = np.nan
    s, fr = fo.align_lattice_np(B, L, rnnt_type)
    assert np.isfinite(s) and fr[0] == 0
    # invalid lengths: NaN
    p = np.zeros((3, 5, 4, 2), np.float32)
    sc, fr = fo.align_pairs_np(p, [0, 6, 5], [2, 2, 4], rnnt_type)
    assert np.isnan(sc).all() and (fr == -1).all()


def test_type0_is_align_oracle():
    rng = np.random.RandomState(0)
    pairs = rng.randn(4, 9, 6, 2).astype(np.float32)
    xn, yn = np.array([9, 5, 7, 1], np.int32), np.array([5, 2, 0, 3], np.int32)
    s, f = fo.align_pairs_np(pairs, xn, yn, 0)
    for n in range(4):
        B, L = fo.lattice(pairs, n, xn[n], yn[n] + 1)
        s0, f0 = align_oracle.align_lattice_np(B, L)
        assert s[n].tobytes() == s0.tobytes() and np.array_equal(f[n, :yn[n]], f0)


def test_delay_pairs_touches_live_label_slots_only():
    rng = np.random.RandomState(1)
    p = rng.randn(2, 6, 5, 2).astype(np.float32)
    q = fo.delay_pairs(p, [4, 7], [2, 3], 0.25)
    assert np.array_equal(q[0, :, :, 0], p[0, :, :, 0]) and np.array_equal(q[0, 4:], p[0, 4:])
    assert np.array_equal(q[0, :4, 2:, 1], p[0, :4, 2:, 1])
    assert np.array_equal(q[1], p[1])                      # xn > T: invalid lengths, untouched
    pen = (np.float32(1.5) - np.arange(4, dtype=np.float32)) * np.float32(0.25)
    assert np.array_equal(q[0, :4, :2, 1], (p[0, :4, :2, 1] + pen[:, None]).astype(np.float32))
