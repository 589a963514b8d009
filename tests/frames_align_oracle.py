"""Viterbi forced alignment on k2's lattices restated in numpy float32: the checker of
warp_rnnt_b200.rnnt_align_from_logits (test infrastructure only).

Types 1 ("modified") and 2 ("constrained") are restated here: the max-plus sweep by frame, in the kernel's order of
additions (alpha + l', with the constrained l' = l + b(t, u+1) formed first), its tie rule (the label edge iff its
candidate is larger or the blank one is NaN; column 0 blank only), its classes and its backtrace.  Type 0 ("regular")
is ``align_oracle``'s.  Everything takes the float32 (blank, label) pairs of the from-logits loss, penalised with
``delay_pairs`` when a delay penalty is given; ``fold`` re-scores a path from its frames and ``brute`` enumerates every
path of a one-symbol-per-frame lattice."""
import itertools

import numpy as np

from tests import align_oracle

F32 = np.float32


def label_weights(B, L, rnnt_type):
    """l' (Tn, Un-1): the label weights of the lattice (constrained: fl(l + b(t, u+1)))"""
    B, L = np.asarray(B, F32), np.asarray(L, F32)
    if rnnt_type == 2:
        with np.errstate(invalid="ignore"):
            return (L + B[:, 1:]).astype(F32)
    return L


def align_lattice_np(B, L, rnnt_type):
    """One lattice: B (Tn,Un) blank and L (Tn,Un-1) label weights, float32 -> (score f32, frames (Un-1,) int32)."""
    B, L = np.asarray(B, F32), np.asarray(L, F32)
    if rnnt_type == 0:
        return align_oracle.align_lattice_np(B, L)
    Tn, Un = B.shape
    frames = np.full(Un - 1, -1, np.int32)
    if Un - 1 > Tn:                                  # more labels than frames: no path
        return F32(-np.inf), frames
    Lp = label_weights(B, L, rnnt_type)
    a = np.full(Un, -np.inf, F32)
    a[0] = 0
    bits = np.zeros((Tn, Un), bool)                  # bits[t, u]: alpha(t+1, u) came by the label edge
    with np.errstate(invalid="ignore"):
        for t in range(Tn):
            skip = (a + B[t]).astype(F32)
            emit = np.full(Un, -np.inf, F32)
            emit[1:] = a[:-1] + Lp[t]
            e = (emit > skip) | np.isnan(skip)
            e[0] = False
            bits[t] = e
            a = np.where(e, emit, skip).astype(F32)
    score = F32(a[Un - 1])
    if not score > -np.inf:                          # -inf or NaN: no alignment
        return score, frames
    u = Un - 1
    for t in range(Tn - 1, -1, -1):
        if bits[t, u]:
            frames[u - 1] = t
            u -= 1
    assert u == 0
    return score, frames


def delay_pairs(pairs, xn, yn, lam):
    """k_delay_pairs: l + ((f32(Tn-1) * 0.5) - f32(t)) * lam at every live label slot, each f32 operation on its own"""
    p = np.array(pairs, dtype=F32, copy=True)
    N, T, U, _ = p.shape
    lam = F32(lam)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not (1 <= Tn <= T and 1 <= Un <= U):
            continue
        half = F32(F32(Tn - 1) * F32(0.5))
        for t in range(Tn):
            pen = F32(F32(half - F32(t)) * lam)
            p[n, t, :Un - 1, 1] = (p[n, t, :Un - 1, 1] + pen).astype(F32)
    return p


def lattice(pairs, n, Tn, Un):
    """B (Tn,Un), L (Tn,Un-1) of lattice n of the (N,T,U,2) pairs"""
    return pairs[n, :Tn, :Un, 0], pairs[n, :Tn, :Un - 1, 1]


def align_pairs_np(pairs, xn, yn, rnnt_type):
    """(N,T,U,2) float32 pairs -> (scores (N,) float32, frames (N,U-1) int32); lengths outside [1,T] / [1,U] for
    xn / yn+1 give score NaN and frames -1."""
    pairs = np.asarray(pairs, F32)
    N, T, U, _ = pairs.shape
    scores = np.full(N, np.nan, F32)
    frames = np.full((N, max(U - 1, 0)), -1, np.int32)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not (1 <= Tn <= T and 1 <= Un <= U):
            continue
        scores[n], frames[n, :Un - 1] = align_lattice_np(*lattice(pairs, n, Tn, Un), rnnt_type)
    return scores, frames


def fold(B, L, frames, rnnt_type, dtype=F32):
    """The left fold acc = acc + w over the edges of the path that emits label u at frame frames[u]"""
    if rnnt_type == 0:
        return align_oracle.path_score_np(B, L, frames)
    Tn, Un = np.shape(B)
    Lp = label_weights(B, L, rnnt_type)
    acc, u = dtype(0), 0
    with np.errstate(invalid="ignore"):
        for t in range(Tn):
            if u < Un - 1 and frames[u] == t:
                acc = dtype(acc + dtype(Lp[t, u]))
                u += 1
            else:
                acc = dtype(acc + dtype(B[t, u]))
    assert u == Un - 1
    return acc


def brute(B, L, rnnt_type):
    """Every path of a one-symbol-per-frame lattice: [(fold, frames)] over every choice of Un-1 label frames"""
    Tn, Un = np.shape(B)
    out = []
    for fr in itertools.combinations(range(Tn), Un - 1):
        fr = np.asarray(fr, np.int32)
        out.append((fold(B, L, fr, rnnt_type), fr))
    return out


def tie_winner(paths, Tn):
    """The best (fold, frames) of ``brute``'s paths (no NaN) under the kernel's tie rule: walking back from frame Tn-1,
    the blank edge wins every tie, so the winner is the least sequence of edges read backwards (blank before label).
    Exact where equal folds have equal prefixes (integer weights)."""
    best = max(s for s, _ in paths)

    def backwards(fr):
        return tuple(int(t in fr) for t in range(Tn - 1, -1, -1))

    return best, min((fr for s, fr in paths if s == best), key=lambda fr: backwards(set(fr.tolist())))


__all__ = ["align_lattice_np", "align_pairs_np", "delay_pairs", "lattice", "fold", "brute", "tie_winner",
           "label_weights"]
