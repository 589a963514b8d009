"""Viterbi forced alignment restated in numpy: the checker of warp_rnnt_b200.rnnt_align (test infrastructure only).

The max-plus recurrence in float32, in the kernel's order of additions, with its predecessor rule (the label edge iff
its candidate is larger or the blank one is NaN), border rules (row 0 the label edge, column 0 the blank edge) and
classes (score -inf or NaN: frames -1; lengths out of range: score NaN), plus the backtrace."""
import numpy as np


def align_lattice_np(B, L):
    """One lattice: B (Tn,Un) blank log-probs, L (Tn,Un-1) label log-probs, float32 -> (score f32, frames (Un-1,))."""
    B = np.asarray(B, dtype=np.float32)
    L = np.asarray(L, dtype=np.float32)
    Tn, Un = B.shape
    a = np.zeros((Tn, Un), np.float32)
    bit = np.zeros((Tn, Un), bool)                   # True: the label predecessor (t, u-1)
    with np.errstate(invalid="ignore", over="ignore"):
        for d in range(1, Tn + Un - 1):              # anti-diagonals t + u = d
            t = np.arange(max(0, d - Un + 1), min(d, Tn - 1) + 1)
            u = d - t
            tp, up = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
            skip = a[tp, u] + B[tp, u]
            emit = a[t, up] + (L[t, up] if Un > 1 else np.float32(0))
            b = (emit > skip) | np.isnan(skip)
            b = (b | (t == 0)) & (u > 0)             # row 0: the label edge; column 0: the blank edge
            bit[t, u] = b
            a[t, u] = np.where(b, emit, skip)
        score = np.float32(a[Tn - 1, Un - 1] + B[Tn - 1, Un - 1])
    frames = np.full(Un - 1, -1, np.int32)
    if not score > -np.inf:                          # -inf or NaN: no alignment
        return score, frames
    t, u = Tn - 1, Un - 1
    while t > 0 or u > 0:
        if t == 0 or (u > 0 and bit[t, u]):
            frames[u - 1] = t
            u -= 1
        else:
            t -= 1
    return score, frames


def align_np(lp, labels, xn, yn, blank=0):
    """Dense (N,T,U,V) log-probs -> (scores (N,) float32, frames (N,U-1) int32); lengths outside [1,T] / [1,U] for
    xn / yn+1 give score NaN and frames -1."""
    lp = np.asarray(lp, dtype=np.float32)
    labels = np.asarray(labels)
    N, T, U, V = lp.shape
    scores = np.full(N, np.nan, np.float32)
    frames = np.full((N, max(U - 1, 0)), -1, np.int32)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not (1 <= Tn <= T and 1 <= Un <= U):
            continue
        B = lp[n, :Tn, :Un, blank]
        L = np.take_along_axis(lp[n, :Tn, :Un - 1], labels[n, :Un - 1].astype(np.int64)[None, :, None], axis=2)[..., 0]
        scores[n], frames[n, :Un - 1] = align_lattice_np(B, L)
    return scores, frames


def path_score_np(B, L, frames):
    """The float32 left-fold of the edges of the path that emits label u at frame frames[u]."""
    Tn, Un = B.shape
    s = np.float32(0)
    t = 0
    for u in range(Un):
        stop = frames[u] if u < Un - 1 else Tn - 1
        while t < stop:
            s = np.float32(s + B[t, u])
            t += 1
        if u < Un - 1:
            s = np.float32(s + L[t, u])
    return np.float32(s + B[Tn - 1, Un - 1])
