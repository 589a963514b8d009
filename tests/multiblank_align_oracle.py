"""Viterbi forced alignment on the multi-blank transducer lattice restated in numpy: the checker of
warp_rnnt_b200.rnnt_align_multiblank (test infrastructure only).

``align_np`` runs the max-plus recurrence along anti-diagonals in float32 in the kernel's order of additions,
``alpha[src] + lp``, with its tie rule (the standard blank, then the big blanks by increasing duration, then the label,
the first of equal values kept), its classes and its backtrace.  It takes the clamped log-probs of every cell, as
``logprobs`` builds them from the logits and the normaliser's lse; with the lse of the kernel's own normaliser
(``_C.rnnt_multiblank_forward``) they are bit for bit the values the kernel reads, because they are plain float32
subtractions.  ``fold`` is a path's score, ``brute`` every path with its score.

An edge is (t, u, k) with k the kernel's decision code: 0 the standard blank, 1 the label, 2 + i big blank i."""
import numpy as np

K_BIG = np.float32(-1.0e30)                 # csrc/common.cuh kBig: log-probs are clamped below at it
DEAD = np.float32(0.5) * K_BIG              # lattice_dead: a best score at or below kBig / 2


def _clamp(v):
    v = np.asarray(v, dtype=np.float32)
    return np.where(v < K_BIG, K_BIG, v).astype(np.float32)      # NaN stays NaN


def lse_np(x):
    """lse per row of x (..., V), float32: NaN for a row with a NaN or +inf, or whose elements are all -inf; else the
    fp64 log-sum-exp rounded to float32 (close to the kernel's, not bit-identical)."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        m = x.max(-1, keepdims=True)
        s = np.exp(x - np.where(np.isfinite(m), m, 0.0)).sum(-1, keepdims=True)
        r = (m + np.log(s))[..., 0]
    bad = np.isnan(x).any(-1) | np.isposinf(x).any(-1) | (x == -np.inf).all(-1)
    return np.where(bad, np.nan, r).astype(np.float32)


def logprobs(x, lse, sigma=0.0):
    """The clamped float32 log-probs of every cell (N,T,U,V): clamp((x - lse) - sigma), the kernel's operations."""
    x = np.asarray(x, dtype=np.float32)
    lse = np.asarray(lse, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        return _clamp((x - lse[..., None]) - np.float32(sigma))


def _col(k, blank, lab_u):
    return blank if k == 0 else lab_u if k == 1 else blank - 1 - (k - 2)


def classify(lp, labels, xn, yn, n):
    """'invalid' or None, Tn, Un: the lengths and the live labels, as the kernel checks them (the NaN class is
    align_np's: a NaN in a live cell's standard blank, label (u < Un - 1) or big-blank log-prob)"""
    N, T, U, V = lp.shape
    Tn, Un = int(xn[n]), int(yn[n]) + 1
    if not (1 <= Tn <= T and 1 <= Un <= U) or any(not 0 <= int(labels[n, u]) < V for u in range(Un - 1)):
        return "invalid", Tn, Un
    return None, Tn, Un


def align_np(lp, labels, xn, yn, durations, blank, dtype=np.float32):
    """lp (N,T,U,V) clamped log-probs (``logprobs``), labels (N,U-1), xn, yn (N,), blank the standard blank's column.
    Returns scores (N,) float32, frames (N,U-1) int32, counts (N,1+B) int32, and the edge list of each lattice's best
    path in path order ([] without one), the last edge the terminal one.  dtype float64: the same recurrence in float64
    on the same values (scores only are meaningful to compare)."""
    lp = np.asarray(lp, dtype=np.float32)
    N, T, U, V = lp.shape
    B = len(durations)
    scores = np.zeros(N, np.float64 if dtype == np.float64 else np.float32)
    frames = np.full((N, max(U - 1, 0)), -1, np.int32)
    counts = np.full((N, 1 + B), -1, np.int32)
    paths = []
    for n in range(N):
        cls, Tn, Un = classify(lp, labels, xn, yn, n)
        paths.append([])
        if cls == "invalid":
            scores[n] = np.nan
            continue
        cell = lp[n, :Tn, :Un]
        S = cell[..., blank]
        L = np.full((Tn, Un), K_BIG, np.float32)
        for u in range(Un - 1):
            L[:, u] = cell[:, u, int(labels[n, u])]
        G = np.stack([cell[..., blank - 1 - i] for i in range(B)], -1)
        if np.isnan(S).any() or np.isnan(L[:, :Un - 1]).any() or np.isnan(G).any():
            scores[n] = np.nan
            continue
        S, L, G = S.astype(dtype), L.astype(dtype), G.astype(dtype)
        big = dtype(K_BIG)
        a = np.full((Tn, Un), big, dtype)
        dec = np.full((Tn, Un), -1, np.int64)
        a[0, 0] = 0
        order = [0] + [2 + i for i in range(B)] + [1]             # the tie rule: the first of equal maxima
        for s in range(1, Tn + Un - 1):
            u = np.arange(max(0, s - Tn + 1), min(s, Un - 1) + 1)
            t = s - u
            c = np.full((2 + B, u.size), -np.inf, dtype)
            tp, up = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
            c[0] = np.where(t > 0, a[tp, u] + S[tp, u], -np.inf)
            c[1] = np.where(u > 0, a[t, up] + L[t, up], -np.inf)
            for i, d in enumerate(durations):
                td = np.maximum(t - d, 0)
                c[2 + i] = np.where(t >= d, a[td, u] + G[td, u, i], -np.inf)
            ranked = c[order]
            r = ranked.argmax(0)
            best = ranked[r, np.arange(u.size)]
            a[t, u] = best
            dec[t, u] = np.asarray(order)[r]
        best, k0, t0 = -np.inf, -1, -1
        cands = [(0, Tn - 1, S)] + [(2 + i, Tn - d, G[..., i]) for i, d in enumerate(durations)]
        for k, tp, w in cands:                                   # the terminal edge, the same rule
            if tp >= 0:
                cand = a[tp, Un - 1] + w[tp, Un - 1]
                if cand > best:
                    best, k0, t0 = cand, k, tp
        if not best > DEAD:
            scores[n] = -np.inf
            continue
        scores[n] = best
        t, u = t0, Un - 1
        edges = [(t, u, k0)]
        for _ in range(Tn + Un - 1):
            k = dec[t, u]
            if k < 0:
                break
            if k == 0:
                t -= 1
            elif k == 1:
                u -= 1
                frames[n, u] = t
            else:
                t -= durations[k - 2]
            edges.append((t, u, int(k)))
        assert (t, u) == (0, 0), (n, t, u)
        counts[n] = [sum(e[2] == k for e in edges) for k in [0] + [2 + i for i in range(B)]]
        paths[-1] = edges[::-1]
    return scores, frames, counts, paths


def fold(edges, lp, labels, n, blank, dtype=np.float32):
    """A path's score: acc = acc + lp over its edges in path order"""
    acc = dtype(0)
    for t, u, k in edges:
        lab = int(labels[n, u]) if k == 1 else -1
        acc = dtype(acc + dtype(lp[n, t, u, _col(k, blank, lab)]))
    return acc


def brute(lp, labels, n, Tn, Un, blank, durations):
    """Every path of lattice n: [(fold, edges)], edges as in align_np"""
    out = []

    def walk(t, u, edges):
        for k, d in [(0, 1)] + [(2 + i, d) for i, d in enumerate(durations)]:
            if t + d < Tn:
                walk(t + d, u, edges + [(t, u, k)])
            elif u == Un - 1 and t + d == Tn:
                e = edges + [(t, u, k)]
                out.append((fold(e, lp, labels, n, blank), e))
        if u < Un - 1:
            walk(t, u + 1, edges + [(t, u, 1)])

    walk(0, 0, [])
    return out


__all__ = ["K_BIG", "DEAD", "lse_np", "logprobs", "align_np", "fold", "brute", "classify"]
