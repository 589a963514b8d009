"""Viterbi forced alignment on the Token-and-Duration Transducer lattice restated in numpy: the checker of
warp_rnnt_b200.rnnt_align_tdt (test infrastructure only).

``align_np`` runs the max-plus recurrence along anti-diagonals in the kernel's order of additions,
``(alpha[src] + lt) + ld``, with its tie rule (blank edges before label edges, each by increasing duration, the first
of equal values kept), its classes and its backtrace.  It takes the clamped log-probs of every cell, as ``logprobs``
builds them from the logits and the normaliser's (lse_tok, lse_dur); with the lse of the kernel's own normaliser
(``_C.rnnt_tdt_forward``) they are bit for bit the values the kernel reads, because they are plain float32
subtractions.  ``fold`` is a path's score, ``brute`` the best score and every path over all paths."""
import numpy as np

K_BIG = np.float32(-1.0e30)                 # csrc/common.cuh kBig: log-probs are clamped below at it
DEAD = np.float32(0.5) * K_BIG              # lattice_dead: a best score at or below kBig / 2


def _clamp(v):
    v = np.asarray(v, dtype=np.float32)
    return np.where(v < K_BIG, K_BIG, v).astype(np.float32)      # NaN stays NaN


def lse_np(x, V):
    """(lse_tok, lse_dur) per row of x (..., V + D), float32, as the kernel's classes need them: NaN for a row with a
    NaN or +inf, or whose elements are all -inf; else the fp64 log-sum-exp rounded to float32 (close to the kernel's,
    not bit-identical)."""
    x = np.asarray(x, dtype=np.float64)
    out = np.zeros(x.shape[:-1] + (2,), np.float32)
    for i, part in enumerate((x[..., :V], x[..., V:])):
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            m = part.max(-1, keepdims=True)
            s = np.exp(part - np.where(np.isfinite(m), m, 0.0)).sum(-1, keepdims=True)
            r = (m + np.log(s))[..., 0]
        bad = np.isnan(part).any(-1) | np.isposinf(part).any(-1) | (part == -np.inf).all(-1)
        out[..., i] = np.where(bad, np.nan, r).astype(np.float32)
    return out


def logprobs(x, lse, V, sigma=0.0):
    """The clamped float32 log-probs of every cell (N,T,U,V+D): clamp((x[k] - lse_tok) - sigma) on the tokens,
    clamp(x[V+j] - lse_dur) on the durations, in the kernel's order of operations."""
    x = np.asarray(x, dtype=np.float32)
    lse = np.asarray(lse, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        tok = (x[..., :V] - lse[..., :1]) - np.float32(sigma)
        dur = x[..., V:] - lse[..., 1:]
    return np.concatenate([_clamp(tok), _clamp(dur)], -1)


def _weights(lp, labels, n, Tn, Un, V, blank):
    """blank (Tn,Un), label (Tn,Un) (kBig in the last column) and duration (Tn,Un,D) log-probs of lattice n"""
    cell = lp[n, :Tn, :Un]
    B = cell[..., blank]
    L = np.full((Tn, Un), K_BIG, np.float32)
    for u in range(Un - 1):
        L[:, u] = cell[:, u, int(labels[n, u])]
    return B, L, cell[..., V:]


def classify(lp, labels, xn, yn, durations, n):
    """'invalid' or None, Tn, Un: the lengths and the live labels, as the kernel checks them (the NaN class is
    align_np's: a NaN in a live cell's blank, label (u < Un - 1) or duration log-prob)"""
    N, T, U, W = lp.shape
    V = W - len(durations)
    Tn, Un = int(xn[n]), int(yn[n]) + 1
    if not (1 <= Tn <= T and 1 <= Un <= U) or any(not 0 <= int(labels[n, u]) < V for u in range(Un - 1)):
        return "invalid", Tn, Un
    return None, Tn, Un


def align_np(lp, labels, xn, yn, durations, blank, dtype=np.float32):
    """lp (N,T,U,V+D) clamped log-probs (``logprobs``), labels (N,U-1), xn, yn (N,).  Returns scores (N,) float32,
    frames and label durations (N,U-1) int32, and the edge list of each lattice's best path ([] without one): edges
    (t, u, kind, d) in path order, kind 'b' (blank) or 'l' (label), the last one the terminal blank.  dtype float64:
    the same recurrence in float64 on the same values (scores only are meaningful to compare)."""
    lp = np.asarray(lp, dtype=np.float32)
    N, T, U, W = lp.shape
    D = len(durations)
    V = W - D
    scores = np.zeros(N, np.float64 if dtype == np.float64 else np.float32)
    frames = np.full((N, max(U - 1, 0)), -1, np.int32)
    fdur = np.full((N, max(U - 1, 0)), -1, np.int32)
    paths = []
    for n in range(N):
        cls, Tn, Un = classify(lp, labels, xn, yn, durations, n)
        paths.append([])
        if cls == "invalid":
            scores[n] = np.nan
            continue
        B, L, Ld = _weights(lp, labels, n, Tn, Un, V, blank)
        if np.isnan(B).any() or np.isnan(L[:, :Un - 1]).any() or np.isnan(Ld).any():
            scores[n] = np.nan
            continue
        B, L, Ld = B.astype(dtype), L.astype(dtype), Ld.astype(dtype)
        big = dtype(K_BIG)
        a = np.full((Tn, Un), big, dtype)
        dec = np.full((Tn, Un), -1, np.int64)               # index into [blank j..., label j...], -1: none
        a[0, 0] = 0
        for s in range(1, Tn + Un - 1):
            u = np.arange(max(0, s - Tn + 1), min(s, Un - 1) + 1)
            t = s - u
            c = np.full((2 * D, u.size), -np.inf, dtype)
            for j, d in enumerate(durations):
                tp = t - d
                ok = tp >= 0
                tq = np.maximum(tp, 0)
                if d > 0:
                    c[j] = np.where(ok, (a[tq, u] + B[tq, u]) + Ld[tq, u, j], -np.inf)
                up = np.maximum(u - 1, 0)
                c[D + j] = np.where(ok & (u > 0), (a[tq, up] + L[tq, up]) + Ld[tq, up, j], -np.inf)
            k = c.argmax(0)                                  # the first of equal maxima: the tie rule
            best = c[k, np.arange(u.size)]
            none = best == -np.inf
            a[t, u] = np.where(none, big, best)
            dec[t, u] = np.where(none, -1, k)
        best, jb = -np.inf, -1
        for j, d in enumerate(durations):                    # the terminal blank edge, the same rule
            if d > 0 and Tn - d >= 0:
                cand = (a[Tn - d, Un - 1] + B[Tn - d, Un - 1]) + Ld[Tn - d, Un - 1, j]
                if cand > best:
                    best, jb = cand, j
        if not best > DEAD:
            scores[n] = -np.inf
            continue
        scores[n] = best
        t, u = Tn - durations[jb], Un - 1
        edges = [(t, u, "b", durations[jb])]
        for _ in range(Tn + Un - 1):
            k = dec[t, u]
            if k < 0:
                break
            j = k % D
            d = durations[j]
            if k < D:
                t -= d
                edges.append((t, u, "b", d))
            else:
                t, u = t - d, u - 1
                edges.append((t, u, "l", d))
                frames[n, u], fdur[n, u] = t, d
        assert (t, u) == (0, 0), (n, t, u)
        paths[-1] = edges[::-1]
    return scores, frames, fdur, paths


def fold(edges, lp, labels, n, blank, durations, dtype=np.float32):
    """A path's score: acc = (acc + lt) + ld over its edges in path order"""
    V = lp.shape[-1] - len(durations)
    acc = dtype(0)
    for t, u, kind, d in edges:
        k = blank if kind == "b" else int(labels[n, u])
        acc = dtype(dtype(acc + dtype(lp[n, t, u, k])) + dtype(lp[n, t, u, V + durations.index(d)]))
    return acc


def brute(lp, labels, n, Tn, Un, blank, durations):
    """Every path of lattice n: [(fold, edges)], edges as in align_np"""
    out = []

    def walk(t, u, edges):
        for d in durations:
            if d > 0:
                if t + d < Tn:
                    walk(t + d, u, edges + [(t, u, "b", d)])
                elif u == Un - 1 and t + d == Tn:
                    e = edges + [(t, u, "b", d)]
                    out.append((fold(e, lp, labels, n, blank, list(durations)), e))
            if u < Un - 1 and t + d < Tn:
                walk(t + d, u + 1, edges + [(t, u, "l", d)])

    walk(0, 0, [])
    return out


__all__ = ["K_BIG", "DEAD", "lse_np", "logprobs", "align_np", "fold", "brute", "classify"]
