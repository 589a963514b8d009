"""fp64 numpy restatement of the multi-blank transducer loss (rnnt_loss_multiblank), and brute force over every path.

``multiblank(...)`` runs alpha and beta along anti-diagonals s = t + u and forms the edge posteriors explicitly;
``multiblank_brute(...)`` enumerates every path of every lattice; ``multiblank_time_major(...)`` is a second
formulation, frame by frame and column by column with pairwise logaddexp as NeMo's ``MultiblankRNNTLossPytorch`` loop
is written, costs only.  The first two return (costs (N,), grads (N,T,U,V)): d cost[n] / d logits, unscaled, with the
degenerate classes of the docstring of ``warp_rnnt_b200.rnnt_loss_multiblank``: invalid lengths or a live label outside
[0, V): cost NaN, zero gradient; a NaN / +inf in a live row, or a live row that is all -inf: cost NaN, NaN on the live
rows; no path above -inf: cost +inf, zero gradient.  ``multiblank`` also returns the per-cell posteriors
(P_std, Pl, P_big[0..B)) and the normalisers lse (N,T,U).  ``blank`` None means V - 1; big blank i is column
blank - 1 - i."""
import numpy as np


def _lse(c):
    c = np.asarray(c, dtype=np.float64)
    if c.size == 0:
        return -np.inf
    if np.isnan(c).any():
        return np.nan
    m = c.max()
    if m == -np.inf:
        return -np.inf
    return m + np.log(np.exp(c - m).sum())


def _log_softmax(x):
    m = x.max()
    if m == -np.inf or np.isnan(x).any() or m == np.inf:
        return np.full_like(x, np.nan), np.nan
    l = m + np.log(np.exp(x - m).sum())
    return x - l, l


def _classify(x, labels, xn, yn, n):
    """'invalid' | 'nan' | None, and Tn, Un"""
    T, U, V = x.shape[1], x.shape[2], x.shape[3]
    Tn, Un = int(xn[n]), int(yn[n]) + 1
    if not (1 <= Tn <= T and 1 <= Un <= U):
        return "invalid", Tn, Un
    if any(not 0 <= int(labels[n, u]) < V for u in range(Un - 1)):
        return "invalid", Tn, Un
    live = x[n, :Tn, :Un]
    if np.isnan(live).any() or np.isposinf(live).any() or (live == -np.inf).all(-1).any():
        return "nan", Tn, Un
    return None, Tn, Un


def _cell_logprobs(x, n, Tn, Un, sigma):
    lp = np.zeros((Tn, Un, x.shape[3]))
    lse = np.zeros((Tn, Un))
    for t in range(Tn):
        for u in range(Un):
            lp[t, u], lse[t, u] = _log_softmax(x[n, t, u])
    return lp - sigma, lse


def _edges(t, u, Tn, Un, durations, blank, lab):
    """(slot, column, dst) for the edges out of (t, u); dst None = terminal; slot 0 standard blank, 1 label, 2 + i big
    blank i"""
    out = []
    for slot, col, d in [(0, blank, 1)] + [(2 + i, blank - 1 - i, d) for i, d in enumerate(durations)]:
        if t + d < Tn:
            out.append((slot, col, (t + d, u)))
        elif u == Un - 1 and t + d == Tn:
            out.append((slot, col, None))
    if u < Un - 1:
        out.append((1, lab[u], (t, u + 1)))
    return out


def _blank(x, blank):
    return x.shape[-1] - 1 if blank is None else blank


def multiblank(x, labels, xn, yn, durations, sigma=0.0, blank=None):
    """Returns costs (N,), grads (N,T,U,V), post (N,T,U,2+B), lse (N,T,U); fp64."""
    x = np.asarray(x, dtype=np.float64)
    N, T, U, V = x.shape
    B = len(durations)
    blank = _blank(x, blank)
    costs = np.zeros(N)
    grads = np.zeros_like(x)
    post = np.zeros((N, T, U, 2 + B))
    lses = np.zeros((N, T, U))
    for n in range(N):
        cls, Tn, Un = _classify(x, labels, xn, yn, n)
        if cls == "invalid":
            costs[n] = np.nan
            continue
        lp, lse = _cell_logprobs(x, n, Tn, Un, sigma)
        lses[n, :Tn, :Un] = lse
        if cls == "nan":
            costs[n] = np.nan
            post[n, :Tn, :Un] = np.nan
            grads[n, :Tn, :Un] = np.nan
            continue
        lab = [int(labels[n, u]) for u in range(Un - 1)]
        edges = {(t, u): _edges(t, u, Tn, Un, durations, blank, lab) for t in range(Tn) for u in range(Un)}
        alpha = np.full((Tn, Un), -np.inf)
        beta = np.full((Tn, Un), -np.inf)
        for s in range(Tn + Un - 1):                       # alpha along anti-diagonals, pulling from the sources
            for u in range(max(0, s - Tn + 1), min(s, Un - 1) + 1):
                t = s - u
                if t == 0 and u == 0:
                    alpha[t, u] = 0.0
                    continue
                c = []
                if t >= 1:
                    c.append(alpha[t - 1, u] + lp[t - 1, u, blank])
                if u >= 1:
                    c.append(alpha[t, u - 1] + lp[t, u - 1, lab[u - 1]])
                for i, d in enumerate(durations):
                    if t >= d:
                        c.append(alpha[t - d, u] + lp[t - d, u, blank - 1 - i])
                alpha[t, u] = _lse(c)
        for s in reversed(range(Tn + Un - 1)):             # beta along anti-diagonals
            for u in range(max(0, s - Tn + 1), min(s, Un - 1) + 1):
                t = s - u
                beta[t, u] = _lse([lp[t, u, col] + (0.0 if dst is None else beta[dst])
                                   for _, col, dst in edges[t, u]])
        lP = beta[0, 0]
        if lP == -np.inf:
            costs[n] = np.inf
            continue
        costs[n] = -lP
        for (t, u), es in edges.items():
            sm = np.exp(x[n, t, u] - lse[t, u])
            g = np.zeros(V)
            for slot, col, dst in es:
                p = np.exp(alpha[t, u] + lp[t, u, col] + (0.0 if dst is None else beta[dst]) - lP)
                post[n, t, u, slot] += p
                g += p * sm
                g[col] -= p
            grads[n, t, u] = g
    return costs, grads, post, lses


def multiblank_brute(x, labels, xn, yn, durations, sigma=0.0, blank=None):
    """Every path enumerated: costs (N,), grads (N,T,U,V)."""
    x = np.asarray(x, dtype=np.float64)
    N, T, U, V = x.shape
    blank = _blank(x, blank)
    costs = np.zeros(N)
    grads = np.zeros_like(x)
    for n in range(N):
        cls, Tn, Un = _classify(x, labels, xn, yn, n)
        if cls is not None:
            costs[n] = np.nan
            if cls == "nan":
                grads[n, :Tn, :Un] = np.nan
            continue
        lp, lse = _cell_logprobs(x, n, Tn, Un, sigma)
        lab = [int(labels[n, u]) for u in range(Un - 1)]
        paths = []                                          # (log weight, [(t, u, column), ...])

        def walk(t, u, score, path):
            for _, col, dst in _edges(t, u, Tn, Un, durations, blank, lab):
                e = path + [(t, u, col)]
                if dst is None:
                    paths.append((score + lp[t, u, col], e))
                else:
                    walk(dst[0], dst[1], score + lp[t, u, col], e)

        walk(0, 0, 0.0, [])
        lP = _lse([p[0] for p in paths])
        if lP == -np.inf:
            costs[n] = np.inf
            continue
        costs[n] = -lP
        for score, path in paths:
            q = np.exp(score - lP)
            if q == 0.0:
                continue
            for t, u, col in path:
                g = np.exp(x[n, t, u] - lse[t, u])
                g[col] -= 1.0
                grads[n, t, u] += q * g
    return costs, grads


def multiblank_time_major(x, labels, xn, yn, durations, sigma=0.0, blank=None):
    """costs (N,) by the time-major loop: for t, for u, alpha[t, u] from the standard blank of (t-1, u), the label of
    (t, u-1) and each big blank of (t-d, u) by pairwise logaddexp; then log P = the standard blank from (Tn-1, Un-1)
    logaddexp'd with each big blank from (Tn-d, Un-1), Tn >= d.  Only for lattices of the None class."""
    x = np.asarray(x, dtype=np.float64)
    N = x.shape[0]
    blank = _blank(x, blank)
    costs = np.zeros(N)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        lp, _ = _cell_logprobs(x, n, Tn, Un, sigma)
        a = np.full((Tn, Un), -np.inf)
        with np.errstate(invalid="ignore"):
            for t in range(Tn):
                for u in range(Un):
                    if t == 0 and u == 0:
                        a[t, u] = 0.0
                        continue
                    v = -np.inf
                    if t > 0:
                        v = a[t - 1, u] + lp[t - 1, u, blank]
                    if u > 0:
                        v = np.logaddexp(v, a[t, u - 1] + lp[t, u - 1, int(labels[n, u - 1])])
                    for i, d in enumerate(durations):
                        if t >= d:
                            v = np.logaddexp(v, a[t - d, u] + lp[t - d, u, blank - 1 - i])
                    a[t, u] = v
            lP = a[Tn - 1, Un - 1] + lp[Tn - 1, Un - 1, blank]
            for i, d in enumerate(durations):
                if Tn >= d:
                    lP = np.logaddexp(lP, a[Tn - d, Un - 1] + lp[Tn - d, Un - 1, blank - 1 - i])
        costs[n] = -lP
    return costs


def random_case(rng, N, T, U, V, B, mask=0.0):
    """logits (N,T,U,V) fp64, labels (N,U-1) tokens in [0, V-1-B) (the columns below NeMo's blanks), lengths with Tn
    in [1, T], yn in [0, U-1]"""
    x = rng.randn(N, T, U, V)
    if mask:
        x[rng.rand(*x.shape) < mask] = -np.inf
    labels = rng.randint(0, max(V - 1 - B, 1), (N, max(U - 1, 0))).astype(np.int32)
    xn = rng.randint(1, T + 1, N).astype(np.int32)
    yn = rng.randint(0, U, N).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    return x, labels, xn, yn


__all__ = ["multiblank", "multiblank_brute", "multiblank_time_major", "random_case"]
