"""fp64 numpy restatement of the Token-and-Duration Transducer loss (rnnt_loss_tdt), and brute force over every path.

``tdt(...)`` runs alpha and beta along anti-diagonals s = t + u and forms the edge posteriors explicitly;
``tdt_brute(...)`` enumerates every path of every lattice.  Both return (costs (N,), grads (N,T,U,V+D)): d cost[n] /
d logits, unscaled, with the degenerate classes of the docstring of ``warp_rnnt_b200.rnnt_loss_tdt``:
invalid lengths or a live label outside [0, V): cost NaN, zero gradient; a NaN / +inf in a live row, or a live row whose
token or duration logits are all -inf: cost NaN, NaN on the live rows; no path above -inf: cost +inf, zero gradient.
``tdt`` also returns the per-cell posteriors (Pb, Pl, Pd[0..D)) and the normalisers (lse_tok, lse_dur)."""
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


def _classify(x, labels, xn, yn, n, V, D):
    """'invalid' | 'nan' | None, and Tn, Un"""
    T, U = x.shape[1], x.shape[2]
    Tn, Un = int(xn[n]), int(yn[n]) + 1
    if not (1 <= Tn <= T and 1 <= Un <= U):
        return "invalid", Tn, Un
    if any(not 0 <= int(labels[n, u]) < V for u in range(Un - 1)):
        return "invalid", Tn, Un
    live = x[n, :Tn, :Un]
    tok, dur = live[..., :V], live[..., V:]
    if np.isnan(live).any() or np.isposinf(live).any() or (tok == -np.inf).all(-1).any() or \
            (dur == -np.inf).all(-1).any():
        return "nan", Tn, Un
    return None, Tn, Un


def _cell_logprobs(x, n, Tn, Un, V, sigma):
    lt = np.zeros((Tn, Un, V))
    ld = np.zeros((Tn, Un, x.shape[3] - V))
    lse = np.zeros((Tn, Un, 2))
    for t in range(Tn):
        for u in range(Un):
            lt[t, u], lse[t, u, 0] = _log_softmax(x[n, t, u, :V])
            ld[t, u], lse[t, u, 1] = _log_softmax(x[n, t, u, V:])
    return lt - sigma, ld, lse


def _edges(t, u, Tn, Un, durations):
    """(kind, j, dst) for the edges out of (t, u); dst None = terminal; kind 'b' blank, 'l' label"""
    out = []
    for j, d in enumerate(durations):
        if d > 0:
            if t + d < Tn:
                out.append(("b", j, (t + d, u)))
            elif u == Un - 1 and t + d == Tn:
                out.append(("b", j, None))
        if u < Un - 1 and t + d < Tn:
            out.append(("l", j, (t + d, u + 1)))
    return out


def _grad_rows(x, n, Tn, Un, V, post, lse, blank, lab):
    """d cost / d logits of lattice n's live rows from the posteriors (Pb, Pl, Pd)"""
    g = np.zeros(x.shape[1:])
    for t in range(Tn):
        for u in range(Un):
            pb, pl, pd = post[t, u, 0], post[t, u, 1], post[t, u, 2:]
            occ = pb + pl
            st = np.exp(x[n, t, u, :V] - lse[t, u, 0])
            sd = np.exp(x[n, t, u, V:] - lse[t, u, 1])
            gt = occ * st
            gt[blank] -= pb
            if u < Un - 1:
                gt[lab[u]] -= pl
            g[t, u, :V] = gt
            g[t, u, V:] = occ * sd - pd
    return g


def tdt(x, labels, xn, yn, durations, sigma=0.0, blank=0):
    """Returns costs (N,), grads (N,T,U,V+D), post (N,T,U,2+D), lse (N,T,U,2); fp64."""
    x = np.asarray(x, dtype=np.float64)
    N, T, U, W = x.shape
    D = len(durations)
    V = W - D
    costs = np.zeros(N)
    grads = np.zeros_like(x)
    post = np.zeros((N, T, U, 2 + D))
    lses = np.zeros((N, T, U, 2))
    for n in range(N):
        cls, Tn, Un = _classify(x, labels, xn, yn, n, V, D)
        if cls == "invalid":
            costs[n] = np.nan
            continue
        lt, ld, lse = _cell_logprobs(x, n, Tn, Un, V, sigma)
        lses[n, :Tn, :Un] = lse
        if cls == "nan":
            costs[n] = np.nan
            post[n, :Tn, :Un] = np.nan
            grads[n, :Tn, :Un] = np.nan
            continue
        lab = [int(labels[n, u]) for u in range(Un - 1)]

        def w(t, u, kind, j):
            return (lt[t, u, blank] if kind == "b" else lt[t, u, lab[u]]) + ld[t, u, j]

        alpha = np.full((Tn, Un), -np.inf)
        beta = np.full((Tn, Un), -np.inf)
        for s in range(Tn + Un - 1):                       # alpha along anti-diagonals, pulling from the sources
            for u in range(max(0, s - Tn + 1), min(s, Un - 1) + 1):
                t = s - u
                if t == 0 and u == 0:
                    alpha[t, u] = 0.0
                    continue
                c = []
                for j, d in enumerate(durations):
                    if t - d >= 0 and d > 0:
                        c.append(alpha[t - d, u] + w(t - d, u, "b", j))
                    if t - d >= 0 and u > 0:
                        c.append(alpha[t - d, u - 1] + w(t - d, u - 1, "l", j))
                alpha[t, u] = _lse(c)
        for s in reversed(range(Tn + Un - 1)):             # beta along anti-diagonals
            for u in range(max(0, s - Tn + 1), min(s, Un - 1) + 1):
                t = s - u
                c = [w(t, u, k, j) + (0.0 if dst is None else beta[dst]) for k, j, dst in _edges(t, u, Tn, Un, durations)]
                beta[t, u] = _lse(c)
        lP = beta[0, 0]
        if lP == -np.inf:
            costs[n] = np.inf
            continue
        costs[n] = -lP
        for t in range(Tn):
            for u in range(Un):
                for k, j, dst in _edges(t, u, Tn, Un, durations):
                    g = np.exp(alpha[t, u] + w(t, u, k, j) + (0.0 if dst is None else beta[dst]) - lP)
                    post[n, t, u, 0 if k == "b" else 1] += g
                    post[n, t, u, 2 + j] += g
        grads[n] = _grad_rows(x, n, Tn, Un, V, post[n], lse, blank, lab)
    return costs, grads, post, lses


def tdt_brute(x, labels, xn, yn, durations, sigma=0.0, blank=0):
    """Every path enumerated: costs (N,), grads (N,T,U,V+D)."""
    x = np.asarray(x, dtype=np.float64)
    N, T, U, W = x.shape
    D = len(durations)
    V = W - D
    costs = np.zeros(N)
    grads = np.zeros_like(x)
    for n in range(N):
        cls, Tn, Un = _classify(x, labels, xn, yn, n, V, D)
        if cls is not None:
            costs[n] = np.nan
            if cls == "nan":
                grads[n, :Tn, :Un] = np.nan
            continue
        lt, ld, lse = _cell_logprobs(x, n, Tn, Un, V, sigma)
        lab = [int(labels[n, u]) for u in range(Un - 1)]
        paths = []                                          # (log weight, [(t, u, kind, j), ...])

        def walk(t, u, score, edges):
            for k, j, dst in _edges(t, u, Tn, Un, durations):
                wt = (lt[t, u, blank] if k == "b" else lt[t, u, lab[u]]) + ld[t, u, j]
                e = edges + [(t, u, k, j)]
                if dst is None:
                    paths.append((score + wt, e))
                else:
                    walk(dst[0], dst[1], score + wt, e)

        walk(0, 0, 0.0, [])
        lP = _lse([p[0] for p in paths])
        if lP == -np.inf:
            costs[n] = np.inf
            continue
        costs[n] = -lP
        for score, edges in paths:
            q = np.exp(score - lP)
            if q == 0.0:
                continue
            for t, u, k, j in edges:
                st = np.exp(x[n, t, u, :V] - lse[t, u, 0])
                sd = np.exp(x[n, t, u, V:] - lse[t, u, 1])
                g = np.zeros(W)
                g[:V] = st
                g[blank if k == "b" else lab[u]] -= 1.0
                g[V:] = sd
                g[V + j] -= 1.0
                grads[n, t, u] += q * g
    return costs, grads


def random_case(rng, N, T, U, V, durations, mask=0.0):
    """logits (N,T,U,V+D) fp64, labels (N,U-1) in [1, V), lengths with Tn in [1, T], yn in [0, U-1]"""
    x = rng.randn(N, T, U, V + len(durations))
    if mask:
        x[rng.rand(*x.shape) < mask] = -np.inf
    labels = rng.randint(1, V, (N, max(U - 1, 0))).astype(np.int32) if V > 1 else np.zeros((N, U - 1), np.int32)
    xn = rng.randint(1, T + 1, N).astype(np.int32)
    yn = rng.randint(0, U, N).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    return x, labels, xn, yn


__all__ = ["tdt", "tdt_brute", "random_case"]
