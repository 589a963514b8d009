"""numpy fp64 restatement of k2's lattice types and delay penalty on (N,T,U,2) (blank, label) pairs, for the tests
(include/rnnt_b200.h states the semantics).

lattice() gives costs, the pair gradients in the kernels' convention (d cost / d pair, the constrained label edge's
occupation folded into the blank slot of the cell it reaches) and the blank slots before that fold.  Log-probs at or
below -1e30 (the kernels' removed-edge sentinel) count as -inf.  penalise() is the delay penalty in the kernels' f32
operation order, and prune_ranges() the windows rule with the step bound of each type, beside simple_oracle's.
brute_force() enumerates every path, for small lattices.

stream() is lattice() for one modified / constrained lattice in O(U) memory, frame by frame from a function that makes
each frame's pair row, so that it reaches the largest lattice the frame sweep takes (U = 25600, 655 M cells);
stream_grads() gives the pair gradients of the frames it kept.  pruned() restates rnnt_loss_pruned for every type:
window rows -> log_softmax -> full pairs with the edges off the windows removed -> penalty -> lattice()."""
import itertools

import numpy as np

from tests.pruned_oracle import _alphas, _betas, log_softmax, window_rows

KBIG = -1.0e30
TYPES = ("regular", "modified", "constrained")


def lengths_ok(Tn, Un, T, U):
    return 1 <= Tn <= T and 1 <= Un <= U


def penalise(pairs, xn, yn, lam):
    """pairs (N,T,U,2) float32 with lam * ((Tn-1)/2 - t) added to every live label slot, in f32, each op rounded."""
    p = np.array(pairs, dtype=np.float32, copy=True)
    N, T, U, _ = p.shape
    lam = np.float32(lam)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U):
            continue
        t = np.arange(Tn, dtype=np.float32)
        pen = (np.float32(Tn - 1) * np.float32(0.5) - t) * lam
        p[n, :Tn, :Un - 1, 1] = p[n, :Tn, :Un - 1, 1] + pen[:, None]
    return p


def _modified(B, L, constrained):
    """(ll, blank occupation (Tn,Un), label occupation (Tn,Un-1)) of one modified / constrained lattice."""
    Tn, Un = B.shape
    Lw = L[:, :Un - 1] + (B[:, 1:] if constrained else 0.0)
    a = np.full((Tn + 1, Un), -np.inf)
    a[0, 0] = 0.0
    for t in range(Tn):
        a[t + 1] = a[t] + B[t]
        a[t + 1, 1:] = np.logaddexp(a[t + 1, 1:], a[t, :-1] + Lw[t])
    b = np.full((Tn + 1, Un), -np.inf)
    b[Tn, Un - 1] = 0.0
    for t in range(Tn - 1, -1, -1):
        b[t] = B[t] + b[t + 1]
        b[t, :-1] = np.logaddexp(b[t, :-1], Lw[t] + b[t + 1, 1:])
    ll = b[0, 0]
    return ll, np.exp(a[:Tn] + B + b[1:] - ll), np.exp(a[:Tn, :-1] + Lw + b[1:, 1:] - ll)


def lattice(pairs, xn, yn, rnnt_type="regular"):
    """-> costs (N,), pair gradients (N,T,U,2) (folded for constrained), blank slots before the fold (N,T,U); fp64.
    Invalid lengths: cost NaN, zeros.  No finite path: +inf, zeros.  A NaN in a live pair: NaN, NaN on the live slots."""
    P = np.asarray(pairs, dtype=np.float64)
    P = np.where(P <= KBIG, -np.inf, P)
    N, T, U, _ = P.shape
    costs = np.zeros(N)
    g = np.zeros((N, T, U, 2))
    raw = np.zeros((N, T, U))
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U):
            costs[n] = np.nan
            continue
        B, L = P[n, :Tn, :Un, 0], P[n, :Tn, :Un, 1]
        if np.isnan(B).any() or np.isnan(L[:, :Un - 1]).any():
            costs[n] = np.nan
            g[n, :Tn, :Un, 0] = np.nan
            g[n, :Tn, :Un - 1, 1] = np.nan
            raw[n, :Tn, :Un] = np.nan
            continue
        with np.errstate(invalid="ignore", divide="ignore"):
            if rnnt_type == "regular":
                a, b = _alphas(B, L), _betas(B, L)
                ll = b[0, 0]
                ob = np.zeros((Tn, Un))
                ob[:-1] = np.exp(a[:-1] + b[1:] + B[:-1] - ll)
                ob[-1, -1] = np.exp(a[-1, -1] + B[-1, -1] - ll)
                ol = np.exp(a[:, :-1] + b[:, 1:] + L[:, :-1] - ll)
            else:
                ll, ob, ol = _modified(B, L, rnnt_type == "constrained")
        if not np.isfinite(ll):
            costs[n] = np.inf
            continue
        costs[n] = -ll
        raw[n, :Tn, :Un] = -ob
        g[n, :Tn, :Un, 0] = -ob
        g[n, :Tn, :Un - 1, 1] = -ol
        if rnnt_type == "constrained":
            g[n, :Tn, 1:Un, 0] -= ol
    return costs, g, raw


def brute_force(pairs, xn, yn, rnnt_type="regular"):
    """lattice() by enumerating every path (small lattices): costs and d cost / d pairs."""
    P = np.asarray(pairs, dtype=np.float64)
    P = np.where(P <= KBIG, -np.inf, P)
    N, T, U, _ = P.shape
    costs = np.full(N, np.inf)
    g = np.zeros((N, T, U, 2))
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        paths = []                       # each: list of (t, u, slot) edges whose log-probs add up
        if rnnt_type == "regular":
            for labs in itertools.combinations(range(Tn - 1 + Un - 1), Un - 1):
                t = u = 0
                e = []
                for k in range(Tn - 1 + Un - 1):
                    if k in labs:
                        e.append((t, u, 1))
                        u += 1
                    else:
                        e.append((t, u, 0))
                        t += 1
                e.append((Tn - 1, Un - 1, 0))
                paths.append(e)
        else:
            for labs in itertools.combinations(range(Tn), Un - 1):
                u = 0
                e = []
                for t in range(Tn):
                    if t in labs:
                        e.append((t, u, 1))
                        if rnnt_type == "constrained":
                            e.append((t, u + 1, 0))
                        u += 1
                    else:
                        e.append((t, u, 0))
                paths.append(e)
        if not paths:
            continue
        scores = np.array([sum(P[n, t, u, k] for t, u, k in e) for e in paths])
        ll = np.logaddexp.reduce(scores)
        if not np.isfinite(ll):
            continue
        costs[n] = -ll
        for e, s in zip(paths, scores):
            w = np.exp(s - ll)
            for t, u, k in e:
                g[n, t, u, k] -= w
    return costs, g


def prune_ranges(pair_grads, xn, yn, S, rnnt_type="regular", raw_blank=None):
    """ranges (N,T) int32 as rnnt_b200_prune_ranges_ex computes them: simple_oracle.prune_ranges' scores (from
    raw_blank's blank slots for constrained), then the suffix-minimum passes with step bound k = S-1 (regular) or 1."""
    pg = np.asarray(pair_grads, np.float32)
    N, T, U, _ = pg.shape
    blank = np.asarray(raw_blank, np.float32).reshape(N, T, U) if rnnt_type == "constrained" else pg[..., 0]
    k = S - 1 if rnnt_type == "regular" else 1
    out = np.zeros((N, T), np.int64)
    tt = np.arange(T, dtype=np.int64)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U) or Un <= S:
            continue
        top = Un - S
        ob, ol = -blank[n], -pg[n, :, :, 1]
        best = np.zeros(T, np.float32)
        best_r = np.zeros(T, np.int64)
        have = np.zeros(T, bool)
        for r in range(top + 1):
            sc = np.zeros(T, np.float32)
            for u in range(r, r + S):
                sc = sc + ob[:, u]
            if r > 0:
                sc = sc - ol[:, r - 1]
            with np.errstate(invalid="ignore"):
                take = ~np.isnan(sc) & (~have | (sc > best))
            best = np.where(take, sc, best)
            best_r = np.where(take, r, best_r)
            have |= take
        r0 = np.full(T, top, np.int64)
        r0[:Tn - 1] = best_r[:Tn - 1]
        b = np.minimum.accumulate(r0[::-1])[::-1]
        c = k * tt - b
        cp = np.minimum.accumulate(c[::-1])[::-1]
        out[n] = k * tt - np.maximum(cp, 0)
    return out.astype(np.int32)


def window_pairs(pairs, ranges, S):
    """pairs with every cell outside its frame's window set to (KBIG, KBIG): the edges out of it removed."""
    p = np.array(pairs, copy=True)
    N, T, U, _ = p.shape
    u = np.arange(U)
    inside = (u[None, None, :] >= ranges[:, :, None]) & (u[None, None, :] < ranges[:, :, None] + S)
    p[~inside] = KBIG
    return p


# ------------------------------------------------------------------------------------------ streaming, O(U) memory
def _frame_ops(row, Un, t, Tn, lam, constrained):
    """(B (Un,), label weight l' (Un-1,)) of one frame from its (Un, 2) pair row, fp64, the penalty added in fp64."""
    r = np.asarray(row, np.float64)[:Un]
    r = np.where(r <= KBIG, -np.inf, r)
    B, L = r[:, 0], r[:Un - 1, 1]
    if lam:
        L = L + lam * ((Tn - 1) / 2.0 - t)
    return B, (L + B[1:] if constrained else L)


def stream(row_fn, Tn, Un, rnnt_type, keep=(), lam=0.0):
    """-> (cost, {t: alpha of frame t}, {t: beta of frame t + 1}) of one modified or constrained lattice, fp64, each
    alpha / beta an (Un,) row, for t in keep.  row_fn(t) gives frame t's (Un, 2) (blank, label) pair row (more columns
    are ignored); it is called twice per frame, once per direction, so the pairs never exist whole.  lam: the delay
    penalty, added in fp64.  Cost +inf when no finite path is left; NaN in a live pair is not classified (see
    lattice())."""
    assert rnnt_type in ("modified", "constrained") and Tn >= 1 and Un >= 1
    con = rnnt_type == "constrained"
    keep = set(int(t) for t in keep)
    alphas, betas = {}, {}
    a = np.full(Un, -np.inf)
    a[0] = 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(Tn):
            if t in keep:
                alphas[t] = a.copy()
            B, Lw = _frame_ops(row_fn(t), Un, t, Tn, lam, con)
            nxt = a + B
            nxt[1:] = np.logaddexp(nxt[1:], a[:-1] + Lw)
            a = nxt
        b = np.full(Un, -np.inf)
        b[Un - 1] = 0.0
        for t in range(Tn - 1, -1, -1):
            if t in keep:
                betas[t] = b.copy()
            B, Lw = _frame_ops(row_fn(t), Un, t, Tn, lam, con)
            nxt = B + b
            nxt[:-1] = np.logaddexp(nxt[:-1], Lw + b[1:])
            b = nxt
    ll = b[0]
    return (-ll if np.isfinite(ll) else np.inf), alphas, betas


def stream_grads(row_fn, Tn, Un, rnnt_type, keep, lam=0.0):
    """-> (cost, {t: (Un, 2) pair gradients of frame t in lattice()'s convention}, the largest |alpha| of the kept
    frames' cells that lie on a path: finite alpha and a finite beta one frame on) from stream()'s rows."""
    cost, alphas, betas = stream(row_fn, Tn, Un, rnnt_type, keep, lam)
    con = rnnt_type == "constrained"
    out = {}
    top = 0.0
    for t in sorted(alphas):
        a, b = alphas[t], betas[t]
        fin = np.isfinite(a) & np.isfinite(b)
        top = max(top, float(np.abs(a[fin]).max()) if fin.any() else 0.0)
        g = np.zeros((Un, 2))
        if np.isfinite(cost):
            B, Lw = _frame_ops(row_fn(t), Un, t, Tn, lam, con)
            with np.errstate(invalid="ignore"):
                ob = np.exp(a + B + b + cost)
                ol = np.exp(a[:-1] + Lw + b[1:] + cost)
            g[:, 0] = -ob
            g[:Un - 1, 1] = -ol
            if con:
                g[1:, 0] -= ol
        out[t] = g
    return cost, out, top


# ------------------------------------------------------------------------------------------ pruned, every type
def pruned(logits, labels, xn, yn, ranges, blank=0, rnnt_type="regular", delay_penalty=0.0, fastemit_lambda=0.0,
           grad_output=None):
    """rnnt_loss_pruned restated for every type: -> (costs (N,), d sum_n grad_output[n] cost[n] / d logits
    (N, T, S, V)), fp64.  The window rows' log_softmax go to their cells of full (N,T,U,2) pairs that are -inf
    everywhere else (window_pairs()), the penalty is added there in fp64, lattice() gives the costs and the pair
    gradients, and each row's gradient is the vector-Jacobian product of log_softmax, gb (e_blank - p) + gl (e_y - p).
    FastEmit (regular only) scales the label gradients by 1 + lambda and leaves the costs, as pruned_oracle.lattice
    does.  Classes are lattice()'s: NaN for invalid lengths, +inf and zero rows when no path is left."""
    assert rnnt_type == "regular" or not fastemit_lambda
    lp = log_softmax(logits)
    labels = np.asarray(labels)
    N, T, S, V = lp.shape
    U = labels.shape[1] + 1
    lab = np.concatenate([labels.astype(np.int64), np.full((N, 1), blank, np.int64)], axis=1)
    n, t, s, u = window_rows(ranges, xn, yn, S)
    cl = lab[n, u]
    P = np.full((N, T, U, 2), -np.inf)
    P[n, t, u, 0] = lp[n, t, s, blank]
    P[n, t, u, 1] = lp[n, t, s, cl]
    if delay_penalty:
        for k in range(N):
            Tn, Un = int(xn[k]), int(yn[k]) + 1
            if lengths_ok(Tn, Un, T, U):
                P[k, :Tn, :Un - 1, 1] += delay_penalty * ((Tn - 1) / 2.0 - np.arange(Tn))[:, None]
    costs, g, _ = lattice(P, xn, yn, rnnt_type)
    g[..., 1] *= 1.0 + fastemit_lambda
    go = np.ones(N) if grad_output is None else np.asarray(grad_output, np.float64)
    qb, ql = g[n, t, u, 0], g[n, t, u, 1]
    grads = np.zeros_like(lp)
    with np.errstate(invalid="ignore"):
        rows = -np.exp(lp[n, t, s]) * (qb + ql)[:, None]
        k = np.arange(len(n))
        rows[k, blank] += qb
        rows[k, cl] += ql
        grads[n, t, s] = rows * go[n][:, None]
    return costs, grads
