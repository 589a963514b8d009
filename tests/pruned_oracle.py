"""numpy fp64 restatement of rnnt_loss_pruned (warp_rnnt_b200/__init__.py), for the tests.

Row (n, t, s) of the (N, T, S, V) logits is cell (t, u = ranges[n, t] + s) of lattice n when t < xn[n] and
0 <= u <= yn[n].  The restatement places log_softmax of each such row into a full (N, T, U, V) tensor that is -inf
everywhere else, so that every edge out of a cell outside its frame's window has probability 0, runs the plain RNN-T
recurrence on it (oracle.ref_transduce_np_batch) and maps the gradient back through log_softmax onto the rows."""
import numpy as np

from oracle import oracle


def cells(ranges, xn, yn, S):
    """-> list of (n, t, s, u) for the rows that are lattice cells."""
    out = []
    N, T = ranges.shape
    for n in range(N):
        Un = int(yn[n]) + 1
        for t in range(int(xn[n])):
            for s in range(S):
                u = int(ranges[n, t]) + s
                if 0 <= u < Un:
                    out.append((n, t, s, u))
    return out


def pruned(logits, labels, xn, yn, ranges, blank=0, fastemit_lambda=0.0, grad_output=None):
    """-> (costs (N,), d sum_n grad_output[n] * cost[n] / d logits (N, T, S, V)), fp64.  A lattice without a path of
    non-zero probability gets cost +inf and NaN gradients on its rows.  As in oracle.from_logits, a label equal to
    blank is not supported (the recurrence's gradient overrides where autograd would add)."""
    x = np.asarray(logits, dtype=np.float64)
    labels = np.asarray(labels)
    ranges = np.asarray(ranges)
    N, T, S, V = x.shape
    U = labels.shape[1] + 1
    m = x.max(axis=-1, keepdims=True)
    lp = x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))
    full = np.full((N, T, U, V), -np.inf)
    rows = cells(ranges, xn, yn, S)
    for n, t, s, u in rows:
        full[n, t, u] = lp[n, t, s]
    with np.errstate(invalid="ignore"):
        costs, g = oracle.ref_transduce_np_batch(full, labels, xn, yn, blank, fastemit_lambda)
    go = np.ones(N) if grad_output is None else np.asarray(grad_output, dtype=np.float64)
    grads = np.zeros_like(x)
    for n, t, s, u in rows:
        gl = g[n, t, u]
        with np.errstate(invalid="ignore"):
            grads[n, t, s] = (gl - np.exp(lp[n, t, s]) * gl.sum()) * go[n]
    return costs, grads


def brute_force(logits, labels, xn, yn, ranges, blank=0):
    """Every monotone path of every lattice enumerated: -> (costs (N,), d costs.sum() / d logits), fp64.  A path from
    (0, 0) takes Tn - 1 blank edges and Un - 1 label edges in some order and ends with the blank out of
    (Tn - 1, Un - 1); an edge out of a cell outside its frame's window has probability 0."""
    import itertools
    x = np.asarray(logits, dtype=np.float64)
    N, T, S, V = x.shape
    m = x.max(axis=-1, keepdims=True)
    lp = x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))
    costs = np.zeros(N)
    grads = np.zeros_like(x)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1

        def row(t, u):
            s = u - int(ranges[n, t])
            return s if 0 <= s < S else None

        paths = []                                          # (log-prob, [(t, s, v) of each edge])
        for lab_pos in itertools.combinations(range(Tn + Un - 2), Un - 1):
            t = u = 0
            edges = []
            for k in range(Tn + Un - 2):
                if k in lab_pos:
                    edges.append((t, u, int(labels[n, u])))
                    u += 1
                else:
                    edges.append((t, u, blank))
                    t += 1
            edges.append((t, u, blank))
            score, used = 0.0, []
            for (t, u, v) in edges:
                s = row(t, u)
                if s is None:
                    score = -np.inf
                    break
                score += lp[n, t, s, v]
                used.append((t, s, v))
            if score > -np.inf:
                paths.append((score, used))
        if not paths:
            costs[n] = np.inf
            continue
        scores = np.array([p[0] for p in paths])
        ll = np.logaddexp.reduce(scores)
        costs[n] = -ll
        glp = np.zeros((T, S, V))
        for score, used in paths:
            w = np.exp(score - ll)
            for (t, s, v) in used:
                glp[t, s, v] -= w
        grads[n] = glp - np.exp(lp[n]) * glp.sum(axis=-1, keepdims=True)
        # rows that are not cells of the lattice carry no gradient
        for t in range(T):
            for s in range(S):
                u = int(ranges[n, t]) + s
                if not (t < Tn and 0 <= u < Un):
                    grads[n, t, s] = 0.0
    return costs, grads
