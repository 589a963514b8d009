"""numpy fp64 restatement of rnnt_loss_pruned (warp_rnnt_b200/__init__.py), for the tests.

Row (n, t, s) of the (N, T, S, V) logits is cell (t, u = ranges[n, t] + s) of lattice n when t < xn[n] and
0 <= u <= yn[n].  The restatement places log_softmax of each such row into a full (N, T, U, V) tensor that is -inf
everywhere else, so that every edge out of a cell outside its frame's window has probability 0, runs the plain RNN-T
recurrence on it (oracle.ref_transduce_np_batch) and maps the gradient back through log_softmax onto the rows.

lattice() is the same restatement on the lattice alone: the (blank, label) log-probs of each cell in (N,T,U,2), the
recurrence along anti-diagonals.  It needs neither the (N,T,U,V) tensor nor a Python loop per cell, so it reaches the
shapes the pruned loss is used at (U in the hundreds, T past a thousand).  The window generators at the end make the
windows the tests run: live ones around a random path, and ones that cut every path."""
import numpy as np

from oracle import oracle

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1


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


def log_softmax(x):
    x = np.asarray(x, dtype=np.float64)
    m = x.max(axis=-1, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))


def window_rows(ranges, xn, yn, S):
    """-> (n, t, s, u) index arrays of the rows that are lattice cells (as cells(), vectorised; 64-bit columns, so
    that ranges near INT32_MAX do not wrap)."""
    N, T = ranges.shape
    u = np.asarray(ranges, np.int64)[:, :, None] + np.arange(S)
    ok = ((np.arange(T)[None, :, None] < np.asarray(xn, np.int64)[:, None, None]) & (u >= 0)
          & (u <= np.asarray(yn, np.int64)[:, None, None]))
    n, t, s = np.nonzero(ok)
    return n, t, s, u[ok]


def _alphas(B, L):
    """alpha (Tn, Un) of one lattice from its blank and label log-probs (Tn, Un), one anti-diagonal per step."""
    Tn, Un = B.shape
    a = np.full((Tn, Un), -np.inf)
    a[0, 0] = 0.0
    for d in range(1, Tn + Un - 1):
        t = np.arange(max(0, d - Un + 1), min(d, Tn - 1) + 1)
        u = d - t
        tp, up = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
        top = np.where(t > 0, a[tp, u] + B[tp, u], -np.inf)
        left = np.where(u > 0, a[t, up] + L[t, up], -np.inf)
        a[t, u] = np.logaddexp(top, left)
    return a


def _betas(B, L):
    """beta (Tn, Un): beta[Tn-1, Un-1] is the final blank's log-prob, as in oracle.ref_transduce_np."""
    Tn, Un = B.shape
    b = np.full((Tn, Un), -np.inf)
    b[Tn - 1, Un - 1] = B[Tn - 1, Un - 1]
    for d in range(Tn + Un - 3, -1, -1):
        t = np.arange(max(0, d - Un + 1), min(d, Tn - 1) + 1)
        u = d - t
        tn, un = np.minimum(t + 1, Tn - 1), np.minimum(u + 1, Un - 1)
        down = np.where(t < Tn - 1, b[tn, u] + B[t, u], -np.inf)
        right = np.where(u < Un - 1, b[t, un] + L[t, u], -np.inf)
        b[t, u] = np.logaddexp(down, right)
    return b


def lattice(logits, labels, xn, yn, ranges, blank=0, fastemit_lambda=0.0, grad_output=None):
    """pruned() on the lattice: the same costs (N,) and gradients (N, T, S, V), fp64, the same dead classes (+inf cost,
    NaN on the rows of the lattice's cells)."""
    lp = log_softmax(logits)
    labels = np.asarray(labels)
    N, T, S, V = lp.shape
    U = labels.shape[1] + 1
    lab = np.concatenate([labels.astype(np.int64), np.full((N, 1), blank, np.int64)], axis=1)       # (N, U)
    n, t, s, u = window_rows(ranges, xn, yn, S)
    cl = lab[n, u]
    pb = np.full((N, T, U), -np.inf)
    pl = np.full((N, T, U), -np.inf)
    pb[n, t, u] = lp[n, t, s, blank]
    pl[n, t, u] = lp[n, t, s, cl]
    costs = np.zeros(N)
    gb = np.zeros((N, T, U))
    gl = np.zeros((N, T, U))
    with np.errstate(invalid="ignore"):
        for k in range(N):
            Tn, Un = int(xn[k]), int(yn[k]) + 1
            B, L = pb[k, :Tn, :Un], pl[k, :Tn, :Un]
            a, b = _alphas(B, L), _betas(B, L)
            ll = b[0, 0]
            costs[k] = -ll
            gb[k, :Tn - 1, :Un] = -np.exp(a[:-1] + b[1:] + B[:-1] - ll)
            gb[k, Tn - 1, Un - 1] = -np.exp(a[-1, -1] + B[-1, -1] - ll)
            gl[k, :Tn, :Un - 1] = -(1.0 + fastemit_lambda) * np.exp(a[:, :-1] + b[:, 1:] + L[:, :-1] - ll)
        go = np.ones(N) if grad_output is None else np.asarray(grad_output, dtype=np.float64)
        qb, ql = gb[n, t, u], gl[n, t, u]
        grads = np.zeros_like(lp)
        rows = -np.exp(lp[n, t, s]) * (qb + ql)[:, None]
        k = np.arange(len(n))
        rows[k, blank] += qb
        rows[k, cl] += ql
        grads[n, t, s] = rows * go[n][:, None]
    return costs, grads


# ------------------------------------------------------------------------------------------ windows
def random_path(rng, Tn, Un, cap):
    """A monotone path through a Tn x Un lattice that emits at most `cap` labels per frame -> (lo, hi) (Tn,): the first
    and last column it visits at frame t."""
    assert Tn * cap >= Un - 1, (Tn, Un, cap)
    per = np.zeros(Tn, np.int64)
    for f in rng.choice(np.repeat(np.arange(Tn), cap), Un - 1, replace=False):
        per[f] += 1
    lo = np.concatenate([[0], np.cumsum(per)[:-1]])
    return lo, lo + per


def live_windows(rng, xn, yn, T, S, cap=2):
    """Arbitrary windows that keep one path alive: with the path at columns [lo_t, hi_t] of frame t (hi_t - lo_t < S),
    r_t is drawn uniformly from [hi_t - S + 1, lo_t], so every window holds its frame's part of the path.  The windows
    are neither monotone nor connected and clip on either side of the lattice wherever that range crosses 0 or Un - S.
    Lattice 0's first frame takes the low end of its range and its last frame the high end, so that with S > cap + 1
    both clip.  Padding frames get anything, INT32_MIN and INT32_MAX among it."""
    cap = min(cap, S - 1)
    N = len(xn)
    r = rng.randint(-S - 2, int(np.max(yn)) + 4, (N, T)).astype(np.int64)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        lo, hi = random_path(rng, Tn, Un, cap)
        r[n, :Tn] = [rng.randint(h - S + 1, l + 1) for l, h in zip(lo, hi)]
        if n == 0:
            r[n, 0], r[n, Tn - 1] = hi[0] - S + 1, lo[Tn - 1]
        if Tn < T:
            r[n, Tn:] = rng.choice([INT32_MIN, INT32_MAX, -S, Un, Un + 7, -1], T - Tn)
    return r.astype(np.int32)


def clipping_frames(r, xn, yn, S):
    """-> (live frames with r < 0, live frames with r + S > Un): how many windows clip on each side."""
    left = right = 0
    for n in range(len(xn)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        rr = r[n, :Tn].astype(np.int64)
        left += int((rr < 0).sum())
        right += int((rr + S > Un).sum())
    return left, right


def cut_windows(rng, r, xn, yn, S, n, kind):
    """Windows of lattice n changed so that no path survives (Tn, Un >= 2 unless named):
      "gap"       frames up to t* keep to columns [0, S - 1], the frame after starts at column S: no path crosses;
      "last"      the last frame misses the last column, so the final blank is removed;
      "int32_max" / "int32_min"  one live frame's window lies wholly outside the lattice;
      "one_frame" Tn = 1: the only window misses column 0;
      "no_labels" Un = 1: one frame's window misses column 0."""
    Tn, Un = int(xn[n]), int(yn[n]) + 1
    if kind == "gap":
        assert Tn >= 2 and Un > S
        ts = rng.randint(0, Tn - 1)
        r[n, :ts + 1] = rng.randint(-S + 1, 1, ts + 1)
        r[n, ts + 1] = rng.randint(S, Un)
    elif kind == "last":
        r[n, Tn - 1] = Un - 1 - S
    elif kind in ("int32_max", "int32_min"):
        r[n, rng.randint(0, Tn)] = INT32_MAX if kind == "int32_max" else INT32_MIN
    elif kind == "one_frame":
        assert Tn == 1
        r[n, 0] = 1
    elif kind == "no_labels":
        assert Un == 1
        r[n, rng.randint(0, Tn)] = 1
    else:
        raise ValueError(kind)
    return r
