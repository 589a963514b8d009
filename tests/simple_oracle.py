"""numpy restatements of rnnt_loss_simple (warp_rnnt_b200/__init__.py) and of its prune ranges, for the tests.

simple() materialises the simple joint am[:, :, None] + lm[:, None] in fp64 and runs the already tested
oracle.from_logits on it; d am and d lm are that logit gradient summed over u and over t.  It needs no recurrence of its
own.

prune_ranges() states the ranges rule of include/rnnt_b200.h (rnnt_b200_prune_ranges) literally, in numpy float32: each
window's score is added in fp32 in increasing u and the subtraction applied last, so sums, NaNs and ties come out as the
kernel's do, bit for bit.  It is vectorised over frames only; every fp32 operation is the kernel's."""
import numpy as np

from oracle import oracle


def simple(am, lm, labels, xn, yn, blank=0, grad_output=None):
    """-> (costs (N,), d sum_n grad_output[n] cost[n] / d am (N,T,V), ... / d lm (N,U,V)), fp64.  As in
    oracle.from_logits, a label equal to blank is not supported."""
    x = np.asarray(am, np.float64)[:, :, None] + np.asarray(lm, np.float64)[:, None]
    costs, g = oracle.from_logits(x, labels, xn, yn, blank, grad_output=grad_output)
    return costs, g.sum(axis=2), g.sum(axis=1)


def lengths_ok(Tn, Un, T, U):
    return 1 <= Tn <= T and 1 <= Un <= U


def prune_ranges(pair_grads, xn, yn, S):
    """ranges (N,T) int32 from pair gradients (N,T,U,2) float32, as rnnt_b200_prune_ranges computes them."""
    pg = np.asarray(pair_grads, np.float32)
    N, T, U, _ = pg.shape
    out = np.zeros((N, T), np.int64)
    tt = np.arange(T, dtype=np.int64)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U) or Un <= S:
            continue
        top = Un - S
        ob, ol = -pg[n, :, :, 0], -pg[n, :, :, 1]
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
        c = (S - 1) * tt - b
        cp = np.minimum.accumulate(c[::-1])[::-1]
        out[n] = (S - 1) * tt - np.maximum(cp, 0)
    return out.astype(np.int32)


def prune_ranges_scalar(pair_grads, xn, yn, S):
    """The same rule with one Python loop per frame and window, np.float32 scalars: the restatement above must equal
    it (vectorising over frames changes no operation)."""
    pg = np.asarray(pair_grads, np.float32)
    N, T, U, _ = pg.shape
    out = np.zeros((N, T), np.int32)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U) or Un <= S:
            continue
        r0 = [Un - S] * T
        for t in range(Tn - 1):
            best, best_r = None, 0
            for r in range(Un - S + 1):
                sc = np.float32(0.0)
                for u in range(r, r + S):
                    sc = np.float32(sc + np.float32(-pg[n, t, u, 0]))
                if r > 0:
                    sc = np.float32(sc - np.float32(-pg[n, t, r - 1, 1]))
                if not np.isnan(sc) and (best is None or sc > best):
                    best, best_r = sc, r
            r0[t] = best_r
        b = [0] * T
        c = [0] * T
        m = None
        for t in range(T - 1, -1, -1):
            m = r0[t] if m is None else min(m, r0[t])
            b[t] = m
        m = None
        for t in range(T - 1, -1, -1):
            ct = (S - 1) * t - b[t]
            m = ct if m is None else min(m, ct)
            c[t] = m
        for t in range(T):
            out[n, t] = (S - 1) * t - max(c[t], 0)
    return out


def reachable(Tn, Un, S):
    """Windows of S columns that start at 0 and move by at most S-1 per frame reach the last label by frame Tn-1."""
    return Un - S <= (S - 1) * (Tn - 1)


def check_ranges(ranges, xn, yn, S, U):
    """The properties every ranges tensor must have; raises AssertionError with the lattice that breaks one."""
    ranges = np.asarray(ranges, np.int64)
    N, T = ranges.shape
    for n in range(N):
        r = ranges[n]
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U):
            assert (r == 0).all(), n
            continue
        top = max(Un - S, 0)
        assert r[0] == 0, n
        d = np.diff(r)
        assert (d >= 0).all() and (d <= S - 1).all(), (n, r)
        assert (r >= 0).all() and (r <= top).all(), (n, r)
        if reachable(Tn, Un, S):
            assert r[Tn - 1] + S - 1 >= Un - 1, (n, r)
        else:
            assert r[Tn - 1] == (S - 1) * (Tn - 1), (n, r)


def pair_grads_of(lp, labels, xn, yn, blank=0):
    """The (N,T,U,2) pair gradients of the fp64 oracle on log-probs (N,T,U,V), in float32: real occupations."""
    _, g = oracle.dense(lp, labels, xn, yn, blank)
    N, T, U, V = lp.shape
    lab = np.concatenate([labels, np.full((N, 1), blank, labels.dtype)], axis=1)
    gb = g[..., blank]
    gl = np.take_along_axis(g, np.broadcast_to(lab[:, None, :, None], (N, T, U, 1)), axis=3)[..., 0]
    gl[:, :, -1] = 0.0
    for n in range(N):
        gl[n, :, int(yn[n]):] = 0.0
    return np.stack([gb, gl], axis=-1).astype(np.float32)
