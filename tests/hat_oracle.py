"""numpy fp64 restatement of the HAT normalisation (Hybrid Autoregressive Transducer, k2's get_hat_logprobs) of
rnnt_loss_from_logits / rnnt_loss_pruned / rnnt_align_from_logits(use_hat_loss=True), for the tests
(include/rnnt_b200.h states the semantics).

hat_logprobs() is the normalised row: logsigmoid(x[blank]) at the blank, log_softmax over the non-blank columns plus
logsigmoid(-x[blank]) elsewhere, so exp of a row sums to 1.  hat_pair() is the (blank, label) pair of
include/rnnt_b200.h for any label y: b = logsigmoid(x[B]) and l = x[y] - lse_nb + logsigmoid(-x[B]), which is
hat_logprobs()[y] for y != blank but not for a label equal to the blank (there l is not b).  dense() and pruned() build the pairs with it, add
the delay penalty in fp64, run path_oracle.lattice() for any rnnt_type and apply the HAT Jacobian, the derivative of
hat_pair(), to the pair gradients (row_grads())."""
import numpy as np

from tests.path_oracle import lattice, lengths_ok
from tests.pruned_oracle import window_rows


def logsigmoid(z):
    z = np.asarray(z, np.float64)
    return np.minimum(z, 0.0) - np.log1p(np.exp(-np.abs(z)))


def sigmoid(z):
    return np.exp(logsigmoid(z))


def lse_nb(x, blank):
    """the normaliser over the columns v != blank, (..., ) fp64"""
    x = np.array(x, np.float64, copy=True)
    x[..., blank] = -np.inf
    m = x.max(axis=-1, keepdims=True)
    with np.errstate(invalid="ignore"):
        return (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))[..., 0]


def hat_logprobs(x, blank):
    """(..., V) HAT log-probs of the rows of x, fp64"""
    x = np.asarray(x, np.float64)
    xb = x[..., blank:blank + 1]
    out = x - lse_nb(x, blank)[..., None] + logsigmoid(-xb)
    out[..., blank] = logsigmoid(xb)[..., 0]
    return out


def hat_pair(x, blank, lab):
    """(b, l) (..., ) fp64 of the rows of x (..., V) with labels lab (...,): b = logsigmoid(x[B]) and
    l = x[y] - lse_nb + logsigmoid(-x[B]) for every y, the blank included"""
    x = np.asarray(x, np.float64)
    xb = x[..., blank]
    xy = np.take_along_axis(x, np.asarray(lab, np.int64)[..., None], -1)[..., 0]
    return logsigmoid(xb), xy - lse_nb(x, blank) + logsigmoid(-xb)


def row_grads(x, blank, lab, qb, ql):
    """(..., V) d / d x of qb * b + ql * l for the rows of x with labels lab (...,): the HAT Jacobian applied to the
    pair gradients, gl ([v == y] - softmax_nb(x)[v]) at v != blank, qb sigmoid(-x[B]) - ql sigmoid(x[B]) at the blank
    (plus ql when the label is the blank)."""
    x = np.asarray(x, np.float64)
    qb, ql = np.asarray(qb, np.float64), np.asarray(ql, np.float64)
    xb = x[..., blank]
    with np.errstate(invalid="ignore"):
        p = np.exp(x - lse_nb(x, blank)[..., None])
        p[..., blank] = 0.0
        g = -ql[..., None] * p
        g[..., blank] += qb * sigmoid(-xb) - ql * sigmoid(xb)
    np.put_along_axis(g, np.asarray(lab, np.int64)[..., None],
                      np.take_along_axis(g, np.asarray(lab, np.int64)[..., None], -1) + ql[..., None], -1)
    return g


def _penalise64(P, xn, yn, lam):
    N, T, U, _ = P.shape
    for k in range(N):
        Tn, Un = int(xn[k]), int(yn[k]) + 1
        if lengths_ok(Tn, Un, T, U):
            P[k, :Tn, :Un - 1, 1] += lam * ((Tn - 1) / 2.0 - np.arange(Tn))[:, None]


def dense_pairs(logits, labels, blank=0):
    """(N,T,U,2) fp64 HAT pairs of dense logits (N,T,U,V), the label on the last column being the blank"""
    x = np.asarray(logits, np.float64)
    N, T, U, V = x.shape
    lab = np.concatenate([np.asarray(labels, np.int64), np.full((N, 1), blank, np.int64)], axis=1)
    lab = np.broadcast_to(lab[:, None, :], (N, T, U))
    return np.stack(hat_pair(x, blank, lab), -1), lab


def dense(logits, labels, xn, yn, blank=0, rnnt_type="regular", delay_penalty=0.0, fastemit_lambda=0.0,
          grad_output=None):
    """-> (costs (N,), d sum_n grad_output[n] cost[n] / d logits (N,T,U,V)), fp64.  FastEmit (regular only) scales the
    label gradients by 1 + lambda and leaves the costs.  Classes are lattice()'s."""
    assert rnnt_type == "regular" or not fastemit_lambda
    x = np.asarray(logits, np.float64)
    P, lab = dense_pairs(x, labels, blank)
    if delay_penalty:
        _penalise64(P, xn, yn, delay_penalty)
    costs, g, _ = lattice(P, xn, yn, rnnt_type)
    g[..., 1] *= 1.0 + fastemit_lambda
    go = np.ones(len(costs)) if grad_output is None else np.asarray(grad_output, np.float64)
    grads = row_grads(x, blank, lab, g[..., 0], g[..., 1]) * go[:, None, None, None]
    return costs, grads


def pruned(logits, labels, xn, yn, ranges, blank=0, rnnt_type="regular", delay_penalty=0.0, fastemit_lambda=0.0,
           grad_output=None):
    """rnnt_loss_pruned(use_hat_loss=True) restated, as path_oracle.pruned restates the log_softmax one: -> (costs (N,),
    d sum_n grad_output[n] cost[n] / d logits (N,T,S,V)), fp64; rows that are not lattice cells get zeros."""
    assert rnnt_type == "regular" or not fastemit_lambda
    x = np.asarray(logits, np.float64)
    labels = np.asarray(labels)
    N, T, S, V = x.shape
    U = labels.shape[1] + 1
    lab = np.concatenate([labels.astype(np.int64), np.full((N, 1), blank, np.int64)], axis=1)
    n, t, s, u = window_rows(ranges, xn, yn, S)
    cl = lab[n, u]
    P = np.full((N, T, U, 2), -np.inf)
    P[n, t, u, 0], P[n, t, u, 1] = hat_pair(x[n, t, s], blank, cl)
    if delay_penalty:
        _penalise64(P, xn, yn, delay_penalty)
    costs, g, _ = lattice(P, xn, yn, rnnt_type)
    g[..., 1] *= 1.0 + fastemit_lambda
    go = np.ones(N) if grad_output is None else np.asarray(grad_output, np.float64)
    grads = np.zeros_like(x)
    grads[n, t, s] = row_grads(x[n, t, s], blank, cl, g[n, t, u, 0], g[n, t, u, 1]) * go[n][:, None]
    return costs, grads
