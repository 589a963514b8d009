"""CPU: tests/hat_oracle.py against brute-force path enumeration and against torch.autograd in float64 of the pairs
as include/rnnt_b200.h states them (logsigmoid, logsumexp over the non-blank columns), for every lattice type, with
the delay penalty, FastEmit, blank != 0, labels equal to the blank in live cells and the pruned rows."""
import numpy as np
import pytest
import torch

from tests import hat_oracle as ho
from tests import path_oracle as po
from tests.pruned_oracle import window_rows


def torch_hat(x, blank):
    """the HAT log-probs of x (..., V) in torch, as k2's get_hat_logprobs composes them"""
    xb = x[..., blank:blank + 1]
    nb = torch.cat([x[..., :blank], x[..., blank + 1:]], -1)
    lab = torch.log_softmax(nb, -1) + torch.nn.functional.logsigmoid(-xb)
    return torch.cat([lab[..., :blank], torch.nn.functional.logsigmoid(xb), lab[..., blank:]], -1)


def torch_pairs(x, blank, lab):
    """(b, l) of the rows of x (..., V) with labels lab (...,) in torch: b = logsigmoid(x[B]),
    l = x[y] - logsumexp_{v != B} x[v] + logsigmoid(-x[B]) for every y, the blank included"""
    xb = x[..., blank]
    col = torch.arange(x.shape[-1])
    lse_nb = torch.logsumexp(torch.where(col == blank, torch.full_like(x, -float("inf")), x), -1)
    xy = x.gather(-1, lab[..., None])[..., 0]
    return torch.nn.functional.logsigmoid(xb), xy - lse_nb + torch.nn.functional.logsigmoid(-xb)


def inputs(N, T, U, V, seed, blank=0, label_blank=False):
    """label_blank: the first label of every lattice is the blank, and every lattice has at least one label, so that
    live cells carry a label equal to the blank"""
    rng = np.random.RandomState(seed)
    x = rng.randn(N, T, U, V) * 2.0
    ys = (rng.randint(1, V, (N, U - 1)) + blank) % V
    xn = rng.randint(max(1, T - 1), T + 1, N)
    yn = rng.randint(0, min(U, T + 1), N)
    if label_blank:
        ys[:, 0] = blank
        yn = np.maximum(yn, 1)
    return x, ys.astype(np.int32), xn.astype(np.int32), yn.astype(np.int32)


def test_label_equal_to_blank_is_the_stated_formula():
    """a label equal to the blank gets l = x[B] - lse_nb + logsigmoid(-x[B]), not the blank's own log-prob"""
    x, ys, xn, yn = inputs(2, 3, 3, 5, seed=6, blank=2, label_blank=True)
    P, lab = ho.dense_pairs(x, ys, blank=2)
    assert (lab[:, :, 0] == 2).all()
    want = x[..., 0, 2] - ho.lse_nb(x[..., 0, :], 2) + ho.logsigmoid(-x[..., 0, 2])
    np.testing.assert_allclose(P[..., 0, 1], want, rtol=1e-13)
    assert not np.allclose(P[..., 0, 1], P[..., 0, 0])


@pytest.mark.parametrize("blank", [0, 3])
def test_rows_sum_to_one(blank):
    x = np.random.RandomState(1).randn(7, 6) * 3
    lp = ho.hat_logprobs(x, blank)
    np.testing.assert_allclose(np.exp(lp).sum(-1), 1.0, rtol=1e-12)
    np.testing.assert_allclose(lp, torch_hat(torch.tensor(x), blank).numpy(), rtol=1e-12, atol=1e-12)


def test_every_nonblank_logit_masked_is_nan():
    x = np.array([[0.5, -np.inf, -np.inf, -np.inf]])
    assert np.isnan(ho.lse_nb(x, 0)).all()
    np.testing.assert_allclose(ho.hat_logprobs(x, 0)[0, 0], ho.logsigmoid(0.5))


@pytest.mark.parametrize("rnnt_type", po.TYPES)
@pytest.mark.parametrize("lam", [0.0, 0.4])
def test_costs_match_brute_force(rnnt_type, lam):
    x, ys, xn, yn = inputs(3, 4, 3, 5, seed=2, blank=1)
    costs, _ = ho.dense(x, ys, xn, yn, blank=1, rnnt_type=rnnt_type, delay_penalty=lam)
    P, _ = ho.dense_pairs(x, ys, blank=1)
    if lam:
        ho._penalise64(P, xn, yn, lam)
    want, _ = po.brute_force(P, xn, yn, rnnt_type)
    np.testing.assert_allclose(costs, want, rtol=1e-12)


# FastEmit is regular-only
@pytest.mark.parametrize("rnnt_type,lam,fe", [(k, lam, 0.0) for k in po.TYPES for lam in (0.0, 0.3)]
                         + [("regular", 0.0, 0.2), ("regular", 0.3, 0.2)])
@pytest.mark.parametrize("blank,label_blank", [(0, False), (2, False), (0, True)])
def test_grads_match_autograd(rnnt_type, lam, fe, blank, label_blank):
    N, T, U, V = 3, 4, 3, 5
    x, ys, xn, yn = inputs(N, T, U, V, seed=3, blank=blank, label_blank=label_blank)
    go = np.array([1.0, 0.5, 2.0])
    costs, grads = ho.dense(x, ys, xn, yn, blank=blank, rnnt_type=rnnt_type, delay_penalty=lam, fastemit_lambda=fe,
                            grad_output=go)
    # autograd of the composition, the lattice's pair gradients as upstream
    P, _ = ho.dense_pairs(x, ys, blank)
    if lam:
        ho._penalise64(P, xn, yn, lam)
    want_costs, g, _ = po.lattice(P, xn, yn, rnnt_type)
    g[..., 1] *= 1.0 + fe
    g *= go[:, None, None, None]
    xt = torch.tensor(x, requires_grad=True)
    lab = torch.tensor(np.concatenate([ys, np.full((N, 1), blank)], 1), dtype=torch.long)
    pairs = torch.stack(torch_pairs(xt, blank, lab[:, None, :].expand(N, T, U)), -1)
    np.testing.assert_allclose(pairs.detach().numpy(), ho.dense_pairs(x, ys, blank)[0], rtol=1e-12, atol=1e-12)
    pairs.backward(torch.tensor(g))
    np.testing.assert_allclose(costs, want_costs, rtol=1e-12)
    np.testing.assert_allclose(grads, xt.grad.numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("rnnt_type", po.TYPES)
def test_pruned_equals_dense_on_full_windows(rnnt_type):
    """windows of S = U starting at column 0 hold every cell: the pruned oracle is the dense one at those rows"""
    N, T, U, V = 2, 4, 3, 6
    x, ys, xn, yn = inputs(N, T, U, V, seed=4, blank=2)
    ranges = np.zeros((N, T), np.int32)
    cd, gd = ho.dense(x, ys, xn, yn, blank=2, rnnt_type=rnnt_type, delay_penalty=0.2)
    cp, gp = ho.pruned(x, ys, xn, yn, ranges, blank=2, rnnt_type=rnnt_type, delay_penalty=0.2)
    np.testing.assert_allclose(cp, cd, rtol=1e-12)
    n, t, s, u = window_rows(ranges, xn, yn, U)
    np.testing.assert_allclose(gp[n, t, s], gd[n, t, u], rtol=1e-12, atol=1e-15)


def test_pruned_grads_match_autograd():
    N, T, S, V, U = 2, 5, 2, 6, 4
    rng = np.random.RandomState(5)
    x = rng.randn(N, T, S, V)
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    ys[:, 1] = 0                                         # a label equal to the blank inside the windows
    xn = np.array([5, 4], np.int32)
    yn = np.array([3, 2], np.int32)
    ranges = np.minimum(np.arange(T)[None, :] // 2, yn[:, None] + 1 - S).astype(np.int32)
    costs, grads = ho.pruned(x, ys, xn, yn, ranges, blank=0, rnnt_type="modified")
    lab = np.concatenate([ys, np.zeros((N, 1), np.int32)], 1)
    n, t, s, u = window_rows(ranges, xn, yn, S)
    assert (lab[n, u] == 0).any() and (u < U - 1)[lab[n, u] == 0].any()
    xt = torch.tensor(x, requires_grad=True)
    it = [torch.tensor(a, dtype=torch.long) for a in (n, t, s)]
    pb, pl = torch_pairs(xt[it[0], it[1], it[2]], 0, torch.tensor(lab[n, u], dtype=torch.long))
    P = np.full((N, T, U, 2), -np.inf)
    P[n, t, u, 0], P[n, t, u, 1] = pb.detach().numpy(), pl.detach().numpy()
    want, g, _ = po.lattice(P, xn, yn, "modified")
    (pb * torch.tensor(g[n, t, u, 0]) + pl * torch.tensor(g[n, t, u, 1])).sum().backward()
    np.testing.assert_allclose(costs, want, rtol=1e-12)
    np.testing.assert_allclose(grads, xt.grad.numpy(), rtol=1e-10, atol=1e-12)
