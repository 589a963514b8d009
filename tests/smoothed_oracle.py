"""fp64 restatement of rnnt_loss_simple with k2's smoothing (lm_only_scale, am_only_scale), for the tests.

Written from the formulas of include/rnnt_b200.h in torch float64 on the CPU; the gradients come from autograd through
an anti-diagonal alpha recursion, so they are independent of the kernels' hand-derived backward:

    Ll[n,u]  = logsumexp_v lm[n,u,v]                 p = exp(lm - Ll)
    uni[v]   = mean over every n < N, u < U of p[n,u,v] + FLT_MIN
    Am[n,t]  = logsumexp_v (am[n,t,v] + log uni[v])
    pair_k   = c (am[t,k] + lm[u,k] - norm[t,u]) + sl (lm[u,k] - Ll[u]) + sa (am[t,k] + log uni[k] - Am[t])

for k in {blank, y_u}, c = 1 - sl - sa, a term with a zero scale left out.  A lattice with invalid lengths has cost NaN
and takes no part in the objective, but with sa > 0 its lm rows still enter the unigram."""
import numpy as np
import torch

FLT_MIN = float(np.finfo(np.float32).tiny)
SENTINEL = -1e30            # alpha outside the lattice: finite, so that logaddexp never meets -inf - (-inf)


def lengths_ok(Tn, Un, T, U):
    return 1 <= Tn <= T and 1 <= Un <= U


def _lae(a, b):
    m = torch.maximum(a, b)
    return m + torch.log(torch.exp(a - m) + torch.exp(b - m))


def lattice_cost(pb, pl, Tn, Un):
    """-log P of lattice (Tn, Un) from its (T,U) blank / label log-probs, alpha over anti-diagonals."""
    t = torch.arange(Tn)
    neg = torch.full((Tn,), SENTINEL, dtype=pb.dtype)
    prev = torch.where(t == 0, torch.zeros((), dtype=pb.dtype), neg)           # diagonal 0: alpha[0,0] = 0
    for d in range(1, Tn + Un - 1):
        u = d - t
        live = (u >= 0) & (u < Un)
        uc = u.clamp(0, Un - 1)
        # blank edge (t-1, u) -> (t, u)
        tm = (t - 1).clamp(min=0)
        from_b = torch.cat([neg[:1], prev[:-1]]) + pb[tm, uc]
        from_b = torch.where(live & (t >= 1), from_b, neg)
        # label edge (t, u-1) -> (t, u)
        from_l = prev + pl[t, (uc - 1).clamp(min=0)]
        from_l = torch.where(live & (u >= 1), from_l, neg)
        prev = torch.where(live, _lae(from_b, from_l), neg)
    return -(prev[Tn - 1] + pb[Tn - 1, Un - 1])


def smoothed(am, lm, labels, xn, yn, blank=0, lm_only_scale=0.0, am_only_scale=0.0, grad_output=None,
             detach_unigram=False, want_pairs=False, round_pairs=False):
    """-> (costs (N,), d sum_n grad_output[n] cost[n] / d am (N,T,V), ... / d lm (N,U,V)) as float64 numpy, and with
    want_pairs the (N,T,U,2) pair gradients d cost[n] / d pair (unscaled).  detach_unigram: the same loss with uni held
    constant in the backward, so that the difference of the two d lm is the unigram's own gradient term.
    round_pairs: run the recurrence on the pairs rounded to float32 (the gradient passes the rounding unchanged), as
    oracle.dense does with its log-probs; only for the comparison with simple_oracle."""
    a = torch.tensor(np.asarray(am, np.float64), requires_grad=True)
    l = torch.tensor(np.asarray(lm, np.float64), requires_grad=True)
    N, T, V = a.shape
    U = l.shape[1]
    sl, sa = float(lm_only_scale), float(am_only_scale)
    c = 1.0 - sl - sa
    go = np.ones(N) if grad_output is None else np.asarray(grad_output, np.float64)
    norm = torch.logsumexp(a[:, :, None, :] + l[:, None, :, :], dim=-1)               # (N,T,U)
    Ll = torch.logsumexp(l, dim=-1)                                                    # (N,U)
    if sa > 0:
        p = torch.exp(l - Ll[..., None])
        uni = p.mean(dim=(0, 1)) + FLT_MIN
        if detach_unigram:
            uni = uni.detach()
        lu = torch.log(uni)
        Am = torch.logsumexp(a + lu, dim=-1)                                           # (N,T)
    y = np.full((N, U), blank, np.int64)
    for n in range(N):
        k = int(yn[n])
        if 0 <= k < U:
            y[n, :k] = np.asarray(labels[n, :k], np.int64)
    yt = torch.from_numpy(y)

    def pair(k):                                                                       # k (N,U) -> (N,T,U)
        am_k = a.gather(2, k[:, None, :].expand(N, T, U))
        lm_k = l.gather(2, k[:, :, None])[:, :, 0]
        out = c * (am_k + lm_k[:, None, :] - norm)
        if sl > 0:
            out = out + sl * (lm_k - Ll)[:, None, :]
        if sa > 0:
            out = out + sa * (am_k + lu[k][:, None, :] - Am[:, :, None])
        return out

    pb = pair(torch.full((N, U), blank, dtype=torch.long))
    pl = pair(yt)
    if round_pairs:
        pb = pb + (pb.float().double() - pb).detach()
        pl = pl + (pl.float().double() - pl).detach()
    pb.retain_grad()
    pl.retain_grad()
    costs = np.full(N, np.nan)
    obj = torch.zeros((), dtype=torch.float64)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not lengths_ok(Tn, Un, T, U):
            continue
        cn = lattice_cost(pb[n], pl[n], Tn, Un)
        costs[n] = cn.item()
        obj = obj + go[n] * cn
    if obj.requires_grad:
        obj.backward()
    dam = a.grad.numpy() if a.grad is not None else np.zeros((N, T, V))
    dlm = l.grad.numpy() if l.grad is not None else np.zeros((N, U, V))
    if not want_pairs:
        return costs, dam, dlm
    pg = np.zeros((N, T, U, 2))
    for n in range(N):                     # the pair gradients of cost[n] alone: divide out grad_output
        if go[n] != 0:
            if pb.grad is not None:
                pg[n, :, :, 0] = pb.grad[n].numpy() / go[n]
                pg[n, :, :, 1] = pl.grad[n].numpy() / go[n]
    for n in range(N):
        Un = int(yn[n]) + 1
        pg[n, :, max(Un - 1, 0):, 1] = 0.0     # the last column has no label edge
    return costs, dam, dlm, pg
