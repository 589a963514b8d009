"""fp64 restatement of rnnt_loss_simple with k2's smoothing (lm_only_scale, am_only_scale), for the tests.

Written from the formulas of include/rnnt_b200.h in torch float64 on the CPU; the gradients come from autograd through
an anti-diagonal alpha recursion, so they are independent of the kernels' hand-derived backward:

    Ll[n,u]  = logsumexp_v lm[n,u,v]                 p = exp(lm - Ll)
    uni[v]   = mean over every n < N, u < U of p[n,u,v] + FLT_MIN
    Am[n,t]  = logsumexp_v (am[n,t,v] + log uni[v])
    pair_k   = c (am[t,k] + lm[u,k] - norm[t,u]) + sl (lm[u,k] - Ll[u]) + sa (am[t,k] + log uni[k] - Am[t])

for k in {blank, y_u}, c = 1 - sl - sa, a term with a zero scale left out.  A lattice with invalid lengths has cost NaN
and takes no part in the objective, but with sa > 0 its lm rows still enter the unigram.

smoothed() takes norm as a logsumexp over the (N,T,U,V) joint and runs autograd through a per-lattice alpha loop, so it
only reaches toy sizes.  factorised() is the same loss from the same pair formula (pairs()) without that tensor: the
normaliser as a per-lattice matrix product, alpha and beta in numpy over anti-diagonals for every lattice at once, and
autograd through the pair formula alone; it reaches the shapes the loss is used at (N=64 T=1500 U=300 V=50).  It
also takes k2's rnnt_type and delay_penalty: the penalty on the fp64 pairs' live label slots, the pair gradients of
the modified and constrained lattices from path_oracle.lattice."""
import numpy as np
import torch

from tests import path_oracle as pa

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


def pairs(a, l, norm, labels, yn, blank, sl, sa, detach_unigram=False, round_pairs=False):
    """The (blank, label) pairs (N,T,U) of every cell from am a (N,T,V), lm l (N,U,V) and the normaliser norm (N,T,U),
    float64 torch tensors in one autograd graph; y_u = labels[u] for u < yn, else blank."""
    N, T, V = a.shape
    U = l.shape[1]
    c = 1.0 - sl - sa
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
    return pb, pl


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
    go = np.ones(N) if grad_output is None else np.asarray(grad_output, np.float64)
    norm = torch.logsumexp(a[:, :, None, :] + l[:, None, :, :], dim=-1)               # (N,T,U)
    pb, pl = pairs(a, l, norm, labels, yn, blank, float(lm_only_scale), float(am_only_scale), detach_unigram,
                   round_pairs)
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


# ------------------------------------------------------------------------------------------ factorised
def alphas(B, L, Tn, Un):
    """alpha (N,T,U) of every lattice from its blank and label log-probs B, L (N,T,U), numpy fp64, one anti-diagonal
    per step for all lattices at once; -inf outside each lattice (Tn, Un), everywhere when Tn = 0."""
    N, T, U = B.shape
    a = np.full((N, T, U), -np.inf)
    a[:, 0, 0] = np.where(Tn > 0, 0.0, -np.inf)
    tt, uu = Tn[:, None], Un[:, None]
    with np.errstate(invalid="ignore"):
        for d in range(1, T + U - 1):
            t = np.arange(max(0, d - U + 1), min(d, T - 1) + 1)
            u = d - t
            tp, up = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
            top = np.where(t > 0, a[:, tp, u] + B[:, tp, u], -np.inf)
            left = np.where(u > 0, a[:, t, up] + L[:, t, up], -np.inf)
            a[:, t, u] = np.where((t < tt) & (u < uu), np.logaddexp(top, left), -np.inf)
    return a


def betas(B, L, Tn, Un):
    """beta (N,T,U), as alphas(): beta[Tn-1, Un-1] is the final blank's log-prob, -inf outside each lattice."""
    N, T, U = B.shape
    b = np.full((N, T, U), -np.inf)
    tt, uu = Tn[:, None], Un[:, None]
    end_t, end_u = np.where(Tn > 0, Tn - 1, -1)[:, None], (Un - 1)[:, None]
    with np.errstate(invalid="ignore"):
        for d in range(T + U - 2, -1, -1):
            t = np.arange(max(0, d - U + 1), min(d, T - 1) + 1)
            u = d - t
            tn, un = np.minimum(t + 1, T - 1), np.minimum(u + 1, U - 1)
            down = np.where(t + 1 < tt, b[:, tn, u] + B[:, t, u], -np.inf)
            right = np.where(u + 1 < uu, b[:, t, un] + L[:, t, u], -np.inf)
            val = np.where((t < tt) & (u < uu), np.logaddexp(down, right), -np.inf)
            b[:, t, u] = np.where((t == end_t) & (u == end_u), B[:, t, u], val)
    return b


def lattice_grads(B, L, Tn, Un):
    """-> (costs (N,), gb, gl (N,T,U)): -log P of every lattice and d cost / d (blank, label) log-prob of every cell,
    from alphas() and betas(); cost NaN and no gradient where Tn = 0 (invalid lengths)."""
    N, T, U = B.shape
    a, b = alphas(B, L, Tn, Un), betas(B, L, Tn, Un)
    ok = Tn > 0
    ll = np.where(ok, b[:, 0, 0], np.nan)
    lk = np.where(ok, ll, 0.0)[:, None, None]
    b_down = np.concatenate([b[:, 1:], np.full((N, 1, U), -np.inf)], axis=1)
    b_right = np.concatenate([b[:, :, 1:], np.full((N, T, 1), -np.inf)], axis=2)
    with np.errstate(invalid="ignore", over="ignore"):
        gb = -np.exp(a + b_down + B - lk)
        gl = -np.exp(a + b_right + L - lk)
        n = np.flatnonzero(ok)
        t, u = Tn[n] - 1, Un[n] - 1
        gb[n, t, u] = -np.exp(a[n, t, u] + B[n, t, u] - ll[n])
    live = (np.arange(T)[None, :, None] < Tn[:, None, None]) & (np.arange(U)[None, None, :] < Un[:, None, None])
    return -ll, np.where(live, gb, 0.0), np.where(live, gl, 0.0)


def factorised(am, lm, labels, xn, yn, blank=0, lm_only_scale=0.0, am_only_scale=0.0, grad_output=None,
               detach_unigram=False, round_pairs=False, rnnt_type="regular", delay_penalty=0.0):
    """smoothed(..., want_pairs=True) without the (N,T,U,V) tensor: -> (costs, d am, d lm, pair gradients), fp64.

    The normaliser is log(exp(am - oa) @ exp(lm - ol)^T) + oa + ol per lattice (oa, ol the rows' maxima, held
    constant: their gradient cancels), the pairs are pairs() above, and the recurrence runs in numpy over
    anti-diagonals for all lattices at once (lattice_grads).  d am and d lm then come from autograd through the pair
    formula with grad_output * (gb, gl) as the pairs' gradient, so the chain rule through the normaliser, Ll and the
    unigram is torch's, not the kernels'.  Arguments and meaning as smoothed()'s.

    rnnt_type, delay_penalty: rnnt_loss_simple's.  The penalty delay_penalty * ((Tn-1)/2 - t) is added in fp64 to the
    label pair of every live label slot (t < Tn, u < Un - 1), a constant that leaves the pairs' gradient alone; the
    modified and constrained lattices take their costs and pair gradients (folded, as the kernels write them) from
    path_oracle.lattice.  At the defaults this is the regular loss, unchanged."""
    a = torch.tensor(np.asarray(am, np.float64), requires_grad=True)
    l = torch.tensor(np.asarray(lm, np.float64), requires_grad=True)
    N, T, V = a.shape
    U = l.shape[1]
    go = np.ones(N) if grad_output is None else np.asarray(grad_output, np.float64)

    def offset(x):
        m = x.detach().amax(dim=-1, keepdim=True)
        return torch.where(torch.isfinite(m), m, torch.zeros_like(m))

    oa, ol = offset(a), offset(l)
    norm = torch.log(torch.exp(a - oa) @ torch.exp(l - ol).transpose(1, 2)) + oa + ol.transpose(1, 2)   # (N,T,U)
    pb, pl = pairs(a, l, norm, labels, yn, blank, float(lm_only_scale), float(am_only_scale), detach_unigram,
                   round_pairs)
    xn, yn = np.asarray(xn, np.int64), np.asarray(yn, np.int64)
    ok = (xn >= 1) & (xn <= T) & (yn >= 0) & (yn < U)
    Tn, Un = np.where(ok, xn, 0), np.where(ok, yn + 1, 0)
    if delay_penalty:
        t, u = np.arange(T)[None, :, None], np.arange(U)[None, None, :]
        tt, uu = Tn[:, None, None], Un[:, None, None]
        pen = np.where((t < tt) & (u < uu - 1), delay_penalty * ((tt - 1) / 2.0 - t), 0.0)
        pl = pl + torch.from_numpy(pen)
    if rnnt_type == "regular":
        costs, gb, gl = lattice_grads(pb.detach().numpy(), pl.detach().numpy(), Tn, Un)
    else:
        costs, g, _ = pa.lattice(np.stack([pb.detach().numpy(), pl.detach().numpy()], -1), xn, yn, rnnt_type)
        gb, gl = g[..., 0], g[..., 1]
    w = go[:, None, None]
    torch.autograd.backward([pb, pl], [torch.from_numpy(w * gb), torch.from_numpy(w * gl)])
    return costs, a.grad.numpy(), l.grad.numpy(), np.stack([gb, gl], axis=-1)
