"""Eager PyTorch restatement of the TDT loss (rnnt_loss_tdt) along anti-diagonals, differentiable by autograd.

It runs on any device and dtype: in float64 it is the reference of the GPU tests on lattices too large for the numpy
oracle (tests/tdt_oracle.py); in float32 it is what a user would write without the library (tools/tdt_time.py).
Masked (-inf) log-probs are clamped to -1e30, as the kernels do, so autograd never forms -inf - -inf.  Lattices with
valid lengths and labels only (a lattice without a path gets +inf, as from the kernels); the other degenerate classes
are the numpy oracle's to check."""
import torch

BIG = -1.0e30


def tdt_costs(x, labels, xn, yn, durations, sigma=0.0, blank=0):
    """x (N,T,U,V+D) -> costs (N,), -log P per lattice; differentiable w.r.t. x."""
    N, T, U, W = x.shape
    D = len(durations)
    V = W - D
    dev = x.device
    lt = torch.log_softmax(x[..., :V], -1) - sigma
    ld = torch.log_softmax(x[..., V:], -1).clamp(min=BIG)
    lab = torch.cat([labels.long(), torch.full((N, 1), blank, dtype=torch.long, device=dev)], 1)   # (N, U)
    lb = lt[..., blank].clamp(min=BIG)                                                              # (N, T, U)
    ll = torch.gather(lt, 3, lab[:, None, :, None].expand(N, T, U, 1))[..., 0].clamp(min=BIG)
    ll = torch.cat([ll[..., :U - 1], torch.full_like(ll[..., U - 1:], BIG)], -1)                   # no label edge at U-1
    u = torch.arange(U, device=dev)
    n_idx = torch.arange(N, device=dev)[:, None]
    big = torch.full((N, U), BIG, dtype=x.dtype, device=dev)

    def on_diag(a, s):
        """a (N,T,U,...) at the cells (s - u, u) of diagonal s, (N, U, ...); BIG off the lattice"""
        t = s - u
        ok = (t >= 0) & (t < T)
        v = a[n_idx, t.clamp(0, T - 1)[None, :], u[None, :]]
        mask = ok[None, :] if v.dim() == 2 else ok[None, :, None]
        return torch.where(mask, v, torch.full_like(v, BIG))

    diags = []                          # alpha along diagonal s, (N, U), indexed by column u
    wdiag = []                          # (blank weights (N,U), label weights (N,U), ld (N,U,D)) of diagonal s
    S = T + U - 1
    for s in range(S):
        wdiag.append((on_diag(lb, s), on_diag(ll, s), on_diag(ld, s)))
        if s == 0:
            diags.append(torch.where(u[None, :] == 0, torch.zeros_like(big), big))
            continue
        c = []
        for j, d in enumerate(durations):
            sp = s - d                                  # blank source (t-d, u) on diagonal s-d, same column
            if d > 0 and sp >= 0:
                b, _, l_d = wdiag[sp]
                c.append(diags[sp] + b + l_d[..., j])
            sq = s - d - 1                              # label source (t-d, u-1) on diagonal s-d-1, column u-1
            if sq >= 0:
                _, lw, l_d = wdiag[sq]
                v = diags[sq] + lw + l_d[..., j]
                c.append(torch.cat([big[:, :1], v[:, :-1]], 1))
        if not c:
            diags.append(big)
            continue
        a = torch.logsumexp(torch.stack(c), 0)
        t = s - u
        diags.append(torch.where(((t >= 0) & (t < T))[None, :], a, big))
    # terminal: blanks of duration d > 0 from (Tn - d, Un - 1)
    Tn, Un = xn.long(), yn.long() + 1
    ends = []
    for j, d in enumerate(durations):
        if d == 0:
            continue
        t0 = Tn - d
        ok = t0 >= 0
        t0c = t0.clamp(min=0)
        s = t0c + Un - 1
        a = torch.stack([diags[int(si)][i, int(ui)] for i, (si, ui) in enumerate(zip(s.tolist(), (Un - 1).tolist()))])
        w = lb[torch.arange(N, device=dev), t0c, Un - 1] + ld[torch.arange(N, device=dev), t0c, Un - 1, j]
        ends.append(torch.where(ok, a + w, torch.full_like(w, BIG)))
    cost = -torch.logsumexp(torch.stack(ends), 0)
    return torch.where(cost >= -0.5 * BIG, torch.full_like(cost, float("inf")), cost)   # no path: +inf
