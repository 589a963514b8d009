"""GPU: compact packing of the joint network's input (SURVEY.md 8(f)3) against the reference's own recipe
(the reference's pytorch_binding/benchmark2.py:37-50: a python loop over the batch + cat) and its autograd backward.
Forward is exact (one fp32 add per element); the backward sums in a fixed order, compared to 1e-5 relative."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def reference_pack(f, g, lf, lg):
    H = f.size(-1)
    return torch.cat([(f[i, :lf[i]].unsqueeze(1) + g[i, :lg[i] + 1].unsqueeze(0)).view(-1, H) for i in range(f.size(0))], dim=0)


@pytest.mark.parametrize("shape", [(3, 11, 5, 8), (4, 37, 20, 640), (2, 50, 9, 30), (5, 16, 33, 129), (1, 7, 1, 4)])
def test_joint_pack_matches_reference_recipe(w, shape):
    N, T, U1, H = shape
    g0 = torch.Generator(device="cuda").manual_seed(N + H)
    f = torch.randn(N, T, H, device="cuda", generator=g0)
    g = torch.randn(N, U1, H, device="cuda", generator=g0)
    lf = torch.randint(max(T // 2, 1), T + 1, (N,), dtype=torch.int, device="cuda", generator=g0)
    lg = torch.randint(0, U1, (N,), dtype=torch.int, device="cuda", generator=g0)
    lf[0], lg[0] = T, U1 - 1
    fa, ga = f.clone().requires_grad_(True), g.clone().requires_grad_(True)
    fb, gb = f.clone().requires_grad_(True), g.clone().requires_grad_(True)
    x = w.joint_pack(fa, ga, lf, lg)
    xr = reference_pack(fb, gb, lf, lg)
    assert x.shape == xr.shape and torch.equal(x, xr)
    wgt = torch.randn(x.shape, device="cuda", generator=g0)
    (x * wgt).sum().backward()
    (xr * wgt).sum().backward()
    np.testing.assert_allclose(fa.grad.cpu().numpy(), fb.grad.cpu().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ga.grad.cpu().numpy(), gb.grad.cpu().numpy(), rtol=1e-5, atol=1e-5)
    # sync-free variant: the caller knows STU
    x2 = w.joint_pack(f, g, lf, lg, stu=int(x.size(0)))
    assert torch.equal(x2, x)


def test_joint_pack_feeds_the_compact_loss(w):
    """joint_pack -> Linear -> log_softmax -> rnnt_loss(compact=True): same loss and parameter gradients as the padded
    joint -> rnnt_loss on the dense layout."""
    N, T, U1, H, V = 3, 14, 6, 16, 9
    g0 = torch.Generator(device="cuda").manual_seed(1)
    f = torch.randn(N, T, H, device="cuda", generator=g0).requires_grad_(True)
    g = torch.randn(N, U1, H, device="cuda", generator=g0).requires_grad_(True)
    lin = torch.nn.Linear(H, V).cuda()
    lf = torch.tensor([14, 9, 12], dtype=torch.int, device="cuda")
    lg = torch.tensor([5, 3, 4], dtype=torch.int, device="cuda")
    ys = torch.randint(1, V, (N, U1 - 1), dtype=torch.int, device="cuda", generator=g0)
    ys_c = torch.cat([ys[i, :lg[i]] for i in range(N)]).contiguous()
    lp_c = torch.log_softmax(lin(torch.tanh(w.joint_pack(f, g, lf, lg))), -1)
    loss_c = w.rnnt_loss(lp_c, ys_c, lf, lg, reduction="sum", compact=True)
    gc = torch.autograd.grad(loss_c, [f, g, lin.weight])
    lp_d = torch.log_softmax(lin(torch.tanh(f.unsqueeze(2) + g.unsqueeze(1))), -1)
    loss_d = w.rnnt_loss(lp_d, ys, lf, lg, reduction="sum")
    gd = torch.autograd.grad(loss_d, [f, g, lin.weight])
    np.testing.assert_allclose(loss_c.item(), loss_d.item(), rtol=1e-5)
    for a, b in zip(gc, gd):
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-4, atol=1e-5)
