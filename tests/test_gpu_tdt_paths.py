"""GPU: every launch configuration the TDT planner can take, on both sides of each of its bounds, each case asserting
its launch record (rnnt_b200_debug_last_tdt_launch) and checking costs and logit gradients against the eager fp64
restatement (tests/tdt_eager.py, autograd on the GPU).

Planner (csrc/tdt.cu, tdt_plan): normaliser lanes 8 when V + D <= 64 else 32, elements per load 4 / 2 / 1 from the row
width and the element alignment; recurrence warps min(ceil(U / 32), 16), column passes ceil(U / 512), ring slots
max(d) + 2 in shared memory while (max(d) + 2) * U * 4 bytes fit the opt-in limit (227 KB on an H100), else 0 (read
back from global memory); candidate slots 5 for D <= 5, else 17."""
import math

import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.tdt_eager import tdt_costs
from tests.test_gpu_tdt import gbound, tdt_record

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMEM_OPTIN = 227 * 1024


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def inputs(N, T, U, V, D, seed, full=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, T, U, V + D, generator=g)
    labels = torch.randint(1, V, (N, U - 1), generator=g, dtype=torch.int32)
    xn = torch.randint(max(1, T // 2), T + 1, (N,), generator=g, dtype=torch.int32)
    yn = torch.randint(max(0, (U - 1) // 2), U, (N,), generator=g, dtype=torch.int32)
    xn[0], yn[0] = T, U - 1
    if full:
        xn[:], yn[:] = T, U - 1
    return x, labels, xn, yn


def run_and_check(N, T, U, V, durations, expect, seed=0, sigma=0.05, blank=0, offset=0):
    D = len(durations)
    x, labels, xn, yn = inputs(N, T, U, V, D, seed)
    buf = torch.empty(x.numel() + offset, device=DEV)
    xd = buf[offset:].view(x.shape)
    xd.copy_(x)
    xd.requires_grad_(True)
    args = [t.to(DEV) for t in (labels, xn, yn)]
    go = torch.rand(N, device=DEV) + 0.5
    c = w.rnnt_loss_tdt(xd, *args, durations, sigma=sigma, blank=blank)
    rec = tdt_record()
    c.backward(go)
    rec.update({k: v for k, v in tdt_record().items() if k.startswith("emit")})
    for k, v in expect.items():
        assert rec[k] == v, (k, rec)
    x64 = x.double().to(DEV).requires_grad_(True)
    c0 = tdt_costs(x64, *args, durations, sigma, blank)
    (c0 * go.double()).sum().backward()
    c0n = c0.detach().cpu().numpy()
    np.testing.assert_allclose(c.detach().cpu().numpy(), c0n, rtol=1e-5)
    err = (xd.grad.double() - x64.grad).abs().max().item()
    assert err <= gbound(T, U, c0n), err
    return rec


@pytest.mark.parametrize("durations,kd", [((1,), 5), ((0, 1, 2, 3, 4), 5), ((0, 1, 2, 3, 4, 5), 17),
                                          (tuple(range(17)), 17)])
def test_candidate_slots(durations, kd):
    run_and_check(3, 40, 6, 7, durations, dict(kd=kd, ring=max(durations) + 2, warps=1, passes=1))


@pytest.mark.parametrize("U,warps,passes", [(32, 1, 1), (33, 2, 1), (512, 16, 1), (513, 16, 2), (2048, 16, 4),
                                            (2049, 16, 5)])
def test_column_passes(U, warps, passes):
    run_and_check(2, 12, U, 6, (0, 1, 2), dict(warps=warps, passes=passes, ring=4, smem=4 * U * 4))


@pytest.mark.parametrize("U", [SMEM_OPTIN // (18 * 4), SMEM_OPTIN // (18 * 4) + 1])
def test_ring_at_its_limit(U):
    """max(d) = 16: 18 ring slots; one column more and the ring reads back from global memory"""
    fits = 18 * U * 4 <= SMEM_OPTIN
    run_and_check(1, 20, U, 4, (0, 1, 16), dict(ring=18 if fits else 0, smem=18 * U * 4 if fits else 0))


def test_long_frames():
    run_and_check(2, 1600, 9, 5, (0, 1, 2, 3, 4), dict(ring=6, warps=1))


@pytest.mark.parametrize("V,D,offset,group,lanes", [
    (28, 4, 0, 4, 8), (28, 4, 1, 1, 8), (28, 4, 2, 2, 8), (29, 5, 0, 2, 8), (27, 5, 1, 1, 8), (27, 3, 0, 2, 8),
    (123, 5, 0, 4, 32), (125, 5, 0, 2, 32), (125, 5, 2, 2, 32), (124, 5, 0, 1, 32),
    (59, 5, 0, 4, 8), (60, 5, 0, 1, 32)])                              # W = 64 and 65: both sides of the lane bound
def test_normaliser_branches(V, D, offset, group, lanes):
    run_and_check(2, 10, 5, V, tuple(range(D)), dict(norm_group=group, norm_lanes=lanes,
                                                     emit_vec=4, emit_xvec=int(offset == 0)),
                  offset=offset, blank=V - 1)


def test_every_row_thread_iterates_its_grid_stride():
    """more rows than the normaliser's and the posterior pass's grids cover (16 CTAs per SM), and more vectors than the
    emit's (32 CTAs per SM): each thread of those kernels runs its grid-stride loop more than once"""
    s = sms()
    T = U = 200
    N = max(2, math.ceil(s * 16 * 256 * 1.5 / (T * U)))
    V, D = 3, 5
    assert N * T * U > s * 16 * 256 and N * T * U * (V + D) / 4 > s * 32 * 256
    x, labels, xn, yn = inputs(N, T, U, V, D, 5, full=True)
    xd = x.to(DEV).requires_grad_(True)
    args = [t.to(DEV) for t in (labels, xn, yn)]
    c = w.rnnt_loss_tdt(xd, *args, (0, 1, 2, 3, 4), blank=0)
    c.sum().backward()
    rec = tdt_record()
    assert rec["norm_lanes"] == 8 and rec["emit_vec"] == 4
    # the stride must not change values: the first lattice alone gives the same bits
    x1 = x[:1].to(DEV).requires_grad_(True)
    c1 = w.rnnt_loss_tdt(x1, *[a[:1] for a in args], (0, 1, 2, 3, 4), blank=0)
    c1.sum().backward()
    assert torch.equal(c1.detach(), c.detach()[:1]) and torch.equal(x1.grad, xd.grad[:1])
    x64 = x[:1].double().to(DEV).requires_grad_(True)
    c0 = tdt_costs(x64, *[a[:1] for a in args], (0, 1, 2, 3, 4), 0.0, 0)
    c0.sum().backward()
    np.testing.assert_allclose(c1.detach().cpu().numpy(), c0.detach().cpu().numpy(), rtol=1e-5)
    assert (x1.grad.double() - x64.grad).abs().max().item() <= gbound(T, U, c0.detach().cpu().numpy())


def test_bf16_beyond_2_31_elements():
    """one bf16 call with more than 2^31 logit elements (int64 offsets throughout): the last lattice, whose rows lie
    past element 2^31, gives the same bits as a call on that lattice alone, and its gradient rows sum to 0"""
    N, T, U, V, D = 4, 1000, 530, 1025, 5
    assert N * T * U * (V + D) > 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(N, T, U, V + D, device=DEV, dtype=torch.bfloat16, generator=g).requires_grad_(True)
    labels = torch.randint(1, V, (N, U - 1), device=DEV, dtype=torch.int32, generator=g)
    xn = torch.full((N,), T, dtype=torch.int32, device=DEV)
    yn = torch.full((N,), U - 1, dtype=torch.int32, device=DEV)
    xn[3], yn[3] = T - 7, U - 12
    c = w.rnnt_loss_tdt(x, labels, xn, yn, (0, 1, 2, 3, 4))
    c.sum().backward()
    assert torch.isfinite(c).all()
    last_c, last_g = c.detach()[3:].clone(), x.grad[3:].clone()
    x.grad = None
    x1 = x.detach()[3:].clone().requires_grad_(True)
    del x
    torch.cuda.empty_cache()
    c1 = w.rnnt_loss_tdt(x1, labels[3:], xn[3:], yn[3:], (0, 1, 2, 3, 4))
    c1.sum().backward()
    assert torch.equal(c1.detach(), last_c) and torch.equal(x1.grad, last_g)
    rows = last_g[0, :T - 7, :U - 11].float()
    assert rows[..., :V].sum(-1).abs().max().item() < 1e-2 and rows[..., V:].sum(-1).abs().max().item() < 1e-2
