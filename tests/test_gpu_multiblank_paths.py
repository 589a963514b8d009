"""GPU: the multi-blank planner's bounds, each side asserted through the launch record (rnnt_b200_debug_last_tdt_launch)
and checked against the fp64 oracle (tests/multiblank_oracle.py).

Planner (csrc/tdt.cu, tdt_plan with multiblank): ring slots max(d) + 1 in shared memory while (max(d) + 1) * U * 4
bytes fit the opt-in limit (227 KB on an H100), else 0 (read back from global memory); recurrence warps
min(ceil(U / 32), 16), column passes ceil(U / 512); candidate slots 5 for B <= 3, else 17."""
import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.multiblank_oracle import multiblank, random_case
from tests.test_gpu_tdt import gbound, tdt_record

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMEM_OPTIN = 227 * 1024


def run_and_check(N, T, U, V, durations, expect, seed=0, sigma=0.05, compact=False):
    B = len(durations)
    x, labels, xn, yn = random_case(np.random.RandomState(seed), N, T, U, V, B)
    xn[:], yn[0] = T, U - 1
    go = np.random.RandomState(seed + 1).uniform(0.5, 1.5, N)
    xt = torch.tensor(x, dtype=torch.float32, device=DEV)
    lab, xn_t, yn_t = (torch.tensor(a, device=DEV) for a in (labels, xn, yn))
    if compact:
        xt = torch.cat([xt[i, :xn[i], :yn[i] + 1].reshape(-1, V) for i in range(N)])
        lab = torch.cat([lab[i, :yn[i]] for i in range(N)])
    xt.requires_grad_(True)
    with w.compact_hints(T, U):
        c = w.rnnt_loss_multiblank(xt, lab, xn_t, yn_t, durations, sigma=sigma, compact=compact)
    rec = tdt_record()
    c.backward(torch.tensor(go, dtype=torch.float32, device=DEV))
    for k, v in expect.items():
        assert rec[k] == v, (k, rec)
    c0, g0, _, _ = multiblank(x.astype(np.float32).astype(np.float64), labels, xn, yn, durations, sigma)
    np.testing.assert_allclose(c.detach().cpu().numpy(), c0, rtol=1e-5)
    g0 = g0 * go[:, None, None, None]
    if compact:
        g0 = np.concatenate([g0[i, :xn[i], :yn[i] + 1].reshape(-1, V) for i in range(N)])
    err = np.abs(xt.grad.cpu().numpy() - g0).max()
    assert err <= gbound(T, U, c0), err
    return rec


@pytest.mark.parametrize("durations,kd", [((2, 4, 8), 5), ((2, 4, 8, 16), 17), (tuple(range(2, 17)), 17)])
def test_candidate_slots(durations, kd):
    run_and_check(3, 40, 6, len(durations) + 6, durations, dict(kd=kd, ring=max(durations) + 1, warps=1, passes=1))


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("U,warps,passes", [(512, 16, 1), (513, 16, 2), (1100, 16, 3)])
def test_column_passes(U, warps, passes, compact):
    run_and_check(2, 8, U, 7, (2, 4), dict(warps=warps, passes=passes, ring=5, smem=5 * U * 4), compact=compact)


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("U", [SMEM_OPTIN // (17 * 4), SMEM_OPTIN // (17 * 4) + 1])
def test_ring_at_its_limit(U, compact):
    """max(d) = 16: 17 ring slots; one column more and the ring reads back from global memory"""
    fits = 17 * U * 4 <= SMEM_OPTIN
    run_and_check(1, 20, U, 6, (2, 16), dict(ring=17 if fits else 0, smem=17 * U * 4 if fits else 0),
                  compact=compact)


def test_long_frames():
    run_and_check(2, 600, 9, 8, (2, 4, 8), dict(ring=9, warps=1))
