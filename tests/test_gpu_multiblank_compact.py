"""GPU: rnnt_loss_multiblank(compact=True), the multi-blank loss on compact (STU, V) logits in joint_pack's row order.

The compact call is checked bit for bit against the dense call on xp, the same rows placed in a padded (N,T,U,V)
tensor at the same element offset modulo 4 with NaN in the padding: costs, lse, the posteriors and the gradient's live
rows are torch.equal.  The dense call is checked against fp64 in test_gpu_multiblank.py; here the compact results are
also compared with the fp64 oracle.  Then the hints, the compact classes, graphs and the one host copy."""
import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.multiblank_oracle import multiblank, random_case
from tests.test_gpu_tdt import gbound, tdt_record
from tests.test_gpu_tdt_compact import layouts, pack

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16


def case(N, T, U, V, B, seed):
    """random_case with ragged lengths, plus a lattice with Tn = 1 and one with yn = 0"""
    x, labels, xn, yn = random_case(np.random.RandomState(seed), N, T, U, V, B)
    if N >= 3:
        xn[1] = 1
        yn[2] = 0
    return x, labels, xn, yn


def rows_of(xn, yn, i):
    start = int(sum(int(xn[k]) * (int(yn[k]) + 1) for k in range(i)))
    return slice(start, start + int(xn[i]) * (int(yn[i]) + 1))


def parity(x, labels, xn, yn, durations, sigma=0.05, blank=None, dtype=torch.float32, offset=0, hints=(0, 0)):
    """compact == dense on xp, bit for bit"""
    b = x.shape[-1] - 1 if blank is None else blank
    xp, xc, ys, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, dtype, offset)
    go = torch.linspace(0.5, 1.5, len(xn), device=DEV)
    cd, ld, pd = w._C.rnnt_multiblank_forward(xp, ys, xn_t, yn_t, list(durations), sigma, b, True)
    gd = w._C.rnnt_multiblank_backward(xp, ld, pd, ys, list(durations), go, b)
    c, l, p, pref = w._C.rnnt_multiblank_compact_forward(xc, ys_c, xn_t, yn_t, list(durations), sigma, b, True, *hints)
    rec = tdt_record()
    g = w._C.rnnt_multiblank_compact_backward(xc, l, p, ys_c, xn_t, yn_t, pref, list(durations), go, b)
    assert torch.equal(c, cd)
    assert torch.equal(l, pack(ld, xn, yn)) and torch.equal(p, pack(pd, xn, yn))
    assert g.dtype == dtype and torch.equal(g, pack(gd, xn, yn))
    return rec, c, g


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("V", [32, 33, 34, 35])                    # V % 4 = 0, 1, 2, 3
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_parity_row_widths_and_offsets(dtype, V, offset):
    x, labels, xn, yn = case(6, 12, 6, V, 3, V * 10 + offset)
    labels[0, 1] = V - 1                                            # a label equal to the standard blank
    parity(x, labels, xn, yn, (2, 4, 8), 0.05, None, dtype, offset)


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("durations", [(2,), (2, 3, 5, 9, 16), (16,)])
@pytest.mark.parametrize("blank", ["default", "B"])
def test_parity_durations_and_blank(dtype, durations, blank):
    B = len(durations)
    x, labels, xn, yn = case(7, 21, 7, B + 8, B, 7 * B + durations[-1])
    b = None if blank == "default" else B
    if b is not None:
        labels = labels + B + 1
    parity(x, labels, xn, yn, durations, 0.05, b, dtype)


def test_against_fp64_with_and_without_hints():
    durations = (2, 4, 8)
    x, labels, xn, yn = case(5, 20, 6, 12, 3, 3)
    go = torch.linspace(0.5, 1.5, 5, device=DEV)
    for hints in ((0, 0), (20, 6), (25, 9)):
        rec, c, g = parity(x, labels, xn, yn, durations, 0.05, None, torch.float32, 0, hints)
        assert rec["ring"] == 9 and rec["kd"] == 5
        c0, g0, _, _ = multiblank(x.astype(np.float32).astype(np.float64), labels, xn, yn, durations, 0.05)
        np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5)
        g0 = g0 * go.cpu().numpy()[:, None, None, None]
        gc = np.concatenate([g0[i, :xn[i], :yn[i] + 1].reshape(-1, 12) for i in range(5)])
        assert np.abs(g.cpu().numpy() - gc).max() <= gbound(20, 6, c0)


def run(xc, ys_c, xn_t, yn_t, durations, hints):
    xt = xc.clone().requires_grad_(True)
    with w.compact_hints(*hints):
        c = w.rnnt_loss_multiblank(xt, ys_c, xn_t, yn_t, durations, compact=True)
    c.sum().backward()
    return c.detach(), xt.grad


def test_sample_exceeding_the_hints():
    """inside compact_hints a sample longer than the hints gets cost NaN and zero rows; every other lattice gives the
    bits of a batch without it"""
    T, U = 12, 6
    x, labels, xn, yn = random_case(np.random.RandomState(6), 4, T, U, 9, 2)
    xn[2], yn[2] = T, U - 1                          # exceeds max_T = T - 1
    xn[[0, 1, 3]] = np.minimum(xn[[0, 1, 3]], T - 1)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    c, g = run(xc, ys_c, xn_t, yn_t, (2, 4), (T - 1, U))
    assert torch.isnan(c[2]) and (g[rows_of(xn, yn, 2)] == 0).all()
    keep = [0, 1, 3]
    _, xk, _, ysk, xnk, ynk = layouts(x[keep], labels[keep], xn[keep], yn[keep], torch.float32, 0)
    ck, gk = run(xk, ysk, xnk, ynk, (2, 4), (T - 1, U))
    assert torch.equal(c[keep], ck) and torch.equal(torch.cat([g[rows_of(xn, yn, i)] for i in keep]), gk)


def test_rows_past_stu_inside_hints():
    """a lattice whose rows would run past the tensor gets cost NaN and is not read; the rows it would own get zeros"""
    x, labels, xn, yn = random_case(np.random.RandomState(12), 3, 8, 5, 9, 2)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    cut = xc.shape[0] - 3
    buf = torch.full((xc.numel() + 64,), float("nan"), device=DEV)
    short = buf[:cut * xc.shape[1]].view(cut, xc.shape[1])
    short.copy_(xc[:cut])
    c, g = run(short, ys_c, xn_t, yn_t, (2, 4), (8, 5))
    assert torch.isnan(c[2]) and torch.isfinite(c[:2]).all()
    assert (g[rows_of(xn, yn, 2).start:] == 0).all() and torch.isfinite(g).all()
    c0, g0 = run(xc, ys_c, xn_t, yn_t, (2, 4), (8, 5))
    s = rows_of(xn, yn, 2).start
    assert torch.equal(c[:2], c0[:2]) and torch.equal(g[:s], g0[:s])


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_graph_capture_and_determinism(dtype):
    T, U, durations = 40, 12, (2, 4, 8)
    x, labels, xn, yn = case(8, T, U, 32, 3, 4)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, dtype, 0)
    xt = xc.clone().requires_grad_(True)

    def step():
        xt.grad = None
        with w.compact_hints(T, U):
            loss = w.rnnt_loss_multiblank(xt, ys_c, xn_t, yn_t, durations, sigma=0.05, reduction="sum", compact=True)
        loss.backward()
        return loss

    l1, g1 = step().detach().clone(), xt.grad.clone()
    l2, g2 = step().detach().clone(), xt.grad.clone()
    assert torch.equal(l1, l2) and torch.equal(g1, g2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    xt.grad = None
    with torch.cuda.graph(graph):
        loss = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss.detach(), l1) and torch.equal(xt.grad, g1)


def test_shape_check_without_hints():
    """without hints the one totals copy checks STU and labels.numel(): a mismatch raises before any loss kernel runs
    (the one launch is the totals pass); inside hints there is no copy (the graph capture test above)"""
    x, labels, xn, yn = case(3, 6, 4, 9, 2, 2)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    for xs, ys, msg in ((xc[:-1], ys_c, r"xs shape mismatch"), (xc, ys_c[:-1], r"ys shape must be equal")):
        torch.cuda.synchronize()
        before = w._C.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            w.rnnt_loss_multiblank(xs.contiguous(), ys.contiguous(), xn_t, yn_t, (2, 4), compact=True)
        assert w._C.launch_count() == before + 1


def test_binding_refuses_before_any_launch():
    x, labels, xn, yn = case(3, 6, 4, 9, 2, 2)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    torch.cuda.synchronize()
    before = w._C.launch_count()
    with pytest.raises(RuntimeError, match=r"blank must be in \[len\(big_blank_durations\), V\)"):
        w._C.rnnt_multiblank_compact_forward(xc, ys_c, xn_t, yn_t, [2, 4], 0.0, 1, True, 6, 4)
    with pytest.raises(RuntimeError):
        w._C.rnnt_multiblank_compact_forward(xc, ys_c.cpu(), xn_t, yn_t, [2, 4], 0.0, 8, True, 6, 4)
    lse = torch.zeros(xc.shape[0], device=DEV)
    pg = torch.zeros(xc.shape[0], 4, device=DEV)
    pref = torch.zeros(6, dtype=torch.long, device=DEV)
    go = torch.ones(3, device=DEV)
    for args in ((xc, lse.cpu(), pg, ys_c, xn_t, yn_t, pref, [2, 4], go, 8),
                 (xc, lse, pg, ys_c, xn_t, yn_t, pref.cpu(), [2, 4], go, 8),
                 (xc, lse, pg[:, :3].contiguous(), ys_c, xn_t, yn_t, pref, [2, 4], go, 8),
                 (xc, lse, pg, ys_c, xn_t, yn_t, pref.int(), [2, 4], go, 8)):
        with pytest.raises(RuntimeError):
            w._C.rnnt_multiblank_compact_backward(*args)
    torch.cuda.synchronize()
    assert w._C.launch_count() == before
