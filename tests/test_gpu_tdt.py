"""GPU: rnnt_loss_tdt against the fp64 oracle (tests/tdt_oracle.py): costs, logit gradients, reductions, bf16 bit
identity with f32, the degenerate classes, determinism, CUDA graphs, argument checks and the C ABI."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.tdt_oracle import random_case, tdt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


# rnntTdtLaunchRecord_t (include/rnnt_b200.h)
TDT_FIELDS = ["seq", "cluster", "warps", "ring", "passes", "kd", "norm_group", "norm_lanes", "smem", "emit_vec",
              "emit_xvec"]
_lib = None


def tdt_record():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
        _lib.rnnt_b200_debug_last_tdt_launch.argtypes = [ctypes.c_void_p]
    buf = (ctypes.c_int32 * len(TDT_FIELDS))()
    _lib.rnnt_b200_debug_last_tdt_launch(buf)
    return dict(zip(TDT_FIELDS, list(buf)))


def gtol(T, U):
    return 2e-5 + 6e-6 * (T + U)


def gbound(T, U, costs):
    fin = np.abs(costs[np.isfinite(costs)])
    big = fin.max() if fin.size else 0.0
    return 1e-4 + max(2 * gtol(T, U), 2.0 ** -23 * big * math.sqrt(T + U))


def run(x, labels, xn, yn, durations, sigma=0.0, blank=0, dtype=torch.float32, go=None, **kw):
    xt = torch.tensor(x, dtype=torch.float32).to(dtype).to(DEV).requires_grad_(True)
    costs = w.rnnt_loss_tdt(xt, torch.tensor(labels, device=DEV), torch.tensor(xn, device=DEV),
                            torch.tensor(yn, device=DEV), durations, sigma=sigma, blank=blank, **kw)
    if go is None:
        go = torch.ones_like(costs)
    costs.backward(go)
    return costs.detach(), xt.grad


def check(x, labels, xn, yn, durations, sigma, blank, go=None):
    c, g = run(x, labels, xn, yn, durations, sigma, blank, go=None if go is None else torch.tensor(go, device=DEV))
    c0, g0, _, _ = tdt(x.astype(np.float32).astype(np.float64), labels, xn, yn, durations, sigma, blank)
    if go is not None:
        g0 = g0 * go[:, None, None, None]
    c = c.cpu().numpy()
    assert np.array_equal(np.isnan(c), np.isnan(c0)) and np.array_equal(np.isinf(c), np.isinf(c0))
    fin = np.isfinite(c0)
    np.testing.assert_allclose(c[fin], c0[fin], rtol=1e-5)
    T, U = x.shape[1], x.shape[2]
    g = g.cpu().numpy().astype(np.float64)
    assert np.array_equal(np.isnan(g), np.isnan(g0))             # NaN exactly where the oracle has it
    fin = np.isfinite(g0)
    err = np.abs(g[fin] - g0[fin])
    assert err.size == 0 or err.max() <= gbound(T, U, c0), err.max()


@pytest.mark.parametrize("durations", [(0, 1, 2, 3, 4), (1,), (0, 2, 5), (2, 3), (0, 1, 2, 4, 8, 16)])
@pytest.mark.parametrize("sigma", [0.0, 0.05])
def test_oracle_agreement(durations, sigma):
    rng = np.random.RandomState(11 + len(durations))
    x, labels, xn, yn = random_case(rng, 5, 18, 7, 9, durations)
    blank = 3
    labels[1, 0] = blank                                     # a label equal to blank
    go = rng.uniform(0.2, 2.0, 5)
    check(x, labels, xn, yn, durations, sigma, blank, go)


@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("average_frames", [False, True])
def test_reductions(reduction, average_frames):
    rng = np.random.RandomState(2)
    durations = (0, 1, 2)
    x, labels, xn, yn = random_case(rng, 4, 12, 5, 6, durations)
    xt = torch.tensor(x, dtype=torch.float32, device=DEV, requires_grad=True)
    args = (torch.tensor(labels, device=DEV), torch.tensor(xn, device=DEV), torch.tensor(yn, device=DEV))
    loss = w.rnnt_loss_tdt(xt, *args, durations, average_frames=average_frames, reduction=reduction)
    (loss if reduction != "none" else loss * torch.arange(1, 5, device=DEV)).sum().backward()
    c0, g0, _, _ = tdt(x.astype(np.float32).astype(np.float64), labels, xn, yn, durations)
    wts = np.ones(4) if reduction != "none" else np.arange(1, 5, dtype=np.float64)
    if average_frames:
        c0, wts = c0 / xn, wts / xn
    if reduction == "mean":
        wts = wts / 4
    ref = {"none": c0, "sum": c0.sum(), "mean": c0.mean()}[reduction]
    np.testing.assert_allclose(loss.detach().cpu().numpy(), ref, rtol=1e-5)
    np.testing.assert_allclose(xt.grad.cpu().numpy(), g0 * wts[:, None, None, None], atol=gbound(12, 5, c0))


@pytest.mark.parametrize("V,D", [(28, 4), (29, 4), (25, 5), (27, 5)])      # (V + D) % 4 = 0, 1, 2, 3
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_bf16_is_f32_rounded(V, D, offset):
    bf16_is_f32_rounded(V, D, offset)


@pytest.mark.parametrize("offset", [0, 2])
def test_bf16_is_f32_rounded_wide_rows(offset):
    """Parakeet's row width, W = 1025 + 5 = 1030 > 64: the 32-lane normaliser, pairs at offset 0 and 2"""
    rec = bf16_is_f32_rounded(1025, 5, offset)
    assert rec["norm_lanes"] == 32 and rec["norm_group"] == 2


def bf16_is_f32_rounded(V, D, offset):
    durations = tuple(range(D))
    rng = np.random.RandomState(V * 10 + offset)
    x, labels, xn, yn = random_case(rng, 3, 10, 6, V, durations)
    W = V + D
    buf = torch.randn(3 * 10 * 6 * W + offset, dtype=torch.float32, device=DEV).to(torch.bfloat16)
    xb = buf[offset:].view(3, 10, 6, W)
    xb.copy_(torch.tensor(x, dtype=torch.float32))
    # xf = xb.float() at the same element offset: the normaliser's branch follows the row width and the element
    # alignment, not the dtype, so both are summed in the same order
    fbuf = torch.empty(3 * 10 * 6 * W + offset, dtype=torch.float32, device=DEV)
    xf = fbuf[offset:].view(3, 10, 6, W)
    xf.copy_(xb.float())
    args = [torch.tensor(a, device=DEV) for a in (labels, xn, yn)]
    cb, lb, pb = w._C.rnnt_tdt_forward(xb, *args, list(durations), 0.05, 1, True)
    rec_b = tdt_record()
    cf, lf, pf = w._C.rnnt_tdt_forward(xf, *args, list(durations), 0.05, 1, True)
    assert tdt_record()["norm_group"] == rec_b["norm_group"]
    assert torch.equal(cb, cf) and torch.equal(lb, lf) and torch.equal(pb, pf)
    go = torch.rand(3, device=DEV) + 0.5
    gb = w._C.rnnt_tdt_backward(xb, lb, pb, args[0], list(durations), go, 1)
    gf = w._C.rnnt_tdt_backward(xf, lf, pf, args[0], list(durations), go, 1)
    assert gb.dtype == torch.bfloat16
    assert torch.equal(gb, gf.to(torch.bfloat16))
    # and the f32 values agree with the oracle
    c0, _, _, _ = tdt(xf.cpu().double().numpy(), labels, xn, yn, durations, 0.05, 1)
    np.testing.assert_allclose(cf.cpu().numpy(), c0, rtol=1e-5)
    return rec_b


def test_degenerate_classes_and_nan_isolation():
    rng = np.random.RandomState(9)
    durations = (1, 2)
    x, labels, xn, yn = random_case(rng, 7, 6, 4, 5, durations)
    xn[:] = 6
    yn[:] = 3
    x[0, :, :, 0] = -np.inf                  # no blank: no path -> +inf
    x[1, :, :, 5:] = [0.0, -np.inf]          # duration 2 masked: a path remains
    xn[2] = 0                                # invalid lengths
    labels[3, 0] = 77                        # live label outside [0, V)
    x[4, 2, 1, 2] = np.nan                   # NaN in a live row
    x[5, :, 3, :] = np.nan                   # NaN only in padding rows (yn = 2)
    yn[5] = 2
    x[6, 1, 1, 5:] = -np.inf                 # a live row whose duration logits are all -inf
    blank = 0
    c, g = run(x, labels, xn, yn, durations, 0.0, blank)
    c, g = c.cpu().numpy(), g.cpu().numpy()
    assert np.isposinf(c[0]) and (g[0] == 0).all()
    assert np.isfinite(c[1])
    assert np.isnan(c[2]) and (g[2] == 0).all()
    assert np.isnan(c[3]) and (g[3] == 0).all()
    assert np.isnan(c[4]) and np.isnan(g[4, :6, :4]).all() and (g[4, :, 4:] == 0).all()
    assert np.isfinite(c[5]) and (g[5, :, 3] == 0).all() and np.isfinite(g[5]).all()
    assert np.isnan(c[6]) and np.isnan(g[6, :6, :4]).all()
    check(np.where(np.isnan(x), 0.0, x)[[1]], labels[[1]], xn[[1]], yn[[1]], durations, 0.0, blank)
    # the other lattices are bit-identical to a batch without the NaN ones
    keep = [0, 1, 2, 3, 5]
    c2, g2 = run(x[keep], labels[keep], xn[keep], yn[keep], durations, 0.0, blank)
    assert np.array_equal(c2.cpu().numpy(), c[keep], equal_nan=True)
    assert np.array_equal(g2.cpu().numpy(), g[keep], equal_nan=True)
    # structurally dead: Tn < min(d > 0)
    xs, ls, xns, yns = random_case(rng, 2, 4, 3, 5, (2, 3))
    xns[:] = 1
    c3, g3 = run(xs, ls, xns, yns, (2, 3))
    assert np.isposinf(c3.cpu().numpy()).all() and (g3 == 0).all()


def test_determinism_and_graph():
    rng = np.random.RandomState(4)
    durations = (0, 1, 2, 3, 4)
    x, labels, xn, yn = random_case(rng, 8, 40, 12, 30, durations)
    xt = torch.tensor(x, dtype=torch.float32, device=DEV, requires_grad=True)
    args = [torch.tensor(a, device=DEV) for a in (labels, xn, yn)]

    def step():
        xt.grad = None
        loss = w.rnnt_loss_tdt(xt, *args, durations, sigma=0.05, reduction="sum")
        loss.backward()
        return loss.detach().clone(), xt.grad.clone()

    l1, g1 = step()
    l2, g2 = step()
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
        loss = w.rnnt_loss_tdt(xt, *args, durations, sigma=0.05, reduction="sum")
        loss.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss.detach(), l1) and torch.equal(xt.grad, g1)


def test_argument_checks():
    x = torch.randn(2, 5, 3, 8, device=DEV, requires_grad=True)
    y = torch.randint(1, 5, (2, 2), dtype=torch.int32, device=DEV)
    xn = torch.full((2,), 5, dtype=torch.int32, device=DEV)
    yn = torch.full((2,), 2, dtype=torch.int32, device=DEV)
    before = w._C.launch_count()
    for bad in ([], [0], [1, 1], [2, 1], [-1, 1], [0, 17], (0, 1.0), "01", None, [True, 2]):
        with pytest.raises(ValueError):
            w.rnnt_loss_tdt(x, y, xn, yn, bad)
    for sigma in (-0.1, float("nan"), float("inf"), True, "0"):
        with pytest.raises(ValueError):
            w.rnnt_loss_tdt(x, y, xn, yn, [0, 1], sigma=sigma)
    with pytest.raises(ValueError):
        w.rnnt_loss_tdt(x, y, xn, yn, list(range(8)))          # logits.size(-1) <= D
    with pytest.raises(ValueError):
        w.rnnt_loss_tdt(x, y, xn, yn, [0, 1], blank=6)           # blank outside [0, V)
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x.double(), y, xn, yn, [0, 1])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x.detach().cpu(), y.cpu(), xn.cpu(), yn.cpu(), [0, 1])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x, y.long(), xn, yn, [0, 1])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x, y, xn.cpu(), yn, [0, 1])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x, y[:, :1].contiguous(), xn, yn, [0, 1])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x, y[:1].contiguous(), xn, yn, [0, 1])        # labels of the wrong batch size
    with pytest.raises(RuntimeError):
        w.rnnt_loss_tdt(x, torch.cat([y, y]), xn, yn, [0, 1])
    torch.cuda.synchronize()
    assert w._C.launch_count() == before


def test_c_abi():
    L = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.rnnt_b200_tdt_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_tdt_workspace_bytes.argtypes = [ci] * 4
    L.rnnt_b200_tdt_forward.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, ci, ctypes.c_float, vp, vp, vp] + \
        [ci] * 6
    L.rnnt_b200_tdt_backward.argtypes = [vp, vp, vp, vp, vp, vp, ci, vp, vp] + [ci] * 6
    rng = np.random.RandomState(1)
    durations = (0, 1, 2)
    N, T, U, V = 3, 9, 4, 6
    x, labels, xn, yn = random_case(rng, N, T, U, V, durations)
    xs = torch.tensor(x, dtype=torch.float32, device=DEV)
    y, a, b = (torch.tensor(t, device=DEV) for t in (labels, xn, yn))
    D = len(durations)
    dur = (ctypes.c_int * D)(*durations)
    wsb = L.rnnt_b200_tdt_workspace_bytes(N, T, U, D)
    ws = torch.empty(wsb + 16, dtype=torch.uint8, device=DEV)
    costs = torch.empty(N, device=DEV)
    lse = torch.empty(N, T, U, 2, device=DEV)
    pg = torch.empty(N, T, U, 2 + D, device=DEV)
    p = lambda t: vp(t.data_ptr())                                            # noqa: E731
    st = vp(torch.cuda.current_stream().cuda_stream)

    def fwd(ws_ptr, nbytes, durs=dur, nd=D, sigma=0.0, eb=4):
        return L.rnnt_b200_tdt_forward(st, ws_ptr, nbytes, p(xs), p(y), p(a), p(b), durs, nd, sigma, p(costs), p(lse),
                                       p(pg), N, T, U, V, 0, eb)

    assert fwd(p(ws), wsb) == 0
    out = torch.empty_like(xs)
    assert L.rnnt_b200_tdt_backward(st, p(xs), p(lse), p(pg), p(y), dur, D, None, p(out), N, T, U, V, 0, 4) == 0
    torch.cuda.synchronize()
    c0, g0, _, _ = tdt(xs.cpu().double().numpy(), labels, xn, yn, durations)
    np.testing.assert_allclose(costs.cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(out.cpu().numpy(), g0, atol=gbound(T, U, c0))
    assert fwd(p(ws), wsb - 1) == 6                                          # RNNT_STATUS_WORKSPACE_TOO_SMALL
    assert fwd(vp(ws.data_ptr() + 8), wsb) == 5                              # workspace not 16-byte aligned
    assert fwd(p(ws), wsb, durs=(ctypes.c_int * 2)(1, 1), nd=2) == 5         # durations not increasing
    assert fwd(p(ws), wsb, durs=(ctypes.c_int * 1)(0), nd=1) == 5            # no duration > 0
    assert fwd(p(ws), wsb, sigma=-1.0) == 5
    assert fwd(p(ws), wsb, eb=3) == 5
    assert L.rnnt_b200_tdt_backward(st, p(xs), p(lse), None, p(y), dur, D, None, p(out), N, T, U, V, 0, 4) == 5
    # lse holds (lse_tok, lse_dur) pairs: a 4-byte aligned lse is refused before any launch
    lse_buf = torch.empty(N * T * U * 2 + 1, device=DEV)
    lse4 = lse_buf[1:]
    before = w._C.launch_count()
    assert L.rnnt_b200_tdt_forward(st, p(ws), wsb, p(xs), p(y), p(a), p(b), dur, D, 0.0, p(costs), p(lse4), p(pg),
                                   N, T, U, V, 0, 4) == 5
    assert L.rnnt_b200_tdt_backward(st, p(xs), p(lse4), p(pg), p(y), dur, D, None, p(out), N, T, U, V, 0, 4) == 5
    assert w._C.launch_count() == before
