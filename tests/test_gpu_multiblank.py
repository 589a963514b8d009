"""GPU: rnnt_loss_multiblank against the fp64 oracle (tests/multiblank_oracle.py): costs, logit gradients, reductions,
bf16 bit identity with f32, the regular transducer when the big blanks are masked, the degenerate classes, determinism,
CUDA graphs, argument checks and the C ABI."""
import ctypes
import os

import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.multiblank_oracle import multiblank, random_case
from tests.test_gpu_tdt import gbound, tdt_record

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
DURATION_SETS = [(2,), (2, 4), (2, 4, 8), (2, 3, 5, 9, 16), (16,)]


def run(x, labels, xn, yn, durations, sigma=0.0, blank=None, dtype=torch.float32, go=None, **kw):
    xt = torch.tensor(x, dtype=torch.float32).to(dtype).to(DEV).requires_grad_(True)
    costs = w.rnnt_loss_multiblank(xt, torch.tensor(labels, device=DEV), torch.tensor(xn, device=DEV),
                                   torch.tensor(yn, device=DEV), durations, sigma=sigma, blank=blank, **kw)
    costs.backward(torch.ones_like(costs) if go is None else go)
    return costs.detach(), xt.grad


def check(x, labels, xn, yn, durations, sigma, blank, go=None):
    c, g = run(x, labels, xn, yn, durations, sigma, blank, go=None if go is None else torch.tensor(go, device=DEV))
    c0, g0, _, _ = multiblank(x.astype(np.float32).astype(np.float64), labels, xn, yn, durations, sigma, blank)
    if go is not None:
        g0 = g0 * go[:, None, None, None]
    c = c.cpu().numpy()
    assert np.array_equal(np.isnan(c), np.isnan(c0)) and np.array_equal(np.isinf(c), np.isinf(c0))
    fin = np.isfinite(c0)
    np.testing.assert_allclose(c[fin], c0[fin], rtol=1e-5)
    g = g.cpu().numpy().astype(np.float64)
    assert np.array_equal(np.isnan(g), np.isnan(g0))
    fin = np.isfinite(g0)
    err = np.abs(g[fin] - g0[fin])
    assert err.size == 0 or err.max() <= gbound(x.shape[1], x.shape[2], c0), err.max()


@pytest.mark.parametrize("durations", DURATION_SETS)
@pytest.mark.parametrize("sigma", [0.0, 0.05])
@pytest.mark.parametrize("blank", ["default", "B"])
def test_oracle_agreement(durations, sigma, blank):
    B = len(durations)
    rng = np.random.RandomState(11 + B + durations[-1])
    x, labels, xn, yn = random_case(rng, 5, 20, 7, B + 8, B)          # ragged lengths
    b = None
    if blank == "B":
        b = B
        labels = labels + B + 1                                        # tokens above the blanks
    labels[1, 0] = B + 7 if b is None else b                           # a label equal to the standard blank
    go = rng.uniform(0.2, 2.0, 5)
    check(x, labels, xn, yn, durations, sigma, b, go)
    rec = tdt_record()
    assert rec["ring"] == max(durations) + 1 and rec["kd"] == (5 if B <= 3 else 17)


@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("average_frames", [False, True])
def test_reductions(reduction, average_frames):
    rng = np.random.RandomState(2)
    durations = (2, 4)
    x, labels, xn, yn = random_case(rng, 4, 12, 5, 8, 2)
    xt = torch.tensor(x, dtype=torch.float32, device=DEV, requires_grad=True)
    args = (torch.tensor(labels, device=DEV), torch.tensor(xn, device=DEV), torch.tensor(yn, device=DEV))
    loss = w.rnnt_loss_multiblank(xt, *args, durations, average_frames=average_frames, reduction=reduction)
    (loss if reduction != "none" else loss * torch.arange(1, 5, device=DEV)).sum().backward()
    c0, g0, _, _ = multiblank(x.astype(np.float32).astype(np.float64), labels, xn, yn, durations)
    wts = np.ones(4) if reduction != "none" else np.arange(1, 5, dtype=np.float64)
    if average_frames:
        c0, wts = c0 / xn, wts / xn
    if reduction == "mean":
        wts = wts / 4
    ref = {"none": c0, "sum": c0.sum(), "mean": c0.mean()}[reduction]
    np.testing.assert_allclose(loss.detach().cpu().numpy(), ref, rtol=1e-5)
    np.testing.assert_allclose(xt.grad.cpu().numpy(), g0 * wts[:, None, None, None], atol=gbound(12, 5, c0))


def bf16_is_f32_rounded(V, offset, durations=(2, 4, 8)):
    B = len(durations)
    rng = np.random.RandomState(V * 10 + offset)
    x, labels, xn, yn = random_case(rng, 3, 10, 6, V, B)
    buf = torch.randn(x.size + offset, dtype=torch.float32, device=DEV).to(torch.bfloat16)
    xb = buf[offset:].view(x.shape)
    xb.copy_(torch.tensor(x, dtype=torch.float32))
    fbuf = torch.empty(x.size + offset, dtype=torch.float32, device=DEV)
    xf = fbuf[offset:].view(x.shape)
    xf.copy_(xb.float())
    args = [torch.tensor(a, device=DEV) for a in (labels, xn, yn)]
    cb, lb, pb = w._C.rnnt_multiblank_forward(xb, *args, list(durations), 0.05, V - 1, True)
    rec_b = tdt_record()
    cf, lf, pf = w._C.rnnt_multiblank_forward(xf, *args, list(durations), 0.05, V - 1, True)
    assert tdt_record()["norm_group"] == rec_b["norm_group"]
    assert torch.equal(cb, cf) and torch.equal(lb, lf) and torch.equal(pb, pf)
    go = torch.rand(3, device=DEV) + 0.5
    gb = w._C.rnnt_multiblank_backward(xb, lb, pb, args[0], list(durations), go, V - 1)
    gf = w._C.rnnt_multiblank_backward(xf, lf, pf, args[0], list(durations), go, V - 1)
    assert gb.dtype == torch.bfloat16
    assert torch.equal(gb, gf.to(torch.bfloat16))
    c0, _, _, _ = multiblank(xf.cpu().double().numpy(), labels, xn, yn, durations, 0.05)
    np.testing.assert_allclose(cf.cpu().numpy(), c0, rtol=1e-5)
    return rec_b


@pytest.mark.parametrize("V", [32, 33, 34, 35])                  # V % 4 = 0, 1, 2, 3
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_bf16_is_f32_rounded(V, offset):
    rec = bf16_is_f32_rounded(V, offset)
    assert rec["norm_lanes"] == 8


@pytest.mark.parametrize("offset", [0, 2])
def test_bf16_is_f32_rounded_wide_rows(offset):
    """V = 1025 + 3 = 1028 > 64: the 32-lane normaliser"""
    rec = bf16_is_f32_rounded(1028, offset)
    assert rec["norm_lanes"] == 32 and rec["norm_group"] == (4 if offset == 0 else 2)


def test_big_blanks_masked_is_the_regular_loss():
    """sigma = 0 and every big-blank logit at -inf: rnnt_loss_from_logits(blank = V - 1), and the big-blank columns'
    gradient is exactly 0"""
    rng = np.random.RandomState(3)
    durations = (2, 4, 8)
    V = 32
    x, labels, xn, yn = random_case(rng, 6, 30, 9, V, 3)
    x[..., V - 4:V - 1] = -np.inf
    args = [torch.tensor(a, device=DEV) for a in (labels, xn, yn)]
    go = torch.rand(6, device=DEV) + 0.5
    xm = torch.tensor(x, dtype=torch.float32, device=DEV, requires_grad=True)
    cm = w.rnnt_loss_multiblank(xm, *args, durations)
    cm.backward(go)
    xr = torch.tensor(x, dtype=torch.float32, device=DEV, requires_grad=True)
    cr = w.rnnt_loss_from_logits(xr, *args, blank=V - 1)
    cr.backward(go)
    np.testing.assert_allclose(cm.detach().cpu().numpy(), cr.detach().cpu().numpy(), rtol=1e-5)
    assert (xm.grad - xr.grad).abs().max().item() <= 1e-4
    assert (xm.grad[..., V - 4:V - 1] == 0).all()


def test_degenerate_classes_and_nan_isolation():
    rng = np.random.RandomState(9)
    durations = (2, 3)
    V = 7
    x, labels, xn, yn = random_case(rng, 8, 6, 4, V, 2)
    xn[:] = 6
    yn[:] = 3
    x[0, :, :, :V - 1] = -np.inf             # only the standard blank: no label edge -> no path, +inf
    x[1, :, :, V - 3:V - 1] = -np.inf        # big blanks masked: a path remains
    xn[2] = 0                                # invalid lengths
    labels[3, 0] = 77                        # live label outside [0, V)
    x[4, 2, 1, 2] = np.nan                   # NaN in a live row
    x[5, :, 3, :] = np.nan                   # NaN only in padding rows (yn = 2)
    yn[5] = 2
    x[6, 1, 1, :] = -np.inf                  # a live row all -inf
    x[7, 3, 2, 0] = np.inf                   # +inf in a live row
    c, g = run(x, labels, xn, yn, durations)
    c, g = c.cpu().numpy(), g.cpu().numpy()
    assert np.isposinf(c[0]) and (g[0] == 0).all()
    assert np.isfinite(c[1])
    assert np.isnan(c[2]) and (g[2] == 0).all()
    assert np.isnan(c[3]) and (g[3] == 0).all()
    assert np.isnan(c[4]) and np.isnan(g[4]).all()
    assert np.isfinite(c[5]) and (g[5, :, 3] == 0).all() and np.isfinite(g[5]).all()
    assert np.isnan(c[6]) and np.isnan(g[6]).all()
    assert np.isnan(c[7]) and np.isnan(g[7]).all()
    check(np.where(np.isnan(x), 0.0, x)[[0, 1, 2, 3]], labels[[0, 1, 2, 3]], xn[[0, 1, 2, 3]], yn[[0, 1, 2, 3]],
          durations, 0.0, None)
    keep = [0, 1, 2, 3, 5]
    c2, g2 = run(x[keep], labels[keep], xn[keep], yn[keep], durations)
    assert np.array_equal(c2.cpu().numpy(), c[keep], equal_nan=True)
    assert np.array_equal(g2.cpu().numpy(), g[keep], equal_nan=True)


def test_determinism_and_graph():
    rng = np.random.RandomState(4)
    durations = (2, 4, 8)
    x, labels, xn, yn = random_case(rng, 8, 40, 12, 32, 3)
    xt = torch.tensor(x, dtype=torch.float32, device=DEV, requires_grad=True)
    args = [torch.tensor(a, device=DEV) for a in (labels, xn, yn)]

    def step():
        xt.grad = None
        loss = w.rnnt_loss_multiblank(xt, *args, durations, sigma=0.05, reduction="sum")
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
        loss = w.rnnt_loss_multiblank(xt, *args, durations, sigma=0.05, reduction="sum")
        loss.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss.detach(), l1) and torch.equal(xt.grad, g1)


def test_argument_checks():
    x = torch.randn(2, 5, 3, 8, device=DEV, requires_grad=True)
    y = torch.randint(0, 4, (2, 2), dtype=torch.int32, device=DEV)
    xn = torch.full((2,), 5, dtype=torch.int32, device=DEV)
    yn = torch.full((2,), 2, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    before = w._C.launch_count()
    for bad in ([], [1], [0, 2], [2, 2], [4, 2], [2, 17], (2, 4.0), "24", None, [True, 2]):
        with pytest.raises(ValueError):
            w.rnnt_loss_multiblank(x, y, xn, yn, bad)
    for sigma in (-0.1, float("nan"), float("inf"), True, "0"):
        with pytest.raises(ValueError):
            w.rnnt_loss_multiblank(x, y, xn, yn, [2, 4], sigma=sigma)
    with pytest.raises(ValueError):
        w.rnnt_loss_multiblank(x, y, xn, yn, list(range(2, 10)))         # V <= B
    for blank in (1, 8, -1, True, 2.0):                                   # outside [B, V), or not an int
        with pytest.raises(ValueError):
            w.rnnt_loss_multiblank(x, y, xn, yn, [2, 4], blank=blank)
    with pytest.raises(ValueError):
        w.rnnt_loss_multiblank(x, y, xn, yn, [2, 4], compact=True)        # not (STU, V)
    with pytest.raises(RuntimeError):
        w.rnnt_loss_multiblank(x.double(), y, xn, yn, [2, 4])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_multiblank(x.detach().cpu(), y.cpu(), xn.cpu(), yn.cpu(), [2, 4])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_multiblank(x, y.long(), xn, yn, [2, 4])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_multiblank(x, y, xn.cpu(), yn, [2, 4])
    with pytest.raises(RuntimeError):
        w.rnnt_loss_multiblank(x, y[:, :1].contiguous(), xn, yn, [2, 4])
    # the operator module: blank below B, and backward tensors of the wrong device, dtype or shape
    with pytest.raises(RuntimeError, match=r"blank must be in \[len\(big_blank_durations\), V\)"):
        w._C.rnnt_multiblank_forward(x.detach(), y, xn, yn, [2, 4], 0.0, 1, True)
    xd = x.detach()
    lse = torch.zeros(2, 5, 3, device=DEV)
    pg = torch.zeros(2, 5, 3, 4, device=DEV)
    go = torch.ones(2, device=DEV)
    for args in ((xd, lse.cpu(), pg, y, [2, 4], go, 7), (xd, lse, pg.cpu(), y, [2, 4], go, 7),
                 (xd, lse, pg, y, [2, 4], go.cpu(), 7), (xd, lse.double(), pg, y, [2, 4], go, 7),
                 (xd, lse, pg[..., :3].contiguous(), y, [2, 4], go, 7), (xd, lse[:1].contiguous(), pg, y, [2, 4], go, 7),
                 (xd, lse, pg, y.cpu(), [2, 4], go, 7)):
        with pytest.raises(RuntimeError):
            w._C.rnnt_multiblank_backward(*args)
    torch.cuda.synchronize()
    assert w._C.launch_count() == before


def test_c_abi():
    L = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.rnnt_b200_multiblank_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_multiblank_workspace_bytes.argtypes = [ci] * 4
    L.rnnt_b200_multiblank_forward.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, ci, ctypes.c_float, vp,
                                               vp, vp] + [ci] * 6
    L.rnnt_b200_multiblank_backward.argtypes = [vp, vp, vp, vp, vp, vp, ci, vp, vp] + [ci] * 6
    rng = np.random.RandomState(1)
    durations = (2, 4)
    N, T, U, V = 3, 9, 4, 8
    B = len(durations)
    x, labels, xn, yn = random_case(rng, N, T, U, V, B)
    xs = torch.tensor(x, dtype=torch.float32, device=DEV)
    y, a, b = (torch.tensor(t, device=DEV) for t in (labels, xn, yn))
    dur = (ctypes.c_int * B)(*durations)
    wsb = L.rnnt_b200_multiblank_workspace_bytes(N, T, U, B)
    ws = torch.empty(wsb + 16, dtype=torch.uint8, device=DEV)
    costs = torch.empty(N, device=DEV)
    lse = torch.empty(N, T, U, device=DEV)
    pg = torch.empty(N, T, U, 2 + B, device=DEV)
    p = lambda t: vp(t.data_ptr())                                            # noqa: E731
    st = vp(torch.cuda.current_stream().cuda_stream)

    def fwd(ws_ptr, nbytes, durs=dur, nb=B, sigma=0.0, eb=4, blank=V - 1):
        return L.rnnt_b200_multiblank_forward(st, ws_ptr, nbytes, p(xs), p(y), p(a), p(b), durs, nb, sigma, p(costs),
                                              p(lse), p(pg), N, T, U, V, blank, eb)

    assert fwd(p(ws), wsb) == 0
    out = torch.empty_like(xs)
    assert L.rnnt_b200_multiblank_backward(st, p(xs), p(lse), p(pg), p(y), dur, B, None, p(out), N, T, U, V, V - 1,
                                           4) == 0
    torch.cuda.synchronize()
    c0, g0, _, _ = multiblank(xs.cpu().double().numpy(), labels, xn, yn, durations)
    np.testing.assert_allclose(costs.cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(out.cpu().numpy(), g0, atol=gbound(T, U, c0))
    before = w._C.launch_count()
    assert fwd(p(ws), wsb - 1) == 6                                          # RNNT_STATUS_WORKSPACE_TOO_SMALL
    assert fwd(vp(ws.data_ptr() + 8), wsb) == 5                              # workspace not 16-byte aligned
    assert fwd(p(ws), wsb, durs=(ctypes.c_int * 2)(2, 2), nb=2) == 5         # durations not increasing
    assert fwd(p(ws), wsb, durs=(ctypes.c_int * 1)(1), nb=1) == 5            # a big blank shorter than 2
    assert fwd(p(ws), wsb, durs=(ctypes.c_int * 1)(17), nb=1) == 5           # longer than 16
    assert fwd(p(ws), wsb, nb=0) == 5
    assert fwd(p(ws), wsb, sigma=-1.0) == 5
    assert fwd(p(ws), wsb, eb=3) == 5
    assert fwd(p(ws), wsb, blank=B - 1) == 5                                 # blank below B
    assert fwd(p(ws), wsb, blank=V) == 5
    assert L.rnnt_b200_multiblank_backward(st, p(xs), p(lse), None, p(y), dur, B, None, p(out), N, T, U, V, V - 1,
                                           4) == 5
    assert L.rnnt_b200_multiblank_backward(st, p(xs), p(lse), p(pg), p(y), dur, B, None, p(out), N, T, U, V, 1,
                                           4) == 5
    assert w._C.launch_count() == before
