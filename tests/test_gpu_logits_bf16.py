"""bfloat16 logits through rnnt_loss_from_logits: bf16 in, bf16 gradient out, float32 normaliser, recurrence and costs.

The contract (include/rnnt_b200.h, DESIGN.md 4): for bf16 logits xb at an 8-byte aligned address and xf = xb.float(),
  costs, lse and pair_grads are torch.equal to the float32 path's on xf (same inputs, same fp32 arithmetic, and the
    normaliser sums each bf16 row in the float32 kernel's order), in both LSE modes, on the fused and general paths;
  the logit gradient is torch.equal to the float32 path's gradient rounded to bf16 once.
Logits only 2- or 4-byte aligned are summed in another order: there the from-logits tolerance against the fp64 oracle
applies, plus one bf16 rounding of the gradient."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.common import apply_mask, assert_same_classes
from tests.test_gpu_logits import gtol, make

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
BF16 = torch.bfloat16
EXACT, FAST = 1, 2

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bf16_inputs(N, T, U, V, seed, blank=0, label_blank=False):
    """make()'s logits rounded to bf16 (xb) and widened back (xf, the same values), labels, lengths on the device."""
    x, ys, xn, yn = make(N, T, U, V, seed=seed, blank=blank)
    if label_blank:
        ys[0, ::3] = blank                       # labels equal to the blank: the two gradients of such a cell add
    xb = cu(x).to(BF16)
    return xb, xb.float(), ys, xn, yn


def both(w, xb, xf, ys, xn, yn, blank, lam, mode, go):
    """(costs, lse, pair_grads, logit gradient) of the bf16 and the float32 path on the same values."""
    out = []
    for x in (xb, xf):
        c, l, p = w._C.rnnt_logits_forward(x, ys, xn, yn, blank, lam, True, mode)
        out.append((c, l, p, w._C.rnnt_logits_backward(x, l, p, ys, go, blank)))
    return out


# One shape per branch of the normaliser (csrc/logits.cu, k_lse_pairs; the float32 kernel takes the same one):
#   V <= 12, V % 4 != 0: one lane per cell       V % 4 == 0, V <= 32: one group of 4 per lane (whole row)
#   12 < V <= 512, V % 4 != 0: 8 lanes online    V % 4 == 0, V > 32: several groups of 4 per lane
#   V > 512, V % 4 != 0: 32 lanes online
# T*U <= 12288 takes the fused kernel on the pairs, larger lattices the general path.
# (N, T, U, V, blank, fastemit_lambda)
PARITY = [(3, 12, 7, 5, 0, 0.0), (2, 31, 18, 7, 2, 0.3), (2, 700, 40, 6, 1, 0.0),
          (4, 150, 40, 28, 0, 0.0), (2, 33, 34, 28, 3, 0.2),
          (2, 33, 34, 30, 5, 0.0), (2, 400, 70, 50, 0, 0.0), (2, 60, 33, 50, 0, 0.25),
          (2, 16, 5, 132, 1, 0.0), (2, 300, 60, 132, 0, 0.1), (2, 30, 12, 1024, 0, 0.0), (2, 25, 9, 5000, 0, 0.1),
          (2, 20, 6, 1026, 4, 0.0), (2, 12, 10, 2001, 0, 0.0)]


@gpu
@pytest.mark.parametrize("label_blank", [False, True])
@pytest.mark.parametrize("shape", PARITY)
def test_bf16_bit_parity_with_f32_path(w, shape, label_blank):
    N, T, U, V, blank, lam = shape
    xb, xf, ys, xn, yn = bf16_inputs(N, T, U, V, seed=T + V, blank=blank, label_blank=label_blank)
    args = (cu(ys), cu(xn), cu(yn))
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    for mode in (EXACT, FAST):
        (cb, lb, pb, gb), (cf, lf, pf, gf) = both(w, xb, xf, *args, blank, lam, mode, go)
        assert cb.dtype == lb.dtype == pb.dtype == torch.float32 and gb.dtype == BF16
        assert torch.equal(cb, cf), (mode, (cb - cf).abs().max().item())
        assert torch.equal(lb, lf), mode
        assert torch.equal(pb, pf), mode
        assert torch.equal(gb, gf.to(BF16)), (mode, (gb.float() - gf).abs().max().item())
        assert torch.isfinite(cb).all()


ORACLE = [s for s in PARITY if s[0] * s[1] * s[2] * s[3] <= 4e6]


@gpu
@pytest.mark.parametrize("shape", ORACLE)
def test_bf16_vs_oracle(w, shape):
    N, T, U, V, blank, lam = shape
    xb, _, ys, xn, yn = bf16_inputs(N, T, U, V, seed=T + V, blank=blank)
    go = np.linspace(0.5, 1.5, N)
    c0, g0 = oracle.from_logits(xb.float().cpu().numpy(), ys, xn, yn, blank, lam, grad_output=go)
    for mode in (EXACT, FAST):
        c, l, p = w._C.rnnt_logits_forward(xb, cu(ys), cu(xn), cu(yn), blank, lam, True, mode)
        g = w._C.rnnt_logits_backward(xb, l, p, cu(ys), cu(go.astype(np.float32)), blank)
        np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5)
        err = np.abs(g.float().cpu().numpy() - g0) - np.abs(g0) * 2.0 ** -8
        assert err.max() <= 1e-4 + 2 * gtol(T, U), (mode, err.max())


@gpu
@pytest.mark.parametrize("V,blank", [(30, 0), (132, 1)])
def test_bf16_masked_vocabulary(w, V, blank):
    """vocab_ninf (tests/common.py): -inf logits at the start of the lanes' online sums; then one cell of -inf only."""
    N, T, U = 3, 12, 9
    x, ys, xn, yn = make(N, T, U, V, seed=7 + V, blank=blank)
    rng = np.random.RandomState(V)
    for n in range(N):
        apply_mask(x, ys, n, int(xn[n]), int(yn[n]) + 1, "vocab_ninf", blank, rng)
    args = (cu(ys), cu(xn), cu(yn))
    go = torch.ones(N, device="cuda")
    for mode in (EXACT, FAST):
        xb = cu(x).to(BF16)
        (cb, lb, pb, gb), (cf, lf, pf, gf) = both(w, xb, xb.float(), *args, blank, 0.0, mode, go)
        assert torch.isfinite(cb).all() and torch.isfinite(lb).all() and torch.isfinite(gb.float()).all()
        assert torch.equal(cb, cf) and torch.equal(lb, lf) and torch.equal(pb, pf)
        assert torch.equal(gb, gf.to(BF16))
        # one cell inside lattice 0 with every logit -inf: NaN normaliser there, NaN gradients in that cell -- as f32
        xd = x.copy()
        xd[0, 1, 1, :] = -np.inf
        xb = cu(xd).to(BF16)
        (cb, lb, pb, gb), (cf, lf, pf, gf) = both(w, xb, xb.float(), *args, blank, 0.0, mode, go)
        assert torch.isnan(lb[0, 1, 1]) and torch.isnan(gb[0, 1, 1].float()).all()
        for got, want, what in ((cb, cf, "costs"), (lb, lf, "lse"), (pb, pf, "pair_grads"),
                                (gb.float(), gf.to(BF16).float(), "grads")):
            assert_same_classes(got.cpu().numpy(), want.cpu().numpy(), what)


@gpu
@pytest.mark.parametrize("offset", [1, 2])
@pytest.mark.parametrize("shape", [(2, 33, 34, 28, 3, 0.2), (2, 16, 5, 132, 1, 0.0), (2, 60, 33, 1024, 0, 0.0)])
def test_bf16_misaligned_view(w, shape, offset):
    """Logits at a 2- (offset 1) or 4-byte (offset 2) aligned address, V % 4 == 0: no groups of 4 then.  NaN on both
    sides of the view: a read outside it would show."""
    N, T, U, V, blank, lam = shape
    xb, _, ys, xn, yn = bf16_inputs(N, T, U, V, seed=T + V, blank=blank)
    n = xb.numel()
    buf = torch.full((n + offset + 1,), float("nan"), dtype=BF16, device="cuda")
    xv = buf[offset:offset + n].view(N, T, U, V)
    xv.copy_(xb)
    assert xv.is_contiguous() and xv.data_ptr() % 8 != 0
    go = np.linspace(0.5, 1.5, N)
    c0, g0 = oracle.from_logits(xb.float().cpu().numpy(), ys, xn, yn, blank, lam, grad_output=go)
    c, l, p = w._C.rnnt_logits_forward(xv, cu(ys), cu(xn), cu(yn), blank, lam, True, EXACT)
    g = w._C.rnnt_logits_backward(xv, l, p, cu(ys), cu(go.astype(np.float32)), blank)
    assert torch.isfinite(c).all() and torch.isfinite(g.float()).all()
    np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5)
    err = np.abs(g.float().cpu().numpy() - g0) - np.abs(g0) * 2.0 ** -8
    assert err.max() <= 1e-4 + 2 * gtol(T, U), err.max()


@gpu
def test_bf16_python_api(w):
    """Frame counts that bf16 cannot represent (601, 513): average_frames divides in float32."""
    N, T, U, V = 2, 601, 5, 12
    xb, xf, ys, _, yn = bf16_inputs(N, T, U, V, seed=3)
    xn = np.array([601, 513], np.int32)
    args = (cu(ys), cu(xn), cu(yn))
    for reduction in ("none", "sum", "mean"):
        for avg in (False, True):
            a = xb.clone().requires_grad_(True)
            b = xf.clone().requires_grad_(True)
            la = w.rnnt_loss_from_logits(a, *args, average_frames=avg, reduction=reduction)
            lb = w.rnnt_loss_from_logits(b, *args, average_frames=avg, reduction=reduction)
            assert la.dtype == torch.float32
            assert torch.equal(la, lb), (reduction, avg, la, lb)
            la.sum().backward()
            lb.sum().backward()
            assert a.grad.dtype == BF16
            assert torch.equal(a.grad, b.grad.to(BF16)), (reduction, avg)
    with torch.no_grad():
        c = w.rnnt_loss_from_logits(xb.clone().requires_grad_(True), *args)
    assert not c.requires_grad
    assert torch.equal(c, w.rnnt_loss_from_logits(xf, *args))
    with pytest.raises(RuntimeError, match="xs must be a Float tensor"):
        w.rnnt_loss_from_logits(xb.half(), *args)


@gpu
def test_bf16_autocast_joint_network(w):
    """A joint network run under torch.autocast hands the loss bf16 logits; its weight gradient stays within bf16
    rounding of the same step in float32."""
    N, T, U, H, V = 3, 40, 9, 64, 36
    gen = torch.Generator().manual_seed(0)
    f = torch.randn(N, T, H, generator=gen).cuda()
    g = torch.randn(N, U, H, generator=gen).cuda()
    _, ys, xn, yn = make(N, T, U, V, seed=1)
    args = (cu(ys), cu(xn), cu(yn))
    torch.manual_seed(0)
    joint = torch.nn.Linear(H, V).cuda()

    def step(enabled):
        joint.zero_grad()
        with torch.autocast("cuda", dtype=BF16, enabled=enabled):
            logits = joint(f[:, :, None] + g[:, None])
            assert logits.dtype == (BF16 if enabled else torch.float32)
            loss = w.rnnt_loss_from_logits(logits, *args, average_frames=True, reduction="mean")
        loss.backward()
        return loss.item(), joint.weight.grad.clone(), joint.bias.grad.clone()

    l32, gw32, gb32 = step(False)
    l16, gw16, gb16 = step(True)
    assert np.isfinite(l16)
    np.testing.assert_allclose(l16, l32, rtol=1e-2)
    assert ((gw16 - gw32).norm() / gw32.norm()).item() < 3e-2
    assert ((gb16 - gb32).norm() / gb32.norm()).item() < 3e-2


@gpu
def test_bf16_cuda_graph_replay(w):
    N, T, U, V = 4, 150, 40, 28
    xb, _, ys, xn, yn = bf16_inputs(N, T, U, V, seed=21)
    xb2 = bf16_inputs(N, T, U, V, seed=22)[0]
    args = (cu(ys), cu(xn), cu(yn))

    def step(x):
        x.grad = None
        loss = w.rnnt_loss_from_logits(x, *args, reduction="sum")
        loss.backward()
        return loss

    def eager(src):
        x = src.clone().requires_grad_(True)
        return step(x).detach(), x.grad

    x = xb.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step(x)
    torch.cuda.current_stream().wait_stream(side)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step(x)
    for src in (xb, xb2):
        with torch.no_grad():
            x.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        l0, g0 = eager(src)
        assert x.grad.dtype == BF16
        assert torch.equal(loss.detach(), l0) and torch.equal(x.grad, g0)


def test_bf16_entry_points_validate_on_host():
    """No GPU needed: T == 0, blank >= V and an odd logits (or gradient) pointer are rejected before any launch
    (status 5).  N == 0 would otherwise return success without a launch, so a missing check shows as 0."""
    import warp_rnnt_b200 as w
    lib = ctypes.CDLL(LIB)
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    fwd = lib.rnnt_b200_logits_forward_bf16
    fwd.restype = I
    fwd.argtypes = [P, P, ctypes.c_size_t] + [P] * 7 + [I] * 5 + [F, I]
    bwd = lib.rnnt_b200_logits_backward_bf16
    bwd.restype = I
    bwd.argtypes = [P] * 7 + [I] * 5
    ptr = [P(0x10000)] * 7

    def f(logits, N, T, U, V, blank):
        return fwd(None, P(0x20000), 1 << 20, P(logits), *ptr[:6], N, T, U, V, blank, 0.0, EXACT)

    def b(logits, out, N, T, U, V, blank):
        return bwd(None, P(logits), ptr[0], ptr[1], ptr[2], ptr[3], P(out), N, T, U, V, blank)

    assert f(0x30000, 4, 0, 3, 5, 0) == 5                           # T == 0
    assert f(0x30000, 4, 2, 3, 5, 7) == 5                           # blank >= V
    assert f(0x30000, 0, 2, 3, 5, 0) == 0                           # nothing to do
    assert f(0x30001, 0, 2, 3, 5, 0) == 5                           # odd logits pointer
    assert b(0x30000, 0x40000, 4, 0, 3, 5, 0) == 5
    assert b(0x30000, 0x40000, 4, 2, 3, 5, 7) == 5
    assert b(0x30000, 0x40000, 0, 2, 3, 5, 0) == 0
    assert b(0x30001, 0x40000, 0, 2, 3, 5, 0) == 5
    assert b(0x30000, 0x40001, 0, 2, 3, 5, 0) == 5                  # odd gradient pointer
    # the operator keeps refusing every other dtype with the float32 message (host tensors: dtype is checked first)
    x = torch.zeros(1, 2, 2, 3, dtype=torch.float16)
    ys, ln = torch.zeros(1, 1, dtype=torch.int), torch.ones(1, dtype=torch.int)
    with pytest.raises(RuntimeError, match="xs must be a Float tensor"):
        w._C.rnnt_logits_forward(x, ys, ln, ln, 0, 0.0, True, 0)
    with pytest.raises(RuntimeError, match="xs must be located in the CUDA"):
        w._C.rnnt_logits_forward(x.to(BF16), ys, ln, ln, 0, 0.0, True, 0)
