"""GPU: use_hat_loss (the HAT normalisation, csrc/logits.cu k_lse_pairs_hat / k_expand_logits_hat) in
rnnt_loss_from_logits, rnnt_loss_pruned and rnnt_align_from_logits.

  1. bit level: the pairs rebuilt in torch f32 from the returned lse_nb, fed to rnnt_b200_loss_pairs_ex, give the HAT
     call's costs and pair gradients bit for bit (every type, penalty, FastEmit, both lse modes); lse_nb is the softmax
     call's lse of the row with the blank logit set to -inf;
  2. bf16 = f32 on the widened logits, compact = dense, pruned = dense at the window rows;
  3. alignment: regular = rnnt_align on the rebuilt pairs as V = 2 log-probs, types 1 and 2 = frames_align_oracle;
  4. against tests/hat_oracle.py in fp64 and against the f32 torch composition fed to rnnt_loss_from_logits;
  5. classes: invalid lengths, no path, NaN in x[B] / in a non-blank column, +-inf blank logits, every non-blank logit
     -inf, isolation from the rest of the batch;
  6. CUDA graphs, determinism, the forward-only path, the empty batch, launch counts;
  7. the ValueErrors, the operator module's refusals and the C ABI's, with no launch."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import frames_align_oracle as fo
from tests import hat_oracle as ho
from tests import path_oracle as pa
from tests.common import to_compact
from tests.test_gpu_logits import gtol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
KIND = {"regular": 0, "modified": 1, "constrained": 2}
INVALID = 5

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


@pytest.fixture(scope="module")
def lib():
    import warp_rnnt_b200  # noqa: F401 (the library next to the package)
    L = ctypes.CDLL(LIB)
    P, I, F, Z = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
    L.rnnt_b200_loss_pairs_ex.restype = I
    L.rnnt_b200_loss_pairs_ex.argtypes = [P, P, Z] + [P] * 5 + [I] * 3 + [F, I, I, F]
    L.rnnt_b200_workspace_bytes.restype = Z
    L.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, I]
    L.rnnt_b200_logits_hat_forward.restype = I
    L.rnnt_b200_logits_hat_forward.argtypes = [P, P, Z] + [P] * 7 + [I] * 5 + [F, I, I, I, F]
    L.rnnt_b200_logits_hat_backward.restype = I
    L.rnnt_b200_logits_hat_backward.argtypes = [P] * 7 + [I] * 6
    L.rnnt_b200_logits_compact_hat_forward.restype = I
    L.rnnt_b200_logits_compact_hat_forward.argtypes = [P, P, Z] + [P] * 9 + [ctypes.c_int64] + [I] * 3 + [F] + [I] * 4
    L.rnnt_b200_logits_compact_hat_backward.restype = I
    L.rnnt_b200_logits_compact_hat_backward.argtypes = [P] * 10 + [ctypes.c_int64] + [I] * 4
    L.rnnt_b200_logits_pruned_hat_backward.restype = I
    L.rnnt_b200_logits_pruned_hat_backward.argtypes = [P] * 8 + [I] * 7
    L.rnnt_b200_logits_pruned_hat_forward.restype = I
    L.rnnt_b200_logits_pruned_hat_forward.argtypes = [P, P, Z] + [P] * 8 + [I] * 6 + [F, I, I, I, F]
    L.rnnt_b200_align_logits_hat_dense.restype = I
    L.rnnt_b200_align_logits_hat_dense.argtypes = [P, P, Z] + [P] * 6 + [I] * 7 + [F]
    L.rnnt_b200_align_logits_hat_compact.restype = I
    L.rnnt_b200_align_logits_hat_compact.argtypes = [P, P, Z] + [P] * 6 + [ctypes.c_int64] + [I] * 6
    L.rnnt_b200_align_logits_workspace_bytes.restype = Z
    L.rnnt_b200_align_logits_workspace_bytes.argtypes = [ctypes.c_int64, I, I, I]
    L.rnnt_b200_launch_count.restype = ctypes.c_uint64
    return L


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(p, q):
    """bit for bit, NaN included"""
    return p.shape == q.shape and p.dtype == q.dtype and torch.equal(p.reshape(-1).view(torch.uint8),
                                                                     q.reshape(-1).view(torch.uint8))


def make(N, T, U, V, seed, xn=None, yn=None, blank=0, scale=2.0, label_blank=False):
    """logits (N,T,U,V) f32, labels other than blank (label_blank: every third label, from the first, is the blank);
    by default most lattices have a modified path"""
    rng = np.random.RandomState(seed)
    x = (rng.randn(N, T, U, V) * scale).astype(np.float32)
    ys = rng.randint(0, V - 1, (N, U - 1)).astype(np.int32)
    ys += (ys >= blank)
    if label_blank:
        ys[:, ::3] = blank
    xn = rng.randint(max(1, T // 2), T + 1, N).astype(np.int32) if xn is None else np.asarray(xn, np.int32)
    yn = np.minimum(rng.randint(0, U, N), xn).astype(np.int32) if yn is None else np.asarray(yn, np.int32)
    return cu(x), cu(ys), cu(xn), cu(yn)


def labels_of(ys, T, blank):
    N, U1 = ys.shape
    return torch.cat([ys, torch.full((N, 1), blank, dtype=torch.int, device=ys.device)], 1).long()


def hat_pairs(x, lse, ys, blank=0):
    """the HAT pairs in torch f32 from the kernel's lse_nb, in include/rnnt_b200.h's operation order"""
    x = x.float()
    N, T, U, _ = x.shape
    lab = labels_of(ys, T, blank)
    xb = x[..., blank]
    xl = x.gather(3, lab[:, None, :, None].expand(N, T, U, 1))[..., 0]
    sp = torch.log1p(torch.exp(-torch.abs(xb)))
    zero = torch.zeros_like(xb)
    b = torch.minimum(xb, zero) - sp
    l = (xl - lse) + (torch.minimum(-xb, zero) - sp)
    return torch.stack([b, l], -1).contiguous()


def torch_hat(x, blank):
    """the HAT log-probs as a user composes them in torch (k2's get_hat_logprobs)"""
    xb = x[..., blank:blank + 1]
    nb = torch.cat([x[..., :blank], x[..., blank + 1:]], -1)
    lab = torch.log_softmax(nb, -1) + torch.nn.functional.logsigmoid(-xb)
    return torch.cat([lab[..., :blank], torch.nn.functional.logsigmoid(xb), lab[..., blank:]], -1)


def loss_pairs(lib, pairs, xn, yn, kind, lam, fe=0.0, lse_mode=0):
    N, T, U, _ = pairs.shape
    c = torch.empty(N, device="cuda")
    pg = torch.empty((N, T, U, 2), device="cuda")
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
    st = lib.rnnt_b200_loss_pairs_ex(torch.cuda.current_stream().cuda_stream, ws.data_ptr(), ws.numel(),
                                     pairs.data_ptr(), xn.data_ptr(), yn.data_ptr(), c.data_ptr(), pg.data_ptr(), N, T,
                                     U, fe, lse_mode, KIND[kind], lam)
    assert st == 0
    return c, pg


def fwd(w, x, ys, xn, yn, blank=0, fe=0.0, kind="regular", lam=0.0, lse_mode=0, want=True):
    return w._C.rnnt_logits_forward(x, ys, xn, yn, blank, fe, want, lse_mode, KIND[kind], lam, True)


# ------------------------------------------------------------------------------------------------ 1. bit level
CASES = [("regular", 0.0, 0.0), ("regular", 0.05, 0.0), ("regular", 0.0, 0.1), ("regular", 0.05, 0.1),
         ("modified", 0.0, 0.0), ("modified", 0.05, 0.0), ("constrained", 0.0, 0.0), ("constrained", 0.05, 0.0)]


# V: SUB = 1 (V <= 12, unaligned), 8 and 32 strided, the VEC4 max-first (V <= 128) and online paths
@pytest.mark.parametrize("V", [5, 12, 37, 28, 128, 515, 1024])
@pytest.mark.parametrize("kind,lam,fe", CASES)
def test_pairs_bit_for_bit(w, lib, V, kind, lam, fe):
    N, T, U = 5, 23, 9
    blank = V // 3                                      # inside a group of 4, at different lanes
    x, ys, xn, yn = make(N, T, U, V, seed=V + U, blank=blank)
    for lse_mode in (0, 1):
        c, lse, pg = fwd(w, x, ys, xn, yn, blank, fe, kind, lam, lse_mode)
        cr, pr = loss_pairs(lib, hat_pairs(x, lse, ys, blank), xn, yn, kind, lam, fe, lse_mode)
        assert same(c, cr) and same(pg, pr)
    # lse_nb is the softmax pass's normaliser of the row with the blank logit -inf, bit for bit
    xm = x.clone()
    xm[..., blank] = -float("inf")
    _, lse_soft, _ = w._C.rnnt_logits_forward(xm, ys, xn, yn, blank, 0.0, False)
    assert same(lse, lse_soft)


# a label equal to the blank: l = x[B] - lse_nb + logsigmoid(-x[B]) (not b), and its gradient collects gl at the blank
@pytest.mark.parametrize("V", [5, 37, 128, 1024])
@pytest.mark.parametrize("kind,lam,fe", [("regular", 0.0, 0.0), ("regular", 0.05, 0.1), ("modified", 0.05, 0.0),
                                         ("constrained", 0.0, 0.0)])
def test_labels_equal_to_blank(w, lib, V, kind, lam, fe):
    N, T, U = 4, 21, 10
    blank = V // 3
    x, ys, xn, yn = make(N, T, U, V, seed=V + 1, blank=blank, label_blank=True)
    xh, yh, ysh = xn.cpu().numpy(), yn.cpu().numpy(), ys.cpu().numpy()
    assert ((ysh == blank) & (np.arange(U - 1)[None, :] < yh[:, None])).any()
    # bit level: the rebuilt pairs through rnnt_b200_loss_pairs_ex
    c, lse, pg = fwd(w, x, ys, xn, yn, blank, fe, kind, lam)
    cr, pr = loss_pairs(lib, hat_pairs(x, lse, ys, blank), xn, yn, kind, lam, fe)
    assert same(c, cr) and same(pg, pr)
    # dense against fp64
    go = np.linspace(0.5, 1.5, N).astype(np.float32)
    xg = x.clone().requires_grad_(True)
    cd = w.rnnt_loss_from_logits(xg, ys, xn, yn, blank=blank, fastemit_lambda=fe, rnnt_type=kind, delay_penalty=lam,
                                 use_hat_loss=True)
    (cd * cu(go)).sum().backward()
    c0, g0 = ho.dense(x.cpu().numpy(), ysh, xh, yh, blank, kind, lam, fe, go)
    fin = np.isfinite(c0)
    assert fin.all()
    np.testing.assert_allclose(cd.detach().cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(xg.grad.cpu().numpy(), g0, rtol=0, atol=1e-4 + 2 * gtol(T, U))
    if kind != "regular" or lam:
        return
    # compact: the dense result, with and without hints
    flat, ysc = to_compact(x.cpu().numpy(), ysh, xh, yh)
    gd, _ = to_compact(xg.grad.cpu().numpy(), ysh, xh, yh)
    for hints in (None, (T, U)):
        xc = cu(flat).requires_grad_(True)
        if hints:
            with w.compact_hints(*hints):
                cc = w.rnnt_loss_from_logits(xc, cu(ysc), xn, yn, blank=blank, fastemit_lambda=fe, compact=True,
                                             use_hat_loss=True)
        else:
            cc = w.rnnt_loss_from_logits(xc, cu(ysc), xn, yn, blank=blank, fastemit_lambda=fe, compact=True,
                                         use_hat_loss=True)
        (cc * cu(go)).sum().backward()
        assert same(cc.detach(), cd.detach()) and np.array_equal(xc.grad.cpu().numpy(), gd)


@pytest.mark.parametrize("kind,lam", [("regular", 0.0), ("regular", 0.03), ("constrained", 0.0)])
def test_pruned_labels_equal_to_blank(w, kind, lam):
    N, T, U, V, S = 4, 30, 10, 24, 4
    rng = np.random.RandomState(17)
    x = rng.randn(N, T, S, V).astype(np.float32) * 2
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    ys[:, ::3] = 0
    xn = np.array([30, 27, 22, 30], np.int32)
    yn = np.array([9, 7, 9, 4], np.int32)
    ranges = np.minimum(np.arange(T)[None, :] * yn[:, None] // xn[:, None], np.maximum(yn[:, None] + 1 - S, 0))
    ranges = ranges.astype(np.int32)
    xd = cu(x).requires_grad_(True)
    c = w.rnnt_loss_pruned(xd, cu(ys), cu(xn), cu(yn), cu(ranges), rnnt_type=kind, delay_penalty=lam,
                           use_hat_loss=True)
    c.sum().backward()
    c0, g0 = ho.pruned(x, ys, xn, yn, ranges, 0, kind, lam)
    fin = np.isfinite(c0)
    assert fin.any()
    np.testing.assert_allclose(c.detach().cpu().numpy()[fin], c0[fin], rtol=1e-5)
    np.testing.assert_allclose(xd.grad.cpu().numpy(), g0, rtol=0, atol=1e-4 + 2 * gtol(T, U))


# ------------------------------------------------------------------------------------------------ 2. parity
@pytest.mark.parametrize("V", [6, 28, 37, 1024])
@pytest.mark.parametrize("kind", ["regular", "modified", "constrained"])
def test_bf16_is_f32_on_widened_logits(w, V, kind):
    N, T, U = 4, 19, 8
    x, ys, xn, yn = make(N, T, U, V, seed=3 * V, blank=1)
    xb = x.to(torch.bfloat16)
    cb, lb, pb = fwd(w, xb, ys, xn, yn, 1, 0.0, kind, 0.02)
    cf, lf, pf = fwd(w, xb.float(), ys, xn, yn, 1, 0.0, kind, 0.02)
    assert same(cb, cf) and same(lb, lf) and same(pb, pf)
    go = torch.rand(N, device="cuda") + 0.5
    gb = w._C.rnnt_logits_backward(xb, lb, pb, ys, go, 1, True)
    gf = w._C.rnnt_logits_backward(xb.float(), lf, pf, ys, go, 1, True)
    assert same(gb, gf.to(torch.bfloat16))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("V", [7, 32, 515])
def test_compact_is_dense(w, dtype, V):
    N, T, U = 5, 17, 7
    x, ys, xn, yn = make(N, T, U, V, seed=V, blank=2)
    x = x.to(dtype)
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    flat, ysc = to_compact(x.float().cpu().numpy(), ys.cpu().numpy(), xh, yh)
    xc = cu(flat).to(dtype)
    ysc = cu(ysc)
    xd = x.clone().requires_grad_(True)
    cd = w.rnnt_loss_from_logits(xd, ys, xn, yn, blank=2, use_hat_loss=True, fastemit_lambda=0.01)
    cd.sum().backward()
    for hints in (None, (T, U)):
        xg = xc.clone().requires_grad_(True)
        if hints:
            with w.compact_hints(*hints):
                cc = w.rnnt_loss_from_logits(xg, ysc, xn, yn, blank=2, compact=True, use_hat_loss=True,
                                             fastemit_lambda=0.01)
        else:
            cc = w.rnnt_loss_from_logits(xg, ysc, xn, yn, blank=2, compact=True, use_hat_loss=True,
                                         fastemit_lambda=0.01)
        cc.sum().backward()
        assert same(cc, cd)
        gd, _ = to_compact(xd.grad.float().cpu().numpy(), ys.cpu().numpy(), xh, yh)
        assert np.array_equal(xg.grad.float().cpu().numpy(), gd)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind,lam", [("regular", 0.0), ("regular", 0.03), ("modified", 0.0), ("constrained", 0.03)])
def test_pruned_is_dense_at_window_rows(w, dtype, kind, lam):
    """windows of S = U from column 0 hold every cell: the pruned call is the dense one"""
    N, T, U, V = 4, 21, 6, 40
    x, ys, xn, yn = make(N, T, U, V, seed=7, blank=3)
    x = x.to(dtype)
    zero = torch.zeros((N, T), dtype=torch.int, device="cuda")
    cd, ld, pd = fwd(w, x, ys, xn, yn, 3, 0.0, kind, lam)
    cp, lp, pp = w._C.rnnt_logits_pruned_forward(x, ys, xn, yn, zero, 3, 0.0, True, 0, KIND[kind], lam, True)
    assert same(cd, cp) and same(pd, pp) and same(ld, lp)
    go = torch.rand(N, device="cuda")
    gd = w._C.rnnt_logits_backward(x, ld, pd, ys, go, 3, True)
    gp = w._C.rnnt_logits_pruned_backward(x, lp, pp, ys, zero, go, 3, True)
    assert same(gd, gp)


# ------------------------------------------------------------------------------------------------ 3. alignment
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_align_regular_is_rnnt_align_on_pairs(w, dtype):
    N, T, U, V = 6, 30, 11, 33
    x, ys, xn, yn = make(N, T, U, V, seed=21, blank=4)
    x = x.to(dtype)
    s, f = w.rnnt_align_from_logits(x, ys, xn, yn, blank=4, use_hat_loss=True)
    _, lse, _ = fwd(w, x, ys, xn, yn, 4, want=False)
    pairs = hat_pairs(x, lse, ys, 4)
    s0, f0 = w.rnnt_align(pairs, torch.ones_like(ys), xn, yn, blank=0)      # V = 2: blank 0, every label 1
    assert same(s, s0) and torch.equal(f, f0)
    # compact: the dense result
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    flat, ysc = to_compact(x.float().cpu().numpy(), ys.cpu().numpy(), xh, yh)
    sc, fc = w.rnnt_align_from_logits(cu(flat).to(dtype), cu(ysc), xn, yn, blank=4, compact=True, use_hat_loss=True)
    assert same(sc, s)
    assert np.array_equal(fc.cpu().numpy(), np.concatenate([f[n, :yh[n]].cpu().numpy() for n in range(N)]))


@pytest.mark.parametrize("kind", ["modified", "constrained"])
@pytest.mark.parametrize("lam", [0.0, 0.04])
def test_align_frames_types_are_the_oracle(w, kind, lam):
    N, T, U, V = 6, 27, 9, 20
    x, ys, xn, yn = make(N, T, U, V, seed=5, blank=0)
    s, f = w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type=kind, delay_penalty=lam, use_hat_loss=True)
    _, lse, _ = fwd(w, x, ys, xn, yn, 0, want=False)
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    P = hat_pairs(x, lse, ys).cpu().numpy()
    if lam:
        P = fo.delay_pairs(P, xh, yh, lam)
    s0, f0 = fo.align_pairs_np(P, xh, yh, KIND[kind])
    assert s.cpu().numpy().tobytes() == s0.tobytes() and np.array_equal(f.cpu().numpy(), f0)


# ------------------------------------------------------------------------------------------------ 4. fp64
@pytest.mark.parametrize("kind,lam,fe", CASES)
@pytest.mark.parametrize("shape", [(4, 33, 12, 29), (2, 120, 40, 256)], ids=lambda s: "x".join(map(str, s)))
def test_against_fp64(w, kind, lam, fe, shape):
    N, T, U, V = shape
    blank = 0 if kind == "regular" else V - 1
    x, ys, xn, yn = make(N, T, U, V, seed=T, blank=blank)
    go = np.linspace(0.5, 1.5, N)
    xg = x.clone().requires_grad_(True)
    c = w.rnnt_loss_from_logits(xg, ys, xn, yn, blank=blank, fastemit_lambda=fe, rnnt_type=kind, delay_penalty=lam,
                                use_hat_loss=True)
    (c * cu(go.astype(np.float32))).sum().backward()
    c0, g0 = ho.dense(x.cpu().numpy(), ys.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy(), blank, kind, lam, fe,
                      go.astype(np.float32))
    fin = np.isfinite(c0)
    np.testing.assert_allclose(c.detach().cpu().numpy()[fin], c0[fin], rtol=1e-5)
    np.testing.assert_allclose(xg.grad.cpu().numpy(), g0, rtol=0, atol=1e-4 + 2 * gtol(T, U))
    # the f32 torch composition fed to rnnt_loss_from_logits (HAT rows sum to 1: log_softmax leaves them)
    xt = x.clone().requires_grad_(True)
    ct = w.rnnt_loss_from_logits(torch_hat(xt, blank), ys, xn, yn, blank=blank, fastemit_lambda=fe, rnnt_type=kind,
                                 delay_penalty=lam)
    (ct * cu(go.astype(np.float32))).sum().backward()
    np.testing.assert_allclose(c.detach().cpu().numpy()[fin], ct.detach().cpu().numpy()[fin], rtol=1e-5)
    np.testing.assert_allclose(xg.grad.cpu().numpy(), xt.grad.cpu().numpy(), rtol=0, atol=1e-4 + 2 * gtol(T, U))


@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("average_frames", [False, True])
def test_reductions(w, reduction, average_frames):
    N, T, U, V = 5, 20, 7, 16
    x, ys, xn, yn = make(N, T, U, V, seed=2, blank=5)
    xg = x.clone().requires_grad_(True)
    out = w.rnnt_loss_from_logits(xg, ys, xn, yn, blank=5, reduction=reduction, average_frames=average_frames,
                                  use_hat_loss=True)
    out.sum().backward()
    c0, _ = ho.dense(x.cpu().numpy(), ys.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy(), 5)
    go = np.ones(N)
    if average_frames:
        c0 = c0 / xn.cpu().numpy()
        go = go / xn.cpu().numpy()
    if reduction == "sum":
        c0 = c0.sum()
    elif reduction == "mean":
        c0, go = c0.mean(), go / N
    _, g0 = ho.dense(x.cpu().numpy(), ys.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy(), 5, grad_output=go)
    np.testing.assert_allclose(out.detach().cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(xg.grad.cpu().numpy(), g0, rtol=0, atol=1e-4 + 2 * gtol(T, U))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind,lam", [("regular", 0.0), ("modified", 0.02), ("constrained", 0.0)])
def test_pruned_against_fp64(w, dtype, kind, lam):
    N, T, U, V, S = 4, 40, 14, 48, 4
    rng = np.random.RandomState(9)
    x = rng.randn(N, T, S, V).astype(np.float32) * 2
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    xn = np.array([40, 37, 30, 40], np.int32)
    yn = np.array([13, 10, 12, 5], np.int32)
    ranges = np.minimum(np.arange(T)[None, :] * yn[:, None] // xn[:, None], np.maximum(yn[:, None] + 1 - S, 0))
    ranges = ranges.astype(np.int32)
    xd = cu(x).to(dtype).requires_grad_(True)
    c = w.rnnt_loss_pruned(xd, cu(ys), cu(xn), cu(yn), cu(ranges), rnnt_type=kind, delay_penalty=lam,
                           use_hat_loss=True)
    c.sum().backward()
    c0, g0 = ho.pruned(xd.detach().float().cpu().numpy(), ys, xn, yn, ranges, 0, kind, lam)
    fin = np.isfinite(c0)
    assert fin.any()
    np.testing.assert_allclose(c.detach().cpu().numpy()[fin], c0[fin], rtol=1e-5)
    atol = 1e-4 + 2 * gtol(T, U) + (2.0 ** -8 if dtype == torch.bfloat16 else 0.0)
    np.testing.assert_allclose(xd.grad.float().cpu().numpy(), g0, rtol=0, atol=atol)


# ------------------------------------------------------------------------------------------------ 5. classes
def test_classes_and_isolation(w):
    N, T, U, V = 9, 8, 5, 10
    inf, nan = float("inf"), float("nan")
    x, ys, xn, yn = make(N, T, U, V, seed=11, xn=[8, 8, 8, 8, 8, 0, 3, 8, 8], yn=[4, 4, 4, 4, 4, 2, 4, 4, 3])
    x[1, 2, 1, 0] = nan                          # NaN blank logit in a live row: NaN lattice
    x[2, 2, 1, 4] = nan                          # NaN non-blank logit in a live row: NaN lattice
    x[3, 7, 4, 4] = nan                          # NaN non-blank logit in a last-column row (u = Un - 1): finite
    x[4, 2, 1, 0] = inf                          # x[B] = +inf: that blank has log-prob 0, its label -inf
    x[4, 3, 2, 0] = -inf                         # x[B] = -inf: blank edge removed, labels keep their softmax
    x[7, 1, 1, 1:] = -inf                        # every non-blank logit -inf: lse_nb NaN, a NaN label
    x[8, :, 4, 2] = nan                          # padding rows of lattice 8 (u = 4 > yn = 3)
    # lattice 5: invalid lengths (NaN); lattice 6: more labels than frames (no path for types 1 and 2)
    for kind in ("regular", "modified", "constrained"):
        xg = x.clone().requires_grad_(True)
        c = w.rnnt_loss_from_logits(xg, ys, xn, yn, rnnt_type=kind, use_hat_loss=True)
        c.sum().backward()
        assert torch.isnan(c[[1, 2, 5, 7]]).all()
        assert torch.isfinite(c[[0, 3, 4, 8]]).all() and torch.isfinite(xg.grad[[0, 4]]).all()
        # lattice 3: l is NaN only in the last column, which no lattice reads; that row's non-blank columns get
        # gl (.. - exp(x - NaN)) with gl = 0, NaN as autograd of the composition gives, everything else is finite
        g3 = xg.grad[3].clone()
        assert torch.isnan(g3[7, 4, 1:]).all() and torch.isfinite(g3[7, 4, 0])
        g3[7, 4] = 0
        assert torch.isfinite(g3).all()
        if kind != "regular":
            assert c[6].item() == inf and (xg.grad[6] == 0).all()
        assert (xg.grad[5] == 0).all()
        # padding rows of lattice 8 (NaN lse_nb, finite blank logit): NaN at the non-blank columns, 0 at the blank
        g8 = xg.grad[8, :, 4]
        assert torch.isnan(g8[:, 1:]).all() and (g8[:, 0] == 0).all()
        # the other lattices are those of a batch without the bad ones
        keep = [0, 3, 4, 8]
        xk = x[keep].clone().requires_grad_(True)
        ck = w.rnnt_loss_from_logits(xk, ys[keep], xn[keep], yn[keep], rnnt_type=kind, use_hat_loss=True)
        ck.sum().backward()
        assert same(c[keep], ck) and same(xg.grad[keep], xk.grad)
    # rows without gradient get exact zeros, NaN at the blank column only where x[B] is NaN
    N, T, U, V = 2, 4, 3, 6
    x, ys, xn, yn = make(N, T, U, V, seed=1, xn=[2, 4], yn=[1, 2])
    x[0, 3, 0, 0] = nan                          # a padding row (t = 3 >= Tn = 2) with a NaN blank logit
    x[0, 3, 1, 2] = nan                          # ... and one with a NaN label logit
    c, lse, pg = fwd(w, x, ys, xn, yn)
    g = w._C.rnnt_logits_backward(x, lse, pg, ys, torch.ones(N, device="cuda"), 0, True)
    assert torch.isnan(g[0, 3, 0, 0]) and (g[0, 3, 0, 1:] == 0).all()
    assert torch.isnan(g[0, 3, 1, 1:]).all() and g[0, 3, 1, 0] == 0
    assert (g[0, 2:][~torch.isnan(g[0, 2:])] == 0).all()


# ------------------------------------------------------------------------------------------------ 6. runtime
@pytest.mark.parametrize("kind", ["regular", "modified"])
def test_cuda_graph_and_determinism(w, kind):
    N, T, U, V = 8, 60, 20, 32
    x, ys, xn, yn = make(N, T, U, V, seed=12)
    src = x.clone().requires_grad_(True)

    def step():
        src.grad = None
        loss = w.rnnt_loss_from_logits(src, ys, xn, yn, reduction="sum", rnnt_type=kind, delay_penalty=0.01,
                                       use_hat_loss=True)
        loss.backward()
        return loss

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    want = step().detach().clone()
    gwant = src.grad.clone()
    again = step().detach().clone()
    assert same(again, want) and same(src.grad, gwant)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert same(out, want) and same(src.grad, gwant)


def test_forward_only_empty_batch_and_launch_counts(w):
    N, T, U, V, S = 4, 20, 7, 24, 3
    x, ys, xn, yn = make(N, T, U, V, seed=13)
    c_full = w.rnnt_loss_from_logits(x.clone().requires_grad_(True), ys, xn, yn, use_hat_loss=True)
    c_fwd = w.rnnt_loss_from_logits(x, ys, xn, yn, use_hat_loss=True)
    assert same(c_full.detach(), c_fwd)
    empty = torch.empty((0, T, U, V), device="cuda")
    e = torch.empty((0, U - 1), dtype=torch.int, device="cuda")
    z = torch.empty((0,), dtype=torch.int, device="cuda")
    assert w.rnnt_loss_from_logits(empty, e, z, z, use_hat_loss=True).shape == (0,)
    ranges = torch.zeros((N, T), dtype=torch.int, device="cuda")
    xp = x[:, :, :S].contiguous()
    flat, ysc = to_compact(x.cpu().numpy(), ys.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy())
    xc, ysc = cu(flat), cu(ysc)

    def launches(fn):
        torch.cuda.synchronize()
        before = w._C.launch_count()
        fn()
        torch.cuda.synchronize()
        return w._C.launch_count() - before

    for call in (
            lambda h: w.rnnt_loss_from_logits(x.clone().requires_grad_(True), ys, xn, yn, use_hat_loss=h,
                                              rnnt_type="constrained", delay_penalty=0.1).sum().backward(),
            lambda h: w.rnnt_loss_from_logits(x.clone().requires_grad_(True), ys, xn, yn, use_hat_loss=h,
                                              fastemit_lambda=0.01).sum().backward(),
            lambda h: w.rnnt_loss_pruned(xp.clone().requires_grad_(True), ys, xn, yn, ranges,
                                         use_hat_loss=h).sum().backward(),
            lambda h: w.rnnt_loss_from_logits(xc.clone().requires_grad_(True), ysc, xn, yn, compact=True,
                                              use_hat_loss=h).sum().backward(),
            lambda h: w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type="modified", use_hat_loss=h),
            lambda h: w.rnnt_align_from_logits(xc, ysc, xn, yn, compact=True, use_hat_loss=h)):
        assert launches(lambda: call(False)) == launches(lambda: call(True))


# ------------------------------------------------------------------------------------------------ 7. refusals
def test_refusals(w, lib):
    x, ys, xn, yn = make(2, 5, 4, 6, seed=1)
    x1 = x[..., :1].contiguous()
    r = torch.zeros((2, 5), dtype=torch.int, device="cuda")
    torch.cuda.synchronize()
    before = w._C.launch_count()
    for bad in (1, 0, None, "yes", np.bool_(True)):
        with pytest.raises(ValueError, match="use_hat_loss"):
            w.rnnt_loss_from_logits(x, ys, xn, yn, use_hat_loss=bad)
        with pytest.raises(ValueError, match="use_hat_loss"):
            w.rnnt_loss_pruned(x, ys, xn, yn, r, use_hat_loss=bad)
        with pytest.raises(ValueError, match="use_hat_loss"):
            w.rnnt_align_from_logits(x, ys, xn, yn, use_hat_loss=bad)
    zero = torch.zeros_like(ys)
    with pytest.raises(ValueError, match="V >= 2"):
        w.rnnt_loss_from_logits(x1, zero, xn, yn, use_hat_loss=True)
    with pytest.raises(ValueError, match="V >= 2"):
        w.rnnt_loss_pruned(x1, zero, xn, yn, r, use_hat_loss=True)
    with pytest.raises(ValueError, match="V >= 2"):
        w.rnnt_align_from_logits(x1, zero, xn, yn, use_hat_loss=True)
    with pytest.raises(ValueError, match="compact"):
        w.rnnt_loss_from_logits(x.view(-1, 6), ys, xn, yn, compact=True, rnnt_type="modified", use_hat_loss=True)
    with pytest.raises(ValueError, match="fastemit_lambda"):
        w.rnnt_loss_from_logits(x, ys, xn, yn, fastemit_lambda=0.1, rnnt_type="modified", use_hat_loss=True)
    # the operator module
    go = torch.ones(2, device="cuda")
    lse = torch.zeros((2, 5, 4), device="cuda")
    pg = torch.zeros((2, 5, 4, 2), device="cuda")
    for fn in (lambda: w._C.rnnt_logits_forward(x1, zero, xn, yn, 0, 0.0, True, 0, 0, 0.0, True),
               lambda: w._C.rnnt_logits_backward(x1, lse, pg, zero, go, 0, True),
               lambda: w._C.rnnt_logits_pruned_forward(x1, zero, xn, yn, r, 0, 0.0, True, 0, 0, 0.0, True),
               lambda: w._C.rnnt_logits_pruned_backward(x1, lse, pg, zero, r, go, 0, True),
               lambda: w._C.rnnt_align_logits_dense(x1, zero, xn, yn, 0, 0, 0.0, True)):
        with pytest.raises(RuntimeError, match="V >= 2"):
            fn()
    # the C ABI
    s = torch.cuda.current_stream().cuda_stream
    N, T, U, V = 2, 5, 4, 6
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
    c = torch.empty(N, device="cuda")
    args = (ws.data_ptr(), ws.numel(), x1.data_ptr(), zero.data_ptr(), xn.data_ptr(), yn.data_ptr(), c.data_ptr(),
            lse.data_ptr(), pg.data_ptr())
    assert lib.rnnt_b200_logits_hat_forward(s, *args, N, T, U, 1, 0, 0.0, 0, 4, 0, 0.0) == INVALID
    assert lib.rnnt_b200_logits_hat_forward(s, *args[:2], x.data_ptr(), *args[3:], N, T, U, V, 0, 0.0, 0, 3, 0,
                                            0.0) == INVALID
    assert lib.rnnt_b200_logits_hat_forward(s, *args[:2], x.data_ptr(), *args[3:], N, T, U, V, 0, 0.0, 0, 4, 3,
                                            0.0) == INVALID
    out = torch.empty_like(x)
    assert lib.rnnt_b200_logits_hat_backward(s, x1.data_ptr(), lse.data_ptr(), pg.data_ptr(), zero.data_ptr(),
                                             go.data_ptr(), out.data_ptr(), N, T, U, 1, 0, 4) == INVALID
    assert lib.rnnt_b200_logits_pruned_hat_forward(s, *args[:6], r.data_ptr(), *args[6:], N, T, U, U, 1, 0, 0.0, 0,
                                                   4, 0, 0.0) == INVALID
    wa = torch.empty(lib.rnnt_b200_align_logits_workspace_bytes(N * T * U, N, T, U), dtype=torch.uint8, device="cuda")
    f = torch.empty((N, U - 1), dtype=torch.int, device="cuda")
    assert lib.rnnt_b200_align_logits_hat_dense(s, wa.data_ptr(), wa.numel(), x1.data_ptr(), zero.data_ptr(),
                                                xn.data_ptr(), yn.data_ptr(), c.data_ptr(), f.data_ptr(), N, T, U, 1,
                                                0, 4, 0, 0.0) == INVALID
    assert lib.rnnt_b200_align_logits_hat_compact(s, wa.data_ptr(), wa.numel(), x1.data_ptr(), zero.data_ptr(),
                                                  xn.data_ptr(), yn.data_ptr(), c.data_ptr(), f.data_ptr(), N * T * U,
                                                  N, 1, 0, 4, T, U) == INVALID
    # compact forward / backward and the pruned backward: V < 2 and a bad element size
    STU = N * T * U
    prefix = torch.zeros(2 * N, dtype=torch.long, device="cuda")
    for V_, eb, xp in ((1, 4, x1), (V, 3, x)):
        assert lib.rnnt_b200_logits_compact_hat_forward(s, ws.data_ptr(), ws.numel(), xp.data_ptr(), zero.data_ptr(),
                                                        xn.data_ptr(), yn.data_ptr(), c.data_ptr(), lse.data_ptr(),
                                                        pg.data_ptr(), prefix.data_ptr(), None, STU, N, V_, 0, 0.0, 0,
                                                        T, U, eb) == INVALID
        assert lib.rnnt_b200_logits_compact_hat_backward(s, xp.data_ptr(), lse.data_ptr(), pg.data_ptr(),
                                                         zero.data_ptr(), xn.data_ptr(), yn.data_ptr(),
                                                         prefix.data_ptr(), go.data_ptr(), out.data_ptr(), STU, N, V_,
                                                         0, eb) == INVALID
        assert lib.rnnt_b200_logits_pruned_hat_backward(s, xp.data_ptr(), lse.data_ptr(), pg.data_ptr(),
                                                        zero.data_ptr(), r.data_ptr(), go.data_ptr(), out.data_ptr(),
                                                        N, T, U, U, V_, 0, eb) == INVALID
    torch.cuda.synchronize()
    assert w._C.launch_count() == before
