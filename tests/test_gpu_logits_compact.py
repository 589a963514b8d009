"""rnnt_loss_from_logits(compact=True): compact (STU,V) logits in joint_pack's row order, float32 or bfloat16.

The contract (include/rnnt_b200.h, DESIGN.md 4), with xp = the compact rows placed in a padded (N,T,U,V) tensor:
  1. lse is torch.equal to the dense from-logits lse of xp on the live rows;
  2. costs and pair_grads are torch.equal to _C.rnnt_loss_compact(x.float() - lse[:, None]) with the same hints and LSE
     mode (fused and general recurrence alike);
  3. the logit gradient is torch.equal, on the live rows, to the dense _C.rnnt_logits_backward on xp, lse and the pair
     gradients padded with zeros;
  4. bf16: costs, lse and pair_grads are torch.equal to the f32 compact path on the widened logits, the gradient is the
     f32 gradient rounded to bf16 once;
  5. against the fp64 oracle and against torch.log_softmax + rnnt_loss(compact=True): costs 1e-5 relative, gradients
     1e-4 + 2 gtol(T,U);
  6. a label equal to blank adds both gradients, a -inf-masked vocabulary stays finite, a lattice without a finite
     alignment gets the compact classes (+inf), a sample exceeding compact_hints gets cost NaN."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.common import apply_mask, assert_same_classes, from_compact, to_compact
from tests.test_gpu_logits import gtol, make
from tests.test_gpu_logits_bf16 import PARITY

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
BF16 = torch.bfloat16
EXACT, FAST = 1, 2
MODES = {EXACT: "exact", FAST: "fast"}

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ragged(N, T, U, V, seed, blank=0, label_blank=False):
    """make()'s batch plus two edge lattices: yn = 0 (Un = 1) and xn = 1.  -> x (N+2,T,U,V) f32, ys, xn, yn (numpy)."""
    x, ys, xn, yn = make(N + 2, T, U, V, seed=seed, blank=blank)
    yn[N] = 0
    xn[N + 1] = 1
    if label_blank:
        ys[0, ::3] = blank                       # labels equal to the blank: the two gradients of such a cell add
    return x, ys, xn, yn


def pack(t, xn, yn):
    """Live rows of a padded (N,T,U,...) tensor in the compact order."""
    return torch.cat([t[i, :int(xn[i]), :int(yn[i]) + 1].reshape(-1, *t.shape[3:]) for i in range(len(xn))])


def unpack(t, xn, yn, T, U):
    """(STU,...) -> zero-padded (N,T,U,...)."""
    out = t.new_zeros((len(xn), T, U) + tuple(t.shape[1:]))
    o = 0
    for i in range(len(xn)):
        Tn, Un = int(xn[i]), int(yn[i]) + 1
        out[i, :Tn, :Un] = t[o:o + Tn * Un].reshape(Tn, Un, *t.shape[1:])
        o += Tn * Un
    return out


class lse_mode:
    """The process default LSE mode (what rnnt_loss_compact runs with) set to `mode` for the block."""

    def __init__(self, w, mode):
        self.w, self.mode = w, mode

    def __enter__(self):
        self.w.set_lse_mode(MODES[self.mode])

    def __exit__(self, *a):
        self.w.set_lse_mode("auto")


def compact_step(w, x, ys_c, xn, yn, blank, lam, mode, hints, go):
    """(costs, lse, pair_grads, prefix, logit gradient) of the compact from-logits operators."""
    c, l, p, pref = w._C.rnnt_logits_compact_forward(x, ys_c, xn, yn, blank, lam, True, mode, *hints)
    g = w._C.rnnt_logits_compact_backward(x, l, p, ys_c, xn, yn, pref, go, blank)
    return c, l, p, pref, g


@gpu
@pytest.mark.parametrize("label_blank", [False, True])
@pytest.mark.parametrize("shape", PARITY)
def test_compact_bit_parity(w, shape, label_blank):
    """Items 1-4 on every normaliser branch, fused-kernel and general-path lattices, with and without hints."""
    N, T, U, V, blank, lam = shape
    x, ys, xn, yn = ragged(N, T, U, V, seed=T + V, blank=blank, label_blank=label_blank)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    xd, ysd, xnd, ynd = cu(from_compact(x_c, xn, yn, T, U)), cu(ys), cu(xn), cu(yn)
    xf, ys_c = cu(x_c), cu(ys_c)
    xb = xf.to(BF16)
    go = torch.linspace(0.5, 1.5, len(xn), device="cuda")
    for mode in (EXACT, FAST):
        # the dense from-logits path on the padded logits
        _, ld, _ = w._C.rnnt_logits_forward(xd, ysd, xnd, ynd, blank, lam, True, mode)
        for hints in ((T, U), (0, 0)):
            cf, lf, pf, pref, gf = compact_step(w, xf, ys_c, xnd, ynd, blank, lam, mode, hints, go)
            assert torch.isfinite(cf).all() and cf.dtype == lf.dtype == pf.dtype == gf.dtype == torch.float32
            assert torch.equal(lf, pack(ld, xn, yn)), (mode, hints)                                   # 1
            with lse_mode(w, mode):
                cr, pr, _ = w._C.rnnt_loss_compact(xf - lf[:, None], ys_c, xnd, ynd, blank, lam, True, *hints)
            assert torch.equal(cf, cr), (mode, hints, (cf - cr).abs().max().item())                    # 2
            assert torch.equal(pf, pr), (mode, hints)
            gd = w._C.rnnt_logits_backward(xd, ld, unpack(pf, xn, yn, T, U), ysd, go, blank)
            assert torch.equal(gf, pack(gd, xn, yn)), (mode, hints)                                   # 3
            # 4: bf16 against the f32 compact path on the widened logits
            cb, lb, pb, _, gb = compact_step(w, xb, ys_c, xnd, ynd, blank, lam, mode, hints, go)
            cw, lw, pw, _, gw = compact_step(w, xb.float(), ys_c, xnd, ynd, blank, lam, mode, hints, go)
            assert cb.dtype == lb.dtype == pb.dtype == torch.float32 and gb.dtype == BF16
            assert torch.equal(cb, cw) and torch.equal(lb, lw) and torch.equal(pb, pw), (mode, hints)
            assert torch.equal(gb, gw.to(BF16)), (mode, hints)
            assert pref.dtype == torch.int64 and pref.shape == (2 * len(xn),)


ORACLE = [s for s in PARITY if s[0] * s[1] * s[2] * s[3] <= 4e6]


@gpu
@pytest.mark.parametrize("shape", ORACLE)
def test_compact_vs_oracle_and_unfused(w, shape):
    """Item 5, both LSE modes, float32 and bfloat16 (one bf16 rounding more on the gradient)."""
    N, T, U, V, blank, lam = shape
    x, ys, xn, yn = ragged(N, T, U, V, seed=T + V, blank=blank)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    go = np.linspace(0.5, 1.5, len(xn))
    args = (cu(ys_c), cu(xn), cu(yn))
    tol = 1e-4 + 2 * gtol(T, U)
    for dtype in (torch.float32, BF16):
        xt = cu(x_c).to(dtype)
        xv = xt.float().cpu().numpy()
        c0, g0 = oracle.from_logits(from_compact(xv, xn, yn, T, U), ys, xn, yn, blank, lam, grad_output=go)
        g0 = to_compact(g0, ys, xn, yn)[0]
        rel = 2.0 ** -8 if dtype == BF16 else 0.0
        for mode in (EXACT, FAST):
            with lse_mode(w, mode):
                a = xt.clone().requires_grad_(True)
                costs = w.rnnt_loss_from_logits(a, *args, blank=blank, fastemit_lambda=lam, compact=True)
                (costs * cu(go.astype(np.float32))).sum().backward()
                b = xt.float().clone().requires_grad_(True)
                cu_ = w.rnnt_loss(torch.log_softmax(b, -1), *args, blank=blank, fastemit_lambda=lam, compact=True)
                (cu_ * cu(go.astype(np.float32))).sum().backward()
            assert a.grad.dtype == dtype and costs.dtype == torch.float32
            got = a.grad.float().cpu().numpy()
            np.testing.assert_allclose(costs.detach().cpu().numpy(), c0, rtol=1e-5)
            np.testing.assert_allclose(costs.detach().cpu().numpy(), cu_.detach().cpu().numpy(), rtol=1e-5)
            for want in (g0, b.grad.cpu().numpy()):
                err = np.abs(got - want) - np.abs(want) * rel
                assert err.max() <= tol, (dtype, mode, err.max())


def classes(a):
    """Finite -> 0, NaN and +-inf kept: compares where two results are non-finite."""
    a = np.asarray(a, np.float32)
    return np.where(np.isfinite(a), np.float32(0), a)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_compact_masked_and_dead_lattices(w, dtype):
    """Item 6: a -inf-masked vocabulary stays finite; a lattice without a finite alignment costs +inf (compact
    classes) and its NaN gradient rows are those of torch.log_softmax + rnnt_loss(compact=True)."""
    N, T, U, V, blank = 3, 12, 9, 30, 0
    x, ys, xn, yn = make(N, T, U, V, seed=11, blank=blank)
    rng = np.random.RandomState(5)
    for n in range(N):
        apply_mask(x, ys, n, int(xn[n]), int(yn[n]) + 1, "vocab_ninf", blank, rng)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    args = (cu(ys_c), cu(xn), cu(yn))
    for hints in ((T, U), (0, 0)):
        with w.compact_hints(*hints) if hints[0] else _null():
            a = cu(x_c).to(dtype).requires_grad_(True)
            w.rnnt_loss_from_logits(a, *args, blank=blank, compact=True).sum().backward()
        assert torch.isfinite(a.grad.float()).all()
    # lattice 1 dead: its label k = 2 masked -inf at every frame
    x2 = x.copy()
    apply_mask(x2, ys, 1, int(xn[1]), int(yn[1]) + 1, "label_all", blank, rng)
    x_c, ys_c = to_compact(x2, ys, xn, yn)
    args = (cu(ys_c), cu(xn), cu(yn))
    for mode in (EXACT, FAST):
        with lse_mode(w, mode):
            a = cu(x_c).to(dtype).requires_grad_(True)
            c = w.rnnt_loss_from_logits(a, *args, blank=blank, compact=True)
            c.sum().backward()
            b = cu(x_c).to(dtype).float().requires_grad_(True)
            cr = w.rnnt_loss(torch.log_softmax(b, -1), *args, blank=blank, compact=True)
            cr.sum().backward()
        assert c[1].item() == np.inf and torch.isfinite(c[[0, 2]]).all()
        assert_same_classes(classes(c.detach().cpu()), classes(cr.detach().cpu()), "costs")
        assert_same_classes(classes(a.grad.float().cpu()), classes(b.grad.cpu()), "grads")
        assert torch.isnan(a.grad.float()).any()


class _null:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


@gpu
def test_compact_sample_exceeding_hints(w):
    """A sample longer than the hints: cost NaN, as rnnt_loss(compact=True) under the same hints; the others agree."""
    N, T, U, V = 3, 20, 8, 12
    x, ys, xn, yn = make(N, T, U, V, seed=4)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    args = (cu(ys_c), cu(xn), cu(yn))
    xt = cu(x_c)
    with w.compact_hints(T - 1, U):                 # lattice 0 has xn = T
        c = w.rnnt_loss_from_logits(xt, *args, compact=True)
        cr = w.rnnt_loss(torch.log_softmax(xt, -1), *args, compact=True)
    assert torch.isnan(c[0]) and torch.isnan(cr[0])
    assert_same_classes(classes(c.cpu()), classes(cr.cpu()), "costs")
    np.testing.assert_allclose(c[1:].cpu().numpy(), cr[1:].cpu().numpy(), rtol=1e-5)


@gpu
def test_compact_forward_only_and_empty_batch(w):
    N, T, U, V = 3, 20, 8, 28
    x, ys, xn, yn = ragged(N, T, U, V, seed=9)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    xt, args = cu(x_c), (cu(ys_c), cu(xn), cu(yn))
    c, l, p, pref = w._C.rnnt_logits_compact_forward(xt, *args, 0, 0.0, False, EXACT)
    assert p.numel() == 0
    c2, l2, _, pref2 = w._C.rnnt_logits_compact_forward(xt, *args, 0, 0.0, True, EXACT)
    assert torch.equal(c, c2) and torch.equal(l, l2) and torch.equal(pref, pref2)
    # the prefix sums: first row and first label of each lattice
    rows = torch.tensor(np.concatenate([[0], np.cumsum(xn * (yn + 1))[:-1]]), device="cuda")
    labs = torch.tensor(np.concatenate([[0], np.cumsum(yn)[:-1]]), device="cuda")
    assert torch.equal(pref, torch.cat([rows, labs]))
    with torch.no_grad():
        c3 = w.rnnt_loss_from_logits(xt.clone().requires_grad_(True), *args, compact=True)
    assert not c3.requires_grad and torch.equal(c3, c)
    # N = 0
    e = torch.zeros(0, V, device="cuda", requires_grad=True)
    z = torch.zeros(0, dtype=torch.int, device="cuda")
    for hints in ((5, 5), None):
        with w.compact_hints(*hints) if hints else _null():
            c0 = w.rnnt_loss_from_logits(e, z, z, z, compact=True)
        assert c0.shape == (0,)
        c0.sum().backward()
        assert e.grad.shape == (0, V)


@gpu
def test_compact_shape_errors_without_hints(w):
    N, T, U, V = 2, 6, 4, 7
    x, ys, xn, yn = make(N, T, U, V, seed=2)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    xt, ys_t, xn_t, yn_t = cu(x_c), cu(ys_c), cu(xn), cu(yn)
    with pytest.raises(RuntimeError, match=r"xs shape mismatch with \(\\sum\{xn\*\(yn\+1\)\}, \)"):
        w.rnnt_loss_from_logits(xt[:-1], ys_t, xn_t, yn_t, compact=True)
    with pytest.raises(RuntimeError, match=r"ys shape must be equal to \(sum\(yn\), \)"):
        w.rnnt_loss_from_logits(xt, ys_t[:-1], xn_t, yn_t, compact=True)
    with pytest.raises(RuntimeError, match="xs must have 2 dimensions"):
        w.rnnt_loss_from_logits(xt[None], ys_t, xn_t, yn_t, compact=True)
    with pytest.raises(RuntimeError, match=r"blank must be in \[0, V\)"):
        w.rnnt_loss_from_logits(xt, ys_t, xn_t, yn_t, blank=V, compact=True)
    with pytest.raises(RuntimeError, match="xs must be a Float tensor"):
        w.rnnt_loss_from_logits(xt.half(), ys_t, xn_t, yn_t, compact=True)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_compact_reductions(w, dtype):
    """average_frames divides in float32 (601 and 513 frames: not bf16 numbers); 'sum' / 'mean' reduce the costs."""
    N, T, U, V = 2, 601, 4, 12
    x, ys, _, yn = make(N, T, U, V, seed=3)
    xn = np.array([601, 513], np.int32)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    args = (cu(ys_c), cu(xn), cu(yn))
    xt = cu(x_c).to(dtype)
    c, l, p, pref = w._C.rnnt_logits_compact_forward(xt, *args, 0, 0.0, True, 0)
    for reduction in ("none", "sum", "mean"):
        for avg in (False, True):
            a = xt.clone().requires_grad_(True)
            loss = w.rnnt_loss_from_logits(a, *args, average_frames=avg, reduction=reduction, compact=True)
            leaf = c.clone().requires_grad_(True)
            want = leaf / cu(xn).float() if avg else leaf
            want = want.sum() if reduction == "sum" else want.mean() if reduction == "mean" else want
            assert loss.dtype == torch.float32 and torch.equal(loss, want.detach()), (reduction, avg)
            loss.sum().backward()
            go, = torch.autograd.grad(want.sum(), leaf)
            g = w._C.rnnt_logits_compact_backward(xt, l, p, args[0], args[1], args[2], pref, go.contiguous(), 0)
            assert a.grad.dtype == dtype and torch.equal(a.grad, g), (reduction, avg)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_compact_cuda_graph_replay(w, dtype):
    """Under compact_hints the forward makes no host sync: a captured loss.backward() step replays to eager's bits."""
    N, T, U, V = 4, 60, 20, 28
    x, ys, xn, yn = make(N, T, U, V, seed=21)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    x2_c = to_compact(make(N, T, U, V, seed=22)[0], ys, xn, yn)[0]
    srcs = [cu(x_c).to(dtype), cu(x2_c).to(dtype)]
    args = (cu(ys_c), cu(xn), cu(yn))

    def step(x):
        x.grad = None
        with w.compact_hints(T, U):
            loss = w.rnnt_loss_from_logits(x, *args, reduction="sum", compact=True)
        loss.backward()
        return loss

    def eager(src):
        x = src.clone().requires_grad_(True)
        return step(x).detach(), x.grad

    x = srcs[0].clone().requires_grad_(True)
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
    for src in srcs:
        with torch.no_grad():
            x.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        l0, g0 = eager(src)
        assert x.grad.dtype == dtype
        assert torch.equal(loss.detach(), l0) and torch.equal(x.grad, g0)


def _abi():
    lib = ctypes.CDLL(LIB)
    P, I, F, L = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int64
    fns = {}
    for name in ("rnnt_b200_logits_compact_forward", "rnnt_b200_logits_compact_forward_bf16"):
        f = getattr(lib, name)
        f.restype = I
        f.argtypes = [P, P, ctypes.c_size_t] + [P] * 9 + [L, I, I, I, F, I, I, I]
        fns[name] = f
    for name in ("rnnt_b200_logits_compact_backward", "rnnt_b200_logits_compact_backward_bf16"):
        f = getattr(lib, name)
        f.restype = I
        f.argtypes = [P] * 10 + [L, I, I, I]
        fns[name] = f
    lib.rnnt_b200_workspace_bytes.restype = ctypes.c_size_t
    lib.rnnt_b200_workspace_bytes.argtypes = [L, I]
    return lib, fns


@gpu
@pytest.mark.parametrize("dtype,V", [(torch.float32, 5), (torch.float32, 6), (torch.float32, 28),
                                     (BF16, 7), (BF16, 6), (BF16, 12), (BF16, 1024)])
def test_compact_abi_writes_every_gradient_element(w, dtype, V):
    """C ABI with NaN-prefilled outputs: the backward writes every element (and lse every row) once, and the result is
    the operator's; vector widths 1, 2, 4 (f32) and 1, 2, 4, 8 (bf16)."""
    lib, fns = _abi()
    sfx = "_bf16" if dtype == BF16 else ""
    N, T, U = 3, 30, 9
    x, ys, xn, yn = ragged(N, T, U, V, seed=V)
    x_c, ys_c = to_compact(x, ys, xn, yn)
    xt, ys_t, xn_t, yn_t = cu(x_c).to(dtype), cu(ys_c), cu(xn), cu(yn)
    STU, Nn = xt.shape[0], len(xn)
    costs = torch.full((Nn,), float("nan"), device="cuda")
    lse = torch.full((STU,), float("nan"), device="cuda")
    pg = torch.full((STU, 2), float("nan"), device="cuda")
    pref = torch.full((2 * Nn,), -1, dtype=torch.int64, device="cuda")
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(STU, Nn), dtype=torch.uint8, device="cuda")
    go = torch.linspace(0.5, 1.5, Nn, device="cuda")
    out = torch.full_like(xt, float("nan"))
    s = torch.cuda.current_stream().cuda_stream
    st = fns["rnnt_b200_logits_compact_forward" + sfx](
        s, ws.data_ptr(), ws.numel(), xt.data_ptr(), ys_t.data_ptr(), xn_t.data_ptr(), yn_t.data_ptr(),
        costs.data_ptr(), lse.data_ptr(), pg.data_ptr(), pref.data_ptr(), None, STU, Nn, V, 0, 0.0, EXACT, T, U)
    assert st == 0
    st = fns["rnnt_b200_logits_compact_backward" + sfx](
        s, xt.data_ptr(), lse.data_ptr(), pg.data_ptr(), ys_t.data_ptr(), xn_t.data_ptr(), yn_t.data_ptr(),
        pref.data_ptr(), go.data_ptr(), out.data_ptr(), STU, Nn, V, 0)
    assert st == 0
    torch.cuda.synchronize()
    assert torch.isfinite(costs).all() and torch.isfinite(lse).all() and torch.isfinite(pg).all()
    assert torch.isfinite(out.float()).all()
    c, l, p, pr, g = compact_step(w, xt, ys_t, xn_t, yn_t, 0, 0.0, EXACT, (T, U), go)
    assert torch.equal(costs, c) and torch.equal(lse, l) and torch.equal(pg, p) and torch.equal(pref, pr)
    assert torch.equal(out, g)


@gpu
@pytest.mark.parametrize("autocast", [False, True])
def test_joint_pack_feeds_the_fused_compact_loss(w, autocast):
    """joint_pack -> Linear -> rnnt_loss_from_logits(compact=True), float32 and under torch.autocast(bfloat16): the
    loss and the gradients of f, g and the weight agree with the padded pipeline joint -> log_softmax -> rnnt_loss."""
    N, T, U1, H, V = 3, 14, 6, 16, 9
    g0 = torch.Generator(device="cuda").manual_seed(1)
    f = torch.randn(N, T, H, device="cuda", generator=g0).requires_grad_(True)
    g = torch.randn(N, U1, H, device="cuda", generator=g0).requires_grad_(True)
    lin = torch.nn.Linear(H, V).cuda()
    lf = torch.tensor([14, 9, 12], dtype=torch.int, device="cuda")
    lg = torch.tensor([5, 3, 4], dtype=torch.int, device="cuda")
    ys = torch.randint(1, V, (N, U1 - 1), dtype=torch.int, device="cuda", generator=g0)
    ys_c = torch.cat([ys[i, :lg[i]] for i in range(N)]).contiguous()
    with torch.autocast("cuda", dtype=BF16, enabled=autocast):
        logits = lin(torch.tanh(w.joint_pack(f, g, lf, lg)))
        assert logits.dtype == (BF16 if autocast else torch.float32)
        loss_c = w.rnnt_loss_from_logits(logits, ys_c, lf, lg, reduction="sum", compact=True)
    gc = torch.autograd.grad(loss_c, [f, g, lin.weight])
    with torch.autocast("cuda", dtype=BF16, enabled=autocast):
        logits_d = lin(torch.tanh(f.unsqueeze(2) + g.unsqueeze(1)))
    lp_d = torch.log_softmax(logits_d.float(), -1)
    loss_d = w.rnnt_loss(lp_d, ys, lf, lg, reduction="sum")
    gd = torch.autograd.grad(loss_d, [f, g, lin.weight])
    # autocast: one more bf16 rounding of the logit gradient (2^-8 relative) in the compact pipeline
    rtol, atol = (1e-5, 1e-5) if not autocast else (1e-2, 1e-2)
    np.testing.assert_allclose(loss_c.item(), loss_d.item(), rtol=max(rtol, 1e-5))
    for a, b in zip(gc, gd):
        np.testing.assert_allclose(a.float().cpu().numpy(), b.float().cpu().numpy(),
                                   rtol=1e-4 if not autocast else rtol, atol=atol)


def test_compact_entry_points_validate_on_host():
    """No GPU needed: V, blank, NULL lse / prefix, a misaligned pair_grads and (bf16) odd logits or gradient pointers
    are rejected before any launch (status 5); N == 0 returns success without a launch."""
    import warp_rnnt_b200 as w
    _, fns = _abi()
    P = ctypes.c_void_p
    ptr = P(0x10000)

    def f(sfx, logits=0x30000, lse=0x40000, pg=0x50000, pref=0x60000, N=4, V=5, blank=0, STU=10):
        return fns["rnnt_b200_logits_compact_forward" + sfx](
            None, P(0x20000), 1 << 20, P(logits), ptr, ptr, ptr, ptr, P(lse), P(pg), P(pref), None, STU, N, V, blank,
            0.0, EXACT, 0, 0)

    def b(sfx, logits=0x30000, out=0x70000, lse=0x40000, pg=0x50000, pref=0x60000, N=4, V=5, blank=0, STU=10):
        return fns["rnnt_b200_logits_compact_backward" + sfx](
            None, P(logits), P(lse), P(pg), ptr, ptr, ptr, P(pref), ptr, P(out), STU, N, V, blank)

    for sfx in ("", "_bf16"):
        for call in (f, b):
            assert call(sfx, V=0) == 5                                 # V < 1
            assert call(sfx, V=1 << 22) == 5                           # V too large
            assert call(sfx, blank=5) == 5                             # blank >= V
            assert call(sfx, blank=-1) == 5
            assert call(sfx, N=-1) == 5
            assert call(sfx, STU=-1) == 5
            assert call(sfx, lse=0) == 5                               # NULL lse
            assert call(sfx, pref=0) == 5                              # NULL prefix
            assert call(sfx, pg=0x50004) == 5                          # pair_grads not 8-byte aligned
            assert call(sfx, N=0) == 0                                 # nothing to do
        assert f(sfx, N=0, pg=0) == 0                                  # forward only
        assert b(sfx, N=0, STU=0) == 0
    assert f("_bf16", N=0, logits=0x30001) == 5                       # odd bf16 logits pointer
    assert b("_bf16", N=0, logits=0x30001) == 5
    assert b("_bf16", N=0, out=0x70001) == 5                           # odd bf16 gradient pointer
    # the operator refuses every other dtype with the float32 message (host tensors: dtype is checked first)
    x = torch.zeros(3, 4, dtype=torch.float16)
    ys, ln = torch.zeros(1, dtype=torch.int), torch.ones(1, dtype=torch.int)
    with pytest.raises(RuntimeError, match="xs must be a Float tensor"):
        w._C.rnnt_logits_compact_forward(x, ys, ln, ln, 0, 0.0, True, 0, 0, 0)
    with pytest.raises(RuntimeError, match="xs must be located in the CUDA"):
        w._C.rnnt_logits_compact_forward(x.to(BF16), ys, ln, ln, 0, 0.0, True, 0, 0, 0)
