"""GPU: k2's rnnt_type ("modified", "constrained") and delay_penalty on rnnt_loss_from_logits, rnnt_loss_pruned and
rnnt_loss_simple (include/rnnt_b200.h, DESIGN.md 3.8).

  1. explicit defaults are today's call, bit for bit, with the same launch record;
  2. regular + penalty is rnnt_b200_loss_pairs on pairs penalised in the kernels' f32 order;
  3. modified / constrained x penalty, f32 and bf16, against the fp64 restatement (tests/path_oracle.py);
  4. bit relations: pruned with S = U windows is from-logits; every forward is rnnt_b200_loss_pairs_ex on its pairs;
     bf16 is f32 on the widened logits;
  5. the ranges rule of the one-symbol-per-frame types, prune_range = 1, and the simple -> ranges -> pruned pipeline;
  6. degenerate lattices, each isolated from the rest of the batch;
  7. k_frames launch shapes against their record; 8. CUDA graph capture; 9. the ValueErrors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import path_oracle as pa
from tests.test_gpu_logits import gtol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
KIND = {"regular": 0, "modified": 1, "constrained": 2}
REC_CONSTRAINED, REC_THREADS, REC_PASSES, REC_SMEM, REC_GRAD_BLOCKS, REC_DELAY = 1, 2, 3, 4, 5, 6

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


@pytest.fixture(scope="module")
def lib():
    L = ctypes.CDLL(LIB)
    P, I, F, Z = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
    L.rnnt_b200_loss_pairs_ex.restype = I
    L.rnnt_b200_loss_pairs_ex.argtypes = [P, P, Z] + [P] * 5 + [I] * 3 + [F, I, I, F]
    L.rnnt_b200_simple_smoothed_forward_ex.restype = I
    L.rnnt_b200_simple_smoothed_forward_ex.argtypes = [P, P, Z] + [P] * 8 + [I] * 6 + [F, F, I, F, P]
    L.rnnt_b200_simple_smoothed_workspace_bytes.restype = Z
    L.rnnt_b200_simple_smoothed_workspace_bytes.argtypes = [I] * 4
    L.rnnt_b200_workspace_bytes.restype = Z
    L.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, I]
    L.rnnt_b200_debug_last_launch.argtypes = [P]
    L.rnnt_b200_debug_last_frames_launch.argtypes = [P]
    return L


def record(lib, frames=False):
    rec = (ctypes.c_int32 * 32)()
    (lib.rnnt_b200_debug_last_frames_launch if frames else lib.rnnt_b200_debug_last_launch)(
        ctypes.cast(rec, ctypes.c_void_p))
    return list(rec)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(p, q):
    """bit for bit, NaN included (a lattice without a path has NaN costs and gradients in the regular classes)"""
    return p.shape == q.shape and p.dtype == q.dtype and torch.equal(p.view(torch.uint8), q.view(torch.uint8))


def make(N, T, U, V, seed, xn=None, yn=None, blank=0):
    rng = np.random.RandomState(seed)
    x = (rng.randn(N, T, U, V) * 2.0).astype(np.float32)
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    xn = rng.randint(max(1, T // 2), T + 1, N).astype(np.int32) if xn is None else np.asarray(xn, np.int32)
    if yn is None:
        yn = np.minimum(rng.randint(0, U, N), xn).astype(np.int32)        # most lattices have a modified path
    return cu(x), cu(ys), cu(xn), cu(np.asarray(yn, np.int32))


def pairs_of(x, lse, ys, blank=0):
    """the f32 pairs the forward built: (x[blank] - lse, x[label] - lse), label = blank on the last column"""
    N, T, U, _ = x.shape
    lab = torch.cat([ys, torch.full((N, 1), blank, dtype=torch.int, device="cuda")], 1).long()
    xl = x.float().gather(3, lab[:, None, :, None].expand(N, T, U, 1))[..., 0]
    return torch.stack([x.float()[..., blank] - lse, xl - lse], -1).contiguous()


def loss_pairs(lib, pairs, xn, yn, kind, lam, want=True):
    N, T, U, _ = pairs.shape
    c = torch.empty(N, device="cuda")
    pg = torch.empty((N, T, U, 2), device="cuda")
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
    st = lib.rnnt_b200_loss_pairs_ex(torch.cuda.current_stream().cuda_stream, ws.data_ptr(), ws.numel(),
                                     pairs.data_ptr(), xn.data_ptr(), yn.data_ptr(), c.data_ptr(),
                                     pg.data_ptr() if want else None, N, T, U, 0.0, 0, KIND[kind], lam)
    assert st == 0
    return c, pg


def simple_inputs(N, T, U, V, seed):
    rng = np.random.RandomState(seed)
    am = cu(rng.randn(N, T, V).astype(np.float32))
    lm = cu(rng.randn(N, U, V).astype(np.float32))
    ys = cu(rng.randint(1, V, (N, U - 1)).astype(np.int32))
    xn = rng.randint(max(1, T // 2), T + 1, N).astype(np.int32)
    yn = np.minimum(rng.randint(1, U, N), xn - 1).clip(0).astype(np.int32)
    return am, lm, ys, cu(xn), cu(yn)


# ------------------------------------------------------------------------------------------------ 1. defaults
def test_explicit_defaults_are_todays_call(w, lib):
    x, ys, xn, yn = make(5, 23, 9, 37, 0)
    for dtype in (torch.float32, torch.bfloat16):
        xs = [x.to(dtype).clone().requires_grad_(True) for _ in range(2)]
        c0 = w.rnnt_loss_from_logits(xs[0], ys, xn, yn)
        r0 = record(lib)
        c1 = w.rnnt_loss_from_logits(xs[1], ys, xn, yn, rnnt_type="regular", delay_penalty=0.0)
        r1 = record(lib)
        assert same(c0, c1) and r0[1:] == r1[1:]
        c0.sum().backward()
        c1.sum().backward()
        assert same(xs[0].grad, xs[1].grad)
    N, T, U, S = 5, 23, 9, 4
    xp = x[:, :, :S].contiguous()
    rng = torch.zeros((N, T), dtype=torch.int, device="cuda")
    a = w._C.rnnt_logits_pruned_forward(xp, ys, xn, yn, rng, 0, 0.0, True, 0)
    b = w._C.rnnt_logits_pruned_forward(xp, ys, xn, yn, rng, 0, 0.0, True, 0, 0, 0.0)
    assert all(same(p, q) for p, q in zip(a, b))
    am, lm, ys2, xn2, yn2 = simple_inputs(4, 30, 12, 40, 1)
    for sl, sa in ((0.0, 0.0), (0.25, 0.0), (0.1, 0.1)):
        a = w._C.rnnt_simple_forward(am, lm, ys2, xn2, yn2, 0, True, 3, 0, sl, sa)
        b = w._C.rnnt_simple_forward(am, lm, ys2, xn2, yn2, 0, True, 3, 0, sl, sa, 0, 0.0)
        assert all(same(p, q) for p, q in zip(a, b))
        c0, r0 = w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, prune_range=3, lm_only_scale=sl, am_only_scale=sa)
        c1, r1 = w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, prune_range=3, lm_only_scale=sl, am_only_scale=sa,
                                    rnnt_type="regular", delay_penalty=0.0)
        assert same(c0, c1) and same(r0, r1)


# ------------------------------------------------------------------------------------------------ 2. regular + penalty
@pytest.mark.parametrize("shape", [(4, 17, 6, 29), (3, 120, 40, 64)])
def test_regular_penalty_is_loss_pairs_on_penalised_pairs(w, lib, shape):
    x, ys, xn, yn = make(*shape, seed=2)
    lam = 0.05
    c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, 0, lam)
    pen = cu(pa.penalise(pairs_of(x, lse, ys).cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy(), lam))
    cr, pr = loss_pairs(lib, pen, xn, yn, "regular", 0.0)
    assert torch.equal(c, cr) and torch.equal(pg, pr)
    go = torch.linspace(0.5, 1.5, shape[0], device="cuda")
    g = w._C.rnnt_logits_backward(x, lse, pg, ys, go, 0)
    assert torch.equal(g, w._C.rnnt_logits_backward(x, lse, pr, ys, go, 0))
    # the _ex entry applies the same penalty itself
    c2, p2 = loss_pairs(lib, pairs_of(x, lse, ys), xn, yn, "regular", lam)
    assert torch.equal(c, c2) and torch.equal(pg, p2)


# ------------------------------------------------------------------------------------------------ 3. against fp64
SHAPES = [(5, 7, 5, 11), (3, 33, 17, 29), (32, 500, 100, 500), (4, 1500, 300, 50)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", ["modified", "constrained"])
@pytest.mark.parametrize("lam", [0.0, 0.05])
def test_against_the_fp64_restatement(w, lib, shape, kind, lam):
    N, T, U, V = shape
    x, ys, xn, yn = make(N, T, U, V, seed=T + U)
    c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    pairs = pairs_of(x, lse, ys).cpu().numpy()
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    c0, g0, _ = pa.lattice(pa.penalise(pairs, xh, yh, lam), xh, yh, kind)
    c = c.cpu().numpy().astype(np.float64)
    fin = np.isfinite(c0)
    assert np.array_equal(np.isinf(c), np.isinf(c0))
    np.testing.assert_allclose(c[fin], c0[fin], rtol=1e-5)
    tol = 1e-4 + max(2 * gtol(T, U), 2.0 ** -23 * np.abs(c0[fin]).max() * np.sqrt(T + U))
    np.testing.assert_allclose(pg.cpu().numpy(), g0, rtol=0, atol=tol)
    # bf16: the f32 call on the widened logits, bit for bit; the gradient rounded once
    xb = x.to(torch.bfloat16)
    cb, lb, pb = w._C.rnnt_logits_forward(xb, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    cf, lf, pf = w._C.rnnt_logits_forward(xb.float(), ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    assert torch.equal(cb, cf) and torch.equal(lb, lf) and torch.equal(pb, pf)
    go = torch.ones(N, device="cuda")
    gb = w._C.rnnt_logits_backward(xb, lb, pb, ys, go, 0)
    assert torch.equal(gb, w._C.rnnt_logits_backward(xb.float(), lf, pf, ys, go, 0).to(torch.bfloat16))


# ------------------------------------------------------------------------------------------------ 4. bit relations
@pytest.mark.parametrize("kind", ["modified", "constrained"])
@pytest.mark.parametrize("lam", [0.0, 0.05])
def test_bit_relations(w, lib, kind, lam):
    N, T, U, V = 6, 41, 13, 33
    x, ys, xn, yn = make(N, T, U, V, seed=5)
    c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    cr, pr = loss_pairs(lib, pairs_of(x, lse, ys), xn, yn, kind, lam)
    assert torch.equal(c, cr) and torch.equal(pg, pr)
    zero = torch.zeros((N, T), dtype=torch.int, device="cuda")
    cp, _, pp = w._C.rnnt_logits_pruned_forward(x, ys, xn, yn, zero, 0, 0.0, True, 0, KIND[kind], lam)
    assert torch.equal(c, cp) and torch.equal(pg, pp)
    am, lm, ys2, xn2, yn2 = simple_inputs(N, T, U, V, 6)
    cs, saved, ps, _ = w._C.rnnt_simple_forward(am, lm, ys2, xn2, yn2, 0, True, 0, 0, 0.0, 0.0, KIND[kind], lam)
    norm = saved[:N * T * U].view(N, T, U)
    lab = torch.cat([ys2, torch.zeros((N, 1), dtype=torch.int, device="cuda")], 1).long()
    al = am.gather(2, lab[:, None, :].expand(N, T, U))
    ll_ = lm.gather(2, lab[:, :, None])[..., 0][:, None, :]
    live = (torch.arange(T, device="cuda")[None, :, None] < xn2[:, None, None]) & \
           (torch.arange(U, device="cuda")[None, None, :] <= yn2[:, None, None])
    sp = torch.stack([(am[..., 0][:, :, None] + lm[..., 0][:, None, :]) - norm, (al + ll_) - norm], -1)
    sp = torch.where(live[..., None], sp, torch.zeros_like(sp)).contiguous()
    cr, pr = loss_pairs(lib, sp, xn2, yn2, kind, lam)
    assert torch.equal(cs, cr) and torch.equal(ps, pr)


# ------------------------------------------------------------------------------------------------ 5. ranges
def simple_ex(lib, am, lm, ys, xn, yn, kind, lam, sl, sa):
    N, T, V = am.shape
    U = lm.shape[1]
    c = torch.empty(N, device="cuda")
    saved = torch.empty(N * T * U + 2 * N * T + 2 * N * U + V, device="cuda")
    pg = torch.empty((N, T, U, 2), device="cuda")
    raw = torch.full((N, T, U), 7.0, device="cuda")
    ws = torch.empty(lib.rnnt_b200_simple_smoothed_workspace_bytes(N, T, U, V), dtype=torch.uint8, device="cuda")
    st = lib.rnnt_b200_simple_smoothed_forward_ex(torch.cuda.current_stream().cuda_stream, ws.data_ptr(), ws.numel(),
                                                  am.data_ptr(), lm.data_ptr(), ys.data_ptr(), xn.data_ptr(),
                                                  yn.data_ptr(), c.data_ptr(), saved.data_ptr(), pg.data_ptr(), N, T,
                                                  U, V, 0, 0, sl, sa, KIND[kind], lam, raw.data_ptr())
    assert st == 0
    return c, pg, raw


@pytest.mark.parametrize("kind", ["modified", "constrained"])
@pytest.mark.parametrize("scales", [(0.0, 0.0), (0.25, 0.0), (0.1, 0.1)])
@pytest.mark.parametrize("S", [1, 2, 5])
def test_ranges_follow_the_rule(w, lib, kind, scales, S):
    am, lm, ys, xn, yn = simple_inputs(16, 60, 20, 48, S)
    sl, sa = scales
    c, r = w.rnnt_loss_simple(am, lm, ys, xn, yn, prune_range=S, lm_only_scale=sl, am_only_scale=sa, rnnt_type=kind,
                              delay_penalty=0.01)
    c2, pg, raw = simple_ex(lib, am, lm, ys, xn, yn, kind, 0.01, sl, sa)
    assert torch.equal(c, c2)
    want = pa.prune_ranges(pg.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy(), S, kind, raw.cpu().numpy())
    assert np.array_equal(r.cpu().numpy(), want)
    if kind == "modified":
        assert torch.equal(raw, pg[..., 0])
    steps = r[:, 1:] - r[:, :-1]
    assert (r[:, 0] == 0).all() and (steps >= 0).all() and (steps <= 1).all()


@pytest.mark.parametrize("kind,S", [("modified", 1), ("modified", 4), ("constrained", 2), ("constrained", 4)])
def test_simple_ranges_pruned_pipeline(w, kind, S):
    N, T, U, V = 12, 50, 16, 24
    am, lm, ys, xn, yn = simple_inputs(N, T, U, V, 11)
    _, r = w.rnnt_loss_simple(am, lm, ys, xn, yn, prune_range=S, rnnt_type=kind)
    full = (am[:, :, None, :] + lm[:, None, :, :]).contiguous()                 # the simple joint, (N,T,U,V)
    idx = (r[:, :, None].long() + torch.arange(S, device="cuda")).clamp(max=U - 1)
    win = full.gather(2, idx[..., None].expand(N, T, S, V)).contiguous()
    cp = w.rnnt_loss_pruned(win, ys, xn, yn, r, rnnt_type=kind)
    cf = w.rnnt_loss_from_logits(full, ys, xn, yn, rnnt_type=kind)
    keep = (yn + 1 - S <= xn - 1)
    assert keep.any() and torch.isfinite(cp[keep]).all()
    assert (cp[keep] >= cf[keep] * (1 - 1e-6)).all()


# ------------------------------------------------------------------------------------------------ 6. degenerate
@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_degenerate_lattices_are_isolated(w, kind):
    N, T, U, V = 6, 9, 7, 12
    x, ys, xn, yn = make(N, T, U, V, seed=9, xn=[9, 9, 4, 9, 0, 9], yn=[3, 6, 6, 2, 2, 4])
    x[3, 2, 1, 5] = float("nan")                        # a live cell of lattice 3 (t = 2 < 9, u = 1 <= 2)
    x[1, :, :, 0] = -float("inf")                       # lattice 1: every blank removed, no path
    xg = x.clone().requires_grad_(True)
    c = w.rnnt_loss_from_logits(xg, ys, xn, yn, rnnt_type=kind, delay_penalty=0.02)
    c.sum().backward()
    assert c[2].item() == float("inf")                  # Un - 1 = 6 > Tn = 4
    assert c[1].item() == float("inf")
    assert torch.isnan(c[3]) and torch.isnan(c[4])
    assert torch.isnan(xg.grad[3, :9, :3]).all() and (xg.grad[[1, 2, 4]] == 0).all()
    keep = [0, 5]
    xk = x[keep].clone().requires_grad_(True)
    ck = w.rnnt_loss_from_logits(xk, ys[keep], xn[keep], yn[keep], rnnt_type=kind, delay_penalty=0.02)
    ck.sum().backward()
    assert torch.equal(c[keep], ck) and torch.equal(xg.grad[keep], xk.grad)


# ------------------------------------------------------------------------------------------------ 7. launch shapes
@pytest.mark.parametrize("T,U", [(1, 1), (2, 2), (5, 32), (7, 33), (40, 1024), (40, 1025), (3, 1600), (700, 3)])
def test_frames_launch_shapes(w, lib, T, U):
    N = 2
    x, ys, xn, yn = make(N, T, U, 5, seed=T * 7 + U, xn=[T, T], yn=[min(U - 1, T), max(0, min(U - 1, T) - 1)])
    for kind in ("modified", "constrained"):
        c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], 0.0)
        rec = record(lib, frames=True)
        threads = min(512, max(32, (U + 31) // 32 * 32))
        assert rec[REC_CONSTRAINED] == (kind == "constrained") and rec[REC_THREADS] == threads
        assert rec[REC_PASSES] == -(-U // threads) and rec[REC_SMEM] == 8 * U and rec[REC_GRAD_BLOCKS] > 0
        assert rec[REC_DELAY] == 0
        xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
        c0, g0, _ = pa.lattice(pairs_of(x, lse, ys).cpu().numpy(), xh, yh, kind)
        np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5)
        np.testing.assert_allclose(pg.cpu().numpy(), g0, atol=1e-4 + 2 * gtol(T, U))


def test_frames_many_waves(w, lib):
    N, T, U, V = 700, 20, 9, 6
    x, ys, xn, yn = make(N, T, U, V, seed=4)
    c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, 1, 0.03)
    assert record(lib, frames=True)[REC_DELAY] == 1
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    c0, g0, _ = pa.lattice(pa.penalise(pairs_of(x, lse, ys).cpu().numpy(), xh, yh, 0.03), xh, yh, "modified")
    np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(pg.cpu().numpy(), g0, atol=1e-4 + 2 * gtol(T, U))


# ------------------------------------------------------------------------------------------------ 8. graphs
@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_cuda_graph_capture(w, kind):
    N, T, U, V = 8, 60, 20, 32
    x, ys, xn, yn = make(N, T, U, V, seed=12)
    src = x.clone().requires_grad_(True)

    def step():
        src.grad = None
        loss = w.rnnt_loss_from_logits(src, ys, xn, yn, reduction="sum", rnnt_type=kind, delay_penalty=0.01)
        loss.backward()
        return loss

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    want = step().detach().clone()
    gwant = src.grad.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want) and torch.equal(src.grad, gwant)


# ------------------------------------------------------------------------------------------------ 9. errors
def test_value_errors(w):
    x, ys, xn, yn = make(2, 5, 4, 6, seed=1)
    am, lm, ys2, xn2, yn2 = simple_inputs(2, 5, 4, 6, 1)
    before = w._C.launch_count()
    for kw in ({"rnnt_type": "warped"}, {"rnnt_type": 1}, {"delay_penalty": -0.1}, {"delay_penalty": float("nan")},
               {"delay_penalty": float("inf")}, {"delay_penalty": True}):
        with pytest.raises(ValueError):
            w.rnnt_loss_from_logits(x, ys, xn, yn, **kw)
        with pytest.raises(ValueError):
            w.rnnt_loss_pruned(x[:, :, :2].contiguous(), ys, xn, yn, torch.zeros_like(x[..., 0, 0], dtype=torch.int),
                               **kw)
        with pytest.raises(ValueError):
            w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, **kw)
    for kind in ("modified", "constrained"):
        with pytest.raises(ValueError, match="fastemit_lambda"):
            w.rnnt_loss_from_logits(x, ys, xn, yn, fastemit_lambda=0.01, rnnt_type=kind)
        with pytest.raises(ValueError, match="fastemit_lambda"):
            w.rnnt_loss_pruned(x, ys, xn, yn, torch.zeros((2, 5), dtype=torch.int, device="cuda"),
                               fastemit_lambda=0.01, rnnt_type=kind)
        with pytest.raises(ValueError, match="compact"):
            w.rnnt_loss_from_logits(x.view(-1, 6), ys, xn, yn, compact=True, rnnt_type=kind)
    with pytest.raises(ValueError, match="compact"):
        w.rnnt_loss_from_logits(x.view(-1, 6), ys, xn, yn, compact=True, delay_penalty=0.1)
    with pytest.raises(ValueError, match=">= 2"):
        w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, prune_range=1)
    with pytest.raises(ValueError, match=">= 1"):
        w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, prune_range=0, rnnt_type="modified")
    assert w._C.launch_count() == before
    # regular + penalty + FastEmit compose
    c = w.rnnt_loss_from_logits(x, ys, xn, yn, fastemit_lambda=0.01, delay_penalty=0.1)
    assert torch.isfinite(c).all()
