"""rnnt_loss_simple: the transducer loss of the factorised joint am[n,t] + lm[n,u], and its prune ranges.

The contract (include/rnnt_b200.h, DESIGN.md 3.6):
  1. costs, d am and d lm agree with the fp64 restatement (tests/simple_oracle.py): costs to 1e-5 relative, each
     gradient element to the per-cell bound of the logit gradients times the occupation it sums (check()), on the fused
     kernel and on the general path (the launch record names the path), across reductions, average_frames and
     blank != 0;
  2. the pairs rebuilt in torch from the saved normaliser with the documented formula give, through
     rnnt_b200_loss_pairs, the same costs and pair gradients bit for bit; the ranges equal the float32 restatement of
     the rule applied to the GPU's own pair gradients;
  3. the windows feed rnnt_loss_pruned: every lattice keeps a finite cost no lower than the full one, and with S >= U
     the pruned cost is the full cost;
  4. two calls give the same bits;
  5. masked vocabulary entries, NaN rows, invalid lengths, N = 0, forward only, CUDA graphs and argument errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import simple_oracle as so
from tests.test_gpu_logits import gtol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
EXACT, FAST = 1, 2
REC_PATH = 1                                          # rnntLaunchRecord_t: 1 fused, 2 general
INVALID, TOO_SMALL = 5, 6

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _abi():
    lib = ctypes.CDLL(LIB)
    P, I, Z = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.rnnt_b200_simple_workspace_bytes.restype = Z
    lib.rnnt_b200_simple_workspace_bytes.argtypes = [I, I, I]
    lib.rnnt_b200_simple_forward.restype = I
    lib.rnnt_b200_simple_forward.argtypes = [P, P, Z] + [P] * 8 + [I] * 6
    lib.rnnt_b200_simple_backward.restype = I
    lib.rnnt_b200_simple_backward.argtypes = [P] * 11 + [I] * 5
    lib.rnnt_b200_prune_ranges.restype = I
    lib.rnnt_b200_prune_ranges.argtypes = [P] * 4 + [I] * 4 + [P]
    lib.rnnt_b200_loss_pairs.restype = I
    lib.rnnt_b200_loss_pairs.argtypes = [P, P, Z] + [P] * 5 + [I] * 3 + [ctypes.c_float, I]
    lib.rnnt_b200_workspace_bytes.restype = Z
    lib.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, I]
    lib.rnnt_b200_debug_last_launch.argtypes = [P]
    return lib


def last_path(lib):
    rec = (ctypes.c_int32 * 32)()
    lib.rnnt_b200_debug_last_launch(ctypes.cast(rec, ctypes.c_void_p))
    return rec[REC_PATH]


def make(N, T, U, V, seed, blank=0, scale=1.5):
    """am (N,T,V), lm (N,U,V) float32; labels never blank (V > 1); ragged lengths with Tn >= Un (lattice 0 full)."""
    rng = np.random.RandomState(seed)
    am = (rng.randn(N, T, V) * scale).astype(np.float32)
    lm = (rng.randn(N, U, V) * scale).astype(np.float32)
    if V > 1:
        ys = rng.randint(0, V - 1, (N, U - 1)).astype(np.int32)
        ys = np.where(ys >= blank, ys + 1, ys).astype(np.int32)
    else:
        ys = np.zeros((N, U - 1), np.int32)
    xn = rng.randint(max(T // 2, 1), T + 1, (N,)).astype(np.int32)
    yn = rng.randint(0, U, (N,)).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    return am, lm, ys, xn, yn


def simple_ref(am, lm, ys, xn, yn, blank, go):
    """The full-joint fp64 restatement -> (costs, d am, d lm, pair gradients) as check() takes them."""
    c0, dam0, dlm0 = so.simple(am, lm, ys, xn, yn, blank, grad_output=go)
    x = np.asarray(am, np.float64)[:, :, None] + np.asarray(lm, np.float64)[:, None]
    m = x.max(axis=-1, keepdims=True)
    lp = x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))
    return c0, dam0, dlm0, so.pair_grads_of(lp, ys, xn, yn, blank)


def bounds(c0, pg0, go):
    """-> (cell, occ, ta, tl): the per-cell bound of tests/test_gpu_pruned_paths.py,
    cell = 1e-4 + max(2 gtol(T,U), 2^-23 max|cost| sqrt(T+U)), the occupation occ (N,T,U) = |gb| + |gl| of the
    reference's pair gradients pg0, and the bounds of d am and d lm: cell times the occupation each element sums.  A
    d am row sums the cells of its frame, a d lm row those of its column (up to Tn / Un frames' worth), and the
    recurrence's fp32 error of each cell's occupation adds up along them."""
    N, T, U, _ = pg0.shape
    occ = np.abs(pg0).sum(axis=3)
    cell = 1e-4 + max(2 * gtol(T, U), 2.0 ** -23 * np.nanmax(np.abs(c0)) * np.sqrt(T + U))
    g = np.abs(np.asarray(go, np.float64)).reshape(N, 1, 1)
    ta = cell * g * np.maximum(1.0, occ.sum(axis=2))[:, :, None]
    tl = cell * g * np.maximum(1.0, occ.sum(axis=1))[:, :, None]
    return cell, occ, ta, tl


def compare(c, dam, dlm, ref, ta, tl):
    """costs to 1e-5 relative, d am and d lm elementwise within ta, tl -> (largest relative cost error, the gradient
    error and bound at the element nearest its bound, their ratio)."""
    c0, dam0, dlm0 = ref[:3]
    np.testing.assert_allclose(c, c0, rtol=1e-5)
    cost_rel = np.nanmax(np.abs(c - c0)) / np.nanmax(np.abs(c0))
    worst = (0.0, 0.0, 1.0)
    for name, got, want, tol in (("d am", dam, dam0, ta), ("d lm", dlm, dlm0, tl)):
        err, tol = np.abs(got - want), np.broadcast_to(tol, got.shape)
        assert (err <= tol).all(), (name, err.max(), np.unravel_index(np.argmax(err - tol), err.shape))
        i = np.unravel_index(np.argmax(err / tol), err.shape)
        if err[i] / tol[i] > worst[0]:
            worst = (err[i] / tol[i], err[i], tol[i])
    return cost_rel, worst[1], worst[2], worst[0]


def check(c, dam, dlm, ref, go):
    """c, dam, dlm against the reference's (costs, d am, d lm, pair gradients) ref: compare() within bounds()."""
    _, _, ta, tl = bounds(ref[0], ref[3], go)
    return compare(c, dam, dlm, ref, ta, tl)


SHAPES = [  # N, T, U, V, blank, path
    (3, 12, 7, 5, 0, 1),
    (2, 33, 34, 28, 3, 1),
    (3, 40, 20, 300, 7, 1),
    (2, 16, 5, 1024, 0, 1),
    (3, 20, 1, 1, 0, 1),              # V = 1: no labels
    (2, 31, 18, 7, 2, 1),
    (2, 150, 140, 16, 0, 2),          # general path (U > 128)
    (2, 220, 200, 33, 1, 2),
]


@pytest.mark.parametrize("mode", [EXACT, FAST])
@pytest.mark.parametrize("shape", SHAPES)
def test_vs_oracle(w, shape, mode):
    """1: costs, d am, d lm against fp64, per-lattice grad_output; the launch record names the recurrence path."""
    lib = _abi()
    N, T, U, V, blank, path = shape
    am, lm, ys, xn, yn = make(N, T, U, V, seed=T + U + V, blank=blank)
    go = np.linspace(0.5, 1.5, N)
    w.set_lse_mode({EXACT: "exact", FAST: "fast"}[mode])
    try:
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), blank=blank)
        assert last_path(lib) == path
        (c * cu(go.astype(np.float32))).sum().backward()
    finally:
        w.set_lse_mode("auto")
    ref = simple_ref(am, lm, ys, xn, yn, blank, go)
    check(c.detach().cpu().numpy(), a.grad.cpu().numpy(), l.grad.cpu().numpy(), ref, go)


@pytest.mark.parametrize("average_frames", [False, True])
@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
@pytest.mark.parametrize("shape", [(3, 24, 11, 40, 5, 1), (2, 150, 140, 12, 3, 2)])
def test_reductions(w, shape, reduction, average_frames):
    N, T, U, V, blank, _ = shape
    am, lm, ys, xn, yn = make(N, T, U, V, seed=7 + V, blank=blank)
    a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
    out = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), average_frames=average_frames, reduction=reduction,
                             blank=blank)
    wts = np.ones(N) / (xn if average_frames else 1.0)
    if reduction == "mean":
        wts = wts / N
    if reduction == "none":
        assert out.shape == (N,)
        wts = wts * np.linspace(1.0, 2.0, N)
        out = (out * cu(np.linspace(1.0, 2.0, N).astype(np.float32))).sum()
    out.backward()
    ref = simple_ref(am, lm, ys, xn, yn, blank, wts)
    np.testing.assert_allclose(out.item(), (ref[0] * wts).sum(), rtol=1e-5)
    check(ref[0], a.grad.cpu().numpy(), l.grad.cpu().numpy(), ref, wts)


def rebuilt_pairs(am, lm, ys, xn, yn, norm, blank):
    """The documented pair formula in torch: ((am[blank] + lm[blank]) - norm, (am[y] + lm[y]) - norm) at the lattice's
    cells, (0, 0) elsewhere."""
    N, T, V = am.shape
    U = lm.shape[1]
    uu = torch.arange(U, device="cuda")
    y = torch.full((N, U), blank, dtype=torch.long, device="cuda")
    y[:, :U - 1] = torch.where(uu[None, :U - 1] < yn[:, None].long(), ys.long(), blank)
    am_y = am.gather(2, y[:, None, :].expand(N, T, U))
    lm_y = lm.gather(2, y[:, :, None])[:, :, 0]
    pb = (am[:, :, blank][:, :, None] + lm[:, :, blank][:, None, :]) - norm
    pl = (am_y + lm_y[:, None, :]) - norm
    live = (torch.arange(T, device="cuda")[None, :, None] < xn[:, None, None]) & (uu[None, None, :] <= yn[:, None, None])
    p = torch.stack([pb, pl], dim=-1)
    return torch.where(live[..., None], p, torch.zeros_like(p)).contiguous()


@pytest.mark.parametrize("shape", [(3, 30, 20, 28, 0, 1), (2, 40, 9, 301, 4, 1), (2, 150, 140, 16, 2, 2)])
def test_bit_parity(w, shape):
    """2: the recurrence sees exactly the documented pairs; the ranges are the rule on the GPU's pair gradients."""
    lib = _abi()
    N, T, U, V, blank, _ = shape
    am, lm, ys, xn, yn = make(N, T, U, V, seed=3 * T + V, blank=blank)
    at, lt, yt, xt, nt = cu(am), cu(lm), cu(ys), cu(xn), cu(yn)
    stream = torch.cuda.current_stream().cuda_stream
    for mode in (EXACT, FAST):
        S = 4
        c, saved, pg, r = w._C.rnnt_simple_forward(at, lt, yt, xt, nt, blank, True, S, mode)
        norm = saved[:N * T * U].view(N, T, U)
        pairs = rebuilt_pairs(at, lt, yt, xt, nt, norm, blank)
        c2 = torch.empty(N, device="cuda")
        pg2 = torch.empty((N, T, U, 2), device="cuda")
        ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
        assert lib.rnnt_b200_loss_pairs(stream, ws.data_ptr(), ws.numel(), pairs.data_ptr(), xt.data_ptr(),
                                        nt.data_ptr(), c2.data_ptr(), pg2.data_ptr(), N, T, U, 0.0, mode) == 0
        torch.cuda.synchronize()
        assert torch.isfinite(c).all()
        assert torch.equal(c, c2) and torch.equal(pg, pg2)
        want = so.prune_ranges(pg.cpu().numpy(), xn, yn, S)
        np.testing.assert_array_equal(r.cpu().numpy(), want)
        so.check_ranges(want, xn, yn, S, U)


@pytest.mark.parametrize("S", [2, 5])
@pytest.mark.parametrize("shape", [(3, 40, 20, 30, 0), (2, 200, 140, 12, 1)])
def test_ranges_feed_the_pruned_loss(w, shape, S):
    """3: the windows keep a path in every lattice; pruning removes paths, so the cost does not go down."""
    N, T, U, V, blank = shape
    am, lm, ys, xn, yn = make(N, T, U, V, seed=11 + S, blank=blank)
    xn = np.maximum(xn, yn + 1)                          # Tn >= Un: every lattice reachable by windows of S >= 2
    at, lt, args = cu(am), cu(lm), (cu(ys), cu(xn), cu(yn))
    _, ranges = w.rnnt_loss_simple(at, lt, *args, blank=blank, prune_range=S)
    x = (at[:, :, None] + lt[:, None]).contiguous()      # the simple joint's full logits, for the check only
    idx = (ranges.long()[:, :, None] + torch.arange(S, device="cuda")).clamp(max=U - 1)
    xw = x.gather(2, idx[..., None].expand(N, T, S, V)).contiguous()
    pruned = w.rnnt_loss_pruned(xw, *args, ranges, blank=blank)
    full = w.rnnt_loss_from_logits(x, *args, blank=blank)
    assert torch.isfinite(pruned).all()
    assert (pruned >= full - 1e-5 * full.abs()).all(), (pruned, full)
    # S >= U: one window covers the lattice (ranges 0) and the pruned loss is the full loss
    _, r_all = w.rnnt_loss_simple(at, lt, *args, blank=blank, prune_range=U)
    assert (r_all == 0).all()
    xa = x[:, :, :U].contiguous()
    np.testing.assert_allclose(w.rnnt_loss_pruned(xa, *args, r_all, blank=blank).cpu().numpy(), full.cpu().numpy(),
                               rtol=1e-5)


def test_deterministic(w):
    """4: two calls, same bits (costs, gradients, ranges)."""
    N, T, U, V = 4, 150, 140, 64
    am, lm, ys, xn, yn = make(N, T, U, V, seed=5)
    outs = []
    for _ in range(2):
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c, r = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), prune_range=5)
        c.sum().backward()
        outs.append((c.detach(), r, a.grad, l.grad))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


def test_masked_vocabulary(w):
    """5: -inf on every vocabulary entry that is neither blank nor one of the lattice's labels."""
    N, T, U, V = 3, 20, 8, 40
    am, lm, ys, xn, yn = make(N, T, U, V, seed=9)
    for n in range(N):
        keep = np.zeros(V, bool)
        keep[0] = True
        keep[ys[n]] = True
        am[n, :, ~keep] = -np.inf
        lm[n, 1::2, ~keep] = -np.inf
    a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
    c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn))
    c.sum().backward()
    check(c.detach().cpu().numpy(), a.grad.cpu().numpy(), l.grad.cpu().numpy(),
          simple_ref(am, lm, ys, xn, yn, 0, np.ones(N)), np.ones(N))


@pytest.mark.parametrize("shape", [(4, 30, 20, 28), (4, 150, 140, 16)])
def test_nan_rows_and_invalid_lengths(w, shape):
    """5: a NaN in a live row makes its lattice's cost NaN, a NaN in a padding row changes nothing; invalid lengths give
    cost NaN, zero gradient rows and ranges 0; the other lattices keep their bits."""
    N, T, U, V = shape
    am, lm, ys, xn, yn = make(N, T, U, V, seed=N + T)
    xn[1], xn[2], yn[3] = T - 2, T + 1, min(int(yn[3]), U - 2)
    S = 3

    def run(am, lm, xn, yn):
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c, r = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), prune_range=S)
        torch.nan_to_num(c, nan=0.0, posinf=0.0).sum().backward()
        return c.detach().cpu().numpy(), r.cpu().numpy(), a.grad.cpu().numpy(), l.grad.cpu().numpy()

    c0, r0, da0, dl0 = run(am, lm, xn, yn)
    assert np.isnan(c0[2]) and (da0[2] == 0).all() and (dl0[2] == 0).all() and (r0[2] == 0).all()
    am2, lm2 = am.copy(), lm.copy()
    am2[0, 3, 5] = np.nan                       # live row of lattice 0
    am2[1, T - 1, :] = np.nan                   # padding frame of lattice 1
    lm2[3, U - 1, :] = np.nan                   # padding column of lattice 3
    c1, r1, da1, dl1 = run(am2, lm2, xn, yn)
    assert np.isnan(c1[0]) and np.isnan(c0[2])
    for n in range(1, N):
        assert np.array_equal(c1[n], c0[n], equal_nan=True) and np.array_equal(r1[n], r0[n])
        assert np.array_equal(da1[n], da0[n]) and np.array_equal(dl1[n], dl0[n])


def test_forward_only_and_empty(w):
    N, T, U, V = 3, 30, 12, 20
    am, lm, ys, xn, yn = make(N, T, U, V, seed=4)
    args = (cu(ys), cu(xn), cu(yn))
    a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
    c, r = w.rnnt_loss_simple(a, l, *args, prune_range=4)
    with torch.no_grad():
        c2 = w.rnnt_loss_simple(cu(am), cu(lm), *args)
        c3, r3 = w.rnnt_loss_simple(cu(am), cu(lm), *args, prune_range=4)
    assert not c2.requires_grad and torch.equal(c.detach(), c2) and torch.equal(c2, c3) and torch.equal(r, r3)
    assert r.dtype == torch.int32 and r.shape == (N, T) and not r.requires_grad
    # only lm needs a gradient: the same d lm
    c.sum().backward()
    l2 = cu(lm).requires_grad_(True)
    w.rnnt_loss_simple(cu(am), l2, *args).sum().backward()
    assert torch.equal(l2.grad, l.grad)
    # N = 0
    e = torch.empty((0, T, V), device="cuda", requires_grad=True)
    f = torch.empty((0, U, V), device="cuda", requires_grad=True)
    z = torch.empty((0,), dtype=torch.int, device="cuda")
    c0, r0 = w.rnnt_loss_simple(e, f, torch.empty((0, U - 1), dtype=torch.int, device="cuda"), z, z, prune_range=3)
    c0.sum().backward()
    assert c0.shape == (0,) and r0.shape == (0, T) and e.grad.shape == (0, T, V) and f.grad.shape == (0, U, V)


def test_cuda_graph_replay(w):
    """No host sync: a captured forward (with ranges) + backward replays to eager's bits on new inputs."""
    N, T, U, V = 4, 60, 30, 48
    srcs = [make(N, T, U, V, seed=s) for s in (21, 22)]
    ys, xn, yn = (cu(x) for x in srcs[0][2:])
    a, l = cu(srcs[0][0]), cu(srcs[0][1])
    go = torch.linspace(0.5, 1.5, N, device="cuda")

    def step():
        c, saved, pg, r = w._C.rnnt_simple_forward(a, l, ys, xn, yn, 0, True, 5, 0)
        dam, dlm = w._C.rnnt_simple_backward(a, l, ys, xn, yn, saved, pg, go, 0)
        return c, r, dam, dlm

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for am, lm, *_ in srcs:
        a.copy_(cu(am))
        l.copy_(cu(lm))
        graph.replay()
        torch.cuda.synchronize()
        want = step()
        for x, y in zip(outs, want):
            assert torch.equal(x, y)


def test_errors(w):
    N, T, U, V = 2, 10, 5, 8
    am, lm, ys, xn, yn = make(N, T, U, V, seed=1)
    a, l, args = cu(am), cu(lm), (cu(ys), cu(xn), cu(yn))
    with pytest.raises(TypeError, match="float32"):
        w.rnnt_loss_simple(a.bfloat16(), l.bfloat16(), *args)
    with pytest.raises(TypeError, match="float32"):
        w.rnnt_loss_simple(a, l.bfloat16(), *args)
    for bad in (1, 0, -3, 2.0, True):
        with pytest.raises(ValueError, match="prune_range"):
            w.rnnt_loss_simple(a, l, *args, prune_range=bad)
    with pytest.raises(RuntimeError, match="blank"):
        w.rnnt_loss_simple(a, l, *args, blank=V)
    with pytest.raises(RuntimeError, match="float32"):
        w._C.rnnt_simple_forward(a.bfloat16(), l.bfloat16(), *args)
    with pytest.raises(RuntimeError, match="ys"):
        w.rnnt_loss_simple(a, l[:, :U - 1].contiguous(), *args)
    with pytest.raises(RuntimeError, match="am must be"):
        w.rnnt_loss_simple(a, l[:, :, :V - 1].contiguous(), *args)
    with pytest.raises(RuntimeError, match="prune_range"):
        w._C.rnnt_prune_ranges(torch.zeros((N, T, U, 2), device="cuda"), args[1], args[2], 1)


def test_cabi_status(w):
    lib = _abi()
    N, T, U, V = 2, 10, 5, 8
    am, lm, ys, xn, yn = make(N, T, U, V, seed=2)
    a, l, y, x, n = cu(am), cu(lm), cu(ys), cu(xn), cu(yn)
    s = torch.cuda.current_stream().cuda_stream
    nbytes = lib.rnnt_b200_simple_workspace_bytes(N, T, U)
    assert nbytes == lib.rnnt_b200_workspace_bytes(N * T * U, N)
    ws = torch.empty(nbytes + 16, dtype=torch.uint8, device="cuda")
    c = torch.empty(N, device="cuda")
    saved = torch.empty(N * T * U + N * T + N * U, device="cuda")
    pg = torch.empty((N, T, U, 2), device="cuda")
    dam, dlm = torch.empty_like(a), torch.empty_like(l)
    r = torch.empty((N, T), dtype=torch.int, device="cuda")
    P = [p.data_ptr() for p in (a, l, y, x, n, c, saved, pg)]

    def fwd(ws_ptr=ws.data_ptr(), nb=nbytes, ptrs=P, Vv=V, blank=0, NN=N):
        return lib.rnnt_b200_simple_forward(s, ws_ptr, nb, *ptrs, NN, T, U, Vv, blank, 0)

    assert fwd() == 0
    assert fwd(nb=nbytes - 1) == TOO_SMALL
    assert fwd(ws_ptr=ws.data_ptr() + 4) == INVALID                         # workspace not 8-byte aligned
    assert fwd(ws_ptr=None, nb=0) == TOO_SMALL
    assert fwd(Vv=0) == INVALID and fwd(blank=V) == INVALID and fwd(NN=-1) == INVALID and fwd(NN=65536) == INVALID
    assert fwd(ptrs=P[:6] + [None] + P[7:]) == INVALID                      # no saved buffer
    assert fwd(ptrs=P[:7] + [pg.data_ptr() + 4]) == INVALID                 # pair_grads not 8-byte aligned
    assert fwd(ptrs=P[:7] + [None]) == 0                                    # costs only
    assert fwd(NN=0) == 0

    def bwd(pgp=pg.data_ptr(), d1=dam.data_ptr(), Uu=U):
        return lib.rnnt_b200_simple_backward(s, a.data_ptr(), l.data_ptr(), y.data_ptr(), x.data_ptr(), n.data_ptr(),
                                             saved.data_ptr(), pgp, None, d1, dlm.data_ptr(), N, T, Uu, V, 0)

    assert fwd() == 0 and bwd() == 0
    assert bwd(pgp=None) == INVALID and bwd(pgp=pg.data_ptr() + 4) == INVALID and bwd(d1=None) == INVALID
    assert bwd(Uu=0) == INVALID

    def rng_(S=3, pgp=pg.data_ptr(), rp=r.data_ptr()):
        return lib.rnnt_b200_prune_ranges(s, pgp, x.data_ptr(), n.data_ptr(), N, T, U, S, rp)

    assert rng_() == 0 and rng_(S=1) == INVALID and rng_(pgp=None) == INVALID and rng_(rp=None) == INVALID
    torch.cuda.synchronize()
    so.check_ranges(r.cpu().numpy(), xn, yn, 3, U)
