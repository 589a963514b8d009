"""rnnt_loss_simple with k2's smoothing: lm_only_scale sl, am_only_scale sa (include/rnnt_b200.h, DESIGN.md 3.6).

  1. zero scales are the plain simple loss: the same bits and the same launches;
  2. costs, d am and d lm agree with the fp64 restatement (tests/smoothed_oracle.py) on the fused and the general
     path, both LSE modes, four scale pairs, per-lattice grad_output, the reductions and average_frames; the gradient
     bound is test_gpu_simple.check's plus a bound on the unigram term, and the test shows that the unigram term is
     larger than the bound somewhere, so that a backward without it fails;
  3. pairs rebuilt in torch from the saved norm, Ll, Am and log uni give the same costs and pair gradients through
     rnnt_b200_loss_pairs bit for bit; the ranges are the rule on those pair gradients and feed rnnt_loss_pruned;
  4. two calls give the same bits where the unigram and G reductions span several CTAs and V % 32 != 0;
  5. the unigram couples the batch exactly when sa > 0 (padding rows, their gradient, NaN);
  6. masked vocabulary, N = 0, forward only, CUDA graphs, bad scales and small workspaces."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import simple_oracle as so
from tests import smoothed_oracle as sm
from tests.test_gpu_simple import (EXACT, FAST, INVALID, SHAPES, TOO_SMALL, _abi, bounds, compare, cu, last_path, make,
                                   rebuilt_pairs)

pytestmark = pytest.mark.gpu

SCALES = [(0.25, 0.0), (0.0, 0.3), (0.1, 0.1), (0.5, 0.45)]


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def abi():
    lib = _abi()
    P, I, Z, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_float
    lib.rnnt_b200_simple_smoothed_workspace_bytes.restype = Z
    lib.rnnt_b200_simple_smoothed_workspace_bytes.argtypes = [I] * 4
    lib.rnnt_b200_simple_smoothed_forward.restype = I
    lib.rnnt_b200_simple_smoothed_forward.argtypes = [P, P, Z] + [P] * 8 + [I] * 6 + [F, F]
    lib.rnnt_b200_simple_smoothed_backward.restype = I
    lib.rnnt_b200_simple_smoothed_backward.argtypes = [P, P, Z] + [P] * 10 + [I] * 5 + [F, F]
    lib.rnnt_b200_launch_count.restype = ctypes.c_uint64
    return lib


def f32(x):
    return float(np.float32(x))


def c_of(sl, sa):
    """c as the host computes it: 1 - sl - sa in double from the float32 scales, rounded to float32 once."""
    return f32(1.0 - f32(sl) - f32(sa))


def saved_len(N, T, U, V, smooth):
    base = N * T * U + N * T + N * U
    return base + N * U + N * T + V if smooth else base


_oracle_cache = {}


def oracle(am, lm, ys, xn, yn, blank, sl, sa, go):
    key = (am.tobytes(), lm.tobytes(), xn.tobytes(), yn.tobytes(), blank, sl, sa, np.asarray(go).tobytes())
    if key not in _oracle_cache:
        c0, da0, dl0, pg0 = sm.smoothed(am, lm, ys, xn, yn, blank, sl, sa, grad_output=go, want_pairs=True)
        du = None
        if sa > 0:
            du = dl0 - sm.smoothed(am, lm, ys, xn, yn, blank, sl, sa, grad_output=go, detach_unigram=True)[2]
        _oracle_cache[key] = (c0, da0, dl0, pg0, du)
    return _oracle_cache[key]


def check(c, dam, dlm, ref, lm, go, sa):
    """c, dam, dlm against the reference's (costs, d am, d lm, pair gradients, unigram term of d lm or None) ref.
    costs to 1e-5 relative.  d am and the c and sl parts of d lm: test_gpu_simple.bounds, the per-cell bound times
    the occupation each element sums (now the smoothed lattice's).  The unigram term of d lm, (1/(N U)) p (G - p.G),
    adds the error of G: G[v] sums go_n times occupations over the whole batch, each divided by uni[v] or weighted by
    exp(am - Am) <= 1/uni[v], so |dG[v]| <= 2 sa cell sum_n |go_n| (sum_{t,u} occ_n) / uni[v].  -> compare()'s
    (cost_rel, grad_err, bound, ratio)."""
    N, U, V = lm.shape
    du = ref[4]
    cell, occ, ta, tl = bounds(ref[0], ref[3], go)
    if sa > 0:
        g = np.abs(np.asarray(go, np.float64))
        l64 = np.asarray(lm, np.float64)
        p = np.exp(l64 - l64.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        uni = p.mean(axis=(0, 1)) + sm.FLT_MIN
        dG = 2 * sa * cell * (g * occ.sum(axis=(1, 2))).sum() / uni
        tu = p * (dG + (p * dG).sum(-1, keepdims=True)) / (N * U)
        tl = tl + tu
        # the unigram term is larger than the whole bound somewhere: a backward without it would fail (with V = 1 the
        # term is identically 0)
        assert V == 1 or (np.abs(du) > tl).any(), (np.abs(du).max(), tl.max())
    return compare(c, dam, dlm, ref, ta, tl)


def test_zero_scales_are_the_simple_loss(w):
    """1: explicit zero scales give the plain call's costs, ranges and gradients bit for bit, with the same launches."""
    lib = abi()
    for shape in ((3, 30, 20, 28), (2, 150, 140, 16)):
        am, lm, ys, xn, yn = make(*shape, seed=sum(shape))
        outs, launches = [], []
        for kw in ({}, {"lm_only_scale": 0.0, "am_only_scale": 0.0}):
            a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
            torch.cuda.synchronize()
            n0 = lib.rnnt_b200_launch_count()
            c, r = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), prune_range=4, **kw)
            (c * torch.linspace(0.5, 1.5, len(c), device="cuda")).sum().backward()
            torch.cuda.synchronize()
            launches.append(lib.rnnt_b200_launch_count() - n0)
            outs.append((c.detach(), r, a.grad, l.grad))
        assert launches[0] == launches[1]
        for x, y in zip(*outs):
            assert torch.equal(x, y)


@pytest.mark.parametrize("scales", SCALES)
@pytest.mark.parametrize("mode", [EXACT, FAST])
@pytest.mark.parametrize("shape", SHAPES)
def test_vs_oracle(w, shape, mode, scales):
    """2: costs, d am, d lm against fp64 with a per-lattice grad_output; the launch record names the path."""
    lib = _abi()
    N, T, U, V, blank, path = shape
    sl, sa = scales
    am, lm, ys, xn, yn = make(N, T, U, V, seed=T + U + V, blank=blank)
    go = np.linspace(0.5, 1.5, N)
    w.set_lse_mode({EXACT: "exact", FAST: "fast"}[mode])
    try:
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), blank=blank, lm_only_scale=sl, am_only_scale=sa)
        assert last_path(lib) == path
        (c * cu(go.astype(np.float32))).sum().backward()
    finally:
        w.set_lse_mode("auto")
    check(c.detach().cpu().numpy(), a.grad.cpu().numpy(), l.grad.cpu().numpy(),
          oracle(am, lm, ys, xn, yn, blank, sl, sa, go), lm, go, sa)


@pytest.mark.parametrize("average_frames", [False, True])
@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
@pytest.mark.parametrize("shape", [(3, 24, 11, 40, 5, 1), (2, 150, 140, 12, 3, 2)])
def test_reductions(w, shape, reduction, average_frames):
    N, T, U, V, blank, _ = shape
    sl, sa = 0.1, 0.1
    am, lm, ys, xn, yn = make(N, T, U, V, seed=7 + V, blank=blank)
    a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
    out = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), average_frames=average_frames, reduction=reduction,
                             blank=blank, lm_only_scale=sl, am_only_scale=sa)
    wts = np.ones(N) / (xn if average_frames else 1.0)
    if reduction == "mean":
        wts = wts / N
    if reduction == "none":
        assert out.shape == (N,)
        wts = wts * np.linspace(1.0, 2.0, N)
        out = (out * cu(np.linspace(1.0, 2.0, N).astype(np.float32))).sum()
    out.backward()
    ref = oracle(am, lm, ys, xn, yn, blank, sl, sa, wts)
    np.testing.assert_allclose(out.item(), (ref[0] * wts).sum(), rtol=1e-5)
    check(ref[0], a.grad.cpu().numpy(), l.grad.cpu().numpy(), ref, lm, wts, sa)


def rebuilt_smoothed_pairs(at, lt, yt, xt, nt, saved, blank, sl, sa):
    """The header's pair formula in torch float32, one rounded operation at a time, from the saved buffer."""
    N, T, V = at.shape
    U = lt.shape[1]
    norm = saved[:N * T * U].view(N, T, U)
    off = N * T * U + N * T + N * U
    Ll = saved[off:off + N * U].view(N, U)
    Am = saved[off + N * U:off + N * U + N * T].view(N, T)
    lu = saved[off + N * U + N * T:]
    simple = rebuilt_pairs(at, lt, yt, xt, nt, norm, blank)
    uu = torch.arange(U, device="cuda")
    y = torch.full((N, U), blank, dtype=torch.long, device="cuda")
    y[:, :U - 1] = torch.where(uu[None, :U - 1] < nt[:, None].long(), yt.long(), blank)
    scalar = lambda x: torch.tensor(x, dtype=torch.float32, device="cuda")       # noqa: E731
    c, s_l, s_a = scalar(c_of(sl, sa)), scalar(sl), scalar(sa)
    out = []
    for j, k in enumerate((torch.full_like(y, blank), y)):
        am_k = at.gather(2, k[:, None, :].expand(N, T, U))
        lm_k = lt.gather(2, k[:, :, None])[:, :, 0]
        p = c * simple[..., j]
        if sl > 0:
            p = p + s_l * (lm_k - Ll)[:, None, :]
        if sa > 0:
            p = p + s_a * ((am_k + lu[k][:, None, :]) - Am[:, :, None])
        out.append(p)
    live = (torch.arange(T, device="cuda")[None, :, None] < xt[:, None, None]) & (uu[None, None, :] <= nt[:, None, None])
    p = torch.stack(out, dim=-1)
    return torch.where(live[..., None], p, torch.zeros_like(p)).contiguous()


@pytest.mark.parametrize("scales", SCALES)
@pytest.mark.parametrize("shape", [(3, 30, 20, 28, 0, 1), (2, 40, 9, 301, 4, 1), (2, 150, 140, 16, 2, 2)])
def test_bit_parity(w, shape, scales):
    """3: the recurrence sees exactly the documented pairs; the ranges are the rule on the GPU's pair gradients and
    feed the pruned loss."""
    lib = _abi()
    N, T, U, V, blank, _ = shape
    sl, sa = scales
    am, lm, ys, xn, yn = make(N, T, U, V, seed=3 * T + V, blank=blank)
    xn = np.maximum(xn, yn + 1)                          # Tn >= Un: windows of S >= 2 reach every lattice's end
    at, lt, yt, xt, nt = cu(am), cu(lm), cu(ys), cu(xn), cu(yn)
    stream = torch.cuda.current_stream().cuda_stream
    S = 4
    for mode in (EXACT, FAST):
        c, saved, pg, r = w._C.rnnt_simple_forward(at, lt, yt, xt, nt, blank, True, S, mode, sl, sa)
        assert saved.numel() == saved_len(N, T, U, V, True)
        pairs = rebuilt_smoothed_pairs(at, lt, yt, xt, nt, saved, blank, sl, sa)
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
    x = (at[:, :, None] + lt[:, None]).contiguous()      # the simple joint's full logits, for the check only
    idx = (r.long()[:, :, None] + torch.arange(S, device="cuda")).clamp(max=U - 1)
    xw = x.gather(2, idx[..., None].expand(N, T, S, V)).contiguous()
    assert torch.isfinite(w.rnnt_loss_pruned(xw, yt, xt, nt, r, blank=blank)).all()


def test_deterministic(w):
    """4: N*U = 1120 lm rows (35 unigram partials), N*T = 480 am rows (15 G partials), V = 1030 (5 CTAs of G)."""
    N, T, U, V = 8, 60, 140, 1030
    am, lm, ys, xn, yn = make(N, T, U, V, seed=5)
    outs = []
    for _ in range(2):
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c, r = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), prune_range=5, lm_only_scale=0.1, am_only_scale=0.1)
        (c * torch.linspace(0.5, 1.5, N, device="cuda")).sum().backward()
        outs.append((c.detach(), r, a.grad, l.grad))
    assert torch.isfinite(outs[0][0]).all()
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("scales", [(0.0, 0.0), (0.25, 0.0), (0.0, 0.3), (0.1, 0.1)])
def test_unigram_couples_the_batch_iff_am_only_scale(w, scales):
    """5: lattice 1's padding lm rows move every cost, and get a gradient, iff sa > 0; a NaN in lattice 2's live lm
    row makes its cost NaN, and every cost NaN iff sa > 0."""
    sl, sa = scales
    N, T, U, V = 4, 30, 20, 28
    am, lm, ys, xn, yn = make(N, T, U, V, seed=12)
    yn[1] = 8
    xn[3] = T + 1                                       # invalid lengths: cost NaN, no cells

    def run(lm):
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), lm_only_scale=sl, am_only_scale=sa)
        torch.nan_to_num(c, nan=0.0).sum().backward()
        return c.detach().cpu().numpy(), l.grad.cpu().numpy()

    c0, dl0 = run(lm)
    assert np.isnan(c0[3]) and np.isfinite(c0[:3]).all()
    pad = np.concatenate([dl0[1, int(yn[1]) + 1:], dl0[3]])
    assert ((pad == 0).all()) == (sa == 0)
    lm2 = lm.copy()
    lm2[1, U - 1] += np.random.RandomState(1).randn(V).astype(np.float32) * 3
    c1, _ = run(lm2)
    for n in range(3):
        assert (c1[n] != c0[n]) == (sa > 0), n
    lm3 = lm.copy()
    lm3[2, 0, 3] = np.nan
    c3, _ = run(lm3)
    assert np.isnan(c3[2])
    if sa > 0:
        assert np.isnan(c3).all()
    else:
        assert np.array_equal(np.delete(c3, 2), np.delete(c0, 2), equal_nan=True)


def test_masked_vocabulary(w):
    """6: -inf on every vocabulary entry that is neither blank nor one of the lattice's labels."""
    N, T, U, V = 3, 20, 8, 40
    am, lm, ys, xn, yn = make(N, T, U, V, seed=9)
    for n in range(N):
        keep = np.zeros(V, bool)
        keep[0] = True
        keep[ys[n]] = True
        am[n, :, ~keep] = -np.inf
        lm[n, 1::2, ~keep] = -np.inf
    for sl, sa in ((0.25, 0.0), (0.1, 0.1)):
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), lm_only_scale=sl, am_only_scale=sa)
        c.sum().backward()
        check(c.detach().cpu().numpy(), a.grad.cpu().numpy(), l.grad.cpu().numpy(),
              oracle(am, lm, ys, xn, yn, 0, sl, sa, np.ones(N)), lm, np.ones(N), sa)


def test_forward_only_and_empty(w):
    N, T, U, V = 3, 30, 12, 20
    am, lm, ys, xn, yn = make(N, T, U, V, seed=4)
    args = (cu(ys), cu(xn), cu(yn))
    kw = {"lm_only_scale": 0.1, "am_only_scale": 0.2}
    a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
    c, r = w.rnnt_loss_simple(a, l, *args, prune_range=4, **kw)
    with torch.no_grad():
        c2 = w.rnnt_loss_simple(cu(am), cu(lm), *args, **kw)
        c3, r3 = w.rnnt_loss_simple(cu(am), cu(lm), *args, prune_range=4, **kw)
    assert not c2.requires_grad and torch.equal(c.detach(), c2) and torch.equal(c2, c3) and torch.equal(r, r3)
    c.sum().backward()
    l2 = cu(lm).requires_grad_(True)
    w.rnnt_loss_simple(cu(am), l2, *args, **kw).sum().backward()
    assert torch.equal(l2.grad, l.grad)
    e = torch.empty((0, T, V), device="cuda", requires_grad=True)
    f = torch.empty((0, U, V), device="cuda", requires_grad=True)
    z = torch.empty((0,), dtype=torch.int, device="cuda")
    c0, r0 = w.rnnt_loss_simple(e, f, torch.empty((0, U - 1), dtype=torch.int, device="cuda"), z, z, prune_range=3,
                                **kw)
    c0.sum().backward()
    assert c0.shape == (0,) and r0.shape == (0, T) and e.grad.shape == (0, T, V) and f.grad.shape == (0, U, V)


def test_cuda_graph_replay(w):
    """No host sync: a captured smoothed forward (with ranges) + backward replays to eager's bits on new inputs."""
    N, T, U, V = 4, 60, 30, 48
    srcs = [make(N, T, U, V, seed=s) for s in (21, 22)]
    ys, xn, yn = (cu(x) for x in srcs[0][2:])
    a, l = cu(srcs[0][0]), cu(srcs[0][1])
    go = torch.linspace(0.5, 1.5, N, device="cuda")

    def step():
        c, saved, pg, r = w._C.rnnt_simple_forward(a, l, ys, xn, yn, 0, True, 5, 0, 0.1, 0.1)
        dam, dlm = w._C.rnnt_simple_backward(a, l, ys, xn, yn, saved, pg, go, 0, 0.1, 0.1)
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


def test_bad_scales(w):
    N, T, U, V = 2, 10, 5, 8
    am, lm, ys, xn, yn = make(N, T, U, V, seed=1)
    a, l, args = cu(am), cu(lm), (cu(ys), cu(xn), cu(yn))
    for sl, sa in ((-0.1, 0.0), (0.0, -1e-9), (1.0, 0.0), (0.5, 0.5), (0.7, 0.4), (math.nan, 0.0), (0.0, math.inf),
                   (True, 0.0), ("0.1", 0.0), (0.5, 0.5 - 1e-12)):
        with pytest.raises(ValueError, match="scale"):
            w.rnnt_loss_simple(a, l, *args, lm_only_scale=sl, am_only_scale=sa)
    with pytest.raises(RuntimeError, match="status 5"):
        w._C.rnnt_simple_forward(a, l, *args, 0, True, 0, 0, 0.6, 0.4)
    # the saved buffer must match the scales
    c, saved, pg, _ = w._C.rnnt_simple_forward(a, l, *args, 0, True, 0, 0, 0.1, 0.0)
    go = torch.ones(N, device="cuda")
    with pytest.raises(RuntimeError, match="saved"):
        w._C.rnnt_simple_backward(a, l, *args, saved, pg, go, 0)
    c, saved, pg, _ = w._C.rnnt_simple_forward(a, l, *args, 0, True, 0, 0)
    with pytest.raises(RuntimeError, match="saved"):
        w._C.rnnt_simple_backward(a, l, *args, saved, pg, go, 0, 0.1, 0.0)


def test_cabi_status(w):
    lib = abi()
    N, T, U, V = 2, 10, 5, 8
    am, lm, ys, xn, yn = make(N, T, U, V, seed=2)
    a, l, y, x, n = cu(am), cu(lm), cu(ys), cu(xn), cu(yn)
    s = torch.cuda.current_stream().cuda_stream
    nbytes = lib.rnnt_b200_simple_smoothed_workspace_bytes(N, T, U, V)
    assert nbytes > lib.rnnt_b200_simple_workspace_bytes(N, T, U)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    c = torch.empty(N, device="cuda")
    saved = torch.empty(saved_len(N, T, U, V, True), device="cuda")
    pg = torch.empty((N, T, U, 2), device="cuda")
    dam, dlm = torch.empty_like(a), torch.empty_like(l)
    P = [p.data_ptr() for p in (a, l, y, x, n, c, saved, pg)]

    def fwd(nb=nbytes, sl=0.1, sa=0.1, wp=ws.data_ptr()):
        return lib.rnnt_b200_simple_smoothed_forward(s, wp, nb, *P, N, T, U, V, 0, 0, sl, sa)

    def bwd(nb=nbytes, sl=0.1, sa=0.1, wp=ws.data_ptr()):
        return lib.rnnt_b200_simple_smoothed_backward(s, wp, nb, *P[:5], saved.data_ptr(), pg.data_ptr(), None,
                                                      dam.data_ptr(), dlm.data_ptr(), N, T, U, V, 0, sl, sa)

    assert fwd() == 0 and bwd() == 0
    assert fwd(sl=0.25, sa=0.0) == 0 and bwd(sl=0.25, sa=0.0) == 0
    for bad in ((-0.5, 0.0), (0.0, -0.5), (0.6, 0.4), (math.nan, 0.0), (0.0, math.inf)):
        assert fwd(*(nbytes,) + bad) == INVALID and bwd(*(nbytes,) + bad) == INVALID
    assert fwd(nb=nbytes - 1) == TOO_SMALL and bwd(nb=nbytes - 1) == TOO_SMALL and bwd(wp=None, nb=0) == TOO_SMALL
    # zero scales: the simple loss's workspace suffices and the backward takes none
    small = lib.rnnt_b200_simple_workspace_bytes(N, T, U)
    assert fwd(nb=small, sl=0.0, sa=0.0) == 0 and bwd(wp=None, nb=0, sl=0.0, sa=0.0) == 0
    torch.cuda.synchronize()
