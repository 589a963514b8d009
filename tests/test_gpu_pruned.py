"""rnnt_loss_pruned: the loss from (N,T,S,V) logits of a joint evaluated in a window of S labels per frame.

The contract (include/rnnt_b200.h, DESIGN.md 3.5 and 4), with xf = a full (N,T,U,V) tensor holding each window row at
its cell (t, ranges[n,t] + s):
  1. a window that is the whole lattice (S = U, ranges = 0) gives rnnt_loss_from_logits's costs and gradients, bit for
     bit, on the fused kernel and on the general path;
  2. lse equals the dense from-logits lse of the same rows; costs and the (N,T,U,2) pair gradients equal
     rnnt_b200_loss_pairs on the pairs rebuilt from lse with (kBig, kBig) off the windows; the logit gradient equals
     _C.rnnt_logits_backward on xf at the window rows -- all bit for bit;
  3. against the fp64 restatement (tests/pruned_oracle.py): costs 1e-5 relative, gradients 1e-4 + 2 gtol(T,U);
  4. bf16 is the f32 result on the widened logits, the gradient rounded to bf16 once;
  5. dead lattices, NaN rows, forward only, N = 0, CUDA graphs, argument errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import pruned_oracle as po
from tests.test_gpu_logits import gtol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
BF16 = torch.bfloat16
EXACT, FAST = 1, 2
MODES = {EXACT: "exact", FAST: "fast"}
KBIG = -1.0e30
REC_PATH = 1                                          # rntLaunchRecord_t: 1 fused, 2 general

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _abi():
    lib = ctypes.CDLL(LIB)
    P, I, F, Z = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
    lib.rnnt_b200_logits_pruned_forward.restype = I
    lib.rnnt_b200_logits_pruned_forward.argtypes = [P, P, Z] + [P] * 8 + [I] * 6 + [F, I, I]
    lib.rnnt_b200_logits_pruned_backward.restype = I
    lib.rnnt_b200_logits_pruned_backward.argtypes = [P] * 8 + [I] * 7
    lib.rnnt_b200_loss_pairs.restype = I
    lib.rnnt_b200_loss_pairs.argtypes = [P, P, Z] + [P] * 5 + [I] * 3 + [F, I]
    lib.rnnt_b200_workspace_bytes.restype = Z
    lib.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, I]
    lib.rnnt_b200_debug_last_launch.argtypes = [P]
    return lib


def last_path(lib):
    rec = (ctypes.c_int32 * 32)()
    lib.rnnt_b200_debug_last_launch(ctypes.cast(rec, ctypes.c_void_p))
    return rec[REC_PATH]


def make(N, T, S, U, V, seed, blank=0, scale=3.0):
    """Raw logits (N,T,S,V), labels never blank, ragged lengths (lattice 0 full), and k2-like monotone windows around
    a random path that emits at most two labels per frame (T >= U / 2): every lattice stays live."""
    rng = np.random.RandomState(seed)
    x = (rng.randn(N, T, S, V) * scale).astype(np.float32)
    ys = rng.randint(0, V - 1, (N, U - 1)).astype(np.int32)
    ys = np.where(ys >= blank, ys + 1, ys).astype(np.int32)
    xn = rng.randint(max(T // 2, 1), T + 1, (N,)).astype(np.int32)
    yn = rng.randint(U // 2, U, (N,)).astype(np.int32)
    xn[0], yn[0] = T, U - 1
    if N > 1:                                    # the last lattice has a padding frame
        xn[N - 1] = min(int(xn[N - 1]), T - 1)
    ranges = rng.randint(-3, U + 3, (N, T)).astype(np.int32)          # padding frames: anything
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        yn[n] = min(int(yn[n]), 2 * Tn)
        Un = int(yn[n]) + 1
        per = np.zeros(Tn, np.int64)
        for f in rng.choice(np.repeat(np.arange(Tn), 2), Un - 1, replace=False):
            per[f] += 1
        lo = np.concatenate([[0], np.cumsum(per)[:-1]])              # first column of the path at frame t
        ranges[n, :Tn] = np.maximum(0, np.minimum(lo - rng.randint(0, 2, Tn), Un - S))
        ranges[n, :Tn] = np.maximum.accumulate(np.minimum(ranges[n, :Tn], lo))
    if N > 1:                                    # ... whose rows reach past U
        ranges[N - 1, T - 1] = U - 1
    return x, ys, xn, yn, ranges


def rows_of(ranges, S, U):
    """(n, t, s, u) index tensors of the rows whose column lies in [0, U)."""
    u = ranges.long()[:, :, None] + torch.arange(S, device=ranges.device)
    ok = (u >= 0) & (u < U)
    n, t, s = ok.nonzero(as_tuple=True)
    return n, t, s, u[ok]


def full_tensor(x, ranges, U, seed):
    """xf (N,T,U,V): random logits with each window row copied to its cell."""
    N, T, S, V = x.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    xf = torch.randn((N, T, U, V), device="cuda", generator=g).to(x.dtype) * 3
    n, t, s, u = rows_of(ranges, S, U)
    xf[n, t, u] = x[n, t, s]
    return xf


SHAPES = [  # N, T, S, U, V, blank, lambda
    (3, 30, 4, 20, 28, 0, 0.0),       # fused kernel
    (4, 40, 5, 33, 7, 2, 0.2),        # fused, rows of 7 logits
    (2, 60, 5, 110, 36, 0, 0.0),      # general path (U > 104)
    (3, 25, 4, 16, 300, 5, 0.1),      # 32 lanes per row
    (2, 20, 5, 12, 1030, 0, 0.0),     # V % 4 == 2
]


class lse_mode:
    def __init__(self, w, mode):
        self.w, self.mode = w, mode

    def __enter__(self):
        self.w.set_lse_mode(MODES[self.mode])

    def __exit__(self, *a):
        self.w.set_lse_mode("auto")


@gpu
@pytest.mark.parametrize("mode", [EXACT, FAST])
@pytest.mark.parametrize("shape,path", [((3, 30, 20, 28), 1), ((2, 30, 110, 8), 2)])
def test_whole_lattice_window_is_from_logits(w, shape, path, mode):
    """1: S = U, ranges = 0: rnnt_loss_from_logits's costs and gradients bit for bit; the launch record names the
    path."""
    lib = _abi()
    N, T, U, V = shape
    x, ys, xn, yn, _ = make(N, T, U, U, V, seed=T + U)
    r = torch.zeros((N, T), dtype=torch.int, device="cuda")
    args = (cu(ys), cu(xn), cu(yn))
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    with lse_mode(w, mode):
        a = cu(x).requires_grad_(True)
        c = w.rnnt_loss_pruned(a, *args, r)
        assert last_path(lib) == path
        (c * go).sum().backward()
        b = cu(x).requires_grad_(True)
        c2 = w.rnnt_loss_from_logits(b, *args)
        (c2 * go).sum().backward()
    assert torch.isfinite(c).all()
    assert torch.equal(c, c2) and torch.equal(a.grad, b.grad)


@gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_bit_parity_with_the_dense_passes(w, shape):
    """2: lse, costs, pair gradients and the logit gradient against the dense kernels on the same values."""
    lib = _abi()
    N, T, S, U, V, blank, lam = shape
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=T + V, blank=blank)
    xt, ys_t, xn_t, yn_t, r_t = cu(x), cu(ys), cu(xn), cu(yn), cu(r)
    xf = full_tensor(xt, r_t, U, seed=V)
    n, t, s, u = rows_of(r_t, S, U)
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    # every row's lse is the dense lse of the same row: here the (N,T,S) lattice of the pruned tensor itself
    _, ls, _ = w._C.rnnt_logits_forward(xt, torch.zeros((N, S - 1), dtype=torch.int, device="cuda"),
                                        xn_t, torch.zeros_like(yn_t), blank, 0.0, False, EXACT)
    stream = torch.cuda.current_stream().cuda_stream
    for mode in (EXACT, FAST):
        c, l, p = w._C.rnnt_logits_pruned_forward(xt, ys_t, xn_t, yn_t, r_t, blank, lam, True, mode)
        assert torch.isfinite(c).all() and l.shape == (N, T, S) and p.shape == (N, T, U, 2)
        assert torch.equal(l, ls)
        _, ld, _ = w._C.rnnt_logits_forward(xf, ys_t, xn_t, yn_t, blank, lam, False, mode)
        assert torch.equal(l[n, t, s], ld[n, t, u])
        # pairs rebuilt from lse: kBig off the windows
        lab = torch.cat([ys_t, torch.full((N, 1), blank, dtype=torch.int, device="cuda")], 1)
        pairs = torch.full((N, T, U, 2), KBIG, device="cuda")
        pairs[n, t, u, 0] = xt[n, t, s, blank] - l[n, t, s]
        pairs[n, t, u, 1] = xt[n, t, s].gather(1, lab[n, u].long()[:, None])[:, 0] - l[n, t, s]
        cr, pr = torch.empty(N, device="cuda"), torch.empty((N, T, U, 2), device="cuda")
        ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
        assert lib.rnnt_b200_loss_pairs(stream, ws.data_ptr(), ws.numel(), pairs.data_ptr(), xn_t.data_ptr(),
                                        yn_t.data_ptr(), cr.data_ptr(), pr.data_ptr(), N, T, U, lam, mode) == 0
        assert torch.equal(c, cr), (mode, (c - cr).abs().max().item())
        assert torch.equal(p, pr), mode
        g = w._C.rnnt_logits_pruned_backward(xt, l, p, ys_t, r_t, go, blank)
        gd = w._C.rnnt_logits_backward(xf, ld, p, ys_t, go, blank)
        assert torch.equal(g[n, t, s], gd[n, t, u]), mode
        # every other row is padding: exact zeros
        pad = torch.ones((N, T, S), dtype=torch.bool, device="cuda")
        pad[n, t, s] = False
        assert pad.any() and g[pad].abs().max().item() == 0
        # rows of padding cells (t >= Tn or u >= Un) too
        live = (t < xn_t.long()[n]) & (u <= yn_t.long()[n])
        assert g[n[~live], t[~live], s[~live]].abs().max().item() == 0 if (~live).any() else True
        assert torch.isfinite(g).all()


@gpu
@pytest.mark.parametrize("shape", SHAPES[:2] + SHAPES[3:4])
def test_against_the_fp64_restatement(w, shape):
    """3: costs 1e-5 relative, gradients 1e-4 + 2 gtol(T,U); every reduction, average_frames, blank != 0, FastEmit."""
    N, T, S, U, V, blank, lam = shape
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=T + V + 1, blank=blank)
    args = (cu(ys), cu(xn), cu(yn), cu(r))
    tol = 1e-4 + 2 * gtol(T, U)
    for mode in (EXACT, FAST):
        for reduction, avg in (("none", False), ("sum", True), ("mean", False), ("mean", True)):
            wgt = (1.0 / xn if avg else np.ones(N)) / (N if reduction == "mean" else 1)
            go = np.linspace(0.5, 1.5, N) if reduction == "none" else np.ones(N)
            c0, g0 = po.pruned(x, ys, xn, yn, r, blank, lam, grad_output=go * wgt)
            with lse_mode(w, mode):
                a = cu(x).requires_grad_(True)
                loss = w.rnnt_loss_pruned(a, *args, average_frames=avg, reduction=reduction, blank=blank,
                                          fastemit_lambda=lam)
                if reduction == "none":
                    (loss * cu(go.astype(np.float32))).sum().backward()
                else:
                    loss.backward()
            want = c0 * (1.0 / xn if avg else 1.0)
            want = want.sum() if reduction == "sum" else want.mean() if reduction == "mean" else want
            np.testing.assert_allclose(loss.detach().cpu().numpy(), want, rtol=1e-5)
            err = np.abs(a.grad.cpu().numpy() - g0).max()
            assert err <= tol, (mode, reduction, avg, err)


@gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_bf16_is_f32_on_the_widened_logits(w, shape):
    """4: bf16 costs equal the f32 call on x.float(), the gradient is the f32 gradient rounded to bf16 once."""
    N, T, S, U, V, blank, lam = shape
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=T + V + 2, blank=blank)
    args = (cu(ys), cu(xn), cu(yn), cu(r))
    xb = cu(x).to(BF16)
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    for mode in (EXACT, FAST):
        with lse_mode(w, mode):
            a = xb.clone().requires_grad_(True)
            c = w.rnnt_loss_pruned(a, *args, blank=blank, fastemit_lambda=lam)
            (c * go).sum().backward()
            b = xb.float().requires_grad_(True)
            c2 = w.rnnt_loss_pruned(b, *args, blank=blank, fastemit_lambda=lam)
            (c2 * go).sum().backward()
        assert c.dtype == torch.float32 and a.grad.dtype == BF16
        assert torch.equal(c, c2) and torch.equal(a.grad, b.grad.to(BF16)), mode


@gpu
def test_dead_lattices_get_the_dense_classes(w):
    """A window that cuts every path: cost NaN (Tn, Un >= 2), +inf with one frame or no labels; NaN gradient rows in
    that lattice only, as the restatement's +inf cost and NaN rows."""
    N, T, S, U, V = 4, 6, 2, 4, 5
    x, ys, _, _, _ = make(N, T, S, U, V, seed=7)
    xn = np.array([6, 6, 1, 6], np.int32)
    yn = np.array([3, 3, 3, 0], np.int32)
    r = np.array([[0, 0, 1, 1, 2, 2],          # live
                  [0, 0, 0, 0, 0, 0],          # never reaches u = 3
                  [0, 0, 0, 0, 0, 0],          # one frame: misses u = 2, 3
                  [0, 0, 1, 0, 0, 0]], np.int32)  # no labels: misses u = 0 at frame 2
    c0, g0 = po.pruned(x, ys, xn, yn, r)
    assert np.isfinite(c0[0]) and np.isinf(c0[1:]).all()
    for mode in (EXACT, FAST):
        with lse_mode(w, mode):
            a = cu(x).requires_grad_(True)
            c = w.rnnt_loss_pruned(a, cu(ys), cu(xn), cu(yn), cu(r))
            c.sum().backward()
        c = c.detach().cpu().numpy()
        assert np.isfinite(c[0]) and np.isnan(c[1]) and c[2] == np.inf and c[3] == np.inf, c
        g = a.grad.cpu().numpy()
        assert np.isfinite(g[0]).all()
        for k in (1, 2, 3):
            assert np.isnan(g[k]).any()
            assert (np.isnan(g[k]) <= np.isnan(g0[k])).all()     # NaN only on rows of lattice cells


@gpu
def test_nan_logits_give_nan_rows(w):
    """NaN logits in padding rows (a frame past the length, a column outside the lattice): those rows' gradients are
    NaN, everything else is what the same call without the NaNs gives."""
    N, T, S, U, V = 2, 12, 4, 8, 9
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=8)
    xn[1] = T - 2
    r[1, T - 2] = -3                             # rows s = 0, 1, 2 of padding frame T-2 lie left of the lattice
    x2 = x.copy()
    x2[1, T - 1, 2, 4] = np.nan
    x2[1, T - 2, 0, 1] = np.nan
    args = (cu(ys), cu(xn), cu(yn), cu(r))
    out = []
    for xx in (x, x2):
        a = cu(xx).requires_grad_(True)
        c = w.rnnt_loss_pruned(a, *args)
        c.sum().backward()
        out.append((c.detach(), a.grad))
    assert torch.equal(out[0][0], out[1][0])
    nan = torch.isnan(out[1][1])
    assert nan[1, T - 1, 2].all() and nan[1, T - 2, 0].all() and nan.sum().item() == 2 * V
    assert torch.equal(out[1][1][~nan], out[0][1][~nan])


@gpu
def test_forward_only_and_empty_batch(w):
    N, T, S, U, V = 3, 20, 4, 10, 12
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=9)
    args = (cu(ys), cu(xn), cu(yn), cu(r))
    c, l, p = w._C.rnnt_logits_pruned_forward(cu(x), *args, 0, 0.0, False, EXACT)
    assert p.numel() == 0
    c2, l2, _ = w._C.rnnt_logits_pruned_forward(cu(x), *args, 0, 0.0, True, EXACT)
    assert torch.equal(c, c2) and torch.equal(l, l2)
    with torch.no_grad():
        c3 = w.rnnt_loss_pruned(cu(x).requires_grad_(True), *args)
    assert not c3.requires_grad and torch.equal(c3, c)
    e = torch.zeros((0, T, S, V), device="cuda", requires_grad=True)
    z = torch.zeros(0, dtype=torch.int, device="cuda")
    c0 = w.rnnt_loss_pruned(e, torch.zeros((0, U - 1), dtype=torch.int, device="cuda"), z, z,
                            torch.zeros((0, T), dtype=torch.int, device="cuda"))
    assert c0.shape == (0,)
    c0.sum().backward()
    assert e.grad.shape == (0, T, S, V)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_cuda_graph_replay(w, dtype):
    """No host sync: a captured loss.backward() step replays to eager's bits."""
    N, T, S, U, V = 4, 50, 5, 30, 28
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=21)
    srcs = [cu(x).to(dtype), cu(make(N, T, S, U, V, seed=22)[0]).to(dtype)]
    args = (cu(ys), cu(xn), cu(yn), cu(r))

    def step(x):
        x.grad = None
        loss = w.rnnt_loss_pruned(x, *args, reduction="sum")
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
        assert torch.equal(loss.detach(), l0) and torch.equal(x.grad, g0)


@gpu
def test_binding_errors(w):
    N, T, S, U, V = 2, 6, 3, 5, 7
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=2)
    xt, ys_t, xn_t, yn_t, r_t = cu(x), cu(ys), cu(xn), cu(yn), cu(r)
    with pytest.raises(RuntimeError, match=r"ranges must be a contiguous Int tensor of shape \(N, T\)"):
        w.rnnt_loss_pruned(xt, ys_t, xn_t, yn_t, r_t[:, :-1].contiguous())
    with pytest.raises(RuntimeError, match=r"ranges must be a contiguous Int tensor of shape \(N, T\)"):
        w.rnnt_loss_pruned(xt, ys_t, xn_t, yn_t, r_t.long())
    with pytest.raises(RuntimeError, match=r"ranges must be a contiguous Int tensor of shape \(N, T\)"):
        w.rnnt_loss_pruned(xt, ys_t, xn_t, yn_t, r_t.t().contiguous().t())
    with pytest.raises(RuntimeError, match="xs must have 4 dimensions"):
        w.rnnt_loss_pruned(xt[0], ys_t, xn_t, yn_t, r_t)
    with pytest.raises(RuntimeError, match="xs must be a Float tensor"):
        w.rnnt_loss_pruned(xt.half(), ys_t, xn_t, yn_t, r_t)
    with pytest.raises(RuntimeError, match=r"blank must be in \[0, V\)"):
        w.rnnt_loss_pruned(xt, ys_t, xn_t, yn_t, r_t, blank=V)
    with pytest.raises(RuntimeError, match="ys must be a Int tensor"):
        w.rnnt_loss_pruned(xt, ys_t.long(), xn_t, yn_t, r_t)
    with pytest.raises(RuntimeError, match=r"ys shape must be \(N, U-1\)"):
        w.rnnt_loss_pruned(xt, ys_t[:1], xn_t, yn_t, r_t)
    with pytest.raises(RuntimeError, match="xs must be contiguous"):
        w.rnnt_loss_pruned(xt.transpose(1, 2), ys_t, xn_t, yn_t, r_t)
    c, l, p = w._C.rnnt_logits_pruned_forward(xt, ys_t, xn_t, yn_t, r_t, 0, 0.0, True, EXACT)
    go = torch.ones(N, device="cuda")
    with pytest.raises(RuntimeError, match=r"pair_grads must be a contiguous Float tensor of shape \(N, T, U, 2\)"):
        w._C.rnnt_logits_pruned_backward(xt, l, p[:, :, :-1].contiguous(), ys_t, r_t, go, 0)
    with pytest.raises(RuntimeError, match=r"lse must be a contiguous Float tensor of shape \(N, T, S\)"):
        w._C.rnnt_logits_pruned_backward(xt, l[:, :-1].contiguous(), p, ys_t, r_t, go, 0)
    with pytest.raises(RuntimeError, match=r"ranges must be a contiguous Int tensor of shape \(N, T\)"):
        w._C.rnnt_logits_pruned_backward(xt, l, p, ys_t, r_t[:1], go, 0)


@gpu
def test_abi_status_codes(w):
    """Element size, alignment, shape and workspace errors come back as status codes before any launch."""
    lib = _abi()
    N, T, S, U, V = 2, 6, 3, 5, 8
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=3)
    xt, ys_t, xn_t, yn_t, r_t = cu(x), cu(ys), cu(xn), cu(yn), cu(r)
    xb = xt.to(BF16)
    costs, lse = torch.empty(N, device="cuda"), torch.empty((N, T, S), device="cuda")
    pg = torch.empty((N, T, U, 2), device="cuda")
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    go = torch.ones(N, device="cuda")

    def fwd(logits=None, eb=4, wsb=None, S_=S, N_=N, pgp=None, lsep=None):
        return lib.rnnt_b200_logits_pruned_forward(
            stream, ws.data_ptr(), ws.numel() if wsb is None else wsb, xt.data_ptr() if logits is None else logits,
            ys_t.data_ptr(), xn_t.data_ptr(), yn_t.data_ptr(), r_t.data_ptr(), costs.data_ptr(),
            lse.data_ptr() if lsep is None else lsep, pg.data_ptr() if pgp is None else pgp, N_, T, S_, U, V, 0, 0.0,
            EXACT, eb)

    def bwd(logits, out, eb):
        return lib.rnnt_b200_logits_pruned_backward(stream, logits, lse.data_ptr(), pg.data_ptr(), ys_t.data_ptr(),
                                                    r_t.data_ptr(), go.data_ptr(), out, N, T, S, U, V, 0, eb)

    assert fwd() == 0
    assert fwd(eb=3) == 5 and fwd(eb=8) == 5
    assert fwd(logits=xb.data_ptr() + 1, eb=2) == 5                       # odd bf16 pointer
    assert fwd(logits=xt.data_ptr() + 2, eb=4) == 5                       # f32 pointer not 4-byte aligned
    assert fwd(S_=0) == 5                                                 # S < 1
    assert fwd(pgp=pg.data_ptr() + 4) == 5                                # pair_grads not 8-byte aligned
    assert fwd(lsep=0) == 5                                               # NULL lse
    assert fwd(N_=-1) == 5
    assert fwd(wsb=ws.numel() - 1) == 6                                    # workspace too small
    assert fwd(N_=0, wsb=0) == 0                                          # nothing to do
    out = torch.empty_like(xt)
    outb = torch.empty_like(xb)
    assert bwd(xt.data_ptr(), out.data_ptr(), 4) == 0
    assert bwd(xt.data_ptr(), out.data_ptr(), 3) == 5
    assert bwd(xb.data_ptr() + 1, outb.data_ptr(), 2) == 5
    assert bwd(xb.data_ptr(), outb.data_ptr() + 1, 2) == 5
    assert bwd(xb.data_ptr(), outb.data_ptr(), 2) == 0
    torch.cuda.synchronize()
    c, l, p = w._C.rnnt_logits_pruned_forward(xt, ys_t, xn_t, yn_t, r_t, 0, 0.0, True, EXACT)
    assert torch.equal(costs, c) and torch.equal(lse, l) and torch.equal(pg, p)
    assert torch.equal(out, w._C.rnnt_logits_pruned_backward(xt, l, p, ys_t, r_t, go, 0))


@gpu
def test_fill_reaches_the_last_cell_of_an_odd_lattice(w):
    """N*T*U odd: k_fill_pairs writes the last cell apart from its 16-byte stores.  The last lattice is full and its last
    frame's window misses its last cell (t = T-1, u = U-1), the lattice's last cell in memory: the blank edge that
    ends every path is removed, so the lattice is dead (cost NaN).  Run through the C ABI with a zero-filled workspace,
    where a last cell left unwritten would read as the pair (0, 0) and give a finite cost; the control window that
    covers the cell gives the restatement's cost."""
    lib = _abi()
    N, T, S, U, V = 3, 7, 3, 5, 6
    assert N * T * U % 2 == 1
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=31)
    xn[2], yn[2] = T, U - 1
    r[2] = [0, 0, 1, 1, 2, 2, 1]                 # frame 6: columns 1..3, not 4
    stream = torch.cuda.current_stream().cuda_stream
    ys_t, xn_t, yn_t = cu(ys), cu(xn), cu(yn)
    for last, dead in ((2, False), (1, True)):
        r[2, T - 1] = last
        c0, _ = po.pruned(x, ys, xn, yn, r)
        assert np.isfinite(c0[:2]).all() and np.isfinite(c0[2]) != dead
        xt, r_t = cu(x), cu(r)
        ws = torch.zeros(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
        costs, lse = torch.empty(N, device="cuda"), torch.empty((N, T, S), device="cuda")
        pg = torch.empty((N, T, U, 2), device="cuda")
        assert lib.rnnt_b200_logits_pruned_forward(
            stream, ws.data_ptr(), ws.numel(), xt.data_ptr(), ys_t.data_ptr(), xn_t.data_ptr(), yn_t.data_ptr(),
            r_t.data_ptr(), costs.data_ptr(), lse.data_ptr(), pg.data_ptr(), N, T, S, U, V, 0, 0.0, EXACT, 4) == 0
        c = costs.cpu().numpy()
        np.testing.assert_allclose(c[:2], c0[:2], rtol=1e-5)
        if dead:
            assert np.isnan(c[2]), c
        else:
            np.testing.assert_allclose(c[2], c0[2], rtol=1e-5)
        cb = w.rnnt_loss_pruned(xt, ys_t, xn_t, yn_t, r_t)
        assert torch.equal(torch.isnan(cb), torch.isnan(costs)) and torch.equal(cb[:2], costs[:2])
