"""rnnt_loss_pruned on every path its calls take, against the fp64 lattice restatement (tests/pruned_oracle.lattice).

Pruning pays at large U, where the fused kernel (U <= 104) no longer runs, and its windows are mostly removed edges
(S = 5 of U = 300 columns).  Each case of the table names the launch record its call must make (path, C, slices,
warps, ring; rnnt_b200_debug_last_launch) and runs two kinds of windows:
  * k2-like: test_gpu_pruned.make's monotone windows around a random path, clipped to [0, Un - S];
  * live: pruned_oracle.live_windows, drawn anywhere around a random path, so non-monotone, with gaps, clipping on
    both sides of the lattice in live frames, INT32_MIN / INT32_MAX in padding frames.
The logits are bf16-representable, so that f32 and bf16 calls see the same values and the same fp64 result.

Checks, in both LSE modes: costs 1e-5 relative, gradients within grad_bound (bf16: plus 2^-8 |g|, its one rounding);
bf16 is the f32 call's result, the gradient rounded once; forward only gives the same costs; a second call gives the
same bits; in exact mode a fused case equals the general path bit for bit (costs, lse, pair and logit gradients).
Then, on the general path: dead lattices, NaN logits in padding rows, CUDA graph capture; the normaliser's branches
and misaligned views on pruned rows; and the pruned forward's workspace alignment through the C ABI.

Every error against the fp64 restatement is printed as "pruned-err <case> <dtype> <mode> ..." next to its bound."""
import os

import numpy as np
import pytest
import torch

from tests import pruned_oracle as po
from tests.test_gpu_fused_emit import subprocess_outputs
from tests.test_gpu_launch_configs import FUSED, GENERAL, Launch, expect, last_launch, sms
from tests.test_gpu_pruned import _abi, make

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
EXACT, FAST = 1, 2
MODES = {EXACT: "exact", FAST: "fast"}
THREADS = 256                                 # kLogitThreads (csrc/logits.cu)


def gtol(T, U):
    return 2e-5 + 6e-6 * (T + U)


def grad_bound(T, U, costs):
    """1e-4 + 2 gtol(T,U), or one fp32 rounding of the log-likelihood per anti-diagonal, adding up as a random walk
    over the T + U of them, when that is larger: alpha + beta - ll cancels terms of the size of the cost, and with
    random logits the cost reaches 5,000-12,000 nats at T = 500-1500.  A plain fp32 restatement of the recurrence on
    the CPU shows the same errors (general_u300: 0.028)."""
    return 1e-4 + max(2 * gtol(T, U), 2.0 ** -23 * float(np.abs(costs).max()) * (T + U) ** 0.5)


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# name -> (N, T, S, U, V, blank, FastEmit lambda, windows, launch record of the forward)
CASES = {
    # the fused kernel's column widths, and one CTA per lattice over several waves
    "fused_c1_u20": (3, 40, 4, 20, 28, 0, 0.0, "k2", dict(path=FUSED, C=1)),
    "fused_c2_u40": (3, 40, 5, 40, 12, 2, 0.2, "live", dict(path=FUSED, C=2)),
    "fused_c4_u80": (3, 40, 5, 80, 36, 1, 0.0, "live", dict(path=FUSED, C=4)),
    "fused_waves_n300": (300, 150, 5, 40, 8, 1, 0.0, "live", dict(path=FUSED, C=2, slices=1)),
    # the profiled regime (tools/pruned_time.py): the general path
    "general_u100": (4, 500, 5, 100, 500, 0, 0.0, "k2", dict(path=GENERAL, warps=4)),
    "general_u300": (2, 1500, 5, 300, 50, 3, 0.1, "live", dict(path=GENERAL, warps=10)),
    # the boundary ring of 16 warps: back-pressure from Tn = 1025
    "ring_t1024": (2, 1024, 5, 481, 6, 1, 0.0, "live", dict(path=GENERAL, warps=16, ring=1024)),
    "ring_t1025": (2, 1025, 5, 481, 6, 1, 0.2, "k2", dict(path=GENERAL, warps=16, ring=1024)),
    # column passes: 2 at U = 513, 3 at U = 1025 (T >= U / 2, so that the windows keep a path)
    "passes_u513": (2, 300, 5, 513, 8, 2, 0.0, "live", dict(path=GENERAL, warps=16)),
    "passes_u1025": (2, 520, 5, 1025, 6, 0, 0.2, "live", dict(path=GENERAL, warps=16)),
    # every thread of the fill, normaliser and expand kernels makes several grid-stride iterations (grid_strides)
    "grid_stride": (16, 400, 5, 200, 500, 0, 0.0, "live", dict(path=GENERAL, warps=7)),
}
FUSED_CASES = [k for k, c in CASES.items() if c[8]["path"] == FUSED]


def case_inputs(name):
    N, T, S, U, V, blank, lam, kind, _ = CASES[name]
    seed = sum(map(ord, name))
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=seed, blank=blank)
    if kind == "live":
        r = po.live_windows(np.random.RandomState(seed), xn, yn, T, S)
        left, right = po.clipping_frames(r, xn, yn, S)
        assert left > 0 and right > 0, (name, left, right)
    x = torch.from_numpy(x).to(BF16).float().numpy()           # bf16-representable
    return x, ys, xn, yn, r, blank, lam


def picked(N):
    """Lattices checked against the fp64 restatement: all of a small batch, eight of a large one."""
    return list(range(N)) if N <= 16 else sorted({0, 1, N // 3, N // 2, N - 2, N - 1, 7, N // 5})


def report(what, dtype, mode, cost_rel, err, bound):
    """err: the largest gradient error, less 2^-8 |g| for bf16; bound: what it must not exceed."""
    print("pruned-err %s %s %s cost_rel=%.3g grad_err=%.3g bound=%.3g ratio=%.3f"
          % (what, dtype, MODES[mode], cost_rel, err, bound, err / bound))


def run(w, x, ys, xn, yn, r, blank, lam, mode, go, dtype=torch.float32):
    """-> (costs, logit gradient, launch record of the forward), through autograd."""
    a = (x if torch.is_tensor(x) else cu(x)).to(dtype).detach().requires_grad_(True)
    w.set_lse_mode(MODES[mode])
    try:
        with Launch() as L:
            c = w.rnnt_loss_pruned(a, cu(ys), cu(xn), cu(yn), cu(r), blank=blank, fastemit_lambda=lam)
        (c * go).sum().backward()
    finally:
        w.set_lse_mode("auto")
    return c.detach(), a.grad, L.rec


def grid_strides(N, T, S, U, V, elem, n_sm):
    """The launches of lse_pairs_as / expand_logits_as (csrc/logits.cu) for pruned rows -> (fill iterates, normaliser
    iterates, expand iterates, expand's stride_v)."""
    cells = N * T * U
    fill_grid = min(-(-(cells // 2 + 1) // THREADS), n_sm * 16)
    rows = N * T * S
    vec4 = V % 4 == 0
    sub = (8 if V <= 32 else 32) if vec4 else (1 if V <= 12 else 8 if V <= 512 else 32)
    per_block = THREADS // sub
    lse_grid = min(-(-rows // per_block), n_sm * 16)
    vec = next(c for c in (16 // elem, 8 // elem, 4 // elem, 2 // elem, 1) if c >= 1 and V % c == 0)
    total = rows * V // vec
    exp_grid = min(-(-total // THREADS), n_sm * 32)
    stride = exp_grid * THREADS * vec
    return cells // 2 > fill_grid * THREADS, rows > lse_grid * per_block, total > exp_grid * THREADS, stride % V


# ------------------------------------------------------------------------------------------ the general path's side
def _general_main(out_dir):
    """Subprocess body (RNNT_B200_PATH=general): exact-mode outputs of the fused cases on the general path."""
    import warp_rnnt_b200 as w
    assert os.environ.get("RNNT_B200_PATH") == "general"
    for name in FUSED_CASES:
        for k, t in fused_side(w, name).items():
            np.save(os.path.join(out_dir, "%s_%s.npy" % (name, k)), t.cpu().numpy())


def fused_side(w, name):
    x, ys, xn, yn, r, blank, lam = case_inputs(name)
    N = len(xn)
    args = (cu(ys), cu(xn), cu(yn), cu(r))
    with Launch() as L:
        c, l, p = w._C.rnnt_logits_pruned_forward(cu(x), *args, blank, lam, True, EXACT)
    want = GENERAL if os.environ.get("RNNT_B200_PATH") == "general" else FUSED
    assert L.rec["path"] == want, (name, L.rec)
    g = w._C.rnnt_logits_pruned_backward(cu(x), l, p, cu(ys), cu(r), torch.linspace(0.5, 1.5, N, device="cuda"), blank)
    return dict(costs=c, lse=l, pairs=p, grads=g)


@pytest.fixture(scope="module")
def general_outputs():
    return subprocess_outputs("RNNT_B200_PATH", "general", "_general_main", module="tests.test_gpu_pruned_paths")


# ------------------------------------------------------------------------------------------ the cases
@pytest.mark.parametrize("name", list(CASES))
def test_pruned_path(w, general_outputs, name):
    N, T, S, U, V, _, _, _, want = CASES[name]
    x, ys, xn, yn, r, blank, lam = case_inputs(name)
    if name == "grid_stride":
        for elem in (4, 2):
            fill, lse, expand, sv = grid_strides(N, T, S, U, V, elem, sms())
            assert fill and lse and expand and sv != 0, (elem, fill, lse, expand, sv)
    pick = picked(N)
    go_np = np.linspace(0.5, 1.5, N)
    go = cu(go_np.astype(np.float32))
    c0, g0 = po.lattice(x[pick], ys[pick], xn[pick], yn[pick], r[pick], blank, lam, grad_output=go_np[pick])
    assert np.isfinite(c0).all()
    tol = grad_bound(T, U, c0)
    for mode in (EXACT, FAST):
        c, g, rec = run(w, x, ys, xn, yn, r, blank, lam, mode, go)
        expect(rec, want, "%s %s f32" % (name, MODES[mode]))
        cn, gn = c.cpu().numpy()[pick], g.cpu().numpy()[pick]
        cost_rel = np.abs(cn - c0).max() / np.abs(c0).max()
        err = np.abs(gn - g0).max()
        report(name, "f32", mode, cost_rel, err, tol)
        np.testing.assert_allclose(cn, c0, rtol=1e-5, err_msg="%s %s" % (name, MODES[mode]))
        assert err <= tol, "%s %s: gradient error %.3g > %.3g" % (name, MODES[mode], err, tol)
        # bf16: the f32 result on the same values, the gradient rounded once
        cb, gb, rec = run(w, x, ys, xn, yn, r, blank, lam, mode, go, BF16)
        expect(rec, want, "%s %s bf16" % (name, MODES[mode]))
        assert torch.equal(cb, c) and torch.equal(gb, g.to(BF16)), (name, MODES[mode])
        errb = (np.abs(gb.float().cpu().numpy()[pick] - g0) - 2.0 ** -8 * np.abs(g0)).max()
        report(name, "bf16", mode, cost_rel, errb, tol)
        assert errb <= tol, "%s %s bf16: gradient error less 2^-8 |g| %.3g > %.3g" % (name, MODES[mode], errb, tol)
        # forward only: the same costs (the general path runs beta alone)
        w.set_lse_mode(MODES[mode])
        with Launch() as L:
            cf = w.rnnt_loss_pruned(cu(x), cu(ys), cu(xn), cu(yn), cu(r), blank=blank, fastemit_lambda=lam)
        w.set_lse_mode("auto")
        if want["path"] == GENERAL:
            expect(L.rec, dict(path=GENERAL, beta_only=1), name + " forward only")
        assert torch.equal(cf, c), (name, MODES[mode])
        # a second call: the same bits
        c2, g2, _ = run(w, x, ys, xn, yn, r, blank, lam, mode, go)
        assert torch.equal(c2, c) and torch.equal(g2, g), (name, MODES[mode])
    if name in FUSED_CASES:
        mine = fused_side(w, name)
        for k, t in mine.items():
            assert t.cpu().numpy().tobytes() == general_outputs["%s_%s.npy" % (name, k)].tobytes(), (name, k)


# ------------------------------------------------------------------------------------------ the general path's edges
def test_dead_lattices_on_the_general_path(w):
    """Windows that cut every path in a U >= 105 batch: NaN for Tn, Un >= 2 (a gap, the last cell, INT32_MAX and
    INT32_MIN in a live frame), +inf for Tn = 1 or Un = 1; NaN rows only on the dead lattices' cells; the live
    lattices are bit for bit a call on a batch of only them."""
    N, T, S, U, V = 8, 60, 5, 110, 12
    x, ys, xn, yn, _ = make(N, T, S, U, V, seed=41)
    x = torch.from_numpy(x).to(BF16).float().numpy()
    rng = np.random.RandomState(41)
    kinds = [None, "gap", "last", "int32_max", "int32_min", "one_frame", None, "no_labels"]
    xn[1] = xn[2] = T
    yn[1] = yn[2] = U - 1
    xn[5], yn[5] = 1, 1
    yn[7] = 0
    r = po.live_windows(rng, xn, yn, T, S)
    for k, kind in enumerate(kinds):
        if kind is not None:
            r = po.cut_windows(rng, r, xn, yn, S, k, kind)
    c0, g0 = po.lattice(x, ys, xn, yn, r)
    live = np.array([k is None for k in kinds])
    assert np.isfinite(c0[live]).all() and np.isinf(c0[~live]).all()
    rows = np.zeros((N, T, S), bool)
    n, t, s, _ = po.window_rows(r, xn, yn, S)
    rows[n, t, s] = True
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    sub = np.flatnonzero(live)
    for mode in (EXACT, FAST):
        c, g, rec = run(w, x, ys, xn, yn, r, 0, 0.0, mode, go)
        expect(rec, dict(path=GENERAL), "dead " + MODES[mode])
        c, g = c.cpu().numpy(), g.cpu().numpy()
        for k, kind in enumerate(kinds):
            if kind in ("one_frame", "no_labels"):
                assert c[k] == np.inf, (kind, c[k])
            elif kind is not None:
                assert np.isnan(c[k]), (kind, c[k])
        assert np.isfinite(c[live]).all() and np.isfinite(g[live]).all()
        for k in np.flatnonzero(~live):
            assert np.isnan(g[k]).any() and (np.isnan(g[k]) <= rows[k][:, :, None]).all(), kinds[k]
        cs, gs, _ = run(w, x[sub], ys[sub], xn[sub], yn[sub], r[sub], 0, 0.0, mode, go[cu(sub).long()])
        assert np.array_equal(c[sub], cs.cpu().numpy()) and np.array_equal(g[sub], gs.cpu().numpy()), MODES[mode]
        np.testing.assert_allclose(c[sub], c0[sub], rtol=1e-5)


def test_nan_logits_in_padding_rows_on_the_general_path(w):
    """NaN logits in padding rows -- a frame past the length, and in live frames a row left of column 0 and a row past
    the lattice's last column: NaN gradient rows there, every other output the same bits as without them."""
    N, T, S, U, V = 3, 60, 5, 110, 10
    x, ys, xn, yn, _ = make(N, T, S, U, V, seed=43)
    xn[1] = T - 3
    r = po.live_windows(np.random.RandomState(43), xn, yn, T, S)
    uu = r.astype(np.int64)[:, :, None] + np.arange(S)
    tt = np.arange(T)[None, :, None]
    live_frame = tt < xn[:, None, None]
    left = np.argwhere(live_frame & (uu < 0))
    right = np.argwhere(live_frame & (uu > yn[:, None, None]))
    assert len(left) and len(right)
    poisoned = [(1, T - 2, 3), tuple(left[0]), tuple(right[-1])]
    x2 = x.copy()
    for n, t, s in poisoned:
        x2[n, t, s, (t + s) % V] = np.nan
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    for mode in (EXACT, FAST):
        c, g, rec = run(w, x, ys, xn, yn, r, 0, 0.0, mode, go)
        expect(rec, dict(path=GENERAL), "nan rows")
        c2, g2, _ = run(w, x2, ys, xn, yn, r, 0, 0.0, mode, go)
        assert torch.isfinite(c).all() and torch.equal(c, c2), MODES[mode]
        nan = torch.isnan(g2)
        for n, t, s in poisoned:
            assert nan[n, t, s].all(), (n, t, s)
        assert nan.sum().item() == len(poisoned) * V
        assert torch.equal(g2[~nan], g[~nan]), MODES[mode]


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_cuda_graph_replay_on_the_general_path(w, dtype):
    """A captured loss.backward() on the general path replays to eager's bits, with new logits each replay."""
    N, T, S, U, V = 3, 80, 5, 110, 28
    x, ys, xn, yn, _ = make(N, T, S, U, V, seed=45)
    r = po.live_windows(np.random.RandomState(45), xn, yn, T, S)
    srcs = [cu(x).to(dtype), cu(make(N, T, S, U, V, seed=46)[0]).to(dtype)]
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
    assert last_launch()["path"] == GENERAL
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
        assert torch.isfinite(l0).all()
        assert torch.equal(loss.detach(), l0) and torch.equal(x.grad, g0)


# ------------------------------------------------------------------------------------------ normaliser branches
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
@pytest.mark.parametrize("V", [2, 12, 13, 32, 36, 50, 128, 132, 511, 512, 513, 1030])
def test_normaliser_branches_on_pruned_rows(w, V, offset):
    """Every SUB / VEC4 branch of the row normaliser and every expand vector (f32 4/2/1, bf16 8/4/2/1), on pruned rows
    with live windows, from contiguous views at element offsets 0-3 (2- and 4-byte aligned rows are summed element by
    element): costs 1e-5 relative, gradients 2^-8 |g| + 1e-4 + 2 gtol(T,U) (DESIGN.md 4, misaligned bf16)."""
    N, T, S, U = 3, 24, 4, 20
    x, ys, xn, yn, _ = make(N, T, S, U, V, seed=V + offset, blank=1)
    r = po.live_windows(np.random.RandomState(V), xn, yn, T, S)
    x = torch.from_numpy(x).to(BF16).float().numpy()
    go_np = np.linspace(0.5, 1.5, N)
    go = cu(go_np.astype(np.float32))
    c0, g0 = po.lattice(x, ys, xn, yn, r, 1, 0.1, grad_output=go_np)
    tol = 1e-4 + 2 * gtol(T, U)
    for dtype in (torch.float32, BF16):
        flat = torch.empty(x.size + offset, dtype=dtype, device="cuda")
        xs = flat[offset:].view(x.shape)
        xs.copy_(cu(x))
        for mode in (EXACT, FAST):
            c, g, _ = run(w, xs, ys, xn, yn, r, 1, 0.1, mode, go, dtype)
            assert g.dtype == dtype
            np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5, err_msg="%s %s" % (dtype, MODES[mode]))
            err = (np.abs(g.float().cpu().numpy() - g0) - 2.0 ** -8 * np.abs(g0)).max()
            assert err <= tol, "V=%d offset=%d %s %s: gradient error %.3g > %.3g" % (V, offset, dtype, MODES[mode],
                                                                                   err, tol)


# ------------------------------------------------------------------------------------------ workspace alignment
def test_pruned_forward_workspace_alignment():
    """The fill writes the workspace's pairs in 16-byte stores: a workspace 16 bytes into an allocation gives the bits
    of an aligned one; one only 8-byte aligned is refused (RNNT_STATUS_INVALID_ARGUMENT) before any launch."""
    lib = _abi()
    N, T, S, U, V = 3, 30, 5, 110, 16
    x, ys, xn, yn, r = make(N, T, S, U, V, seed=47)
    xt, ys_t, xn_t, yn_t, r_t = cu(x), cu(ys), cu(xn), cu(yn), cu(r)
    stream = torch.cuda.current_stream().cuda_stream
    need = lib.rnnt_b200_workspace_bytes(N * T * U, N)
    ws = torch.empty(need + 16, dtype=torch.uint8, device="cuda")
    assert ws.data_ptr() % 16 == 0
    out = []
    for off in (0, 16, 8):
        costs, lse = torch.full((N,), 7.0, device="cuda"), torch.full((N, T, S), 7.0, device="cuda")
        pg = torch.full((N, T, U, 2), 7.0, device="cuda")
        st = lib.rnnt_b200_logits_pruned_forward(
            stream, ws.data_ptr() + off, need, xt.data_ptr(), ys_t.data_ptr(), xn_t.data_ptr(), yn_t.data_ptr(),
            r_t.data_ptr(), costs.data_ptr(), lse.data_ptr(), pg.data_ptr(), N, T, S, U, V, 0, 0.0, EXACT, 4)
        torch.cuda.synchronize()
        out.append((st, costs, lse, pg))
    (s0, *a), (s16, *b), (s8, *c) = out
    assert s0 == 0 and s16 == 0 and s8 == 5, (s0, s16, s8)
    assert torch.isfinite(a[0]).all()
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    assert all((t == 7.0).all() for t in c)                                 # nothing was launched
