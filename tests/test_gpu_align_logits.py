"""GPU: rnnt_align_from_logits (Viterbi forced alignment from joint logits on k2's lattices, csrc/frames.cu
k_frames_align and csrc/wavefront.cu k_align).

  1. regular: rnnt_align on x - lse (penalised as k_delay_pairs does), bit for bit, dense and compact, f32 and bf16;
  2. modified / constrained, with and without a penalty: tests/frames_align_oracle.py on the kernel's own pairs, bit
     for bit; the re-fold of the returned frames; the loss of the same type and an fp64 max-plus as bounds;
  3. both sides of every thread-layout bound, with the launch record; long T;
  4. degenerate lattices isolated from the rest of the batch; bf16, compact, CUDA graphs, determinism;
  5. the ValueErrors, the operator module's refusals and the C ABI's, with no launch."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import frames_align_oracle as fo
from tests.common import to_compact

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
KIND = {"regular": 0, "modified": 1, "constrained": 2}
REC = dict(seq=0, constrained=1, threads=2, passes=3, smem=4, blocks=5, delay=6)
INVALID, SMALL = 5, 6

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
    L.rnnt_b200_align_logits_workspace_bytes.restype = Z
    L.rnnt_b200_align_logits_workspace_bytes.argtypes = [ctypes.c_int64, I, I, I]
    L.rnnt_b200_align_logits_dense.restype = I
    L.rnnt_b200_align_logits_dense.argtypes = [P, P, Z] + [P] * 6 + [I] * 7 + [F]
    L.rnnt_b200_align_logits_compact.restype = I
    L.rnnt_b200_align_logits_compact.argtypes = [P, P, Z] + [P] * 6 + [ctypes.c_int64] + [I] * 6
    L.rnnt_b200_debug_last_frames_align_launch.argtypes = [P]
    L.rnnt_b200_launch_count.restype = ctypes.c_uint64
    return L


def record(lib):
    rec = (ctypes.c_int32 * 16)()
    lib.rnnt_b200_debug_last_frames_align_launch(ctypes.cast(rec, ctypes.c_void_p))
    return {k: rec[i] for k, i in REC.items()}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make(N, T, U, V, seed, xn=None, yn=None, blank=0, scale=2.0):
    """logits (N,T,U,V) f32, labels in [0,V) other than blank; by default most lattices have a modified path"""
    rng = np.random.RandomState(seed)
    x = (rng.randn(N, T, U, V) * scale).astype(np.float32)
    ys = rng.randint(0, V - 1, (N, U - 1)).astype(np.int32)
    ys += (ys >= blank)
    xn = rng.randint(max(1, T // 2), T + 1, N).astype(np.int32) if xn is None else np.asarray(xn, np.int32)
    yn = np.minimum(rng.randint(0, U, N), xn).astype(np.int32) if yn is None else np.asarray(yn, np.int32)
    return cu(x), cu(ys), cu(xn), cu(yn)


def lse_of(w, x, ys, xn, yn, blank=0):
    """the normaliser of the from-logits loss's own pass"""
    return w._C.rnnt_logits_forward(x, ys, xn, yn, blank, 0.0, False)[1]


def pairs_of(x, lse, ys, blank=0):
    """(x[blank] - lse, x[label] - lse) in f32, label = blank on the last column: the loss's pairs"""
    N, T, U, _ = x.shape
    lab = torch.cat([ys, torch.full((N, 1), blank, dtype=torch.int, device="cuda")], 1).long()
    xl = x.float().gather(3, lab[:, None, :, None].expand(N, T, U, 1))[..., 0]
    return torch.stack([x.float()[..., blank] - lse, xl - lse], -1).contiguous()


def penalty(xn, yn, T, U, lam):
    """(N,T,U) f32: ((f32(Tn-1) * 0.5) - f32(t)) * lam on live label slots, 0 elsewhere (k_delay_pairs' order), and
    the mask of those slots"""
    N = xn.numel()
    t = torch.arange(T, device="cuda", dtype=torch.float32)[None, :, None]
    u = torch.arange(U, device="cuda")[None, None, :]
    half = (xn.float() - 1.0) * 0.5
    pen = (half[:, None, None] - t) * torch.tensor(lam, dtype=torch.float32, device="cuda")
    live = (torch.arange(T, device="cuda")[None, :, None] < xn[:, None, None]) & (u < yn[:, None, None]) & \
        ((xn >= 1) & (xn <= T) & (yn >= 0) & (yn + 1 <= U))[:, None, None]
    return pen.expand(N, T, U), live


def same(p, q):
    return p.shape == q.shape and p.dtype == q.dtype and torch.equal(p.view(torch.uint8), q.view(torch.uint8))


def alignf(w, x, ys, xn, yn, kind="regular", lam=0.0, blank=0):
    s, f = w.rnnt_align_from_logits(x, ys, xn, yn, blank=blank, rnnt_type=kind, delay_penalty=lam)
    assert s.dtype == torch.float32 and f.dtype == torch.int32 and f.shape == (x.shape[0], x.shape[2] - 1)
    return s, f


# ------------------------------------------------------------------------------------------------ 1. regular
def regular_reference(w, x, ys, xn, yn, lam, blank=0):
    """rnnt_align on the f32 log-probs x - lse, the penalty added to the non-blank columns of live label slots"""
    lp = x.float() - lse_of(w, x, ys, xn, yn, blank)[..., None]
    if lam:
        pen, live = penalty(xn, yn, x.shape[1], x.shape[2], lam)
        cols = torch.arange(x.shape[3], device="cuda") != blank
        lp = torch.where(live[..., None] & cols, lp + pen[..., None], lp)
    return w.rnnt_align(lp.contiguous(), ys, xn, yn, blank=blank)


@pytest.mark.parametrize("lam", [0.0, 0.05])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(6, 40, 20, 12, 0), (3, 70, 45, 300, 2), (4, 150, 40, 28, 0)])
def test_regular_is_rnnt_align_on_log_probs(w, shape, dtype, lam):
    N, T, U, V, blank = shape
    x, ys, xn, yn = make(N, T, U, V, seed=T + U, blank=blank)
    yn = torch.randint(0, U, (N,), device="cuda", dtype=torch.int32)       # regular: more labels than frames is fine
    x = x.to(dtype)
    s, f = alignf(w, x, ys, xn, yn, lam=lam, blank=blank)
    s0, f0 = regular_reference(w, x, ys, xn, yn, lam, blank)
    assert same(s, s0) and torch.equal(f, f0)
    assert torch.isfinite(s).all()


def compact_of(x, ys, xn, yn):
    xc, yc = to_compact(x.float().cpu().numpy(), ys.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy())
    return cu(xc).to(x.dtype), cu(yc)


def padded_frames(f, yn, U):
    out = torch.full((len(yn), U - 1), -1, dtype=torch.int32, device="cuda")
    o = 0
    for n, y in enumerate(yn.tolist()):
        out[n, :y] = f[o:o + y]
        o += y
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_regular_compact_is_rnnt_align_on_log_probs(w, dtype):
    N, T, U, V = 6, 50, 24, 33
    x, ys, xn, yn = make(N, T, U, V, seed=5)
    x = x.to(dtype)
    xc, yc = compact_of(x, ys, xn, yn)
    lse = w._C.rnnt_logits_compact_forward(xc, yc, xn, yn, 0, 0.0, False, 0, 0, 0)[1]
    s0, f0 = w.rnnt_align((xc.float() - lse[:, None]).contiguous(), yc, xn, yn, compact=True)
    s, f = w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True)
    assert same(s, s0) and torch.equal(f, f0) and f.shape == (int(yn.sum()),)


# ------------------------------------------------------------------------------------------------ 2. modified / constrained
def f64_maxplus(B, L, rnnt_type):
    """the same sweep in float64 on the same f32 weights (scores only)"""
    B, L = B.astype(np.float64), L.astype(np.float64)
    Tn, Un = B.shape
    Lp = L + B[:, 1:] if rnnt_type == 2 else L
    a = np.full(Un, -np.inf)
    a[0] = 0
    for t in range(Tn):
        nxt = a + B[t]
        nxt[1:] = np.maximum(nxt[1:], a[:-1] + Lp[t])
        a = nxt
    return a[Un - 1]


def check_typed(w, x, ys, xn, yn, kind, lam, blank=0, loss=True):
    """scores and frames equal the oracle on the kernel's pairs bit for bit, re-fold, and lie below -cost and near
    fp64.  -> scores, frames (torch)"""
    k = KIND[kind]
    s, f = alignf(w, x, ys, xn, yn, kind, lam, blank)
    pairs = pairs_of(x, lse_of(w, x, ys, xn, yn, blank), ys, blank).cpu().numpy()
    xn_h, yn_h = xn.cpu().numpy(), yn.cpu().numpy()
    if lam:
        pairs = fo.delay_pairs(pairs, xn_h, yn_h, lam)
    s0, f0 = fo.align_pairs_np(pairs, xn_h, yn_h, k)
    sh, fh = s.cpu().numpy(), f.cpu().numpy()
    assert sh.tobytes() == s0.tobytes(), (sh, s0)
    assert np.array_equal(fh, f0)
    cost = None
    if loss:
        with torch.no_grad():
            cost = w.rnnt_loss_from_logits(x, ys, xn, yn, blank=blank, rnnt_type=kind, delay_penalty=lam)
        cost = cost.cpu().numpy()
    for n in range(len(xn_h)):
        Tn, Un = int(xn_h[n]), int(yn_h[n]) + 1
        if not s0[n] > -np.inf:
            assert (fh[n] == -1).all()
            continue
        fr = fh[n, :Un - 1]
        assert (fh[n, Un - 1:] == -1).all()
        assert (np.diff(fr) > 0).all() and (fr >= 0).all() and (fr <= Tn - 1).all()
        B, L = fo.lattice(pairs, n, Tn, Un)
        assert fo.fold(B, L, fr, k).tobytes() == sh[n].tobytes(), n
        s64 = f64_maxplus(B, L, k)
        # f32 rounding of each of the Tn additions: at most half an ulp of the running |sum| <= sum of |w|
        bound = Tn * 2.0 ** -24 * (np.abs(B).sum() + np.abs(L).sum() + 1.0)
        assert abs(float(sh[n]) - s64) <= bound, (n, sh[n], s64)
        if cost is not None and np.isfinite(cost[n]):
            # the best path's probability is at most the total: score <= -cost, up to the loss's f32 LSE rounding
            assert sh[n] <= -cost[n] + 1e-5 * (1.0 + abs(cost[n])), (n, sh[n], cost[n])
    return s, f


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("lam", [0.0, 0.05])
@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_types_against_the_oracle(w, kind, lam, dtype):
    x, ys, xn, yn = make(7, 60, 25, 29, seed=KIND[kind] + int(lam * 100))
    check_typed(w, x.to(dtype), ys, xn, yn, kind, lam)


@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_types_blank_not_zero_and_large_vocabulary(w, kind):
    x, ys, xn, yn = make(3, 40, 18, 1024, seed=9, blank=1023)
    check_typed(w, x, ys, xn, yn, kind, 0.05, blank=1023)


@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_minus_inf_exactly_where_the_cost_is_inf(w, kind):
    N, T, U, V = 6, 20, 9, 7
    x, ys, xn, yn = make(N, T, U, V, seed=21)
    xn[:] = 20
    yn[:] = torch.tensor([8, 8, 8, 5, 8, 8], dtype=torch.int32)
    xn[3] = 4                                                  # 5 labels, 4 frames: no path
    lab = int(ys[1, 2])
    x[1, :, 2, lab] = -float("inf")                            # label 2 masked on every frame
    x[4, :, 8, 0] = -float("inf")                              # the last column's blank masked (modified: dead)
    x[4, :, 7, 0] = -float("inf")
    s, _ = check_typed(w, x, ys, xn, yn, kind, 0.0)
    with torch.no_grad():
        c = w.rnnt_loss_from_logits(x, ys, xn, yn, rnnt_type=kind)
    assert torch.equal(torch.isneginf(s), torch.isposinf(c)), (s, c)
    assert torch.isneginf(s[[1, 3]]).all()


def test_unique_path_when_labels_fill_the_frames(w):
    x, ys, xn, yn = make(2, 12, 13, 6, seed=4, xn=[12, 9], yn=[12, 9])
    for kind in ("modified", "constrained"):
        _, f = check_typed(w, x, ys, xn, yn, kind, 0.0)
        assert f[0].tolist() == list(range(12)) and f[1, :9].tolist() == list(range(9))


# ------------------------------------------------------------------------------------------------ 3. thread layout
def threads_for(U):
    return min(512, max(32, (U + 31) // 32 * 32))


# U -> (T, xn, yn): columns in prefetch slot 0 (33), slot 1 (513), the in-step loop (1100, 2100), the largest U
LAYOUTS = {
    33: (40, [40, 33, 20], [32, 30, 20]),
    513: (520, [520, 513], [512, 400]),
    1100: (1100, [1100], [1099]),
    2100: (2101, [2101], [2099]),
    25600: (40, [40, 40], [30, 25599]),
}


@pytest.mark.parametrize("kind", ["modified", "constrained"])
@pytest.mark.parametrize("U", list(LAYOUTS))
def test_thread_layout_bounds(w, lib, U, kind):
    T, xn, yn = LAYOUTS[U]
    lam = 0.05 if U % 2 else 0.0
    x, ys, xnd, ynd = make(len(xn), T, U, 4, seed=U, xn=xn, yn=yn, scale=1.0)
    check_typed(w, x, ys, xnd, ynd, kind, lam, loss=U < 25600)
    th = threads_for(U)
    rec = record(lib)
    want = dict(constrained=KIND[kind] == 2, threads=th, passes=(U + th - 1) // th, smem=8 * U, blocks=(U + 31) // 32,
                delay=int(lam != 0))
    assert {k: rec[k] for k in want} == want, rec


def test_u_above_the_frame_sweep_bound(w):
    x, ys, xn, yn = make(1, 2, 25601, 2, seed=1, xn=[2], yn=[1])
    for kind in ("modified", "constrained"):
        with pytest.raises(RuntimeError, match="status 5"):
            w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type=kind)
    s, f = alignf(w, x, ys, xn, yn)
    s0, f0 = regular_reference(w, x, ys, xn, yn, 0.0)
    assert same(s, s0) and torch.equal(f, f0) and torch.isfinite(s).all()


@pytest.mark.parametrize("kind", ["regular", "modified", "constrained"])
def test_long_lattices(w, kind):
    """T >= 3000: the backtrace crosses many 32-frame blocks and column blocks"""
    x, ys, xn, yn = make(2, 3000, 150, 6, seed=30, xn=[3000, 2777], yn=[149, 120], scale=1.0)
    if kind == "regular":
        s, f = alignf(w, x, ys, xn, yn, lam=0.05)
        s0, f0 = regular_reference(w, x, ys, xn, yn, 0.05)
        assert same(s, s0) and torch.equal(f, f0)
    else:
        check_typed(w, x, ys, xn, yn, kind, 0.05)


# ------------------------------------------------------------------------------------------------ 4. isolation, layouts
@pytest.mark.parametrize("lam", [0.0, 0.05])
@pytest.mark.parametrize("kind", ["regular", "modified", "constrained"])
def test_degenerate_lattices_are_isolated(w, kind, lam):
    N, T, U, V = 6, 30, 10, 9
    x, ys, xn, yn = make(N, T, U, V, seed=40, xn=[30] * 6, yn=[9, 5, 7, 8, 6, 9])
    s0, f0 = alignf(w, x, ys, xn, yn, kind, lam)
    xb, xnb, ynb = x.clone(), xn.clone(), yn.clone()
    xb[1] = float("nan")                                     # every path NaN
    xnb[3] = 0                                               # invalid lengths
    xb[4, :, :, 0] = -float("inf")                           # no blank anywhere: dead (regular and types 1/2)
    s, f = alignf(w, xb, ys, xnb, ynb, kind, lam)
    keep = [0, 2, 5]
    assert same(s[keep], s0[keep]) and torch.equal(f[keep], f0[keep])
    assert torch.isnan(s[1]) and torch.isnan(s[3]) and torch.isneginf(s[4])
    assert (f[[1, 3, 4]] == -1).all()


@pytest.mark.parametrize("kind,lam", [("regular", 0.0), ("regular", 0.05), ("modified", 0.05), ("constrained", 0.0)])
def test_bf16_equals_f32_on_the_widened_logits(w, kind, lam):
    x, ys, xn, yn = make(5, 45, 21, 40, seed=50)
    xb = x.to(torch.bfloat16)
    s16, f16 = alignf(w, xb, ys, xn, yn, kind, lam)
    s32, f32 = alignf(w, xb.float(), ys, xn, yn, kind, lam)
    assert same(s16, s32) and torch.equal(f16, f32)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_compact_equals_dense(w, dtype):
    N, T, U, V = 7, 40, 20, 12
    x, ys, xn, yn = make(N, T, U, V, seed=60)
    yn = torch.randint(0, U, (N,), device="cuda", dtype=torch.int32)
    x = x.to(dtype)
    x[N - 1, :, 0, int(ys[N - 1, 0])] = -float("inf")          # one dead lattice
    sd, fd = alignf(w, x, ys, xn, yn)
    xc, yc = compact_of(x, ys, xn, yn)
    exact = (int(xn.max()), int(yn.max()) + 1)
    for hints in (exact, (T + 13, U + 40), None):
        if hints is None:
            s, f = w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True)
        else:
            with w.compact_hints(*hints):
                s, f = w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True)
        assert same(s, sd) and torch.equal(padded_frames(f, yn, U), fd), hints
    # rows past the last lattice (a tensor sized for more than the lengths use) are never read
    extra = torch.full((37, V), float("nan"), device="cuda").to(dtype)
    with w.compact_hints(*exact):
        s, f = w.rnnt_align_from_logits(torch.cat([xc, extra]), yc, xn, yn, compact=True)
    assert same(s, sd) and torch.equal(padded_frames(f, yn, U), fd)
    # lattices above the hints: NaN, the others unchanged
    with w.compact_hints(exact[0] - 1, exact[1]):
        s, f = w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True)
    over = xn == exact[0]
    assert torch.isnan(s[over]).all() and same(s[~over], sd[~over])


@pytest.mark.parametrize("mode", ["regular", "modified", "constrained", "compact"])
def test_cuda_graph_capture_and_repeats(w, mode):
    N, T, U, V = 5, 60, 30, 10
    x, ys, xn, yn = make(N, T, U, V, seed=70)
    if mode == "compact":
        xc, yc = compact_of(x, ys, xn, yn)

    def call():
        if mode == "compact":
            with w.compact_hints(T, U):
                return w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True)
        return w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type=mode, delay_penalty=0.05)

    runs = [call() for _ in range(3)]
    for s, f in runs[1:]:
        assert same(s, runs[0][0]) and torch.equal(f, runs[0][1])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s_g, f_g = call()
    for _ in range(2):
        s_g.fill_(0.0)
        f_g.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        assert same(s_g, runs[0][0]) and torch.equal(f_g, runs[0][1])


# ------------------------------------------------------------------------------------------------ 5. refusals
def test_value_errors_and_binding_refusals_launch_nothing(w):
    x, ys, xn, yn = make(3, 10, 6, 5, seed=80)
    xc, yc = compact_of(x, ys, xn, yn)
    before = w._C.launch_count()
    for kw in ({"rnnt_type": "warped"}, {"rnnt_type": 1}, {"delay_penalty": -0.1}, {"delay_penalty": float("nan")},
               {"delay_penalty": float("inf")}, {"delay_penalty": True}):
        with pytest.raises(ValueError):
            w.rnnt_align_from_logits(x, ys, xn, yn, **kw)
    for kw in ({"rnnt_type": "modified"}, {"rnnt_type": "constrained"}, {"delay_penalty": 0.05}):
        with pytest.raises(ValueError):
            w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        w.rnnt_align_from_logits(x.cpu(), ys, xn, yn)
    with pytest.raises(RuntimeError, match="Float"):
        w.rnnt_align_from_logits(x.double(), ys, xn, yn, rnnt_type="modified")
    with pytest.raises(RuntimeError, match="Int"):
        w.rnnt_align_from_logits(x, ys.long(), xn, yn)
    with pytest.raises(RuntimeError, match="xn must be located in the CUDA"):
        w.rnnt_align_from_logits(x, ys, xn.cpu(), yn)
    with pytest.raises(RuntimeError, match="Float"):
        w.rnnt_align_from_logits(xc.half(), yc, xn, yn, compact=True)
    with pytest.raises(RuntimeError, match="blank"):
        w.rnnt_align_from_logits(x, ys, xn, yn, blank=5)
    assert w._C.launch_count() == before


def test_c_abi_refusals(w, lib):
    N, T, U, V = 3, 10, 6, 5
    x, ys, xn, yn = make(N, T, U, V, seed=90)
    sc = torch.full((N,), 5.0, device="cuda")
    fr = torch.full((N, U - 1), 5, dtype=torch.int32, device="cuda")
    need = lib.rnnt_b200_align_logits_workspace_bytes(N * T * U, N, T, U)
    ws = torch.empty(need + 64, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    xb = x.to(torch.bfloat16)

    def dense(ws_ptr=None, nbytes=need, xs=None, eb=4, kind=0, lam=0.0, Ux=U, s_ptr=None, f_ptr=None, blank=0):
        return lib.rnnt_b200_align_logits_dense(
            st, ws.data_ptr() if ws_ptr is None else ws_ptr, nbytes, x.data_ptr() if xs is None else xs,
            ys.data_ptr(), xn.data_ptr(), yn.data_ptr(), sc.data_ptr() if s_ptr is None else s_ptr,
            fr.data_ptr() if f_ptr is None else f_ptr, N, T, Ux, V, blank, eb, kind, lam)

    before = lib.rnnt_b200_launch_count()
    bad = {"type3": dict(kind=3), "type-1": dict(kind=-1), "lam<0": dict(lam=-0.5), "lam_nan": dict(lam=float("nan")),
           "lam_inf": dict(lam=float("inf")), "U>25600_modified": dict(kind=1, Ux=25601),
           "U>25600_constrained": dict(kind=2, Ux=25601), "scores": dict(s_ptr=0), "frames": dict(f_ptr=0),
           "eb3": dict(eb=3), "eb8": dict(eb=8), "misaligned_f32": dict(xs=x.data_ptr() + 2),
           "misaligned_bf16": dict(xs=xb.data_ptr() + 1, eb=2), "ws_misaligned": dict(ws_ptr=ws.data_ptr() + 8),
           "blank": dict(blank=V)}
    for name, kw in bad.items():
        assert dense(**kw) == INVALID, name
    assert dense(nbytes=need - 1) == SMALL and dense(nbytes=0) == SMALL
    xc, yc = compact_of(x, ys, xn, yn)
    STU = xc.shape[0]
    needc = lib.rnnt_b200_align_logits_workspace_bytes(STU, N, T, U)
    fc = torch.full((yc.numel(),), 5, dtype=torch.int32, device="cuda")

    def compact(nbytes=needc, eb=4, bounds=(T, U), s_ptr=None, ws_ptr=None):
        return lib.rnnt_b200_align_logits_compact(
            st, ws.data_ptr() if ws_ptr is None else ws_ptr, nbytes, xc.data_ptr(), yc.data_ptr(), xn.data_ptr(),
            yn.data_ptr(), sc.data_ptr() if s_ptr is None else s_ptr, fc.data_ptr(), STU, N, V, 0, eb, *bounds)

    assert compact(bounds=(0, U)) == INVALID and compact(bounds=(T, 0)) == INVALID and compact(eb=1) == INVALID
    assert compact(s_ptr=0) == INVALID and compact(ws_ptr=ws.data_ptr() + 4) == INVALID
    assert compact(nbytes=needc - 1) == SMALL
    assert lib.rnnt_b200_launch_count() == before
    torch.cuda.synchronize()
    assert (sc == 5.0).all() and (fr == 5).all() and (fc == 5).all()
    # and the valid calls run
    for kind in (0, 1, 2):
        assert dense(kind=kind, lam=0.05) == 0
        s0, f0 = w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type=list(KIND)[kind], delay_penalty=0.05)
        torch.cuda.synchronize()
        assert same(sc, s0) and torch.equal(fr, f0)
    assert dense(xs=xb.data_ptr(), eb=2) == 0
    assert compact() == 0
    torch.cuda.synchronize()
    s0, f0 = w.rnnt_align_from_logits(x, ys, xn, yn)
    assert same(sc, s0) and torch.equal(padded_frames(fc, yn, U), f0)
