"""GPU: rnnt_align_tdt, the Viterbi alignment on the TDT lattice, against the numpy restatement
(tests/tdt_align_oracle.py) bit for bit -- scores, frames and label durations -- on the kernel's own normaliser output;
every planner bound of tdt_plan with its launch record; self-consistency with rnnt_loss_tdt and an fp64 max-plus at
every shape; degenerate input; bf16 and compact parity; CUDA graphs, determinism, the C ABI and argument errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.tdt_align_oracle import align_np, logprobs
from tests.tdt_oracle import random_case
from tests.test_gpu_tdt import tdt_record
from tests.test_gpu_tdt_compact import at_offset, pack, pack_labels

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
SMEM_OPTIN = 227 * 1024
BF16 = torch.bfloat16


def dev(*ts):
    return [torch.as_tensor(t).to(DEV) for t in ts]


def kernel_lp(xd, labels, xn, yn, durations, sigma, blank):
    """the clamped log-probs the kernel reads, from the lse of its own normaliser (float32 subtractions)"""
    _, lse, _ = w._C.rnnt_tdt_forward(xd, labels, xn, yn, list(durations), sigma, blank, False)
    V = xd.shape[-1] - len(durations)
    return logprobs(xd.float().cpu().numpy(), lse.cpu().numpy(), V, sigma)


def same(a, b):
    """bit-identical float arrays, NaN where the other has NaN (of any payload)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and a[~nan].tobytes() == b[~nan].tobytes()


def consistency(xd, labels, xn, yn, durations, sigma, blank, scores, frames, fdur, lp):
    """frames in [0, Tn-1], label edges in order and inside the lattice, durations from the set; score <= -cost of
    the loss, the same classes; within 2^-23 (Tn + Un) |s64| of the fp64 max-plus over the same log-probs"""
    costs = w.rnnt_loss_tdt(xd, labels, xn, yn, durations, sigma=sigma, blank=blank).cpu().numpy().astype(np.float64)
    xn, yn = xn.cpu().numpy(), yn.cpu().numpy()
    s64 = align_np(lp, labels.cpu().numpy(), xn, yn, durations, blank, dtype=np.float64)[0]
    assert np.array_equal(np.isnan(scores), np.isnan(costs)), (scores, costs)
    assert np.array_equal(scores == -np.inf, costs == np.inf), (scores, costs)
    for n in range(len(scores)):
        if not np.isfinite(scores[n]):
            assert (frames[n] == -1).all() and (fdur[n] == -1).all()
            continue
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        f, d = frames[n, :Un - 1].astype(np.int64), fdur[n, :Un - 1].astype(np.int64)
        assert (f >= 0).all() and (f <= Tn - 1).all()
        assert np.isin(d, durations).all()
        assert (f[:-1] + d[:-1] <= f[1:]).all() and (Un == 1 or f[-1] + d[-1] <= Tn - 1)
        assert (frames[n, Un - 1:] == -1).all() and (fdur[n, Un - 1:] == -1).all()
        c = costs[n]
        assert scores[n] <= -c + 2e-6 * (1 + abs(c)), (n, scores[n], c)
        assert abs(float(scores[n]) - s64[n]) <= 2.0 ** -23 * (Tn + Un) * abs(s64[n]), (n, scores[n], s64[n])


def check(x, labels, xn, yn, durations, sigma=0.0, blank=0, expect=None):
    """f32 call on the device against align_np on the kernel's log-probs, bit for bit, plus the consistency checks;
    expect: launch record fields to assert"""
    xd = torch.as_tensor(x, dtype=torch.float32).to(DEV)
    ys, xnd, ynd = dev(labels, xn, yn)
    s, f, d = w.rnnt_align_tdt(xd, ys, xnd, ynd, durations, sigma=sigma, blank=blank)
    rec = tdt_record()
    for k, v in (expect or {}).items():
        assert rec[k] == v, (k, rec)
    assert rec["emit_vec"] == 0 and rec["emit_xvec"] == 0
    s, f, d = s.cpu().numpy(), f.cpu().numpy(), d.cpu().numpy()
    lp = kernel_lp(xd, ys, xnd, ynd, durations, sigma, blank)
    s0, f0, d0, paths = align_np(lp, np.asarray(labels), np.asarray(xn), np.asarray(yn), durations, blank)
    assert same(s, s0), (s, s0)
    assert np.array_equal(f, f0) and np.array_equal(d, d0)
    consistency(xd, ys, xnd, ynd, durations, sigma, blank, s, f, d, lp)
    return s, f, d, paths


# ---- 1. the oracle, bit for bit ---------------------------------------------------------------------------------

@pytest.mark.parametrize("durations", [(1,), (0, 1, 2, 3, 4), (0, 1, 2, 3, 4, 5), (0, 1, 16), tuple(range(17))])
@pytest.mark.parametrize("sigma", [0.0, 0.05])
def test_oracle(durations, sigma):
    rng = np.random.RandomState(len(durations) + int(sigma * 100))
    V = 9
    x, labels, xn, yn = random_case(rng, 6, 24, 7, V, durations)
    labels[1, 0] = 0                                   # a label equal to blank
    xn[2] = 1                                          # T = 1
    yn[3] = 0                                          # no labels
    check(x, labels, xn, yn, durations, sigma=sigma, blank=0)


@pytest.mark.parametrize("durations", [(0, 1, 2, 3, 4), (0, 1, 2, 3, 4, 5)])
def test_blank_last_and_label_equal_to_blank(durations):
    rng = np.random.RandomState(7)
    V = 11
    x, labels, xn, yn = random_case(rng, 5, 30, 8, V, durations)
    labels[0, 2] = V - 1
    check(x, labels, xn, yn, durations, sigma=0.05, blank=V - 1)


def test_no_labels_and_single_frame():
    rng = np.random.RandomState(8)
    x, labels, xn, yn = random_case(rng, 4, 10, 1, 6, (0, 1, 2))   # U = 1: no labels at all
    s, f, d, _ = check(x, labels, xn, yn, (0, 1, 2))
    assert f.shape == (4, 0) and np.isfinite(s).all()
    x, labels, xn, yn = random_case(rng, 4, 1, 5, 6, (0, 1, 2))    # T = 1: every label at frame 0 with d = 0
    s, f, d, _ = check(x, labels, xn, yn, (0, 1, 2))
    live = np.arange(4)[None, :] < yn[:, None]
    assert (f[live] == 0).all() and (d[live] == 0).all() and (f[~live] == -1).all()


def test_dead_lattices():
    rng = np.random.RandomState(18)
    durations = (0, 2, 3)
    x, labels, xn, yn = random_case(rng, 4, 12, 4, 6, durations)
    xn[1] = 1                                          # Tn < min(d > 0)
    x[2, :, :, 0] = -np.inf                            # every blank masked: no path above the dead threshold
    s, f, d, _ = check(x, labels, xn, yn, durations)
    assert s[1] == -np.inf and s[2] == -np.inf and np.isfinite(s[[0, 3]]).all()


def test_random_lengths():
    rng = np.random.RandomState(9)
    x, labels, xn, yn = random_case(rng, 12, 60, 15, 20, (0, 1, 2, 3, 4))
    check(x, labels, xn, yn, (0, 1, 2, 3, 4), sigma=0.05)


def test_c2_like_batch():
    rng = np.random.RandomState(10)
    x, labels, xn, yn = random_case(rng, 8, 150, 40, 28, (0, 1, 2, 3, 4))
    xn[:] = np.maximum(xn, 100)
    check(x, labels, xn, yn, (0, 1, 2, 3, 4))


def test_c4_batch():
    g = torch.Generator().manual_seed(11)
    N, T, U, V, durations = 4, 1500, 300, 50, (0, 1, 2, 3, 4)
    x = torch.randn(N, T, U, V + 5, generator=g)
    labels = torch.randint(1, V, (N, U - 1), generator=g, dtype=torch.int32)
    xn = torch.tensor([T, T - 37, T - 400, T - 3], dtype=torch.int32)
    yn = torch.tensor([U - 1, U - 20, U - 1, U - 150], dtype=torch.int32)
    check(x.numpy(), labels.numpy(), xn.numpy(), yn.numpy(), durations)


# ---- 2. every planner bound of tdt_plan, with its launch record ------------------------------------------------

def planner(N, T, U, V, durations, expect, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, T, U, V + len(durations), generator=g)
    labels = torch.randint(1, V, (N, U - 1), generator=g, dtype=torch.int32)
    xn = torch.randint(max(1, T // 2), T + 1, (N,), generator=g, dtype=torch.int32)
    yn = torch.randint(max(0, (U - 1) // 2), U, (N,), generator=g, dtype=torch.int32)
    xn[0], yn[0] = T, U - 1
    check(x.numpy(), labels.numpy(), xn.numpy(), yn.numpy(), durations, sigma=0.05, expect=expect)


@pytest.mark.parametrize("durations,kd", [((0, 1, 2, 3, 4), 5), ((0, 1, 2, 3, 4, 5), 17)])
def test_candidate_slots(durations, kd):
    planner(3, 40, 6, 7, durations, dict(kd=kd, ring=max(durations) + 2, warps=1, passes=1))


@pytest.mark.parametrize("U,warps,passes", [(32, 1, 1), (33, 2, 1), (512, 16, 1), (513, 16, 2), (2048, 16, 4),
                                            (2049, 16, 5)])
def test_column_passes(U, warps, passes):
    planner(2, 12, U, 6, (0, 1, 2), dict(warps=warps, passes=passes, ring=4, smem=4 * U * 4, kd=5))


@pytest.mark.parametrize("U", [SMEM_OPTIN // (18 * 4), SMEM_OPTIN // (18 * 4) + 1])
def test_ring_at_its_limit(U):
    """max(d) = 16: 18 ring slots; one column more and the sweep reads back from global memory"""
    fits = 18 * U * 4 <= SMEM_OPTIN
    planner(1, 20, U, 4, (0, 1, 16), dict(ring=18 if fits else 0, smem=18 * U * 4 if fits else 0))


def test_long_frames():
    planner(2, 1600, 9, 5, (0, 1, 2, 3, 4), dict(ring=6, warps=1))


# ---- 3. degenerate input ------------------------------------------------------------------------------------------

def align(x, labels, xn, yn, durations, **kw):
    s, f, d = w.rnnt_align_tdt(torch.as_tensor(x, dtype=torch.float32).to(DEV), *dev(labels, xn, yn), durations, **kw)
    return s.cpu().numpy(), f.cpu().numpy(), d.cpu().numpy()


def base_case():
    rng = np.random.RandomState(12)
    x, labels, xn, yn = random_case(rng, 5, 30, 8, 10, (0, 1, 2, 3, 4))
    xn[2], yn[2] = 25, 5
    return x, labels, xn, yn


def test_minus_inf_on_the_path_moves_it_and_off_the_path_not():
    durations = (0, 1, 2, 3, 4)
    x, labels, xn, yn = base_case()
    s0, f0, d0, paths = check(x, labels, xn, yn, durations)
    n = 2
    t, u, _, _ = next(e for e in paths[n] if e[2] == "l")
    on = x.copy()
    on[n, t, u, labels[n, u]] = -np.inf
    s1, f1, d1, _ = check(on, labels, xn, yn, durations)
    assert f1[n, u] != t and s1[n] <= s0[n]
    visited = {(e[0], e[1]) for e in paths[n]}
    tt, uu = next((a, b) for a in range(int(xn[n])) for b in range(int(yn[n])) if (a, b) not in visited)
    off = x.copy()
    off[n, tt, uu, labels[n, uu]] = -np.inf
    s2, f2, d2, _ = check(off, labels, xn, yn, durations)
    assert same(s2, s0) and np.array_equal(f2, f0) and np.array_equal(d2, d0)


def test_nan_in_a_row_no_path_visits():
    durations = (0, 1, 2, 3, 4)
    x, labels, xn, yn = base_case()
    _, _, _, paths = check(x, labels, xn, yn, durations)
    n = 2
    visited = {(e[0], e[1]) for e in paths[n]}
    t, u = next((a, b) for a in range(int(xn[n])) for b in range(int(yn[n]) + 1) if (a, b) not in visited)
    bad = x.copy()
    bad[n, t, u, 3] = np.nan
    s, f, d, _ = check(bad, labels, xn, yn, durations)
    assert np.isnan(s[n]) and (f[n] == -1).all() and (d[n] == -1).all()


def test_padding_nan_all_minus_inf_durations_invalid_lengths_and_isolation():
    durations = (0, 1, 2, 3, 4)
    x, labels, xn, yn = base_case()
    s0, f0, d0 = align(x, labels, xn, yn, durations)
    pad = x.copy()
    pad[2, 25:, :, :] = np.nan                          # padding rows of lattice 2 (Tn = 25, Un = 6)
    pad[2, :, 6:, :] = np.nan
    s, f, d = align(pad, labels, xn, yn, durations)
    assert same(s, s0) and np.array_equal(f, f0) and np.array_equal(d, d0)
    for kind in ("durations", "lengths"):
        bad, bxn = x.copy(), xn.copy()
        if kind == "durations":
            bad[2, 3, 1, 10:] = -np.inf
        else:
            bxn[2] = 31
        s, f, d, _ = check(bad, labels, bxn, yn, durations)
        assert np.isnan(s[2]) and (f[2] == -1).all() and (d[2] == -1).all()
        keep = np.arange(5) != 2
        sk, fk, dk = align(x[keep], labels[keep], xn[keep], yn[keep], durations)
        assert same(s[keep], sk) and np.array_equal(f[keep], fk) and np.array_equal(d[keep], dk)


# ---- 4. bf16 and compact parity -----------------------------------------------------------------------------------

@pytest.mark.parametrize("V,D", [(28, 4), (29, 4), (30, 4), (27, 4)])           # (V + D) % 4 = 0, 1, 2, 3
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_bf16_equals_f32_on_widened_logits(V, D, offset):
    durations = tuple(range(D))
    rng = np.random.RandomState(V + offset)
    x, labels, xn, yn = random_case(rng, 4, 20, 6, V, durations)
    xb = at_offset(torch.tensor(x, dtype=torch.float32).to(BF16).to(DEV), offset)
    xf = at_offset(xb.float(), offset)
    args = dev(labels, xn, yn)
    rb = w.rnnt_align_tdt(xb, *args, durations, sigma=0.05, blank=V - 1)
    rf = w.rnnt_align_tdt(xf, *args, durations, sigma=0.05, blank=V - 1)
    for a, b in zip(rb, rf):
        assert torch.equal(a, b)


def compact_case(seed, N=8, T=30, U=9, V=12, durations=(0, 1, 2, 3, 4), dtype=torch.float32):
    rng = np.random.RandomState(seed)
    x, labels, xn, yn = random_case(rng, N, T, U, V, durations)
    xn[1], yn[2] = 1, 0
    xt = torch.tensor(x, dtype=torch.float32).to(dtype).to(DEV)
    return xt, labels, xn, yn


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("hints", [False, True])
def test_compact_equals_dense(dtype, hints):
    durations = (0, 1, 2, 3, 4)
    T, U = 30, 9
    xt, labels, xn, yn = compact_case(13, T=T, U=U, dtype=dtype)
    ys, xnd, ynd = dev(labels, xn, yn)
    dense = w.rnnt_align_tdt(xt, ys, xnd, ynd, durations, sigma=0.05)
    xc, ysc = pack(xt, xn, yn), pack_labels(labels, yn).to(DEV)
    if hints:
        with w.compact_hints(T, U):
            comp = w.rnnt_align_tdt(xc, ysc, xnd, ynd, durations, sigma=0.05, compact=True)
    else:
        comp = w.rnnt_align_tdt(xc, ysc, xnd, ynd, durations, sigma=0.05, compact=True)
    assert torch.equal(comp[0], dense[0])
    yl = yn.tolist()
    for c, d in zip(comp[1:], dense[1:]):
        assert torch.equal(c, torch.cat([d[i, :yl[i]] for i in range(len(yl))]))


def test_compact_sample_exceeding_the_hints():
    durations = (0, 1, 2, 3, 4)
    xt, labels, xn, yn = compact_case(14, T=30, U=9)
    xn[0] = 29                                          # inside the hints below
    xn[3], yn[3] = 30, 8                                # above them
    ys, xnd, ynd = dev(labels, xn, yn)
    dense = w.rnnt_align_tdt(xt, ys, xnd, ynd, durations)
    with w.compact_hints(29, 9):
        s, f, d = w.rnnt_align_tdt(pack(xt, xn, yn), pack_labels(labels, yn).to(DEV), xnd, ynd, durations,
                                   compact=True)
    assert torch.isnan(s[3]) and torch.equal(s[:3], dense[0][:3]) and torch.equal(s[4:], dense[0][4:])
    lo, hi = int(yn[:3].sum()), int(yn[:4].sum())
    assert (f[lo:hi] == -1).all() and (d[lo:hi] == -1).all()


def test_compact_graph_capture_and_determinism():
    durations = (0, 1, 2, 3, 4)
    T, U = 30, 9
    xt, labels, xn, yn = compact_case(15, T=T, U=U)
    xc, ysc = pack(xt, xn, yn), pack_labels(labels, yn).to(DEV)
    xnd, ynd = dev(xn, yn)

    def call():
        with w.compact_hints(T, U):
            return w.rnnt_align_tdt(xc, ysc, xnd, ynd, durations, sigma=0.05, compact=True)

    r1, r2 = call(), call()
    for a, b in zip(r1, r2):
        assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = call()
    for k in range(2):
        for o in out:
            o.fill_(7)
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(out, r1):
            assert torch.equal(a, b), k


# ---- 5. determinism, the C ABI, argument errors -------------------------------------------------------------------

def test_dense_determinism_and_no_autograd():
    xt, labels, xn, yn = compact_case(16)
    xg = xt.clone().requires_grad_(True)
    r1 = w.rnnt_align_tdt(xg, *dev(labels, xn, yn), (0, 1, 2, 3, 4))
    r2 = w.rnnt_align_tdt(xt, *dev(labels, xn, yn), (0, 1, 2, 3, 4))
    for a, b in zip(r1, r2):
        assert torch.equal(a, b) and not a.requires_grad


def test_python_argument_errors():
    xt, labels, xn, yn = compact_case(17)
    args = dev(labels, xn, yn)
    for durations in ([], (0,), (2, 1), (0, 17), (1.0,)):
        with pytest.raises(ValueError, match="rnnt_align_tdt: durations"):
            w.rnnt_align_tdt(xt, *args, durations)
    for sigma in (-0.1, float("nan"), float("inf"), True):
        with pytest.raises(ValueError, match="rnnt_align_tdt: sigma"):
            w.rnnt_align_tdt(xt, *args, (0, 1), sigma=sigma)
    for blank in (-1, 12, True):
        with pytest.raises(ValueError, match="rnnt_align_tdt: blank"):
            w.rnnt_align_tdt(xt, *args, (0, 1, 2, 3, 4), blank=blank)
    with pytest.raises(ValueError, match="rnnt_align_tdt: logits"):
        w.rnnt_align_tdt(xt[0], *args, (0, 1, 2, 3, 4))
    with pytest.raises(ValueError, match=r"rnnt_loss_tdt: sigma must be a finite number >= 0, got -0\.1"):
        w.rnnt_loss_tdt(xt, *args, (0, 1), sigma=-0.1)


def test_c_abi_refuses_before_any_launch():
    lib = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    ws_bytes = lib.rnnt_b200_tdt_align_workspace_bytes
    ws_bytes.restype = ctypes.c_size_t
    ws_bytes.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int]
    fd = lib.rnnt_b200_tdt_align_dense
    fd.restype = ctypes.c_int
    head = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 5 + [ctypes.c_int, ctypes.c_float] + \
        [ctypes.c_void_p] * 3
    fd.argtypes = head + [ctypes.c_int] * 6
    fc = lib.rnnt_b200_tdt_align_compact
    fc.restype = ctypes.c_int
    fc.argtypes = head + [ctypes.c_int64] + [ctypes.c_int] * 6
    N, T, U, V = 2, 5, 3, 6
    durs = (ctypes.c_int * 3)(0, 1, 2)
    x = torch.zeros(N, T, U, V + 3, device=DEV)
    i32 = torch.zeros(N * U, dtype=torch.int32, device=DEV)
    sc = torch.full((N,), 5.0, device=DEV)
    fr = torch.full((N * U,), 5, dtype=torch.int32, device=DEV)
    need = ws_bytes(N * T * U, N, 3)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    base = [None, p(ws), need, p(x), p(i32), p(i32), p(i32), durs, 3, 0.0, p(sc), p(fr), p(fr), N, T, U, V, 0, 4]
    before = w._C.launch_count()
    bad = {"T": (14, 0), "blank": (17, V), "elem_bytes": (18, 3), "durations": (7, None), "sigma": (9, -1.0),
           "scores": (10, None), "frames": (11, None), "label_durations": (12, None), "ws_align": (1, ws.data_ptr() + 8)}
    for name, (i, v) in bad.items():
        a = list(base)
        a[i] = ctypes.c_void_p(v) if name == "ws_align" else v
        assert fd(*a) == 5, name
    a = list(base)
    a[2] = need - 1
    assert fd(*a) == 6
    cbase = [None, p(ws), need, p(x), p(i32), p(i32), p(i32), durs, 3, 0.0, p(sc), p(fr), p(fr), N * T * U, N, V, 0, 4,
             T, U]
    for i, v in ((18, 0), (19, 0), (11, None), (10, None)):
        a = list(cbase)
        a[i] = v
        assert fc(*a) == 5, i
    a = list(cbase)
    a[2] = need - 1
    assert fc(*a) == 6
    torch.cuda.synchronize()
    assert w._C.launch_count() == before
    assert (sc == 5.0).all() and (fr == 5).all()
