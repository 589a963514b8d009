"""GPU: rnnt_align_multiblank, the Viterbi alignment on the multi-blank lattice, against the numpy restatement
(tests/multiblank_align_oracle.py) bit for bit -- scores, frames and blank counts -- on the kernel's own normaliser
output; rnnt_align on the same log-probs when the big blanks are masked; self-consistency with rnnt_loss_multiblank and
an fp64 max-plus at every shape; the degenerate classes; bf16 and compact parity; CUDA graphs, determinism; every
planner bound with its launch record; the C ABI and argument errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.multiblank_align_oracle import align_np, logprobs
from tests.multiblank_oracle import random_case
from tests.test_gpu_tdt import tdt_record
from tests.test_gpu_tdt_compact import at_offset, pack, pack_labels

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
SMEM_OPTIN = 227 * 1024
BF16 = torch.bfloat16
DURATION_SETS = [(2,), (2, 4), (2, 4, 8), (2, 3, 5, 9, 16), (16,)]


def dev(*ts):
    return [torch.as_tensor(t).to(DEV) for t in ts]


def kernel_lp(xd, labels, xn, yn, durations, sigma, blank):
    """the clamped log-probs the kernel reads, from the lse of its own normaliser (float32 subtractions)"""
    _, lse, _ = w._C.rnnt_multiblank_forward(xd, labels, xn, yn, list(durations), sigma, blank, False)
    return logprobs(xd.float().cpu().numpy(), lse.cpu().numpy(), sigma)


def same(a, b):
    """bit-identical float arrays, NaN where the other has NaN (of any payload)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and a[~nan].tobytes() == b[~nan].tobytes()


def consistency(xd, labels, xn, yn, durations, sigma, blank, scores, frames, counts, lp):
    """frames in [0, Tn-1] and non-decreasing; counts[0] + sum_i d_i counts[1+i] = Tn; score <= -cost of the loss, the
    same classes; within 2^-23 (Tn + Un) |s64| of the fp64 max-plus over the same log-probs"""
    with torch.no_grad():
        costs = w.rnnt_loss_multiblank(xd, labels, xn, yn, durations, sigma=sigma, blank=blank)
    costs = costs.cpu().numpy().astype(np.float64)
    xn, yn = xn.cpu().numpy(), yn.cpu().numpy()
    s64 = align_np(lp, labels.cpu().numpy(), xn, yn, durations, blank, dtype=np.float64)[0]
    assert np.array_equal(np.isnan(scores), np.isnan(costs)), (scores, costs)
    assert np.array_equal(scores == -np.inf, costs == np.inf), (scores, costs)
    for n in range(len(scores)):
        if not np.isfinite(scores[n]):
            assert (frames[n] == -1).all() and (counts[n] == -1).all()
            continue
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        f = frames[n, :Un - 1].astype(np.int64)
        assert (f >= 0).all() and (f <= Tn - 1).all() and (np.diff(f) >= 0).all()
        assert (frames[n, Un - 1:] == -1).all()
        assert (counts[n] >= 0).all()
        assert counts[n, 0] + sum(d * counts[n, 1 + i] for i, d in enumerate(durations)) == Tn
        c = costs[n]
        assert scores[n] <= -c + 2e-6 * (1 + abs(c)), (n, scores[n], c)
        assert abs(float(scores[n]) - s64[n]) <= 2.0 ** -23 * (Tn + Un) * abs(s64[n]), (n, scores[n], s64[n])


def check(x, labels, xn, yn, durations, sigma=0.0, blank=None, expect=None):
    """f32 call on the device against align_np on the kernel's log-probs, bit for bit, plus the consistency checks;
    expect: launch record fields to assert"""
    xd = torch.as_tensor(x, dtype=torch.float32).to(DEV)
    b = x.shape[-1] - 1 if blank is None else blank
    ys, xnd, ynd = dev(labels, xn, yn)
    s, f, c = w.rnnt_align_multiblank(xd, ys, xnd, ynd, durations, sigma=sigma, blank=blank)
    rec = tdt_record()
    for k, v in (expect or {}).items():
        assert rec[k] == v, (k, rec)
    assert rec["emit_vec"] == 0 and rec["emit_xvec"] == 0
    assert s.dtype == torch.float32 and f.dtype == c.dtype == torch.int32 and c.shape == (len(xn), 1 + len(durations))
    s, f, c = s.cpu().numpy(), f.cpu().numpy(), c.cpu().numpy()
    lp = kernel_lp(xd, ys, xnd, ynd, durations, sigma, b)
    s0, f0, c0, paths = align_np(lp, np.asarray(labels), np.asarray(xn), np.asarray(yn), durations, b)
    assert same(s, s0), (s, s0)
    assert np.array_equal(f, f0) and np.array_equal(c, c0), (f, f0, c, c0)
    consistency(xd, ys, xnd, ynd, durations, sigma, b, s, f, c, lp)
    return s, f, c, paths


# ---- 1. the oracle, bit for bit ---------------------------------------------------------------------------------

@pytest.mark.parametrize("durations", DURATION_SETS)
@pytest.mark.parametrize("sigma", [0.0, 0.05])
@pytest.mark.parametrize("blank", ["default", "B"])
def test_oracle(durations, sigma, blank):
    B = len(durations)
    rng = np.random.RandomState(3 + B + durations[-1] + int(sigma * 100))
    V = B + 8
    x, labels, xn, yn = random_case(rng, 6, 24, 7, V, B)                 # ragged lengths
    b = None
    if blank == "B":
        b = B
        labels = labels + B + 1                                           # tokens above the blanks
    labels[1, 0] = V - 1 if b is None else b                              # a label equal to the standard blank
    xn[2] = 1                                                             # T = 1
    yn[3] = 0                                                             # no labels
    check(x, labels, xn, yn, durations, sigma=sigma, blank=b)
    rec = tdt_record()
    assert rec["ring"] == max(durations) + 1 and rec["kd"] == (5 if B <= 3 else 17)


def test_random_lengths():
    rng = np.random.RandomState(9)
    x, labels, xn, yn = random_case(rng, 12, 60, 15, 20, 3)
    check(x, labels, xn, yn, (2, 4, 8), sigma=0.05)


def test_c2_like_batch():
    rng = np.random.RandomState(10)
    x, labels, xn, yn = random_case(rng, 8, 150, 40, 32, 3)
    xn[:] = np.maximum(xn, 100)
    _, _, c, _ = check(x, labels, xn, yn, (2, 4, 8))
    assert (c[:, 1:] > 0).any()                                           # the big blanks are used


@pytest.mark.parametrize("durations", [(2, 4, 8), (2, 3, 5, 9, 16)])
def test_masked_big_blanks_equal_rnnt_align(durations):
    """every big blank at -inf, sigma = 0: scores and frames are rnnt_align's on the same log-probs, bit for bit"""
    B = len(durations)
    rng = np.random.RandomState(20 + B)
    V = B + 10
    x, labels, xn, yn = random_case(rng, 8, 40, 12, V, B)
    x[..., V - 1 - B:V - 1] = -np.inf
    xd = torch.tensor(x, dtype=torch.float32, device=DEV)
    ys, xnd, ynd = dev(labels, xn, yn)
    s, f, c = w.rnnt_align_multiblank(xd, ys, xnd, ynd, durations)
    _, lse, _ = w._C.rnnt_multiblank_forward(xd, ys, xnd, ynd, list(durations), 0.0, V - 1, False)
    s0, f0 = w.rnnt_align(xd - lse[..., None], ys, xnd, ynd, blank=V - 1)
    assert torch.equal(s, s0) and torch.equal(f, f0)
    assert torch.equal(c[:, 0], xnd) and (c[:, 1:] == 0).all()


# ---- 2. every planner bound, with its launch record -----------------------------------------------------------

def planner(N, T, U, V, durations, expect, seed=0):
    """the dense call against the oracle, then the compact call on the same rows: the same results and record"""
    B = len(durations)
    x, labels, xn, yn = random_case(np.random.RandomState(seed), N, T, U, V, B)
    xn[:], yn[0] = T, U - 1
    s, f, c, _ = check(x, labels, xn, yn, durations, sigma=0.05, expect=expect)
    xt = torch.tensor(x, dtype=torch.float32, device=DEV)
    with w.compact_hints(T, U):
        sc, fc, cc = w.rnnt_align_multiblank(pack(xt, xn, yn), pack_labels(labels, yn).to(DEV), *dev(xn, yn),
                                             durations, sigma=0.05, compact=True)
    rec = tdt_record()
    for k, v in expect.items():
        assert rec[k] == v, (k, rec)
    assert same(sc.cpu().numpy(), s) and np.array_equal(cc.cpu().numpy(), c)
    assert np.array_equal(fc.cpu().numpy(), np.concatenate([f[i, :yn[i]] for i in range(N)]))


@pytest.mark.parametrize("durations,kd", [((2, 4, 8), 5), ((2, 4, 8, 16), 17)])
def test_candidate_slots(durations, kd):
    planner(3, 40, 6, len(durations) + 6, durations, dict(kd=kd, ring=max(durations) + 1, warps=1, passes=1))


@pytest.mark.parametrize("U,warps,passes", [(512, 16, 1), (513, 16, 2), (1100, 16, 3)])
def test_column_passes(U, warps, passes):
    planner(2, 8, U, 7, (2, 4), dict(warps=warps, passes=passes, ring=5, smem=5 * U * 4))


@pytest.mark.parametrize("U", [SMEM_OPTIN // (17 * 4), SMEM_OPTIN // (17 * 4) + 1])
def test_ring_at_its_limit(U):
    """max(d) = 16: 17 ring slots; one column more and the sweep reads back from global memory"""
    fits = 17 * U * 4 <= SMEM_OPTIN
    planner(1, 20, U, 6, (2, 16), dict(ring=17 if fits else 0, smem=17 * U * 4 if fits else 0))


def test_long_frames():
    planner(2, 600, 9, 8, (2, 4, 8), dict(ring=9, warps=1))


# ---- 3. degenerate input ------------------------------------------------------------------------------------------

def align(x, labels, xn, yn, durations, **kw):
    r = w.rnnt_align_multiblank(torch.as_tensor(x, dtype=torch.float32).to(DEV), *dev(labels, xn, yn), durations, **kw)
    return [t.cpu().numpy() for t in r]


def base_case():
    rng = np.random.RandomState(12)
    x, labels, xn, yn = random_case(rng, 5, 30, 8, 11, 3)
    xn[2], yn[2] = 25, 5
    return x, labels, xn, yn


def test_minus_inf_on_the_path_moves_it_and_off_the_path_not():
    durations = (2, 4, 8)
    x, labels, xn, yn = base_case()
    s0, f0, c0, paths = check(x, labels, xn, yn, durations)
    n = 2
    t, u, _ = next(e for e in paths[n] if e[2] == 1)
    on = x.copy()
    on[n, t, u, labels[n, u]] = -np.inf
    _, f1, _, _ = check(on, labels, xn, yn, durations)
    assert f1[n, u] != t
    # off the path: the row's least likely token, so its other log-probs move by no more than about 0.005
    visited = {(e[0], e[1]) for e in paths[n]}
    tt, uu = next((a, b) for a in range(int(xn[n])) for b in range(int(yn[n])) if (a, b) not in visited)
    off = x.copy()
    off[n, tt, uu, int(np.argmin(x[n, tt, uu, :x.shape[-1] - 4]))] = -np.inf
    s2, f2, c2, _ = check(off, labels, xn, yn, durations)
    assert same(s2, s0) and np.array_equal(f2, f0) and np.array_equal(c2, c0)


@pytest.mark.parametrize("kind", ["lengths", "label", "nan", "posinf", "all_minus_inf", "nan_off_path", "dead"])
def test_degenerate_classes_and_isolation(kind):
    """each class on lattice 2: its score, frames and counts; every other lattice as in a batch without it"""
    durations = (2, 4, 8)
    x, labels, xn, yn = base_case()
    _, _, _, paths = check(x, labels, xn, yn, durations)
    n, V = 2, x.shape[-1]
    bad, bxn, blab = x.copy(), xn.copy(), labels.copy()
    if kind == "lengths":
        bxn[n] = 31
    elif kind == "label":
        blab[n, 1] = V
    elif kind == "nan":
        bad[n, 3, 1, 5] = np.nan
    elif kind == "posinf":
        bad[n, 0, 0, 0] = np.inf
    elif kind == "all_minus_inf":
        bad[n, 24, 5, :] = -np.inf
    elif kind == "nan_off_path":
        visited = {(e[0], e[1]) for e in paths[n]}
        t, u = next((a, b) for a in range(int(xn[n])) for b in range(int(yn[n]) + 1) if (a, b) not in visited)
        bad[n, t, u, 3] = np.nan
    else:
        bad[n, :, :, V - 4:] = -np.inf                                    # every blank masked: no path
    s, f, c, _ = check(bad, blab, bxn, yn, durations)
    assert (s[n] == -np.inf) if kind == "dead" else np.isnan(s[n])
    assert (f[n] == -1).all() and (c[n] == -1).all()
    keep = np.arange(5) != n
    sk, fk, ck = align(x[keep], labels[keep], xn[keep], yn[keep], durations)
    assert same(s[keep], sk) and np.array_equal(f[keep], fk) and np.array_equal(c[keep], ck)


def test_padding_rows_are_never_read():
    durations = (2, 4, 8)
    x, labels, xn, yn = base_case()
    s0, f0, c0 = align(x, labels, xn, yn, durations)
    pad = x.copy()
    pad[2, 25:, :, :] = np.nan                          # padding rows of lattice 2 (Tn = 25, Un = 6)
    pad[2, :, 6:, :] = np.nan
    s, f, c = align(pad, labels, xn, yn, durations)
    assert same(s, s0) and np.array_equal(f, f0) and np.array_equal(c, c0)


# ---- 4. bf16 and compact parity -----------------------------------------------------------------------------------

@pytest.mark.parametrize("V", [32, 33, 34, 35])                  # V % 4 = 0, 1, 2, 3
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_bf16_equals_f32_on_widened_logits(V, offset):
    durations = (2, 4, 8)
    rng = np.random.RandomState(V + offset)
    x, labels, xn, yn = random_case(rng, 4, 20, 6, V, 3)
    xb = at_offset(torch.tensor(x, dtype=torch.float32).to(BF16).to(DEV), offset)
    xf = at_offset(xb.float(), offset)
    args = dev(labels, xn, yn)
    rb = w.rnnt_align_multiblank(xb, *args, durations, sigma=0.05)
    rec_b = tdt_record()
    rf = w.rnnt_align_multiblank(xf, *args, durations, sigma=0.05)
    assert tdt_record()["norm_group"] == rec_b["norm_group"]
    for a, b in zip(rb, rf):
        assert torch.equal(a, b)


def compact_case(seed, N=8, T=30, U=9, V=12, B=3, dtype=torch.float32):
    rng = np.random.RandomState(seed)
    x, labels, xn, yn = random_case(rng, N, T, U, V, B)
    xn[1], yn[2] = 1, 0
    xt = torch.tensor(x, dtype=torch.float32).to(dtype).to(DEV)
    return xt, labels, xn, yn


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("hints", [False, True])
def test_compact_equals_dense(dtype, hints):
    durations = (2, 4, 8)
    T, U = 30, 9
    xt, labels, xn, yn = compact_case(13, T=T, U=U, dtype=dtype)
    ys, xnd, ynd = dev(labels, xn, yn)
    dense = w.rnnt_align_multiblank(xt, ys, xnd, ynd, durations, sigma=0.05)
    xc, ysc = pack(xt, xn, yn), pack_labels(labels, yn).to(DEV)
    if hints:
        with w.compact_hints(T, U):
            comp = w.rnnt_align_multiblank(xc, ysc, xnd, ynd, durations, sigma=0.05, compact=True)
    else:
        comp = w.rnnt_align_multiblank(xc, ysc, xnd, ynd, durations, sigma=0.05, compact=True)
    assert torch.equal(comp[0], dense[0]) and torch.equal(comp[2], dense[2])
    yl = yn.tolist()
    assert torch.equal(comp[1], torch.cat([dense[1][i, :yl[i]] for i in range(len(yl))]))


def test_compact_sample_exceeding_the_hints_and_rows_past_stu():
    durations = (2, 4, 8)
    xt, labels, xn, yn = compact_case(14, T=30, U=9)
    xn[0] = 29                                          # inside the hints below
    xn[3], yn[3] = 30, 8                                # above them
    ys, xnd, ynd = dev(labels, xn, yn)
    dense = w.rnnt_align_multiblank(xt, ys, xnd, ynd, durations)
    xc, ysc = pack(xt, xn, yn), pack_labels(labels, yn).to(DEV)
    with w.compact_hints(29, 9):
        s, f, c = w.rnnt_align_multiblank(xc, ysc, xnd, ynd, durations, compact=True)
    ok = torch.arange(8, device=DEV) != 3
    assert torch.isnan(s[3]) and torch.equal(s[ok], dense[0][ok]) and torch.equal(c[ok], dense[2][ok])
    lo, hi = int(yn[:3].sum()), int(yn[:4].sum())
    assert (f[lo:hi] == -1).all() and (c[3] == -1).all()
    # the last lattice's rows run past STU: NaN there, the others as dense
    rows = int(xn[7]) * (int(yn[7]) + 1)
    with w.compact_hints(30, 9):
        s, f, c = w.rnnt_align_multiblank(xc[:xc.shape[0] - (rows + 1) // 2], ysc, xnd, ynd, durations, compact=True)
    assert torch.isnan(s[7]) and torch.equal(s[:7], dense[0][:7]) and (c[7] == -1).all()
    assert (f[int(yn[:7].sum()):] == -1).all()


def test_compact_graph_capture_and_determinism():
    durations = (2, 4, 8)
    T, U = 30, 9
    xt, labels, xn, yn = compact_case(15, T=T, U=U)
    xc, ysc = pack(xt, xn, yn), pack_labels(labels, yn).to(DEV)
    xnd, ynd = dev(xn, yn)

    def call():
        with w.compact_hints(T, U):
            return w.rnnt_align_multiblank(xc, ysc, xnd, ynd, durations, sigma=0.05, compact=True)

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
    r1 = w.rnnt_align_multiblank(xg, *dev(labels, xn, yn), (2, 4, 8))
    r2 = w.rnnt_align_multiblank(xt, *dev(labels, xn, yn), (2, 4, 8))
    for a, b in zip(r1, r2):
        assert torch.equal(a, b) and not a.requires_grad


def test_python_argument_errors():
    xt, labels, xn, yn = compact_case(17)
    args = dev(labels, xn, yn)
    for durations in ([], (1,), (4, 2), (2, 17), (2.0,), (True,)):
        with pytest.raises(ValueError, match="rnnt_align_multiblank: big_blank_durations"):
            w.rnnt_align_multiblank(xt, *args, durations)
    for sigma in (-0.1, float("nan"), float("inf"), True):
        with pytest.raises(ValueError, match="rnnt_align_multiblank: sigma"):
            w.rnnt_align_multiblank(xt, *args, (2, 4), sigma=sigma)
    for blank in (-1, 2, 12, True):
        with pytest.raises(ValueError, match="rnnt_align_multiblank: blank"):
            w.rnnt_align_multiblank(xt, *args, (2, 4, 8), blank=blank)
    with pytest.raises(ValueError, match="rnnt_align_multiblank: logits"):
        w.rnnt_align_multiblank(xt[0], *args, (2, 4, 8))
    with pytest.raises(ValueError, match="rnnt_align_multiblank: logits"):
        w.rnnt_align_multiblank(xt, *args, (2, 4, 8), compact=True)


def test_c_abi_refuses_before_any_launch():
    lib = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    ws_bytes = lib.rnnt_b200_multiblank_align_workspace_bytes
    ws_bytes.restype = ctypes.c_size_t
    ws_bytes.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int]
    fd = lib.rnnt_b200_multiblank_align_dense
    fd.restype = ctypes.c_int
    head = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 5 + [ctypes.c_int, ctypes.c_float] + \
        [ctypes.c_void_p] * 3
    fd.argtypes = head + [ctypes.c_int] * 6
    fc = lib.rnnt_b200_multiblank_align_compact
    fc.restype = ctypes.c_int
    fc.argtypes = head + [ctypes.c_int64] + [ctypes.c_int] * 6
    N, T, U, V, B = 2, 5, 3, 8, 3
    durs = (ctypes.c_int * B)(2, 4, 8)
    bad_durs = (ctypes.c_int * B)(2, 8, 4)
    x = torch.zeros(N, T, U, V, device=DEV)
    i32 = torch.zeros(N * U, dtype=torch.int32, device=DEV)
    sc = torch.full((N,), 5.0, device=DEV)
    fr = torch.full((N * (1 + B) + N * U,), 5, dtype=torch.int32, device=DEV)
    need = ws_bytes(N * T * U, N, B)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    base = [None, p(ws), need, p(x), p(i32), p(i32), p(i32), durs, B, 0.0, p(sc), p(fr), p(fr), N, T, U, V, V - 1, 4]
    before = w._C.launch_count()
    bad = {"T": (14, 0), "blank_high": (17, V), "blank_low": (17, B - 1), "elem_bytes": (18, 3), "durations": (7, None),
           "order": (7, bad_durs), "B": (8, 0), "sigma": (9, -1.0), "sigma_nan": (9, float("nan")),
           "scores": (10, None), "frames": (11, None), "counts": (12, None), "ws_align": (1, ws.data_ptr() + 8)}
    for name, (i, v) in bad.items():
        a = list(base)
        a[i] = ctypes.c_void_p(v) if name == "ws_align" else v
        assert fd(*a) == 5, name
    a = list(base)
    a[2] = need - 1
    assert fd(*a) == 6
    cbase = [None, p(ws), need, p(x), p(i32), p(i32), p(i32), durs, B, 0.0, p(sc), p(fr), p(fr), N * T * U, N, V,
             V - 1, 4, T, U]
    for i, v in ((18, 0), (19, 0), (16, V), (7, bad_durs), (12, None), (11, None), (10, None)):
        a = list(cbase)
        a[i] = v
        assert fc(*a) == 5, i
    a = list(cbase)
    a[2] = need - 1
    assert fc(*a) == 6
    torch.cuda.synchronize()
    assert w._C.launch_count() == before
    assert (sc == 5.0).all() and (fr == 5).all()
