"""k2's rnnt_type ("modified", "constrained") and delay_penalty on every path their calls take, against fp64
(tests/path_oracle.py, tests/smoothed_oracle.factorised), at the shapes and edges where the kernels could go wrong.

  B. k_frames (csrc/frames.cu) where its columns are live.  A CTA has min(512, roundup32(U)) threads and a thread
     handles three kinds of columns, each with its own load code: u < bd (prefetch slot 0), bd <= u < 2 bd (prefetch
     slot 1, loaded one frame ahead) and u >= 2 bd (loaded in their own step).  The case table reaches each of them
     with a live lattice, and the largest shared memory (U = 25600, 50 column passes) with padding columns; every case
     asserts its frames launch record and checks the flow identities on every frame.  Then: U = 25600 with every
     column live against the streaming fp64 sweep, U = 25601 refused before any launch, NaN isolation in the high
     columns, padding invariance across thread counts and passes, and bf16 in the in-step columns.
  C. rnnt_loss_pruned with the new types on real windows (rnnt_loss_simple's, and random monotone ones around a
     modified path) against path_oracle.pruned, f32 and bf16, and its dead lattices.
  D. regular + delay_penalty on rnnt_loss_pruned (fused and general path), rnnt_loss_from_logits (c4, with FastEmit)
     and rnnt_loss_simple; and rnnt_loss_simple with the new types, d am and d lm against the extended factorised().

Every case prints one "types-err <case> <kind> <lambda> <dtype> ... ratio=" line: its largest error over its bound."""
import ctypes
import os
import time

import numpy as np
import pytest
import torch

from tests import path_oracle as pa
from tests import smoothed_oracle as sm
from tests.test_gpu_fused_emit import subprocess_outputs
from tests.test_gpu_launch_configs import FUSED, GENERAL, Launch, expect
from tests.test_gpu_path_types import (KIND, REC_CONSTRAINED, REC_DELAY, REC_GRAD_BLOCKS, REC_PASSES, REC_SMEM,
                                       REC_THREADS, cu, lib, loss_pairs, make, pairs_of, record, simple_ex,
                                       simple_inputs, w)  # noqa: F401 (lib, w: the fixtures)
from tests.test_gpu_pruned_paths import CASES as PRUNED_CASES
from tests.test_gpu_pruned_paths import case_inputs as pruned_case_inputs
from tests.test_gpu_pruned_paths import grad_bound, picked
from tests.test_gpu_simple import check as check_plain
from tests.test_gpu_simple_paths import CASES as SIMPLE_CASES
from tests.test_gpu_simple_paths import case_inputs as simple_case_inputs
from tests.test_gpu_simple_paths import scales_name
from tests.test_gpu_simple_smoothed import check as check_smoothed

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
EXACT, FAST = 1, 2
MODES = {EXACT: "exact", FAST: "fast"}
INVALID = 5                                   # RNNT_STATUS_INVALID_ARGUMENT
TYPES = ["modified", "constrained"]
LAMS = [0.0, 0.05]


def report(case, kind, lam, dtype, **kv):
    """one "types-err" line; kv ends with err and bound, whose ratio closes the line and must be <= 1"""
    err, bound = kv.pop("err"), kv.pop("bound")
    rest = " ".join("%s=%.3g" % (k, v) for k, v in kv.items())
    print("types-err %s %s %g %s %s err=%.3g bound=%.3g ratio=%.3f" % (case, kind, lam, dtype, rest, err, bound,
                                                                       err / bound))
    return err / bound


def threads_for(U):
    return min(512, max(32, (U + 31) // 32 * 32))


def expect_frames(lib, kind, U, lam, what):
    """the frames launch record of the last call: its type, threads, column passes, shared memory, grad grid, delay"""
    rec = record(lib, frames=True)
    th = threads_for(U)
    got = dict(constrained=rec[REC_CONSTRAINED], threads=rec[REC_THREADS], passes=rec[REC_PASSES],
               smem=rec[REC_SMEM], delay=rec[REC_DELAY])
    want = dict(constrained=int(kind == "constrained"), threads=th, passes=-(-U // th), smem=8 * U,
                delay=int(lam != 0))
    assert got == want and rec[REC_GRAD_BLOCKS] > 0, (what, got, want, rec)
    return rec


def walk(A, steps):
    """2^-23 A sqrt(steps): one fp32 rounding of a log-value of size A per step, adding up as a random walk"""
    return 2.0 ** -23 * A * steps ** 0.5


def flow_bound(Un, A, Tn):
    """1e-5 sqrt(Un), plus walk(A, Tn) with A the size of alpha and beta along the paths.  Every occupation of a frame
    is exp(alpha + w + beta - ll) with alpha, beta and ll from separate fp32 sweeps of Tn steps, so a frame's sum is
    off by their common error, about walk(A, Tn), whatever the kernel's columns do (without a penalty, A is about the
    cost: 0.7e-3 to 2e-3 at the 800-3,000 nats of the random-logit cases below, past 1e-5 sqrt(Un) = 2.5e-4)."""
    return 1e-5 * Un ** 0.5 + walk(A, Tn)


def flow_error(pg, Tn, Un, kind, chunk=2048):
    """Largest deviation, in fp64 over the GPU's own pair gradients (N,T,U,2) of one lattice, from the identities that
    hold for any pairs: modified -sum_u (gb + gl)(t, u) = 1 and constrained -sum_u gb(t, u) = 1 (the fold puts the
    label edge into the blank slot) on every frame t < Tn, each taking exactly one edge; and -sum_t gl(t, u) = 1 on
    every label column u < Un - 1, each label emitted once (so -sum gl = Un - 1)."""
    worst = 0.0
    col = torch.zeros(max(Un - 1, 0), dtype=torch.float64, device=pg.device)
    for t0 in range(0, Tn, chunk):
        g = pg[t0:min(t0 + chunk, Tn), :Un].double()
        frame = -(g[..., 0] + g[..., 1]).sum(1) if kind == "modified" else -g[..., 0].sum(1)
        worst = max(worst, (frame - 1).abs().max().item())
        col -= g[:, :Un - 1, 1].sum(0)
    if Un > 1:
        worst = max(worst, (col - 1).abs().max().item())
    return worst


# ================================================================================ B. the frame sweep's columns
# name -> (N, T, U, V, xn, yn): what it reaches
FRAMES = {
    # bd = 512: columns 512-639 through prefetch slot 1 (lattice 1: 512-560)
    "slot1": (2, 700, 640, 4, [700, 660], [639, 560]),
    # columns 1024-1099 through the in-step loop, one iteration (lattice 1: 1024-1060)
    "instep": (2, 1200, 1100, 4, [1200, 1150], [1099, 1060]),
    # columns 1024-2099: the in-step loop iterating three times (u = tid + 1024, + 1536, + 2048)
    "instep3": (1, 2200, 2100, 4, [2200], [2099]),
    # the largest shared memory (200 KB) and 50 column passes, every column past 301 padding
    "pad_25600": (2, 300, 25600, 2, [300, 280], [300, 250]),
}


@pytest.mark.parametrize("lam", LAMS)
@pytest.mark.parametrize("kind", TYPES)
@pytest.mark.parametrize("name", list(FRAMES))
def test_frames_columns(w, lib, name, kind, lam):
    """From logits, against the fp64 restatement on the same f32 pairs: costs within 1e-5 |c| + walk(A, Tn), pair
    gradients within test_gpu_pruned_paths.grad_bound, and the flow identities on every frame of the GPU's pair
    gradients within flow_bound, where A = |cost| + lam Tn^2 / 8 is the size of alpha and beta along the paths: the
    penalty piles up lam ((Tn-1)/2 - t) over the first half of the frames (nearly every frame emits a label here) and
    gives it back over the second, so at lam = 0.05 alpha reaches 3,000-30,000 nats while the costs are a few hundred,
    and 1e-5 relative alone is below one fp32 rounding of alpha (slot1: 1.6e-3 on a cost of -35)."""
    N, T, U, V, xn_, yn_ = FRAMES[name]
    x, ys, xn, yn = make(N, T, U, V, seed=sum(map(ord, name)), xn=xn_, yn=yn_)
    c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    expect_frames(lib, kind, U, lam, name)
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    c0, g0, _ = pa.lattice(pa.penalise(pairs_of(x, lse, ys).cpu().numpy(), xh, yh, lam), xh, yh, kind)
    assert np.isfinite(c0).all()
    c = c.cpu().numpy().astype(np.float64)
    A = np.abs(c0) + lam * xh.astype(np.float64) ** 2 / 8
    cost_err = (np.abs(c - c0) / (1e-5 * np.abs(c0) + walk(A, xh))).max()
    Tm, Um = int(xh.max()), int(yh.max()) + 1
    bound = grad_bound(Tm, Um, A)
    err = np.abs(pg.cpu().numpy() - g0).max()
    ratio = report(name, kind, lam, "f32", cost_ratio=cost_err, err=err, bound=bound)
    fl, fb = 0.0, 0.0
    for n in range(N):
        Tn, Un = int(xh[n]), int(yh[n]) + 1
        fl = max(fl, flow_error(pg[n], Tn, Un, kind))
        fb = max(fb, flow_bound(Un, A[n], Tn))
    fratio = report(name + "/flow", kind, lam, "f32", err=fl, bound=fb)
    assert cost_err <= 1 and ratio <= 1 and fratio <= 1, (name, kind, lam, cost_err, err, bound, fl, fb)


def big_row(seed, t, U):
    """frame t's (U, 2) pair row of the U = 25600 case, from its own seed, in [-2e-3, 0]"""
    return -np.random.default_rng([seed, t]).uniform(0.0, 2e-3, (U, 2)).astype(np.float32)


@pytest.mark.parametrize("lam", [0.0, 1e-5])
@pytest.mark.parametrize("kind", TYPES)
def test_the_bound_u25600(w, lib, kind, lam):
    """rnnt_b200_loss_pairs_ex at U = kFramesMaxU = 25600 with every column live: N = 1, Tn = 25600, Un = 25598 (3
    blank frames, C(25600, 3) = 2.8e12 paths), pairs drawn per frame in [-2e-3, 0], delay_penalty 0 and 1e-5, against
    path_oracle.stream on the same rows.  Along the paths alpha stays within a few tens of nats without the penalty;
    the penalty moves it by up to lam Tn^2 / 8 = 820 nats at mid-sweep (cancelled again by beta), where one fp32
    rounding is 6e-5.  Each bound therefore adds 4 walk(A, Tn), A the largest |alpha| on a path in the kept frames:
    costs 1e-5 |c| + 4 walk(A, Tn); pair gradients of frames {0, 1, 12799, 25597, 25598, 25599} within
    1e-6 + (1e-3 + 4 walk(A, Tn)) |g0|; the flow identities on every frame within 1e-5 sqrt(Un) + 4 walk(A, Tn).
    The factor 4: 25,600 LSE roundings of the same sign-biased kind add up faster than a random walk.  A plain numpy
    float32 restatement of the sweep (the kernel's clamp and exact LSE) misses the fp64 cost by 0.0526 (modified) and
    0.0451 (constrained) at lam = 1e-5, exactly what this kernel misses it by on an H100, against walk(A, Tn) = 0.0158;
    at lam = 0 both errors are below 1e-4.  About 21 GB of device memory, freed afterwards."""
    T = U = 25600
    Tn, Un, seed = 25600, 25598, 7 + KIND[kind]
    keep = [0, 1, 12799, 25597, 25598, 25599]
    start = time.time()
    pairs = torch.empty((1, T, U, 2), device="cuda")
    for t0 in range(0, T, 512):
        rows = np.stack([big_row(seed, t, U) for t in range(t0, min(t0 + 512, T))])
        pairs[0, t0:t0 + len(rows)].copy_(torch.from_numpy(rows))
    xn = torch.tensor([Tn], dtype=torch.int, device="cuda")
    yn = torch.tensor([Un - 1], dtype=torch.int, device="cuda")
    try:
        c, pg = loss_pairs(lib, pairs, xn, yn, kind, lam)
        torch.cuda.synchronize()
        expect_frames(lib, kind, U, lam, "u25600")
        del pairs
        gpu_done = time.time()
        c0, g0, A = pa.stream_grads(lambda t: big_row(seed, t, U), Tn, Un, kind, keep, lam)
        cpu_done = time.time()
        assert np.isfinite(c0)
        A = max(A, abs(c0))
        cerr, cb = abs(float(c.item()) - c0), 1e-5 * abs(c0) + 4 * walk(A, Tn)
        report("u25600/cost", kind, lam, "f32", cost=c0, alpha_max=A, err=cerr, bound=cb)
        gerr = 0.0
        for t in keep:
            g = pg[0, t, :Un].double().cpu().numpy()
            gerr = max(gerr, (np.abs(g - g0[t]) / (1e-6 + (1e-3 + 4 * walk(A, Tn)) * np.abs(g0[t]))).max())
        report("u25600/grads", kind, lam, "f32", err=gerr, bound=1.0)
        fl, fb = flow_error(pg[0], Tn, Un, kind), flow_bound(Un, 4 * A, Tn)
        report("u25600/flow", kind, lam, "f32", err=fl, bound=fb)
        print("types-time u25600 %s gpu+upload %.1f s, fp64 stream %.1f s" % (kind, gpu_done - start,
                                                                             cpu_done - gpu_done))
        assert cerr <= cb and gerr <= 1 and fl <= fb, (cerr, cb, gerr, fl, fb)
    finally:
        pairs = c = pg = None
        torch.cuda.empty_cache()


def test_u25601_is_refused_before_any_launch(w, lib):
    """U = kFramesMaxU + 1 is refused by every entry of the new types before any launch; regular takes it."""
    N, T, U, V = 1, 3, 25601, 2
    x, ys, xn, yn = make(N, T, U, V, seed=3, xn=[3], yn=[2])
    am, lm, ys2, xn2, yn2 = simple_inputs(N, T, U, 5, 4)
    rng = torch.zeros((N, T), dtype=torch.int, device="cuda")
    pairs = pairs_of(x, torch.zeros((N, T, U), device="cuda"), ys)
    nbytes = lib.rnnt_b200_workspace_bytes(N * T * U, N)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    c = torch.full((N,), 7.0, device="cuda")
    pg = torch.full((N, T, U, 2), 7.0, device="cuda")
    sbytes = lib.rnnt_b200_simple_smoothed_workspace_bytes(N, T, U, 5)
    sws = torch.empty(sbytes, dtype=torch.uint8, device="cuda")
    saved = torch.empty(N * T * U + 2 * N * T + 2 * N * U + 5, device="cuda")
    torch.cuda.synchronize()
    before = w._C.launch_count()
    for kind in TYPES:
        for lam in LAMS:
            kw = dict(rnnt_type=kind, delay_penalty=lam)
            with pytest.raises(RuntimeError):
                w.rnnt_loss_from_logits(x, ys, xn, yn, **kw)
            with pytest.raises(RuntimeError):
                w.rnnt_loss_pruned(x[:, :, :2].contiguous(), ys, xn, yn, rng, **kw)
            with pytest.raises(RuntimeError):
                w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, **kw)
            st = lib.rnnt_b200_loss_pairs_ex(s, ws.data_ptr(), nbytes, pairs.data_ptr(), xn.data_ptr(),
                                             yn.data_ptr(), c.data_ptr(), pg.data_ptr(), N, T, U, 0.0, 0, KIND[kind],
                                             lam)
            assert st == INVALID, st
            st = lib.rnnt_b200_simple_smoothed_forward_ex(s, sws.data_ptr(), sbytes, am.data_ptr(), lm.data_ptr(),
                                                          ys2.data_ptr(), xn2.data_ptr(), yn2.data_ptr(), c.data_ptr(),
                                                          saved.data_ptr(), pg.data_ptr(), N, T, U, 5, 0, 0, 0.0, 0.0,
                                                          KIND[kind], lam, None)
            assert st == INVALID, st
    torch.cuda.synchronize()
    assert w._C.launch_count() == before
    assert (c == 7.0).all() and (pg == 7.0).all()
    for lam in LAMS:
        cr = w.rnnt_loss_from_logits(x, ys, xn, yn, delay_penalty=lam)
        cs = w.rnnt_loss_simple(am, lm, ys2, xn2, yn2, delay_penalty=lam)
        assert torch.isfinite(cr).all() and torch.isfinite(cs).all()


@pytest.mark.parametrize("kind", TYPES)
def test_nan_in_high_columns_is_isolated(w, lib, kind):
    """A NaN logit in a live cell at column 600 (prefetch slot 1) of lattice 0 and at column 1050 (the in-step loop)
    of lattice 2: those two get cost NaN and NaN on every live pair slot; lattices 1 and 3 are bit for bit a batch of
    only them."""
    N, T, U, V = 4, 1100, 1100, 4
    x, ys, xn, yn = make(N, T, U, V, seed=61, xn=[700, 1100, 1100, 900], yn=[650, 1080, 1099, 850])
    x[0, 300, 600, 2] = float("nan")
    x[2, 500, 1050, 0] = float("nan")
    lam = 0.05
    c, _, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    expect_frames(lib, kind, U, lam, "nan")
    for n in (0, 2):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        assert torch.isnan(c[n]), (n, c[n])
        assert torch.isnan(pg[n, :Tn, :Un, 0]).all() and torch.isnan(pg[n, :Tn, :Un - 1, 1]).all(), n
    keep = [1, 3]
    ck, _, pk = w._C.rnnt_logits_forward(x[keep].contiguous(), ys[keep], xn[keep], yn[keep], 0, 0.0, True, 0,
                                         KIND[kind], lam)
    assert torch.isfinite(ck).all()
    assert torch.equal(c[keep], ck) and torch.equal(pg[keep], pk)


@pytest.mark.parametrize("kind", TYPES)
def test_padding_invariance(w, lib, kind):
    """The same lattice (Tn = 150, Un = 100) at U = 100, 1100 and 25600 -- 128 / 512 / 512 threads, 1 / 3 / 50 column
    passes, different row strides, random padding columns: the same costs, normalisers and live pair gradients, bit
    for bit."""
    T, Un, V, lam = 150, 100, 4, 0.05
    base, ys0, xn, yn = make(1, T, Un, V, seed=71, xn=[T], yn=[Un - 1])
    out = []
    for U in (100, 1100, 25600):
        x, ys, _, _ = make(1, T, U, V, seed=U)
        x[:, :, :Un] = base
        ys[:, :Un - 1] = ys0
        c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
        expect_frames(lib, kind, U, lam, "U=%d" % U)
        out.append((c, lse[:, :, :Un], pg[:, :, :Un]))
    assert torch.isfinite(out[0][0]).all()
    for o in out[1:]:
        assert all(torch.equal(p, q) for p, q in zip(out[0], o))


@pytest.mark.parametrize("lam", LAMS)
@pytest.mark.parametrize("kind", TYPES)
def test_bf16_in_the_instep_columns(w, lib, kind, lam):
    """bf16 logits at the instep case: the f32 call on the widened logits, bit for bit; the gradient rounded once."""
    N, T, U, V, xn_, yn_ = FRAMES["instep"]
    x, ys, xn, yn = make(N, T, U, V, seed=81, xn=xn_, yn=yn_)
    xb = x.to(BF16)
    cb, lb, pb = w._C.rnnt_logits_forward(xb, ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    expect_frames(lib, kind, U, lam, "bf16")
    cf, lf, pf = w._C.rnnt_logits_forward(xb.float(), ys, xn, yn, 0, 0.0, True, 0, KIND[kind], lam)
    assert torch.isfinite(cb).all()
    assert torch.equal(cb, cf) and torch.equal(lb, lf) and torch.equal(pb, pf)
    go = torch.linspace(0.5, 1.5, N, device="cuda")
    gb = w._C.rnnt_logits_backward(xb, lb, pb, ys, go, 0)
    assert gb.dtype == BF16
    assert torch.equal(gb, w._C.rnnt_logits_backward(xb.float(), lf, pf, ys, go, 0).to(BF16))


# ================================================================================ C. pruned with the new types
# name -> (kind, S, N, T, U, V)
PRUNED = {
    "m_s1": ("modified", 1, 12, 50, 16, 24),
    "m_s4": ("modified", 4, 12, 50, 16, 24),
    "c_s2": ("constrained", 2, 12, 50, 16, 24),
    "c_s5": ("constrained", 5, 12, 50, 16, 24),
    # the profiled pipeline shape (tools/path_types_time.py): 8 picked lattices against fp64
    "m_profiled": ("modified", 5, 32, 500, 100, 500),
    "c_profiled": ("constrained", 5, 32, 500, 100, 500),
}


def step_windows(rng, xn, yn, T, S, kind):
    """Monotone windows moving by at most one column a frame around a random modified path (one label or none per
    frame): r_t = clip(u_t - d_t, 0, Un - S), u_t the path's column at frame t, the offset d_t in [0, S - 1] (S - 2
    constrained, whose label edge also reads the blank of the cell it reaches) moving only where that keeps the step
    in {0, 1}.  So every window holds its frame's part of the path, and the constrained one the cell reached."""
    top = S - 1 - (kind == "constrained")
    N = len(xn)
    r = np.zeros((N, T), np.int64)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        e = np.zeros(Tn, np.int64)
        e[rng.choice(Tn, Un - 1, replace=False)] = 1
        u = np.concatenate([[0], np.cumsum(e)[:-1]])
        d = np.zeros(Tn, np.int64)
        d[0] = rng.randint(0, top + 1)
        for t in range(1, Tn):
            d[t] = d[t - 1]
            if rng.rand() < 0.3:
                d[t] = min(d[t] + 1, top) if e[t - 1] else max(d[t] - 1, 0)
        r[n, :Tn] = np.maximum(np.minimum(u - d, Un - S), 0)
        r[n, Tn:] = r[n, Tn - 1]
    assert (np.diff(r, axis=1) >= 0).all() and (np.diff(r, axis=1) <= 1).all()
    return r.astype(np.int32)


def pruned_inputs(name, windows, w):
    """-> (x (N,T,S,V) bf16-representable, ys, xn, yn, ranges) as numpy: the windows of rnnt_loss_simple(...,
    rnnt_type=kind, prune_range=S) on random am / lm, or step_windows()."""
    kind, S, N, T, U, V = PRUNED[name]
    seed = sum(map(ord, name + windows))
    am, lm, ys, xn, yn = simple_inputs(N, T, U, V, seed)
    if windows == "simple":
        _, r = w.rnnt_loss_simple(am, lm, ys, xn, yn, prune_range=S, rnnt_type=kind)
        r = r.cpu().numpy()
    else:
        r = step_windows(np.random.RandomState(seed), xn.cpu().numpy(), yn.cpu().numpy(), T, S, kind)
    rng = np.random.RandomState(seed + 1)
    x = torch.from_numpy((rng.randn(N, T, S, V) * 2).astype(np.float32)).to(BF16).float().numpy()
    return x, ys.cpu().numpy(), xn.cpu().numpy(), yn.cpu().numpy(), r


def pruned_call(w, x, ys, xn, yn, r, go, dtype=torch.float32, **kw):
    """rnnt_loss_pruned through autograd -> (costs, logit gradient)"""
    a = (x if torch.is_tensor(x) else cu(x)).to(dtype).detach().requires_grad_(True)
    c = w.rnnt_loss_pruned(a, cu(ys), cu(xn), cu(yn), cu(r), **kw)
    (c * go).sum().backward()
    return c.detach(), a.grad


@pytest.mark.parametrize("lam", LAMS)
@pytest.mark.parametrize("windows", ["simple", "step"])
@pytest.mark.parametrize("name", list(PRUNED))
def test_pruned_types(w, lib, name, windows, lam):
    """Costs 1e-5 relative and the window-logit gradient within grad_bound of path_oracle.pruned (bf16: plus
    2^-8 |g|, and the f32 result on the same values with the gradient rounded once), non-uniform grad_output."""
    kind, S, N, T, U, V = PRUNED[name]
    x, ys, xn, yn, r = pruned_inputs(name, windows, w)
    pick = picked(N)
    go_np = np.linspace(0.5, 1.5, N)
    go = cu(go_np.astype(np.float32))
    c0, g0 = pa.pruned(x[pick], ys[pick], xn[pick], yn[pick], r[pick], 0, kind, lam, grad_output=go_np[pick])
    fin = np.isfinite(c0)
    assert fin.all(), c0                                           # both kinds of windows keep a path
    tol = grad_bound(T, U, c0[fin])
    c, g = pruned_call(w, x, ys, xn, yn, r, go, rnnt_type=kind, delay_penalty=lam)
    expect_frames(lib, kind, U, lam, name)
    cn, gn = c.cpu().numpy()[pick].astype(np.float64), g.cpu().numpy()[pick]
    assert np.array_equal(np.isinf(cn), ~fin)
    np.testing.assert_allclose(cn[fin], c0[fin], rtol=1e-5)
    cost_rel = np.abs(cn[fin] - c0[fin]).max() / np.abs(c0[fin]).max()
    err = np.abs(gn - g0).max()
    ratio = report("%s/%s" % (name, windows), kind, lam, "f32", S=S, cost_rel=cost_rel, err=err, bound=tol)
    cb, gb = pruned_call(w, x, ys, xn, yn, r, go, BF16, rnnt_type=kind, delay_penalty=lam)
    assert torch.equal(cb, c) and torch.equal(gb, g.to(BF16))
    errb = (np.abs(gb.float().cpu().numpy()[pick] - g0) - 2.0 ** -8 * np.abs(g0)).max()
    ratio_b = report("%s/%s" % (name, windows), kind, lam, "bf16", S=S, cost_rel=cost_rel, err=errb, bound=tol)
    assert ratio <= 1 and ratio_b <= 1, (err, errb, tol)


@pytest.mark.parametrize("kind", TYPES)
def test_pruned_types_dead_lattices(w, lib, kind):
    """Windows with a gap, more labels than frames, and (constrained) S = 1: cost +inf and exactly zero gradient rows,
    as path_oracle.pruned says; the live lattices are bit for bit a batch of only them and match fp64."""
    N, T, S, U, V, lam = 6, 30, 4, 12, 10, 0.05
    rng = np.random.RandomState(91 + KIND[kind])
    xn = np.array([30, 25, 5, 30, 28, 20], np.int32)
    yn = np.array([11, 9, 8, 11, 6, 10], np.int32)              # lattice 2: Un - 1 = 8 > Tn = 5
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    batches = []
    r = step_windows(rng, np.where(xn > yn, xn, yn + 1), yn, T, S, kind)
    for n, ts in ((1, 10), (5, 3)):                              # gaps: frames <= ts in [0, S), after it from S + 1 on
        r[n, :ts + 1] = 0
        r[n, ts + 1:] = S + 1
    batches.append((S, r, [1, 2, 5]))
    if kind == "constrained":                                    # S = 1: no label edge keeps its reached blank
        yn1 = yn.copy()
        yn1[[0, 4]] = 0                                          # Un = 1: the lattices that keep their path
        batches.append((1, np.zeros((N, T), np.int32), [1, 2, 3, 5]))
    for S_, r_, dead in batches:
        yy = yn1 if S_ == 1 else yn
        x = torch.from_numpy((rng.randn(N, T, S_, V) * 2).astype(np.float32)).to(BF16).float().numpy()
        go_np = np.linspace(0.5, 1.5, N)
        go = cu(go_np.astype(np.float32))
        c, g = pruned_call(w, x, ys, xn, yy, r_, go, rnnt_type=kind, delay_penalty=lam)
        c0, g0 = pa.pruned(x, ys, xn, yy, r_, 0, kind, lam, grad_output=go_np)
        live = np.setdiff1d(np.arange(N), dead)
        assert np.isinf(c0[dead]).all() and np.isfinite(c0[live]).all()
        c, g = c.cpu().numpy(), g.cpu().numpy()
        assert (c[dead] == np.inf).all() and (g[dead] == 0).all(), (S_, c)
        cs, gs = pruned_call(w, x[live], ys[live], xn[live], yy[live], r_[live], go[cu(live).long()], rnnt_type=kind,
                             delay_penalty=lam)
        assert np.array_equal(c[live], cs.cpu().numpy()) and np.array_equal(g[live], gs.cpu().numpy())
        np.testing.assert_allclose(c[live], c0[live], rtol=1e-5)
        assert np.abs(g[live] - g0[live]).max() <= grad_bound(T, U, c0[live])


# ================================================================================ D. regular + penalty, simple types
PRUNED_REGULAR = ["general_u300", "fused_c2_u40"]
LAM_REG = 0.05


def _general_main(out_dir):
    """Subprocess body (RNNT_B200_PATH=general): exact-mode outputs of fused_c2_u40 with the penalty on the general
    path."""
    import warp_rnnt_b200 as w_
    assert os.environ.get("RNNT_B200_PATH") == "general"
    for k, t in fused_with_penalty(w_, "fused_c2_u40").items():
        np.save(os.path.join(out_dir, "%s.npy" % k), t.cpu().numpy())


def fused_with_penalty(w_, name):
    x, ys, xn, yn, r, blank, fe = pruned_case_inputs(name)
    N = len(xn)
    args = (cu(ys), cu(xn), cu(yn), cu(r))
    with Launch() as L:
        c, l, p = w_._C.rnnt_logits_pruned_forward(cu(x), *args, blank, fe, True, EXACT, 0, LAM_REG)
    want = GENERAL if os.environ.get("RNNT_B200_PATH") == "general" else FUSED
    assert L.rec["path"] == want, (name, L.rec)
    g = w_._C.rnnt_logits_pruned_backward(cu(x), l, p, cu(ys), cu(r), torch.linspace(0.5, 1.5, N, device="cuda"),
                                          blank)
    return dict(costs=c, lse=l, pairs=p, grads=g)


@pytest.fixture(scope="module")
def general_outputs():
    return subprocess_outputs("RNNT_B200_PATH", "general", "_general_main",
                              module="tests.test_gpu_path_types_paths")


@pytest.mark.parametrize("name", PRUNED_REGULAR)
def test_pruned_regular_penalty(w, general_outputs, name):
    """rnnt_loss_pruned, regular, delay_penalty 0.05 (with the case's FastEmit) on test_gpu_pruned_paths' cases: the
    case's launch record, costs 1e-5 relative and gradients within grad_bound of path_oracle.pruned, in both LSE
    modes; in exact mode the fused case equals the general path bit for bit."""
    N, T, S, U, V, _, _, _, want = PRUNED_CASES[name]
    x, ys, xn, yn, r, blank, fe = pruned_case_inputs(name)
    pick = picked(N)
    go_np = np.linspace(0.5, 1.5, N)
    go = cu(go_np.astype(np.float32))
    c0, g0 = pa.pruned(x[pick], ys[pick], xn[pick], yn[pick], r[pick], blank, "regular", LAM_REG, fe,
                       grad_output=go_np[pick])
    assert np.isfinite(c0).all()
    tol = grad_bound(T, U, c0)
    for mode in (EXACT, FAST):
        a = cu(x).requires_grad_(True)
        w.set_lse_mode(MODES[mode])
        try:
            with Launch() as L:
                c = w.rnnt_loss_pruned(a, cu(ys), cu(xn), cu(yn), cu(r), blank=blank, fastemit_lambda=fe,
                                       delay_penalty=LAM_REG)
            (c * go).sum().backward()
        finally:
            w.set_lse_mode("auto")
        c, g = c.detach(), a.grad
        expect(L.rec, want, "%s %s" % (name, MODES[mode]))
        cn, gn = c.cpu().numpy()[pick], g.cpu().numpy()[pick]
        cost_rel = np.abs(cn - c0).max() / np.abs(c0).max()
        np.testing.assert_allclose(cn, c0, rtol=1e-5)
        err = np.abs(gn - g0).max()
        ratio = report("%s/%s" % (name, MODES[mode]), "regular", LAM_REG, "f32", fastemit=fe, cost_rel=cost_rel,
                       err=err, bound=tol)
        assert ratio <= 1
    if want["path"] == FUSED:
        for k, t in fused_with_penalty(w, name).items():
            assert t.cpu().numpy().tobytes() == general_outputs["%s.npy" % k].tobytes(), (name, k)


@pytest.mark.parametrize("fe", [0.0, 0.01])
def test_from_logits_regular_penalty_c4(w, lib, fe):
    """rnnt_loss_from_logits at c4's size (N=4 T=1500 U=300 V=50), regular, delay_penalty 0.05, with and without
    FastEmit, on the general path: costs 1e-5 relative, pair gradients within grad_bound of path_oracle.lattice on the
    penalised pairs, the label gradients scaled by 1 + fastemit_lambda (pruned_oracle.lattice's rule)."""
    N, T, U, V = 4, 1500, 300, 50
    x, ys, xn, yn = make(N, T, U, V, seed=1850)
    with Launch() as L:
        c, lse, pg = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, fe, True, 0, 0, LAM_REG)
    expect(L.rec, dict(path=GENERAL), "c4")
    xh, yh = xn.cpu().numpy(), yn.cpu().numpy()
    c0, g0, _ = pa.lattice(pa.penalise(pairs_of(x, lse, ys).cpu().numpy(), xh, yh, LAM_REG), xh, yh, "regular")
    g0[..., 1] *= 1.0 + fe
    assert np.isfinite(c0).all()
    c = c.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(c, c0, rtol=1e-5)
    cost_rel = np.abs(c - c0).max() / np.abs(c0).max()
    tol = grad_bound(T, U, c0)
    err = np.abs(pg.cpu().numpy() - g0).max()
    assert report("c4", "regular", LAM_REG, "f32", fastemit=fe, cost_rel=cost_rel, err=err, bound=tol) <= 1


SIMPLE_NAMES = ["v_small", "profiled_b", "tile_129"]
SIMPLE_TYPES = [("regular", LAM_REG), ("modified", 0.0), ("modified", LAM_REG), ("constrained", 0.0),
                ("constrained", LAM_REG)]
SCALES = [(0.0, 0.0), (0.25, 0.0), (0.1, 0.1)]


@pytest.mark.parametrize("kind,lam", SIMPLE_TYPES, ids=["%s-%g" % k for k in SIMPLE_TYPES])
@pytest.mark.parametrize("scales", SCALES, ids=scales_name)
@pytest.mark.parametrize("name", SIMPLE_NAMES)
def test_simple_types(w, lib, name, scales, kind, lam):
    """rnnt_loss_simple with a type and a penalty on test_gpu_simple_paths' cases, both LSE modes: costs, d am and
    d lm against factorised(..., rnnt_type=, delay_penalty=) within test_gpu_simple.check's /
    test_gpu_simple_smoothed.check's bounds; the launch record of the case (regular) or of the frame sweep."""
    N, T, U, V, _, _, _, want, _ = SIMPLE_CASES[name]
    am, lm, ys, xn, yn, blank = simple_case_inputs(name)
    go = np.linspace(0.5, 1.5, N)
    ref = sm.factorised(am, lm, ys, xn, yn, blank, *scales, grad_output=go, rnnt_type=kind, delay_penalty=lam)
    assert np.isfinite(ref[0]).all()
    du = None
    if scales[1] > 0:
        du = ref[2] - sm.factorised(am, lm, ys, xn, yn, blank, *scales, grad_output=go, detach_unigram=True,
                                    rnnt_type=kind, delay_penalty=lam)[2]
    ref = tuple(ref) + (du,)
    for mode in (EXACT, FAST):
        a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
        w.set_lse_mode(MODES[mode])
        try:
            if kind == "regular":
                with Launch() as L:
                    c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), blank=blank, lm_only_scale=scales[0],
                                           am_only_scale=scales[1], delay_penalty=lam)
                expect(L.rec, want, "%s %s" % (name, MODES[mode]))
            else:
                c = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), blank=blank, lm_only_scale=scales[0],
                                       am_only_scale=scales[1], rnnt_type=kind, delay_penalty=lam)
                expect_frames(lib, kind, U, lam, name)
            (c * cu(go.astype(np.float32))).sum().backward()
        finally:
            w.set_lse_mode("auto")
        c, dam, dlm = c.detach().cpu().numpy(), a.grad.cpu().numpy(), l.grad.cpu().numpy()
        if scales == (0.0, 0.0):
            cost_rel, err, bound, ratio = check_plain(c, dam, dlm, ref, go)
        else:
            cost_rel, err, bound, ratio = check_smoothed(c, dam, dlm, ref, lm, go, scales[1])
        report("simple/%s/%s/%s" % (name, scales_name(scales), MODES[mode]), kind, lam, "f32", cost_rel=cost_rel,
               err=err, bound=bound)
        assert ratio <= 1


@pytest.mark.parametrize("S,scales", [(2, (0.0, 0.0)), (5, (0.25, 0.0)), (5, (0.1, 0.1))])
def test_simple_regular_penalty_ranges(w, lib, S, scales):
    """rnnt_loss_simple(..., delay_penalty=0.05, prune_range=S) at profiled_b: the ranges are path_oracle.prune_ranges
    on the GPU's own pair gradients of the penalised lattice, bit for bit, and they move."""
    am, lm, ys, xn, yn, blank = simple_case_inputs("profiled_b")
    assert blank == 0
    args = [cu(t) for t in (am, lm, ys, xn, yn)]
    c, r = w.rnnt_loss_simple(*args, prune_range=S, lm_only_scale=scales[0], am_only_scale=scales[1],
                              delay_penalty=LAM_REG)
    c2, pg, _ = simple_ex(lib, *args, "regular", LAM_REG, *scales)
    assert torch.equal(c, c2)
    c3 = w.rnnt_loss_simple(*args, lm_only_scale=scales[0], am_only_scale=scales[1])
    assert (c != c3).any()                                       # the penalty reached the costs
    want = pa.prune_ranges(pg.cpu().numpy(), xn, yn, S, "regular")
    r = r.cpu().numpy()
    assert np.array_equal(r, want)
    assert (np.diff(r, axis=1) > 0).sum() > len(xn)
