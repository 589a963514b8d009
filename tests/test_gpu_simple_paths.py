"""rnnt_loss_simple, plain and smoothed, on every path its calls take, against the factorised fp64 restatement
(tests/smoothed_oracle.factorised), which needs no (N,T,U,V) tensor and so reaches the shapes the loss is used at.

Each case of the table names the launch record its forward must make and sits on an edge of the kernels of
csrc/simple.cu:
  * k_simple_mm's 64 x 64 tiles and K steps of 16: T, U, Tn and Un just below, on and just above a multiple of 64, so
    that whole tiles lie past a lattice (they must still write their zeros), V below one K step and one past a multiple
    of it, and kMmDlm's reduction over K = Tn up to 1500;
  * the grid-stride loops of the row kernels (row_grid caps their grids at 16 CTAs per SM): grid_strides() derives each
    launch from the device's SM count and every case asserts which loops it makes iterate;
  * N = 65535, the largest batch (its contractions put N on gridDim.z), with k_prune_ranges' and k_smooth_G's largest
    grids and scans; T = 1500 for k_prune_ranges' 47 passes of 32 frames and its suffix minima across 32-frame blocks;
  * labels equal to blank (they take both terms, as in autograd), on the fused and the general path.

Checks, for the plain loss, (lm_only_scale, am_only_scale) = (0.25, 0) (icefall's) and (0.1, 0.1) (k2's), both LSE
modes, a per-lattice grad_output: costs 1e-5 relative and d am, d lm within test_gpu_simple.check's /
test_gpu_simple_smoothed.check's bounds, printed as "simple-err <case> <mode> <scales> ..." lines; in exact mode a
fused case equals the general path bit for bit (costs, saved, pair gradients, ranges, d am, d lm); at the largest
cases a second call gives the same bits.  Then: the ranges at scale are the rule on the GPU's own pair gradients and
keep a path for rnnt_loss_pruned; and the C ABI writes every output element, checked on buffers filled with NaN."""
import os

import numpy as np
import pytest
import torch

from tests import simple_oracle as so
from tests import smoothed_oracle as sm
from tests.test_gpu_fused_emit import subprocess_outputs
from tests.test_gpu_launch_configs import FUSED, GENERAL, Launch, expect, sms
from tests.test_gpu_simple import check as check_plain
from tests.test_gpu_simple import make
from tests.test_gpu_simple_smoothed import abi
from tests.test_gpu_simple_smoothed import check as check_smoothed

pytestmark = pytest.mark.gpu
EXACT, FAST = 1, 2
MODES = {EXACT: "exact", FAST: "fast"}
SCALES = [(0.0, 0.0), (0.25, 0.0), (0.1, 0.1)]
ROW_THREADS = 256                             # kRowThreads (csrc/simple.cu)
ROW_CAP = 16                                  # row_grid: at most 16 CTAs per SM


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# name -> (N, T, U, V, blank, (xn, yn) or None, share of labels set to blank, launch record of the forward, row-kernel
#          loops that iterate more than once (grid_strides))
CASES = {
    # (Tn, Un) = (64, 64), (63, 63), (1, 1): one whole tile, one short of it, one cell; V = one K step
    "tile_64": (3, 64, 64, 16, 0, ([64, 63, 1], [63, 62, 0]), 0.0, dict(path=FUSED, C=2), ()),
    # (65, 65), (64, 64), (2, 1): the second row / column tile holds one row / column, or lies wholly past the lattice
    "tile_65": (3, 65, 65, 17, 1, ([65, 64, 2], [64, 63, 0]), 0.0, dict(path=FUSED, C=4), ()),
    # (129, 129), (128, 128), (65, 1): three tiles each way; V = one 64-wide tile of d am / d lm plus one column and
    # 4 K steps + 1; a quarter of the labels equal to blank
    "tile_129": (3, 129, 129, 65, 2, ([129, 128, 65], [128, 127, 0]), 0.25, dict(path=GENERAL, warps=5), ()),
    # V < 16: one partial K step; a quarter of the labels equal to blank
    "v_small": (4, 40, 20, 15, 3, None, 0.25, dict(path=FUSED, C=1), ()),
    # DESIGN.md 3.6's shapes
    "profiled_b": (32, 500, 100, 500, 0, None, 0.0, dict(path=GENERAL, warps=4), ("row_offsets", "mix")),
    "profiled_v1024": (32, 600, 150, 1024, 0, None, 0.0, dict(path=GENERAL, warps=5),
                       ("row_offsets", "am_norm", "mix")),
    "c4": (64, 1500, 300, 50, 0, None, 0.0, dict(path=GENERAL, warps=10),
           ("row_offsets", "am_norm", "lm_rows_bwd", "mix")),
    # gridDim.z = 65535; every row kernel's loop iterates
    "n65535": (65535, 6, 9, 16, 0, None, 0.0, dict(path=FUSED, C=1),
               ("row_offsets", "am_norm", "lm_rows_bwd", "sparse", "cols", "mix")),
}
FUSED_CASES = [k for k, c in CASES.items() if c[7]["path"] == FUSED]


def case_inputs(name):
    N, T, U, V, blank, lens, share, _, _ = CASES[name]
    seed = sum(map(ord, name))
    am, lm, ys, xn, yn = make(N, T, U, V, seed=seed, blank=blank)
    if lens is not None:
        xn, yn = np.asarray(lens[0], np.int32), np.asarray(lens[1], np.int32)
    if share:
        rng = np.random.RandomState(seed)
        ys[rng.rand(*ys.shape) < share] = blank
        assert (ys[0] == blank).any()
    return am, lm, ys, xn, yn, blank


def grid_strides(N, T, U, n_sm):
    """The grid-stride loops of csrc/simple.cu's row kernels on n_sm SMs -> the set of those in which a thread
    iterates more than once.  row_grid(rows, per_cta) = min(ceil(rows / per_cta), 16 n_sm): a warp per row
    (k_row_offsets over N(T+U) rows, k_smooth_am_norm over N T, k_smooth_lm_rows_bwd over N U; 8 rows per CTA) or a
    thread per row (k_simple_sparse over N(T+U), k_smooth_cols over N U columns, k_smooth_mix over N T U cells)."""
    out = set()
    for name, rows, per in (("row_offsets", N * (T + U), ROW_THREADS // 32), ("am_norm", N * T, ROW_THREADS // 32),
                            ("lm_rows_bwd", N * U, ROW_THREADS // 32), ("sparse", N * (T + U), ROW_THREADS),
                            ("cols", N * U, ROW_THREADS), ("mix", N * T * U, ROW_THREADS)):
        grid = max(1, min(-(-rows // per), ROW_CAP * n_sm))
        if rows > grid * per:
            out.add(name)
    return out


def scales_name(scales):
    return "plain" if scales == (0.0, 0.0) else "sl=%g,sa=%g" % scales


def reference(name, scales):
    """factorised() on the case at these scales, with grad_output linspace(0.5, 1.5, N), and with sa > 0 the
    unigram's own term of d lm (the difference to the detached-unigram d lm) -> (costs, d am, d lm, pair grads, du)."""
    am, lm, ys, xn, yn, blank = case_inputs(name)
    go = np.linspace(0.5, 1.5, len(xn))
    c0, da0, dl0, pg0 = sm.factorised(am, lm, ys, xn, yn, blank, *scales, grad_output=go)
    du = None
    if scales[1] > 0:
        du = dl0 - sm.factorised(am, lm, ys, xn, yn, blank, *scales, grad_output=go, detach_unigram=True)[2]
    return c0, da0, dl0, pg0, du


def run(w, am, lm, ys, xn, yn, blank, scales, mode, S=None):
    """-> (costs, ranges or None, d am, d lm, launch record of the forward), through autograd."""
    N = len(xn)
    a, l = cu(am).requires_grad_(True), cu(lm).requires_grad_(True)
    w.set_lse_mode(MODES[mode])
    try:
        with Launch() as L:
            out = w.rnnt_loss_simple(a, l, cu(ys), cu(xn), cu(yn), blank=blank, prune_range=S,
                                     lm_only_scale=scales[0], am_only_scale=scales[1])
        c, r = out if S is not None else (out, None)
        (c * torch.linspace(0.5, 1.5, N, device="cuda")).sum().backward()
    finally:
        w.set_lse_mode("auto")
    return c.detach(), r, a.grad, l.grad, L.rec


# ------------------------------------------------------------------------------------------ the general path's side
def _general_main(out_dir):
    """Subprocess body (RNNT_B200_PATH=general): exact-mode outputs of the fused cases on the general path."""
    import warp_rnnt_b200 as w
    assert os.environ.get("RNNT_B200_PATH") == "general"
    for name in FUSED_CASES:
        for scales in SCALES:
            for k, t in exact_outputs(w, name, scales).items():
                np.save(os.path.join(out_dir, "%s_%s_%s.npy" % (name, scales_name(scales), k)), t.cpu().numpy())


def exact_outputs(w, name, scales, S=4):
    """The forward (with ranges of S) and the backward of the case in exact mode, through the operator module."""
    am, lm, ys, xn, yn, blank = case_inputs(name)
    N = len(xn)
    a, l, args = cu(am), cu(lm), (cu(ys), cu(xn), cu(yn))
    with Launch() as L:
        c, saved, pg, r = w._C.rnnt_simple_forward(a, l, *args, blank, True, S, EXACT, *scales)
    want = GENERAL if os.environ.get("RNNT_B200_PATH") == "general" else FUSED
    assert L.rec["path"] == want, (name, L.rec)
    dam, dlm = w._C.rnnt_simple_backward(a, l, *args, saved, pg, torch.linspace(0.5, 1.5, N, device="cuda"), blank,
                                         *scales)
    return dict(costs=c, saved=saved, pair_grads=pg, ranges=r, dam=dam, dlm=dlm)


@pytest.fixture(scope="module")
def general_outputs():
    return subprocess_outputs("RNNT_B200_PATH", "general", "_general_main", module="tests.test_gpu_simple_paths")


# ------------------------------------------------------------------------------------------ the cases
@pytest.mark.parametrize("scales", SCALES, ids=scales_name)
@pytest.mark.parametrize("name", list(CASES))
def test_simple_path(w, general_outputs, name, scales):
    N, T, U, V, _, _, _, want, strides = CASES[name]
    am, lm, ys, xn, yn, blank = case_inputs(name)
    got = grid_strides(N, T, U, sms())
    assert set(strides) <= got, (name, sorted(got))
    ref = reference(name, scales)
    assert np.isfinite(ref[0]).all()
    go = np.linspace(0.5, 1.5, N)
    for mode in (EXACT, FAST):
        c, _, dam, dlm, rec = run(w, am, lm, ys, xn, yn, blank, scales, mode)
        expect(rec, want, "%s %s %s" % (name, MODES[mode], scales_name(scales)))
        c, dam, dlm = c.cpu().numpy(), dam.cpu().numpy(), dlm.cpu().numpy()
        if scales == (0.0, 0.0):
            cost_rel, err, bound, ratio = check_plain(c, dam, dlm, ref, go)
        else:
            cost_rel, err, bound, ratio = check_smoothed(c, dam, dlm, ref, lm, go, scales[1])
        print("simple-err %s %s %s cost_rel=%.3g grad_err=%.3g bound=%.3g ratio=%.3f"
              % (name, MODES[mode], scales_name(scales), cost_rel, err, bound, ratio))
        if name in ("c4", "n65535"):
            # a second call, with ranges: the same bits
            c2, r2, dam2, dlm2, _ = run(w, am, lm, ys, xn, yn, blank, scales, mode, S=5)
            c3, r3, dam3, dlm3, _ = run(w, am, lm, ys, xn, yn, blank, scales, mode, S=5)
            assert c2.cpu().numpy().tobytes() == c.tobytes()
            assert torch.equal(c2, c3) and torch.equal(r2, r3) and torch.equal(dam2, dam3) and torch.equal(dlm2, dlm3)
    if name in FUSED_CASES:
        for k, t in exact_outputs(w, name, scales).items():
            theirs = general_outputs["%s_%s_%s.npy" % (name, scales_name(scales), k)]
            assert t.cpu().numpy().tobytes() == theirs.tobytes(), (name, scales, k)


# ------------------------------------------------------------------------------------------ ranges at scale
@pytest.mark.parametrize("name,S,scales", [("profiled_b", 2, (0.0, 0.0)), ("profiled_b", 5, (0.25, 0.0)),
                                           ("c4", 2, (0.0, 0.0)), ("c4", 5, (0.25, 0.0)), ("c4", 40, (0.1, 0.1))])
def test_ranges_at_scale(w, name, S, scales):
    """The ranges are the rule (simple_oracle.prune_ranges) on the GPU's own pair gradients bit for bit and have its
    properties; on the simple joint's windows rnnt_loss_pruned keeps every cost finite and no lower than the full
    cost (the plain simple loss's: pruning removes paths)."""
    am, lm, ys, xn, yn, blank = case_inputs(name)
    N, T, U, _, _, _, _, want, _ = CASES[name]
    assert all(so.reachable(int(x), int(y) + 1, S) for x, y in zip(xn, yn))
    at, lt, args = cu(am), cu(lm), (cu(ys), cu(xn), cu(yn))
    with Launch() as L:
        c, saved, pg, r = w._C.rnnt_simple_forward(at, lt, *args, blank, True, S, EXACT, *scales)
    expect(L.rec, want, name)
    r = r.cpu().numpy()
    np.testing.assert_array_equal(r, so.prune_ranges(pg.cpu().numpy(), xn, yn, S))
    so.check_ranges(r, xn, yn, S, U)
    assert (np.diff(r, axis=1) > 0).sum() > N                   # the windows move
    full = w.rnnt_loss_simple(at, lt, *args, blank=blank)
    idx = (cu(r).long()[:, :, None] + torch.arange(S, device="cuda")).clamp(max=U - 1)          # (N,T,S)
    n = torch.arange(N, device="cuda")[:, None, None]
    xw = (at[:, :, None, :] + lt[n, idx]).contiguous()           # the simple joint's rows in the windows
    pruned = w.rnnt_loss_pruned(xw, *args, cu(r), blank=blank)
    assert torch.isfinite(pruned).all() and torch.isfinite(full).all()
    assert (pruned >= full - 1e-5 * full.abs()).all(), (pruned, full)


# ------------------------------------------------------------------------------------------ every output written
def cabi_call(lib, am, lm, ys, xn, yn, blank, scales, fill, want, S=3):
    """The C ABI forward (with pair gradients; its launch record must be `want`), prune ranges and backward, every
    output buffer and the workspace filled with `fill` beforehand -> dict of the outputs as numpy arrays."""
    N, T, V = am.shape
    U = lm.shape[1]
    smooth = scales[0] > 0 or scales[1] > 0
    a, l, y, x, n = cu(am), cu(lm), cu(ys), cu(xn), cu(yn)
    s = torch.cuda.current_stream().cuda_stream
    nbytes = lib.rnnt_b200_simple_smoothed_workspace_bytes(N, T, U, V)
    ws = torch.full((nbytes // 4,), fill, device="cuda")
    saved = torch.full((N * T * U + N * T + N * U + (N * T + N * U + V if smooth else 0),), fill, device="cuda")
    out = dict(costs=torch.full((N,), fill, device="cuda"), saved=saved,
               pair_grads=torch.full((N, T, U, 2), fill, device="cuda"),
               ranges=torch.full((N, T), -7 if np.isnan(fill) else 0, dtype=torch.int, device="cuda"),
               dam=torch.full((N, T, V), fill, device="cuda"), dlm=torch.full((N, U, V), fill, device="cuda"))
    go = cu(np.linspace(0.5, 1.5, N).astype(np.float32))
    P = [t.data_ptr() for t in (a, l, y, x, n)]
    with Launch() as L:
        assert lib.rnnt_b200_simple_smoothed_forward(s, ws.data_ptr(), nbytes, *P, out["costs"].data_ptr(),
                                                     saved.data_ptr(), out["pair_grads"].data_ptr(), N, T, U, V,
                                                     blank, EXACT, *scales) == 0
    expect(L.rec, want, "C ABI")
    assert lib.rnnt_b200_prune_ranges(s, out["pair_grads"].data_ptr(), x.data_ptr(), n.data_ptr(), N, T, U, S,
                                      out["ranges"].data_ptr()) == 0
    assert lib.rnnt_b200_simple_smoothed_backward(s, ws.data_ptr(), nbytes, *P, saved.data_ptr(),
                                                  out["pair_grads"].data_ptr(), go.data_ptr(), out["dam"].data_ptr(),
                                                  out["dlm"].data_ptr(), N, T, U, V, blank, *scales) == 0
    torch.cuda.synchronize()
    return {k: t.cpu().numpy() for k, t in out.items()}


@pytest.mark.parametrize("scales", SCALES, ids=scales_name)
@pytest.mark.parametrize("shape", [(4, 100, 65, 70, 1, FUSED), (4, 150, 140, 70, 2, GENERAL)],
                         ids=["fused", "general"])
def test_every_output_written(w, shape, scales):
    """On NaN-filled buffers the C ABI writes what it writes on zero-filled ones, bit for bit, and outside the
    lattices what the header states: costs NaN for invalid lengths; norm, pairs' gradients, d am rows 0 past a
    lattice (d lm rows too when am_only_scale = 0); Ll 0 on rows past Un and Am 0 on frames past Tn when
    am_only_scale = 0, Am and log uni 0 when it is 0; ranges 0 for invalid lengths.  The batch has whole 64-row and
    64-column tiles past Tn / Un and a lattice with invalid lengths."""
    lib = abi()
    N, T, U, V, blank, path = shape
    sl, sa = scales
    am, lm, ys, xn, yn = make(N, T, U, V, seed=T + U + V, blank=blank)
    xn[:] = [T, 30, T - 1, T + 1]                       # lattice 3: invalid lengths
    yn[:] = [U - 1, 19, 62, 10]
    got = cabi_call(lib, am, lm, ys, xn, yn, blank, scales, np.nan, dict(path=path))
    clean = cabi_call(lib, am, lm, ys, xn, yn, blank, scales, 0.0, dict(path=path))
    for k in got:
        assert got[k].tobytes() == clean[k].tobytes(), k
    smooth = sl > 0 or sa > 0
    assert np.isnan(got["costs"][3]) and np.isfinite(got["costs"][:3]).all()
    nan = {k: int(np.isnan(v).sum()) for k, v in got.items() if v.dtype != np.int32}
    assert nan == dict(costs=1, saved=0, pair_grads=0, dam=0, dlm=0), nan
    assert (got["ranges"][3] == 0).all() and (got["ranges"] >= 0).all()
    live = np.zeros((N, T, U), bool)
    frames = np.arange(T)[None, :] < np.where(np.arange(N) < 3, xn, 0)[:, None]
    cols = np.arange(U)[None, :] < np.where(np.arange(N) < 3, yn + 1, 0)[:, None]
    live[:] = frames[:, :, None] & cols[:, None, :]
    sv = got["saved"]
    norm = sv[:N * T * U].reshape(N, T, U)
    assert (norm[~live] == 0).all() and (norm[live] != 0).all()
    assert (got["pair_grads"][~live] == 0).all()
    assert (got["dam"][~frames] == 0).all()
    assert (got["dlm"][~cols] == 0).all() == (sa == 0)
    if smooth:
        off = N * T * U + N * T + N * U
        Ll = sv[off:off + N * U].reshape(N, U)
        Am = sv[off + N * U:off + N * U + N * T].reshape(N, T)
        lu = sv[off + N * U + N * T:]
        assert (Ll[~cols] == 0).all() == (sa == 0)
        assert (Am[~frames] == 0).all() and ((Am == 0).all() and (lu == 0).all()) == (sa == 0)
