"""GPU: the two orders in which the fused kernel (csrc/fused.cu) writes the dense gradient.

A gradient larger than L2 whose rows are whole 16-byte vectors of at most COMPOSE_MAX_ROW_BYTES is composed after
beta[0,0] and written once; otherwise it is zero-filled while the recurrence runs and patched afterwards.  The order
a launch took is read back from the kernel's phase stamps (rnnt_b200_debug_fused_trace): slot 11 is stamped only by
the composed emit, slot 6 only by the zero-fill.

  * Every element is written by the composed emit: the gradient buffer is pre-filled with NaN, on shapes with ragged
    lengths, several CTAs per lattice, a label equal to blank, FastEmit and a per-sample scale, one lattice with
    invalid lengths and one whose mismatch guard fires (both all zeros).  Rows that are not whole vectors (unaligned
    heads and tails) are composed only when RNNT_B200_EMIT=compose forces it: a subprocess does that, and its output
    must equal the default order's bit for bit.
  * Both sides of each selection bound (row size, whole vectors, gradient against L2) give what the general path
    gives on the same inputs, bit for bit in exact mode (RNNT_B200_PATH=general in a subprocess: the switches are
    read once per process).
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.common import make_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMPOSE_MAX_ROW_BYTES = 4096            # kComposeMaxRowBytes in csrc/fused.cu
EXACT = 1
BLANK = 1
LAM = 0.3


def gtol(T, U):
    return 2e-5 + 6e-6 * (T + U)


def load_lib():
    import warp_rnnt_b200  # noqa: F401 (the library next to the package)
    L = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    L.rnnt_b200_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int]
    L.rnnt_b200_debug_guard_poison.argtypes = [ctypes.c_int, ctypes.c_float]
    L.rnnt_b200_debug_guard_poison.restype = None
    L.rnnt_b200_debug_fused_trace.argtypes = [ctypes.c_void_p]
    L.rnnt_b200_debug_fused_trace.restype = None
    return L


@pytest.fixture(scope="module")
def lib():
    return load_lib()


def p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def inputs(N, T, U, V, seed):
    """Ragged lengths, blank = 1, and labels equal to the blank in two lattices."""
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=seed, random_lengths=True, blank=BLANK)
    ys[N - 1, 0] = BLANK
    ys[N - 2, min(3, U - 2)] = BLANK
    return lp, ys, xn, yn


def run_dense(L, lp, ys, xn, yn, scale, bf16, fill=float("nan"), trace=False):
    """One rnnt_b200_loss_dense(_bf16) call in exact mode -> (costs, grads as float32 numpy, stamps or None)."""
    N, T, U, V = lp.shape
    dev = "cuda"
    xs = torch.from_numpy(lp).to(dev)
    if bf16:
        xs = xs.to(torch.bfloat16)
    y, a, b = (torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (ys, xn, yn))
    sc = torch.from_numpy(scale).to(dev)
    ws = torch.empty(L.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device=dev)
    costs = torch.empty(N, device=dev)
    grads = torch.full(xs.shape, fill, dtype=xs.dtype, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    stamps = torch.zeros(8192 * 16, dtype=torch.int64, device=dev) if trace else None
    if trace:
        L.rnnt_b200_debug_fused_trace(p(stamps))
    try:
        if bf16:
            loss = torch.zeros(1, device=dev)
            counter = torch.zeros(1, dtype=torch.int32, device=dev)
            st = L.rnnt_b200_loss_dense_bf16(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b),
                                             p(costs), p(grads), p(sc), p(loss), p(counter), N, T, U, V, BLANK,
                                             ctypes.c_float(LAM), EXACT)
        else:
            st = L.rnnt_b200_loss_dense(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b),
                                        p(costs), p(grads), p(sc), N, T, U, V, BLANK, ctypes.c_float(LAM), EXACT)
        torch.cuda.synchronize()
    finally:
        if trace:
            L.rnnt_b200_debug_fused_trace(None)
    assert st == 0
    g = grads.float().cpu().numpy() if bf16 else grads.cpu().numpy()
    if trace:
        stamps = stamps.view(-1, 16).cpu().numpy()
        stamps = stamps[stamps[:, 0] > 0]
    return costs.cpu().numpy(), g, stamps


def emit_order(stamps):
    assert stamps is not None and len(stamps) > 0, "the fused kernel did not run"
    composed, filled = (stamps[:, 11] > 0).all(), (stamps[:, 6] > 0).any()
    assert composed != filled, "mixed emit orders"
    return "compose" if composed else "patch"


# ------------------------------------------------------------------------------------------ every element written
VICTIM = 1


def dead_and_poisoned_inputs(N, T, U, V, bf16):
    """inputs() with invalid lengths in lattice 0 (dead) and bf16-representable values for bf16."""
    lp, ys, xn, yn = inputs(N, T, U, V, seed=11)
    if bf16:
        lp = torch.from_numpy(lp).to(torch.bfloat16).float().numpy()   # bf16-representable: same inputs on both paths
    xn[0] = T + 1
    return lp, ys, xn, yn, np.linspace(0.5, 2.0, N).astype(np.float32)


def run_poisoned(L, lp, ys, xn, yn, scale, bf16, trace=False):
    """run_dense with the mismatch guard of lattice VICTIM fired."""
    L.rnnt_b200_debug_guard_poison(VICTIM, ctypes.c_float(-1.0e4))
    try:
        return run_dense(L, lp, ys, xn, yn, scale, bf16, trace=trace)
    finally:
        L.rnnt_b200_debug_guard_poison(-1, ctypes.c_float(0.0))


# gradients > L2 (50 MB on an H100): 4 KB rows (LDG gather) at N = 4, short rows through the TMA row gather at N = 40;
# several CTAs per lattice in both
@pytest.mark.parametrize("shape,bf16", [((4, 150, 40, 1020), False), ((40, 150, 40, 56), False),
                                        ((4, 150, 40, 2040), True), ((40, 150, 40, 112), True)])
def test_composed_emit_writes_every_element(lib, shape, bf16):
    N, T, U, V = shape
    lp, ys, xn, yn, scale = dead_and_poisoned_inputs(N, T, U, V, bf16)

    def run(bf16_io, trace=False):
        return run_poisoned(lib, lp, ys, xn, yn, scale, bf16_io, trace)
    costs, g, stamps = run(bf16, trace=True)
    assert emit_order(stamps) == "compose"
    assert len(stamps) > N, "expected several CTAs per lattice"
    assert not np.isnan(g).any(), "%d elements left unwritten" % int(np.isnan(g).sum())
    assert not g[0].any() and not g[VICTIM].any()
    if bf16:
        # the fp32 path on the same inputs, rounded once: bit for bit (either emit order); checked against the oracle below
        costs32, g32, _ = run(False)
        assert costs.tobytes() == costs32.tobytes()
        assert g.tobytes() == torch.from_numpy(g32).to(torch.bfloat16).float().numpy().tobytes()
        g = g32
    ok = list(range(2, N))
    c0, g0 = oracle.dense(lp[ok], ys[ok], xn[ok], yn[ok], blank=BLANK, fastemit_lambda=LAM)
    np.testing.assert_allclose(costs[ok], c0, rtol=1e-5)
    np.testing.assert_allclose(g[ok], g0 * scale[ok].reshape(-1, 1, 1, 1), atol=2 * gtol(T, U), rtol=0)


# rows that are not whole 16-byte vectors: f32 V=7 (LDG gather) and V=50, bf16 V=28 (TMA gather) and V=5
FORCED = [((4, 20, 9, 7), False), ((3, 24, 10, 50), False), ((4, 30, 12, 28), True), ((3, 20, 9, 5), True)]


def _forced_compose_main(out_dir):
    """Subprocess body (RNNT_B200_EMIT=compose): the composed emit's outputs for every entry of FORCED."""
    assert os.environ.get("RNNT_B200_EMIT") == "compose"
    L = load_lib()
    for i, (shape, bf16) in enumerate(FORCED):
        lp, ys, xn, yn, scale = dead_and_poisoned_inputs(*shape, bf16)
        costs, g, stamps = run_poisoned(L, lp, ys, xn, yn, scale, bf16, trace=True)
        assert emit_order(stamps) == "compose"
        np.save(os.path.join(out_dir, "costs_%d.npy" % i), costs)
        np.save(os.path.join(out_dir, "grads_%d.npy" % i), g)


def subprocess_outputs(env_name, env_value, main, module="tests.test_gpu_fused_emit"):
    """Run module.main(out_dir) in a fresh process with env_name=env_value -> {file name: array} it saved."""
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, **{env_name: env_value})
        code = "import sys; sys.path.insert(0, %r); from %s import %s; %s(%r)" % (ROOT, module, main, main, d)
        r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        return {k: np.load(os.path.join(d, k)) for k in os.listdir(d)}


def test_forced_composed_emit_on_partial_vector_rows(lib):
    out = subprocess_outputs("RNNT_B200_EMIT", "compose", "_forced_compose_main")
    for i, (shape, bf16) in enumerate(FORCED):
        lp, ys, xn, yn, scale = dead_and_poisoned_inputs(*shape, bf16)
        costs, g, stamps = run_poisoned(lib, lp, ys, xn, yn, scale, bf16, trace=True)
        assert emit_order(stamps) == "patch"                   # small gradients: the default order
        gc = out["grads_%d.npy" % i]
        assert not np.isnan(gc).any(), "%d elements left unwritten" % int(np.isnan(gc).sum())
        assert not gc[0].any() and not gc[VICTIM].any()
        assert costs.tobytes() == out["costs_%d.npy" % i].tobytes()
        assert g.tobytes() == gc.tobytes(), shape


# ------------------------------------------------------------------------------------------ both sides of the selection
def l2_lattices():
    """Largest N at T=150 U=40 V=28 f32 whose gradient fits in L2 (patched); one more lattice is composed."""
    return torch.cuda.get_device_properties(0).L2_cache_size // (150 * 40 * 28 * 4)


# (bf16, N, T, U, V, expected order): the row-size and whole-vector bounds at a gradient > L2, then the L2 bound
SIDES = [(False, 4, 150, 40, COMPOSE_MAX_ROW_BYTES // 4, "compose"),
         (False, 4, 150, 40, COMPOSE_MAX_ROW_BYTES // 4 + 4, "patch"),
         (True, 4, 150, 40, COMPOSE_MAX_ROW_BYTES // 2, "compose"),
         (True, 4, 150, 40, COMPOSE_MAX_ROW_BYTES // 2 + 8, "patch"),
         (False, 4, 150, 40, COMPOSE_MAX_ROW_BYTES // 4 - 2, "patch"),      # not whole 16-byte vectors
         (False, "l2", 150, 40, 28, "patch"),
         (False, "l2+1", 150, 40, 28, "compose")]


def side_inputs(side):
    bf16, N, T, U, V, _ = side
    if N in ("l2", "l2+1"):
        N = l2_lattices() + (N == "l2+1")
    lp, ys, xn, yn = inputs(N, T, U, V, seed=V)
    if bf16:
        lp = torch.from_numpy(lp).to(torch.bfloat16).float().numpy()
    return lp, ys, xn, yn, np.linspace(0.5, 2.0, N).astype(np.float32)


def side_key(side):
    return "%d_%s_%d" % (side[0], side[1], side[4])


def _general_main(out_dir):
    """Subprocess body: the general path's outputs for every entry of SIDES."""
    assert os.environ.get("RNNT_B200_PATH") == "general"
    L = load_lib()
    for side in SIDES:
        lp, ys, xn, yn, scale = side_inputs(side)
        costs, g, stamps = run_dense(L, lp, ys, xn, yn, scale, side[0], trace=True)
        assert len(stamps) == 0, "the general path ran the fused kernel"
        np.save(os.path.join(out_dir, "costs_%s.npy" % side_key(side)), costs)
        np.save(os.path.join(out_dir, "grads_%s.npy" % side_key(side)), g)


@pytest.fixture(scope="module")
def general_outputs():
    return subprocess_outputs("RNNT_B200_PATH", "general", "_general_main")


@pytest.mark.parametrize("side", SIDES, ids=side_key)
def test_both_orders_match_general_path(lib, general_outputs, side):
    lp, ys, xn, yn, scale = side_inputs(side)
    costs, g, stamps = run_dense(lib, lp, ys, xn, yn, scale, side[0], trace=True)
    assert emit_order(stamps) == side[5]
    assert costs.tobytes() == general_outputs["costs_%s.npy" % side_key(side)].tobytes()
    assert g.tobytes() == general_outputs["grads_%s.npy" % side_key(side)].tobytes()
