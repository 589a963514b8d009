"""GPU: call the C ABI (lib/librnnt_b200.so) directly through ctypes -- plain pointers and sizes,
no torch types in the signatures -- and check it against the oracle.  This is the binding a
non-PyTorch host (cgo / JNI / a TF custom op) would write; see INTEGRATION.md section 3."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.common import make_inputs, to_compact

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import warp_rnnt_b200  # noqa: F401 (builds the library if needed)
    L = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    L.rnnt_b200_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int]
    return L


def p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("shape", [(3, 20, 9, 7), (2, 40, 70, 300), (2, 700, 40, 5)])
def test_native_dense_and_gather(lib, shape):
    N, T, U, V = shape
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=5, random_lengths=True, blank=1)
    xs, y, a, b = cu(lp), cu(ys), cu(xn), cu(yn)
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device="cuda")
    costs, grads = torch.empty(N, device="cuda"), torch.empty_like(xs)
    scale = torch.linspace(0.5, 2.0, N).cuda()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    st = lib.rnnt_b200_loss_dense(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b), p(costs),
                                  p(grads), p(scale), N, T, U, V, 1, ctypes.c_float(0.3), 2)
    assert st == 0
    c0, g0 = oracle.dense(lp, ys, xn, yn, blank=1, fastemit_lambda=0.3)
    tol = 2e-5 + 6e-6 * (T + U)
    np.testing.assert_allclose(costs.cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(grads.cpu().numpy(), g0 * scale.cpu().numpy().reshape(-1, 1, 1, 1), atol=2 * tol)
    # gather forward / backward pair
    pg = torch.empty(N, T, U, 2, device="cuda")
    st = lib.rnnt_b200_gather_forward(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b), p(costs),
                                      p(pg), N, T, U, V, 1, ctypes.c_float(0.3), 2)
    assert st == 0
    out = torch.empty_like(xs)
    for lengths in (None, b):                       # label liveness by value (no lengths) / structural (with yn)
        out.fill_(7.0)
        st = lib.rnnt_b200_gather_backward(stream, p(pg), p(y), p(scale), p(out), N, T, U, V, 1, 0, p(lengths))
        assert st == 0
        np.testing.assert_allclose(out.cpu().numpy(), g0 * scale.cpu().numpy().reshape(-1, 1, 1, 1), atol=2 * tol)
    # too-small workspace is refused for shapes that need one; invalid arguments are refused
    st = lib.rnnt_b200_loss_dense(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b), p(costs),
                                  p(grads), None, N, T, U, V, V, ctypes.c_float(0.0), 0)
    assert st == 5
    # without a workspace (6 = too small): the dense, pairs and gather forwards need none when the fused kernel takes
    # the shape (700 frames do not fit its shared memory); the from-logits and compact forwards always need one
    fused_status = 0 if T < 700 else 6
    no_ws, lam = (stream, p(ws), ctypes.c_size_t(0)), ctypes.c_float(0.0)
    xb, gb = xs.bfloat16(), torch.empty(N, T, U, V, dtype=torch.bfloat16, device="cuda")
    pairs, lse = xs[..., :2].contiguous(), torch.empty(N, T, U, device="cuda")
    assert lib.rnnt_b200_loss_dense(*no_ws, p(xs), p(y), p(a), p(b), p(costs), p(grads), None, N, T, U, V, 1, lam,
                                    0) == fused_status
    assert lib.rnnt_b200_loss_dense_bf16(*no_ws, p(xb), p(y), p(a), p(b), p(costs), p(gb), None, None, None, N, T, U,
                                         V, 1, lam, 0) == fused_status
    assert lib.rnnt_b200_loss_pairs(*no_ws, p(pairs), p(a), p(b), p(costs), p(pg), N, T, U, lam, 0) == fused_status
    assert lib.rnnt_b200_gather_forward(*no_ws, p(xs), p(y), p(a), p(b), p(costs), p(pg), N, T, U, V, 1, lam,
                                        0) == fused_status
    for fwd, x in ((lib.rnnt_b200_logits_forward, xs), (lib.rnnt_b200_logits_forward_bf16, xb)):
        assert fwd(*no_ws, p(x), p(y), p(a), p(b), p(costs), p(lse), p(pg), N, T, U, V, 1, lam, 0) == 6
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    STU = xs_c.shape[0]
    xc, yc = cu(xs_c), cu(ys_c)
    pgc, lsec = torch.empty(STU, 2, device="cuda"), torch.empty(STU, device="cuda")
    loc, prefix = torch.empty(STU, dtype=torch.int64, device="cuda"), torch.empty(2 * N, dtype=torch.int64, device="cuda")
    assert lib.rnnt_b200_compact_forward(*no_ws, p(xc), p(yc), p(a), p(b), p(costs), p(pgc), p(loc), None,
                                         ctypes.c_int64(STU), N, V, 1, lam, 0, T, U) == 6
    for fwd, x in ((lib.rnnt_b200_logits_compact_forward, xc), (lib.rnnt_b200_logits_compact_forward_bf16, xc.bfloat16())):
        assert fwd(*no_ws, p(x), p(yc), p(a), p(b), p(costs), p(lsec), p(pgc), p(prefix), None, ctypes.c_int64(STU), N,
                   V, 1, lam, 0, T, U) == 6


def test_reference_abi_symbols_direct(lib):
    """run_warp_rnnt (core.h:29-33) called as the reference's binding calls it."""
    N, T, U, V = 3, 25, 12, 6
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=6, random_lengths=True)
    xs, y, a, b = cu(lp), cu(ys), cu(xn), cu(yn)
    counts = torch.zeros(N, 2 * U, dtype=torch.int32, device="cuda")
    alphas, betas = torch.empty(N, T, U, device="cuda"), torch.empty(N, T, U, device="cuda")
    grads, costs = torch.zeros_like(xs), torch.empty(N, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    st = lib.run_warp_rnnt(stream, p(counts), p(alphas), p(betas), p(y), p(xs), p(grads), p(costs), p(a), p(b),
                           N, T, U, V, 0, ctypes.c_float(0.0))
    assert st == 0
    c0, g0, al0, be0 = oracle.dense(lp, ys, xn, yn, want_ab=True)
    np.testing.assert_allclose(costs.cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(grads.cpu().numpy(), g0, atol=1e-4)
    # alphas / betas land in the caller's (N,T,U) buffers like the reference's
    m = ~np.isnan(al0)
    np.testing.assert_allclose(alphas.cpu().numpy()[m], al0[m], rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(betas.cpu().numpy()[m], be0[m], rtol=1e-4, atol=1e-3)


def test_native_compact(lib):
    N, T, U, V = 4, 30, 11, 9
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=8, random_lengths=True, blank=2)
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    STU = xs_c.shape[0]
    xs, y, a, b = cu(xs_c), cu(ys_c), cu(xn), cu(yn)
    ws = torch.empty(lib.rnnt_b200_workspace_bytes(STU, N), dtype=torch.uint8, device="cuda")
    costs, pg = torch.empty(N, device="cuda"), torch.empty(STU, 2, device="cuda")
    loc = torch.empty(STU, dtype=torch.int64, device="cuda")
    totals = torch.empty(4, dtype=torch.int32, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    st = lib.rnnt_b200_compact_forward(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b), p(costs),
                                       p(pg), p(loc), p(totals), ctypes.c_int64(STU), N, V, 2, ctypes.c_float(0.0), 0, 0, 0)
    assert st == 0
    assert totals.cpu().tolist() == [STU, int(yn.sum()), int(xn.max()), int(yn.max()) + 1]
    c0, pg0, loc0 = oracle.compact(xs_c, ys_c, xn, yn, blank=2)
    np.testing.assert_allclose(costs.cpu().numpy(), c0, rtol=1e-5)
    np.testing.assert_allclose(pg.cpu().numpy(), pg0, atol=1e-4)
    assert np.array_equal(loc.cpu().numpy(), loc0)
    cum = cu(np.cumsum(xn.astype(np.int64) * (yn + 1)).astype(np.int32))
    go = torch.ones(N, device="cuda")
    out = torch.empty(STU, V, device="cuda")
    st = lib.rnnt_b200_compact_backward(stream, p(go), p(pg), p(loc), p(cum), p(out), ctypes.c_int64(STU), N, V, 2)
    assert st == 0
    np.testing.assert_allclose(out.cpu().numpy(), oracle.compact_scatter(np.ones(N), pg0, loc0, cum.cpu().numpy(), V, 2),
                               atol=1e-4)
