"""GPU: rnnt_loss_tdt(compact=True), the TDT loss on compact (STU, V+D) logits in joint_pack's row order.

The compact call is checked bit for bit against the dense call on xp, the same rows placed in a padded (N,T,U,V+D)
tensor at the same element offset modulo 4 with NaN in the padding: costs, lse, the posteriors and the gradient's live
rows are torch.equal.  The dense call is itself checked against fp64 in test_gpu_tdt.py / test_gpu_tdt_paths.py; here
the compact results are also compared with the fp64 oracle (tests/tdt_oracle.py) and the eager restatement
(tests/tdt_eager.py).  Then every planner bound driven by max_U (from compact_hints or the totals), the degenerate
classes, graphs, determinism, the one host copy without hints, joint_pack end to end, and the C ABI."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import warp_rnnt_b200 as w
from tests.tdt_eager import tdt_costs
from tests.tdt_oracle import random_case, tdt
from tests.test_gpu_tdt import gbound, tdt_record

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
BF16 = torch.bfloat16
SMEM_OPTIN = 227 * 1024


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pack(t, xn, yn):
    """live rows of a padded (N,T,U,...) tensor in the compact order"""
    return torch.cat([t[i, :int(xn[i]), :int(yn[i]) + 1].reshape(-1, *t.shape[3:]) for i in range(len(xn))])


def pack_labels(labels, yn):
    return torch.cat([torch.as_tensor(labels[i, :int(yn[i])]) for i in range(len(yn))]).to(torch.int32)


def at_offset(t, offset, fill=float("nan")):
    """a copy of t whose first element lies `offset` elements past an allocation (so at offset mod 4 of 16 bytes)"""
    buf = torch.full((t.numel() + offset,), fill, dtype=t.dtype, device=DEV)
    v = buf[offset:].view(t.shape)
    v.copy_(t)
    return v


def case(N, T, U, V, durations, seed, edges=True):
    """random_case with ragged lengths, plus a lattice with Tn = 1 and one with yn = 0"""
    rng = np.random.RandomState(seed)
    x, labels, xn, yn = random_case(rng, N, T, U, V, durations)
    if edges and N >= 3:
        xn[1] = 1
        yn[2] = 0
    return x, labels, xn, yn


def layouts(x, labels, xn, yn, dtype, offset):
    """(xp, xc, labels (N,U-1), labels (sum yn), xn, yn) on the device: xp padded with NaN outside the live rows, xc the
    compact rows; both at element offset `offset`"""
    xt = torch.tensor(x, dtype=torch.float32).to(dtype).to(DEV)
    mask = torch.zeros(xt.shape[:3], dtype=torch.bool, device=DEV)
    for i in range(len(xn)):
        mask[i, :int(xn[i]), :int(yn[i]) + 1] = True
    xt = torch.where(mask[..., None], xt, torch.full_like(xt, float("nan")))
    xp = at_offset(xt, offset)
    xc = at_offset(pack(xt, xn, yn), offset)
    return (xp, xc, torch.tensor(labels, device=DEV), pack_labels(labels, yn).to(DEV), torch.tensor(xn, device=DEV),
            torch.tensor(yn, device=DEV))


def compact_call(xc, ys_c, xn, yn, durations, sigma, blank, go, hints=(0, 0)):
    c, l, p, pref = w._C.rnnt_tdt_compact_forward(xc, ys_c, xn, yn, list(durations), sigma, blank, True, *hints)
    rec = tdt_record()
    g = w._C.rnnt_tdt_compact_backward(xc, l, p, ys_c, xn, yn, pref, list(durations), go, blank)
    rec.update({k: v for k, v in tdt_record().items() if k.startswith("emit")})
    return c, l, p, g, rec


def parity(x, labels, xn, yn, durations, sigma=0.05, blank=0, dtype=torch.float32, offset=0, hints=(0, 0)):
    """compact == dense on xp, bit for bit; returns the compact call's launch record and outputs"""
    xp, xc, ys, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, dtype, offset)
    go = torch.linspace(0.5, 1.5, len(xn), device=DEV)           # lattice 0 gets 0.5 whatever N
    cd, ld, pd = w._C.rnnt_tdt_forward(xp, ys, xn_t, yn_t, list(durations), sigma, blank, True)
    gd = w._C.rnnt_tdt_backward(xp, ld, pd, ys, list(durations), go, blank)
    c, l, p, g, rec = compact_call(xc, ys_c, xn_t, yn_t, durations, sigma, blank, go, hints)
    assert torch.equal(c, cd)
    assert torch.equal(l, pack(ld, xn, yn)) and torch.equal(p, pack(pd, xn, yn))
    assert g.dtype == dtype and torch.equal(g, pack(gd, xn, yn))
    return rec, (c, g, xc, ys_c, xn_t, yn_t, go)


# ---- 1. bit parity with the dense call ----------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("V,D", [(28, 4), (29, 4), (25, 5), (27, 5)])      # (V + D) % 4 = 0, 1, 2, 3
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_parity_row_widths_and_offsets(dtype, V, D, offset):
    x, labels, xn, yn = case(6, 9, 6, V, tuple(range(D)), V * 10 + offset)
    labels[0, 1] = V - 1                                    # a label equal to blank
    parity(x, labels, xn, yn, tuple(range(D)), 0.05, V - 1, dtype, offset)


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
@pytest.mark.parametrize("durations", [(0, 1, 2, 3, 4), (1,), (2, 3), (0, 1, 2, 4, 8, 16)])
@pytest.mark.parametrize("sigma", [0.0, 0.05])
@pytest.mark.parametrize("blank", ["first", "last"])
def test_parity_durations_sigma_blank(dtype, durations, sigma, blank):
    V = 11
    b = 0 if blank == "first" else V - 1
    x, labels, xn, yn = case(7, 21, 7, V, durations, len(durations) * 7 + int(sigma * 100))
    labels[3, :2] = b
    parity(x, labels, xn, yn, durations, sigma, b, dtype)


# ---- 2. against fp64 ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("durations", [(0, 1, 2, 3, 4), (1,), (0, 2, 5), (0, 1, 2, 4, 8, 16)])
def test_oracle_small_lattices(durations):
    x, labels, xn, yn = case(5, 18, 7, 9, durations, 3 + len(durations))
    x = x.astype(np.float32).astype(np.float64)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    go = np.random.RandomState(1).uniform(0.2, 2.0, 5)
    c, _, _, g, _ = compact_call(xc, ys_c, xn_t, yn_t, durations, 0.05, 3, torch.tensor(go, dtype=torch.float32,
                                                                                         device=DEV))
    c0, g0, _, _ = tdt(x, labels, xn, yn, durations, 0.05, 3)
    np.testing.assert_allclose(c.cpu().numpy(), c0, rtol=1e-5)
    g0 = pack(torch.tensor(g0 * go[:, None, None, None]), xn, yn).numpy()
    assert np.abs(g.cpu().numpy() - g0).max() <= gbound(18, 7, c0)


def test_eager_large_lattices():
    N, T, U, V, durations = 3, 300, 60, 40, (0, 1, 2, 3, 4)
    x, labels, xn, yn = case(N, T, U, V, durations, 17)
    xt = torch.tensor(x, dtype=torch.float32)
    _, xc, ys, ys_c, xn_t, yn_t = layouts(xt.numpy(), labels, xn, yn, torch.float32, 0)
    xc.requires_grad_(True)
    loss = w.rnnt_loss_tdt(xc, ys_c, xn_t, yn_t, durations, sigma=0.05, blank=0, compact=True)
    loss.sum().backward()
    x64 = xt.double().to(DEV).requires_grad_(True)
    c0 = tdt_costs(x64, ys, xn_t, yn_t, durations, 0.05, 0)
    c0.sum().backward()
    c0n = c0.detach().cpu().numpy()
    np.testing.assert_allclose(loss.detach().cpu().numpy(), c0n, rtol=1e-5)
    err = (xc.grad.double() - pack(x64.grad, xn, yn)).abs().max().item()
    assert err <= gbound(T, U, c0n), err


# ---- 3. every planner bound, on both sides, driven by max_U -------------------------------------------------------

def planner_case(N, T, U, V, durations, expect, seed=0, offset=0, blank=0, hints=True, dtype=torch.float32):
    x, labels, xn, yn = case(N, T, U, V, durations, seed, edges=False)
    rec, out = parity(x, labels, xn, yn, durations, 0.05, blank, dtype, offset, (T, U) if hints else (0, 0))
    for k, v in expect.items():
        assert rec[k] == v, (k, rec)
    return rec, out


@pytest.mark.parametrize("durations,kd", [((1,), 5), ((0, 1, 2, 3, 4), 5), ((0, 1, 2, 3, 4, 5), 17),
                                          (tuple(range(17)), 17)])
def test_candidate_slots(durations, kd):
    planner_case(3, 40, 6, 7, durations, dict(kd=kd, ring=max(durations) + 2, warps=1, passes=1))


@pytest.mark.parametrize("U,warps,passes", [(32, 1, 1), (33, 2, 1), (512, 16, 1), (513, 16, 2), (2048, 16, 4),
                                            (2049, 16, 5)])
def test_column_passes_from_the_hints(U, warps, passes):
    planner_case(2, 12, U, 6, (0, 1, 2), dict(warps=warps, passes=passes, ring=4, smem=4 * U * 4))


def test_column_passes_from_the_totals():
    """without hints max_U is the batch's max yn + 1: lattice 0 has U = 513 columns"""
    planner_case(2, 12, 513, 6, (0, 1, 2), dict(warps=16, passes=2, ring=4, smem=4 * 513 * 4), hints=False)


def test_hints_do_not_change_values():
    """a larger max_U changes the plan (warps, ring bytes), not one bit"""
    x, labels, xn, yn = case(4, 30, 20, 9, (0, 1, 2, 3, 4), 8)
    _, (c, g, xc, ys_c, xn_t, yn_t, go) = parity(x, labels, xn, yn, (0, 1, 2, 3, 4))
    c2, _, _, g2, rec = compact_call(xc, ys_c, xn_t, yn_t, (0, 1, 2, 3, 4), 0.05, 0, go, (64, 700))
    assert rec["warps"] == 16 and rec["passes"] == 2
    assert torch.equal(c, c2) and torch.equal(g, g2)


@pytest.mark.parametrize("U", [SMEM_OPTIN // (18 * 4), SMEM_OPTIN // (18 * 4) + 1])
def test_ring_at_its_limit(U):
    """max(d) = 16: 18 ring slots of max_U columns; one column more and the ring reads back from global memory"""
    fits = 18 * U * 4 <= SMEM_OPTIN
    planner_case(1, 20, U, 4, (0, 1, 16), dict(ring=18 if fits else 0, smem=18 * U * 4 if fits else 0))


def test_long_frames():
    planner_case(2, 1600, 9, 5, (0, 1, 2, 3, 4), dict(ring=6, warps=1))


@pytest.mark.parametrize("V,D,offset,group,lanes", [
    (28, 4, 0, 4, 8), (28, 4, 1, 1, 8), (28, 4, 2, 2, 8), (29, 5, 0, 2, 8), (27, 5, 1, 1, 8), (27, 3, 0, 2, 8),
    (123, 5, 0, 4, 32), (125, 5, 0, 2, 32), (125, 5, 2, 2, 32), (124, 5, 0, 1, 32),
    (59, 5, 0, 4, 8), (60, 5, 0, 1, 32)])                              # W = 64 and 65: both sides of the lane bound
def test_normaliser_and_emit_branches(V, D, offset, group, lanes):
    planner_case(3, 10, 5, V, tuple(range(D)), dict(norm_group=group, norm_lanes=lanes, emit_vec=4,
                                                    emit_xvec=int(offset == 0)), offset=offset, blank=V - 1)


def test_emit_scalar_stores():
    """a gradient tensor that is not 16-byte aligned: the emit stores element by element (C ABI, out at offset 1)"""
    rec, (c, g, xc, ys_c, xn_t, yn_t, go) = planner_case(3, 10, 5, 12, (0, 1, 2), {})
    L, fns = _abi()
    _, l, p, pref = w._C.rnnt_tdt_compact_forward(xc, ys_c, xn_t, yn_t, [0, 1, 2], 0.05, 0, True, 10, 5)
    out = at_offset(torch.zeros_like(xc), 1)
    st = fns["bwd"](_stream(), _p(xc), _p(l), _p(p), _p(ys_c), _p(yn_t), _durs((0, 1, 2)), 3, _p(pref), _p(go), _p(out),
                    xc.shape[0], len(xn_t), 12, 0, 4)
    assert st == 0
    torch.cuda.synchronize()
    assert tdt_record()["emit_vec"] == 1 and torch.equal(out, g)


def test_every_row_thread_iterates_its_grid_stride():
    """more rows than the normaliser's and the posterior pass's grids cover, and more vectors than the emit's: each
    thread of those kernels runs its grid-stride loop more than once; lattice 0 alone gives the same bits"""
    s = sms()
    T = U = 200
    N = max(2, math.ceil(s * 16 * 256 * 1.5 / (T * U)))
    V, D = 3, 5
    g0 = torch.Generator().manual_seed(5)
    x = torch.randn(N, T, U, V + D, generator=g0)
    labels = torch.randint(1, V, (N, U - 1), generator=g0, dtype=torch.int32).numpy()
    xn = np.full(N, T, np.int32)
    yn = np.full(N, U - 1, np.int32)
    assert N * T * U > s * 16 * 256 and N * T * U * (V + D) / 4 > s * 32 * 256
    rec, (c, g, *_) = parity(x.numpy(), labels, xn, yn, (0, 1, 2, 3, 4), 0.0, 0, torch.float32, 0, (T, U))
    assert rec["norm_lanes"] == 8 and rec["emit_vec"] == 4
    _, (c1, g1, *_) = parity(x[:1].numpy(), labels[:1], xn[:1], yn[:1], (0, 1, 2, 3, 4), 0.0, 0)
    assert torch.equal(c1, c[:1]) and torch.equal(g1, g[:T * U])


def test_bf16_beyond_2_31_elements():
    """one bf16 call with STU * (V+D) > 2^31: the last lattice, whose rows lie past element 2^31, gives the same bits as
    a call on that lattice alone, and its gradient rows sum to 0"""
    N, T, U, V, D = 4, 1000, 530, 1025, 5
    xn = torch.tensor([T, T, T, T - 7], dtype=torch.int32, device=DEV)
    yn = torch.tensor([U - 1, U - 1, U - 1, U - 12], dtype=torch.int32, device=DEV)
    STU = int((xn.long() * (yn.long() + 1)).sum())
    assert STU * (V + D) > 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(STU, V + D, device=DEV, dtype=BF16, generator=g).requires_grad_(True)
    ys = torch.randint(1, V, (int(yn.sum()),), device=DEV, dtype=torch.int32, generator=g)
    with w.compact_hints(T, U):
        c = w.rnnt_loss_tdt(x, ys, xn, yn, (0, 1, 2, 3, 4), compact=True)
    c.sum().backward()
    assert torch.isfinite(c).all()
    first = 3 * T * U
    last_c, last_g = c.detach()[3:].clone(), x.grad[first:].clone()
    x.grad = None
    x1 = x.detach()[first:].clone().requires_grad_(True)
    del x
    torch.cuda.empty_cache()
    c1 = w.rnnt_loss_tdt(x1, ys[3 * (U - 1):], xn[3:], yn[3:], (0, 1, 2, 3, 4), compact=True)
    c1.sum().backward()
    assert torch.equal(c1.detach(), last_c) and torch.equal(x1.grad, last_g)
    rows = last_g.float()
    assert rows[:, :V].sum(-1).abs().max().item() < 1e-2 and rows[:, V:].sum(-1).abs().max().item() < 1e-2


# ---- 4. degenerate classes ----------------------------------------------------------------------------------------

def run(xc, ys_c, xn, yn, durations, hints=(0, 0), blank=0, grad=True):
    x = xc.clone().requires_grad_(grad)
    if hints[0]:
        with w.compact_hints(*hints):
            c = w.rnnt_loss_tdt(x, ys_c, xn, yn, durations, blank=blank, compact=True)
    else:
        c = w.rnnt_loss_tdt(x, ys_c, xn, yn, durations, blank=blank, compact=True)
    if grad:
        c.sum().backward()
    return c.detach(), x.grad


def rows_of(xn, yn, i):
    lens = [int(a) * (int(b) + 1) for a, b in zip(xn, yn)]
    o = sum(lens[:i])
    return slice(o, o + lens[i])


def test_degenerate_classes_and_isolation():
    durations = (1, 2)
    rng = np.random.RandomState(9)
    x, labels, xn, yn = random_case(rng, 7, 6, 4, 5, durations)
    xn[:], yn[:] = 6, 3
    x[0, :, :, 0] = -np.inf                  # no blank: no path -> +inf
    labels[1, 0] = 77                        # live label outside [0, V)
    x[2, 2, 1, 2] = np.nan                   # NaN in a live row
    x[3, 1, 2, 1] = np.inf                   # +inf in a live row
    x[4, 1, 1, 5:] = -np.inf                 # a live row whose duration logits are all -inf
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    c, g = run(xc, ys_c, xn_t, yn_t, durations)
    c = c.cpu().numpy()
    assert np.isposinf(c[0]) and (g[rows_of(xn, yn, 0)] == 0).all()
    assert np.isnan(c[1]) and (g[rows_of(xn, yn, 1)] == 0).all()
    for i in (2, 3, 4):
        assert np.isnan(c[i]) and torch.isnan(g[rows_of(xn, yn, i)]).all()
    assert np.isfinite(c[5:]).all()
    keep = [0, 1, 5, 6]
    _, xk, _, ysk, xnk, ynk = layouts(x[keep], labels[keep], xn[keep], yn[keep], torch.float32, 0)
    ck, gk = run(xk, ysk, xnk, ynk, durations)
    assert np.array_equal(ck.cpu().numpy(), c[keep], equal_nan=True)
    assert torch.equal(gk, torch.cat([g[rows_of(xn, yn, i)] for i in keep]))
    # structurally dead: Tn < min(d > 0)
    xs, ls, xns, yns = random_case(rng, 2, 4, 3, 5, (2, 3))
    xns[:] = 1
    _, xc2, _, ys2, xn2, yn2 = layouts(xs, ls, xns, yns, torch.float32, 0)
    c2, g2 = run(xc2, ys2, xn2, yn2, (2, 3))
    assert np.isposinf(c2.cpu().numpy()).all() and (g2 == 0).all()


def test_invalid_lengths():
    """xn < 1 or yn < 0: cost NaN and no rows (their xn * (yn + 1) is 0); the others as in a batch without them.  yn < 0
    is on the last lattice: the label prefix sums count it, so the labels of a later lattice would start earlier."""
    x, labels, xn, yn = case(5, 8, 5, 6, (0, 1, 2), 4, edges=False)
    xn[1], yn[4] = 0, -1
    keep = [0, 2, 3]
    _, xc, _, _, _, _ = layouts(x[keep], labels[keep], xn[keep], yn[keep], torch.float32, 0)
    ys_c = pack_labels(labels, np.maximum(yn, 0)).to(DEV)        # inside hints nothing compares its size with sum yn
    c, g = run(xc, ys_c, torch.tensor(xn, device=DEV), torch.tensor(yn, device=DEV), (0, 1, 2), hints=(8, 5))
    assert torch.isnan(c[[1, 4]]).all()
    _, xk, _, ysk, xnk, ynk = layouts(x[keep], labels[keep], xn[keep], yn[keep], torch.float32, 0)
    ck, gk = run(xk, ysk, xnk, ynk, (0, 1, 2), hints=(8, 5))
    assert torch.equal(c[keep], ck) and torch.equal(g, gk)


def test_sample_exceeding_the_hints():
    """inside compact_hints a sample longer than the hints gets cost NaN and zero rows; every other lattice gives the
    bits of a batch without it"""
    T, U = 12, 6
    x, labels, xn, yn = case(4, T, U, 7, (0, 1, 2), 6, edges=False)
    xn[2], yn[2] = T, U - 1                          # exceeds max_T = T - 1
    xn[[0, 1, 3]] = np.minimum(xn[[0, 1, 3]], T - 1)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    c, g = run(xc, ys_c, xn_t, yn_t, (0, 1, 2), hints=(T - 1, U))
    assert torch.isnan(c[2]) and (g[rows_of(xn, yn, 2)] == 0).all()
    keep = [0, 1, 3]
    _, xk, _, ysk, xnk, ynk = layouts(x[keep], labels[keep], xn[keep], yn[keep], torch.float32, 0)
    ck, gk = run(xk, ysk, xnk, ynk, (0, 1, 2), hints=(T - 1, U))
    assert torch.equal(c[keep], ck) and torch.equal(torch.cat([g[rows_of(xn, yn, i)] for i in keep]), gk)


def test_rows_past_stu_inside_hints():
    """inside hints nothing checks STU on the host: a lattice whose rows would run past the tensor gets cost NaN and
    is not read (the rows after the tensor are NaN in its allocation); the rows it would own get zeros"""
    x, labels, xn, yn = case(3, 8, 5, 6, (0, 1, 2), 12, edges=False)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    cut = xc.shape[0] - 3
    buf = torch.full((xc.numel() + 64,), float("nan"), device=DEV)
    short = buf[:cut * xc.shape[1]].view(cut, xc.shape[1])
    short.copy_(xc[:cut])
    c, g = run(short, ys_c, xn_t, yn_t, (0, 1, 2), hints=(8, 5))
    assert torch.isnan(c[2]) and torch.isfinite(c[:2]).all()
    assert (g[rows_of(xn, yn, 2).start:] == 0).all() and torch.isfinite(g).all()
    c0, g0 = run(xc, ys_c, xn_t, yn_t, (0, 1, 2), hints=(8, 5))
    assert torch.equal(c[:2], c0[:2]) and torch.equal(g[:rows_of(xn, yn, 2).start], g0[:rows_of(xn, yn, 2).start])


def test_forward_without_grad_and_empty_batch():
    x, labels, xn, yn = case(4, 9, 5, 6, (0, 1, 2), 3)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    c_grad, _ = run(xc, ys_c, xn_t, yn_t, (0, 1, 2))
    c, g = run(xc, ys_c, xn_t, yn_t, (0, 1, 2), grad=False)
    assert g is None and torch.equal(c, c_grad)
    e = torch.empty(0, 9, device=DEV, requires_grad=True)
    ei = torch.empty(0, dtype=torch.int32, device=DEV)
    loss = w.rnnt_loss_tdt(e, ei, ei, ei, (0, 1, 2), compact=True, reduction="sum")
    loss.backward()
    assert loss.item() == 0 and e.grad.shape == e.shape


def test_shape_errors_without_hints():
    """without hints the totals copy checks STU and labels.numel(): a mismatch raises before any loss kernel runs
    (the one launch is the totals pass)"""
    x, labels, xn, yn = case(3, 6, 4, 7, (0, 1, 2), 2)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    for xs, ys, msg in ((xc[:-1], ys_c, r"xs shape mismatch"), (xc, ys_c[:-1], r"ys shape must be equal")):
        torch.cuda.synchronize()
        before = w._C.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            w.rnnt_loss_tdt(xs.contiguous(), ys.contiguous(), xn_t, yn_t, (0, 1, 2), compact=True)
        assert w._C.launch_count() == before + 1
    with pytest.raises(ValueError):
        w.rnnt_loss_tdt(xc[None], ys_c, xn_t, yn_t, (0, 1, 2), compact=True)       # not (STU, V + D)
    with pytest.raises(RuntimeError, match=r"blank must be in \[0, V\)"):
        w._C.rnnt_tdt_compact_forward(xc, ys_c, xn_t, yn_t, [0, 1, 2], 0.0, 7, True, 0, 0)


# ---- 5. graphs, determinism, host copies --------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_graph_capture_and_determinism(dtype):
    T, U, durations = 40, 12, (0, 1, 2, 3, 4)
    x, labels, xn, yn = case(8, T, U, 30, durations, 4)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, dtype, 0)
    xt = xc.clone().requires_grad_(True)

    def step():
        xt.grad = None
        with w.compact_hints(T, U):
            loss = w.rnnt_loss_tdt(xt, ys_c, xn_t, yn_t, durations, sigma=0.05, reduction="sum", compact=True)
        loss.backward()
        return loss

    l1, g1 = step().detach().clone(), xt.grad.clone()
    l2, g2 = step().detach().clone(), xt.grad.clone()
    assert torch.equal(l1, l2) and torch.equal(g1, g2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    xt.grad = None
    with torch.cuda.graph(graph):
        loss = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss.detach(), l1) and torch.equal(xt.grad, g1)


def test_one_host_copy_without_hints():
    from torch.profiler import ProfilerActivity, profile
    x, labels, xn, yn = case(4, 20, 6, 9, (0, 1, 2), 5)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, torch.float32, 0)
    xt = xc.clone().requires_grad_(True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        w.rnnt_loss_tdt(xt, ys_c, xn_t, yn_t, (0, 1, 2), reduction="sum", compact=True).backward()
        torch.cuda.synchronize()
    d2h = [e for e in prof.events() if "Memcpy DtoH" in e.name and e.device_type.name == "CUDA"]
    assert len(d2h) == 1, [e.name for e in d2h]


# ---- 6. end to end ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("autocast", [False, True])
def test_joint_pack_feeds_the_compact_tdt_loss(autocast):
    """joint_pack -> Linear -> rnnt_loss_tdt(compact=True), float32 and under bf16 autocast: the loss and the gradients
    of f, g and the Linear weights agree with the padded pipeline"""
    N, T, U1, H, V, durations = 3, 14, 6, 16, 9, (0, 1, 2, 3)
    W = V + len(durations)
    g0 = torch.Generator(device=DEV).manual_seed(1)
    f = torch.randn(N, T, H, device=DEV, generator=g0).requires_grad_(True)
    g = torch.randn(N, U1, H, device=DEV, generator=g0).requires_grad_(True)
    lin = torch.nn.Linear(H, W).to(DEV)
    lf = torch.tensor([14, 9, 12], dtype=torch.int, device=DEV)
    lg = torch.tensor([5, 3, 4], dtype=torch.int, device=DEV)
    ys = torch.randint(1, V, (N, U1 - 1), dtype=torch.int, device=DEV, generator=g0)
    ys_c = torch.cat([ys[i, :lg[i]] for i in range(N)]).contiguous()
    with torch.autocast("cuda", dtype=BF16, enabled=autocast):
        logits = lin(torch.tanh(w.joint_pack(f, g, lf, lg)))
        assert logits.dtype == (BF16 if autocast else torch.float32)
        loss_c = w.rnnt_loss_tdt(logits, ys_c, lf, lg, durations, reduction="sum", compact=True)
    gc = torch.autograd.grad(loss_c, [f, g, lin.weight])
    with torch.autocast("cuda", dtype=BF16, enabled=autocast):
        logits_d = lin(torch.tanh(f.unsqueeze(2) + g.unsqueeze(1)))
        loss_d = w.rnnt_loss_tdt(logits_d, ys, lf, lg, durations, reduction="sum")
    gd = torch.autograd.grad(loss_d, [f, g, lin.weight])
    tol = 1e-4 if not autocast else 2e-2
    np.testing.assert_allclose(loss_c.item(), loss_d.item(), rtol=1e-5 if not autocast else 1e-3)
    for a, b in zip(gc, gd):
        np.testing.assert_allclose(a.float().cpu().numpy(), b.float().cpu().numpy(), rtol=tol, atol=tol)


# ---- 7. C ABI -----------------------------------------------------------------------------------------------------

def _abi():
    L = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    P, I, F, L64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int64
    L.rnnt_b200_tdt_compact_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_tdt_compact_workspace_bytes.argtypes = [L64, I, I]
    fwd, bwd = L.rnnt_b200_tdt_compact_forward, L.rnnt_b200_tdt_compact_backward
    fwd.restype = bwd.restype = I
    fwd.argtypes = [P, P, ctypes.c_size_t, P, P, P, P, P, I, F, P, P, P, P, P, L64, I, I, I, I, I, I]
    bwd.argtypes = [P, P, P, P, P, P, P, I, P, P, P, L64, I, I, I, I]
    return L, {"fwd": fwd, "bwd": bwd}


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _durs(d):
    return (ctypes.c_int * len(d))(*d)


@pytest.mark.parametrize("dtype", [torch.float32, BF16])
def test_c_abi_writes_every_element_and_refuses(dtype):
    """NaN-poisoned outputs: the forward writes costs, the prefix and every posterior row, the backward every gradient
    element -- the rows past the last lattice (STU larger than the lattices need, inside bounds) as zeros; then each
    refusal returns RNNT_STATUS_INVALID_ARGUMENT without a launch"""
    L, fns = _abi()
    durations = (0, 1, 2, 3)
    N, T, U, V = 4, 11, 6, 13
    x, labels, xn, yn = case(N, T, U, V, durations, 31)
    _, xc, _, ys_c, xn_t, yn_t = layouts(x, labels, xn, yn, dtype, 0)
    extra = 5
    xs = torch.cat([xc, torch.randn(extra, xc.shape[1], device=DEV).to(dtype)])
    STU, D = xs.shape[0], len(durations)
    eb = 2 if dtype == BF16 else 4
    wsb = L.rnnt_b200_tdt_compact_workspace_bytes(STU, N, D)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    costs = torch.full((N,), float("nan"), device=DEV)
    lse = torch.full((STU, 2), float("nan"), device=DEV)
    pg = torch.full((STU, 2 + D), float("nan"), device=DEV)
    pref = torch.full((2 * N,), -1, dtype=torch.int64, device=DEV)
    totals = torch.full((4,), -1, dtype=torch.int32, device=DEV)
    go = torch.linspace(0.5, 1.5, N, device=DEV)
    out = torch.full_like(xs, float("nan"))
    dur = _durs(durations)

    def fwd(ws_ptr=None, nbytes=wsb, nd=D, durs=dur, sigma=0.0, prefix=pref, STU_=STU, mT=T, mU=U, e=eb, lse_=lse):
        return fns["fwd"](_stream(), ws_ptr if ws_ptr is not None else _p(ws), nbytes, _p(xs), _p(ys_c), _p(xn_t),
                          _p(yn_t), durs, nd, sigma, _p(costs), _p(lse_), _p(pg),
                          None if prefix is None else _p(prefix), _p(totals), STU_, N, V, 0, e, mT, mU)

    def bwd(prefix=pref, e=eb, grads=pg):
        return fns["bwd"](_stream(), _p(xs), _p(lse), None if grads is None else _p(grads), _p(ys_c), _p(yn_t), dur, D,
                          None if prefix is None else _p(prefix), _p(go), _p(out), STU, N, V, 0, e)

    assert fwd() == 0 and bwd() == 0
    torch.cuda.synchronize()
    assert torch.isfinite(costs).all() and torch.isfinite(pg).all() and torch.isfinite(out.float()).all()
    assert (out[STU - extra:] == 0).all() and (pg[STU - extra:] == 0).all()
    assert totals[0].item() == STU - extra and totals[1].item() == ys_c.numel()
    c, l, p, g, _ = compact_call(xc, ys_c, xn_t, yn_t, durations, 0.0, 0, go, (T, U))
    assert torch.equal(costs, c) and torch.equal(pg[:STU - extra], p) and torch.equal(out[:STU - extra], g)
    assert torch.equal(lse[:STU - extra], l)
    torch.cuda.synchronize()
    before = w._C.launch_count()
    assert fwd(nbytes=wsb - 1) == 6                                       # RNNT_STATUS_WORKSPACE_TOO_SMALL
    assert fwd(ws_ptr=ctypes.c_void_p(ws.data_ptr() + 8)) == 5            # workspace not 16-byte aligned
    assert fwd(durs=_durs((1, 1)), nd=2) == 5                             # durations not increasing
    assert fwd(durs=_durs((0,)), nd=1) == 5                               # no duration > 0
    assert fwd(sigma=-1.0) == 5
    assert fwd(sigma=float("nan")) == 5
    assert fwd(e=3) == 5
    assert fwd(prefix=None) == 5
    assert fwd(mT=0) == 5 and fwd(mU=0) == 5
    assert fwd(STU_=2 ** 31) == 5
    lse_buf = torch.empty(STU * 2 + 1, device=DEV)
    assert fwd(lse_=lse_buf[1:]) == 5                                     # lse not 8-byte aligned
    assert bwd(prefix=None) == 5 and bwd(grads=None) == 5 and bwd(e=3) == 5
    assert w._C.launch_count() == before
