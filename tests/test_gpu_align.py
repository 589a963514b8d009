"""GPU: rnnt_align (Viterbi forced alignment, csrc/wavefront.cu k_align) against its numpy restatement
(tests/align_oracle.py), bit for bit; the self-consistency of its outputs at every shape; the launch configurations of
the general wavefront it runs, on both sides of each bound; the bf16 and compact layouts; CUDA-graph capture; and the C
ABI's argument checks."""
import ctypes

import numpy as np
import pytest
import torch

from tests import align_oracle
from tests.common import GOLDEN, assert_same_classes, golden_case, make_inputs, to_compact
from tests.test_gpu_fused_emit import load_lib
from tests.test_gpu_launch_configs import Launch, expect

pytestmark = pytest.mark.gpu
GENERAL = 2


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def align(w, lp, ys, xn, yn, blank, bf16=False):
    xs = cu(lp).to(torch.bfloat16) if bf16 else cu(lp)
    with Launch() as L:
        s, f = w.rnnt_align(xs, cu(ys), cu(xn), cu(yn), blank=blank)
    assert s.dtype == torch.float32 and f.dtype == torch.int32 and f.shape == (len(xn), lp.shape[2] - 1)
    return s.cpu().numpy(), f.cpu().numpy(), L.rec


def lattice(lp, ys, n, Tn, Un, blank):
    B = lp[n, :Tn, :Un, blank]
    L = np.take_along_axis(lp[n, :Tn, :Un - 1], ys[n, :Un - 1].astype(np.int64)[None, :, None], axis=2)[..., 0]
    return B, L


def check(w, lp, ys, xn, yn, blank, want=None):
    """rnnt_align equals align_np bit for bit, its paths are consistent with its scores, and the scores lie below the
    log-likelihood.  -> scores, frames."""
    s, f, rec = align(w, lp, ys, xn, yn, blank)
    if want is not None:
        expect(rec, dict(want, path=GENERAL), "align")
    s0, f0 = align_oracle.align_np(lp, ys, xn, yn, blank)
    assert_same_classes(s, s0, "scores")
    np.testing.assert_array_equal(f, f0)
    T, U = lp.shape[1:3]
    costs, _ = w._C.rnnt_loss_dense(cu(lp), cu(ys), cu(xn), cu(yn), blank=blank, want_grads=False)
    costs = costs.cpu().numpy()
    for n in range(len(xn)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        if not (1 <= Tn <= T and 1 <= Un <= U):
            assert np.isnan(s[n]) and (f[n] == -1).all()
            continue
        if not s[n] > -np.inf:
            assert (f[n] == -1).all()
            continue
        fr = f[n, :Un - 1]
        assert (f[n, Un - 1:] == -1).all()
        assert (np.diff(fr) >= 0).all() and (fr >= 0).all() and (fr <= Tn - 1).all()
        B, L = lattice(lp, ys, n, Tn, Un, blank)
        assert align_oracle.path_score_np(B, L, fr).tobytes() == s[n].tobytes(), n
        if np.isfinite(costs[n]):
            assert s[n] <= -costs[n] + 2e-6 * (1.0 + abs(costs[n])), (n, s[n], costs[n])
    return s, f


# ------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_golden(w, name):
    g = golden_case(name)
    check(w, g["lp"], g["ys"], g["xn"], g["yn"], 0)


# name -> (N, T, U, V, blank, random lengths)
SHAPES = {
    "random_lengths": (6, 40, 20, 12, 0, True),
    "u1": (3, 17, 1, 5, 0, False),
    "t1": (3, 1, 9, 5, 1, False),
    "t1_u1": (2, 1, 1, 4, 0, False),
    "blank3": (4, 25, 14, 9, 3, True),
    "cfg2": (8, 150, 40, 28, 0, True),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_shapes(w, name):
    N, T, U, V, blank, rl = SHAPES[name]
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=len(name), random_lengths=rl, blank=blank)
    check(w, lp, ys, xn, yn, blank)


def test_label_equal_to_blank(w):
    lp, ys, xn, yn = make_inputs(3, 12, 8, 6, seed=3, blank=2)
    ys[:, 2] = 2
    ys[1, :] = 2
    check(w, lp, ys, xn, yn, 2)


def test_masked_and_nonfinite(w):
    """-inf on a label edge of the best path and off it, one NaN log-prob, a dead lattice (score -inf), a lattice
    whose every path is NaN, invalid lengths."""
    N, T, U, V, blank = 9, 10, 7, 6, 1
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=11, blank=blank)
    _, f0 = align_oracle.align_np(lp, ys, xn, yn, blank)
    lp[0, f0[0, 3], 3, ys[0, 3]] = -np.inf                    # on the best path: another path wins
    t_off = (f0[1, 3] + 2) % T
    lp[1, t_off, 3, ys[1, 3]] = -np.inf                       # off it: the same path
    lp[2, 4, 2, blank] = np.nan                               # one NaN
    lp[3, :, 2, ys[3, 2]] = -np.inf                           # label 2 never emitted: no alignment, score -inf
    lp[4, T - 1, U - 1, blank] = np.nan                       # every path NaN
    xn[5], xn[6], yn[7], yn[8] = 0, T + 1, U, -1              # invalid lengths
    s, f = check(w, lp, ys, xn, yn, blank)
    assert f[0, 3] != f0[0, 3] and (f[1] == f0[1]).all()
    assert s[3] == -np.inf and np.isnan(s[4]) and np.isnan(s[5:]).all()
    assert (f[3:] == -1).all()


def test_ties_put_every_label_at_frame_zero(w):
    N, T, U, V = 3, 30, 12, 5
    lp = np.full((N, T, U, V), -1.0, np.float32)
    ys = np.random.RandomState(0).randint(1, V, (N, U - 1)).astype(np.int32)
    xn, yn = np.array([30, 17, 1], np.int32), np.array([11, 6, 11], np.int32)
    s, f = check(w, lp, ys, xn, yn, 0)
    assert (f[0] == 0).all() and (f[1, :6] == 0).all() and (f[2] == 0).all()
    assert list(s) == [-(29 + 11 + 1.0), -(16 + 6 + 1.0), -(11 + 1.0)]


# ------------------------------------------------------------------------------------------ launch configurations
# name -> (N, T, U, V, (xn, yn) or None, expected warps / ring).  Warp and column-pass seams (32/33, 512/513, 1024/1025
# columns), the 16-warp ring at Tn = 1024/1025 (back-pressure from 1025), one warp at Tn = 128/129, and a lattice whose
# Un is no multiple of 32 with full-warp blocks of Tn + 31 steps, no multiple of the unroll (8): a word stored past the
# last step would land in the next column block's first words, which the backtrace reads.
SEAMS = {
    "u32": (3, 20, 32, 5, ([20, 19, 20], [31, 31, 20]), dict(warps=1, ring=128)),
    "u33": (3, 20, 33, 5, ([20, 19, 20], [32, 31, 32]), dict(warps=2, ring=128)),
    "u512": (2, 6, 512, 3, ([6, 5], [511, 480]), dict(warps=16, ring=128)),
    "u513": (2, 6, 513, 3, ([6, 6], [512, 511]), dict(warps=16, ring=128)),
    "u1024": (2, 5, 1024, 3, ([5, 4], [1023, 991]), dict(warps=16, ring=128)),
    "u1025": (3, 5, 1025, 3, ([5, 3, 5], [1024, 1023, 512]), dict(warps=16, ring=128)),
    "t1024_w16": (2, 1024, 481, 3, ([1024, 1000], [480, 470]), dict(warps=16, ring=1024)),
    "t1025_w16": (2, 1025, 481, 3, ([1025, 1024], [480, 449]), dict(warps=16, ring=1024)),
    "t128_w1": (2, 128, 20, 4, ([128, 100], [19, 12]), dict(warps=1, ring=128)),
    "t129_w1": (2, 129, 20, 4, ([129, 129], [19, 12]), dict(warps=1, ring=128)),
    "stray_store": (3, 42, 70, 5, ([42, 42, 41], [69, 60, 37]), dict(warps=3, ring=128)),
}


@pytest.mark.parametrize("name", list(SEAMS))
def test_seams(w, name):
    N, T, U, V, lens, want = SEAMS[name]
    lp, ys, _, _ = make_inputs(N, T, U, V, seed=sum(map(ord, name)), blank=0)
    xn, yn = np.asarray(lens[0], np.int32), np.asarray(lens[1], np.int32)
    check(w, lp, ys, xn, yn, 0, want)


# ------------------------------------------------------------------------------------------ layouts
def bf16_exact(lp):
    return torch.from_numpy(lp).to(torch.bfloat16).float().numpy()


@pytest.mark.parametrize("shape", [(5, 40, 20, 12), (2, 30, 70, 7)])
def test_bf16_equals_f32_on_the_widened_tensor(w, shape):
    N, T, U, V = shape
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=T + U, random_lengths=True)
    lp = bf16_exact(lp)
    lp[0, 3, 2, 0] = np.nan
    s32, f32, _ = align(w, lp, ys, xn, yn, 0)
    s16, f16, _ = align(w, lp, ys, xn, yn, 0, bf16=True)
    assert s16.tobytes() == s32.tobytes() and np.array_equal(f16, f32)


def compact_align(w, lp, ys, xn, yn, blank, hints, bf16=False):
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    xs = cu(xs_c).to(torch.bfloat16) if bf16 else cu(xs_c)
    args = (xs, cu(ys_c), cu(xn), cu(yn))
    with Launch() as L:
        if hints is None:
            s, f = w.rnnt_align(*args, blank=blank, compact=True)
        else:
            with w.compact_hints(*hints):
                s, f = w.rnnt_align(*args, blank=blank, compact=True)
    assert f.shape == (int(yn.sum()),)
    return s.cpu().numpy(), f.cpu().numpy(), L.rec


def padded_frames(f, yn, U):
    out = np.full((len(yn), U - 1), -1, np.int32)
    o = 0
    for n, y in enumerate(yn):
        out[n, :y] = f[o:o + y]
        o += y
    return out


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("shape", [(6, 40, 20, 12, 0), (3, 130, 75, 6, 2), (2, 9, 600, 4, 1)])
def test_compact_equals_dense(w, shape, bf16):
    N, T, U, V, blank = shape
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=N * T, random_lengths=True, blank=blank)
    lp = bf16_exact(lp)
    lp[N - 1, :, 0, ys[N - 1, 0]] = -np.inf                    # one dead lattice
    sd, fd, rd = align(w, lp, ys, xn, yn, blank, bf16=bf16)
    exact = (int(xn.max()), int(yn.max()) + 1)
    for hints in (exact, (T + 13, U + 40), None):
        s, f, rec = compact_align(w, lp, ys, xn, yn, blank, hints, bf16=bf16)
        assert s.tobytes() == sd.tobytes(), hints
        assert np.array_equal(padded_frames(f, yn, U), fd), hints
        if hints == exact or hints is None:
            expect(rec, {k: rd[k] for k in ("path", "warps", "ring")}, "compact %s" % (hints,))


def test_compact_sample_over_the_hints(w):
    N, T, U, V = 4, 30, 12, 6
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=5)
    xn[:] = [30, 20, 25, 20]
    yn[:] = [5, 11, 9, 3]
    sd, fd, _ = align(w, lp, ys, xn, yn, 0)
    s, f, _ = compact_align(w, lp, ys, xn, yn, 0, (25, 10))    # lattice 0 too long, lattice 1 too many labels
    pf = padded_frames(f, yn, U)
    assert np.isnan(s[:2]).all() and (pf[:2] == -1).all()
    assert s[2:].tobytes() == sd[2:].tobytes() and np.array_equal(pf[2:], fd[2:])


# ------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("compact", [False, True])
def test_cuda_graph_capture(w, compact):
    N, T, U, V = 5, 60, 30, 10
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=7, random_lengths=True)
    if compact:
        xs_c, ys_c = to_compact(lp, ys, xn, yn)
        args = (cu(xs_c), cu(ys_c), cu(xn), cu(yn))
    else:
        args = (cu(lp), cu(ys), cu(xn), cu(yn))

    def call():
        if compact:
            with w.compact_hints(T, U):
                return w.rnnt_align(*args, compact=True)
        return w.rnnt_align(*args)

    s_e, f_e = call()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()                                               # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s_g, f_g = call()
    for _ in range(2):
        s_g.fill_(0.0)
        f_g.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(s_g, s_e) and torch.equal(f_g, f_e)


# ------------------------------------------------------------------------------------------ C ABI
def abi():
    L = load_lib()
    L.rnnt_b200_align_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_align_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    vp = ctypes.c_void_p
    L.rnnt_b200_align_dense.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, vp] + [ctypes.c_int] * 6
    L.rnnt_b200_align_compact.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, vp, ctypes.c_int64] + \
        [ctypes.c_int] * 6
    return L


def test_c_abi_checks(w):
    L = abi()
    INVALID, SMALL = 5, 6
    N, T, U, V = 3, 10, 6, 5
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=2)
    xs, y, a, b = cu(lp), cu(ys), cu(xn), cu(yn)
    s = torch.empty(N, device="cuda")
    f = torch.empty(N, U - 1, dtype=torch.int32, device="cuda")
    need = L.rnnt_b200_align_workspace_bytes(N * T * U, N, T, U)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())              # noqa: E731

    def dense(nbytes=need, eb=4, blank=0, n=N, x=xs):
        return L.rnnt_b200_align_dense(st, p(ws), nbytes, p(x), p(y), p(a), p(b), p(s), p(f), n, T, U, V, blank, eb)

    assert dense(eb=3) == INVALID and dense(eb=8) == INVALID
    assert dense(blank=V) == INVALID and dense(blank=-1) == INVALID
    assert dense(nbytes=need - 1) == SMALL
    assert dense(n=0) == 0
    assert dense() == 0
    torch.cuda.synchronize()
    s0, f0 = align_oracle.align_np(lp, ys, xn, yn, 0)
    assert s.cpu().numpy().tobytes() == s0.tobytes() and np.array_equal(f.cpu().numpy(), f0)
    xbf = xs.to(torch.bfloat16)
    assert dense(eb=2, x=xbf) == 0

    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    STU = xs_c.shape[0]
    xc, yc = cu(xs_c), cu(ys_c)
    fc = torch.empty(ys_c.size, dtype=torch.int32, device="cuda")
    needc = L.rnnt_b200_align_workspace_bytes(STU, N, T, U)

    def compact(nbytes=needc, eb=4, bounds=(T, U), blank=0):
        return L.rnnt_b200_align_compact(st, p(ws), nbytes, p(xc), p(yc), p(a), p(b), p(s), p(fc), STU, N, V, blank,
                                         eb, bounds[0], bounds[1])

    assert compact(bounds=(0, 0)) == INVALID and compact(bounds=(T, 0)) == INVALID and compact(bounds=(0, U)) == INVALID
    assert compact(eb=1) == INVALID and compact(blank=V) == INVALID
    assert compact(nbytes=needc - 1) == SMALL
    assert compact() == 0
    torch.cuda.synchronize()
    assert s.cpu().numpy().tobytes() == s0.tobytes()
    assert np.array_equal(padded_frames(fc.cpu().numpy(), yn, U), f0)
