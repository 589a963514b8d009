"""GPU: every launch configuration the fused kernel (csrc/fused.cu) and the general path (csrc/wavefront.cu, api.cu)
can take, each case on one side of one planner bound with the case on the other side next to it.

The configuration a call ran with is read back from the library (rnnt_b200_debug_last_launch); every case asserts the
configuration it names.  The bounds, from fused_plan / launch_fused, launch_wavefront_kp and pipeline_groups:

  * fused column width C: 1 for U <= 32, 2 for U <= 64, 4 for U <= 128; C = 1 with odd U pads one phantom column
  * fused or general: staged lattice <= 220 KB of shared memory (U = 104 only for T <= 10, never U >= 105; along T:
    U = 1 at T = 5412, U = 33 at 342, U = 65 at 114), and at most 96 gather chunks of 128 cells (U = 16 at T = 768)
  * two CTAs per SM when the staged lattice takes <= 110 KB (U = 64 at T = 20), then the occupancy query (one on an
    H100 80GB HBM3: the register count of 512 threads allows no second CTA)
  * CTAs per lattice (slices) above a lattice's length, and one CTA per lattice over several waves of CTAs
  * the row gather: TMA with two buffers per warp, TMA with fewer buffer warps than gather warps, or LDG (row not a
    16-byte multiple, row > 32 KB, misaligned base, or four buffers do not fit); bf16 rows flip at other V
  * general: ceil(U/32) warps per CTA, at most 16 (column passes at U = 513 and 1025, lattices ending on a warp or
    pass seam); boundary ring of 1024 slots with 16 warps (back-pressure from Tn = 1025), 128 slots for a compact call
    without max_T / max_U (from Tn = 129); beta alone without gradients
  * the stream pipeline of the general path: 4 lattice groups for 8 <= N < 32, 8 from N = 32

Every case runs the dense f32 layout, the gathered (N,T,U,2) layout, compact with exact hints, with loose hints (max_T,
max_U larger than any lattice) and without hints; fused cases also dense bf16.  Checks: the fp64 oracle in both LSE
modes (costs 1e-5 relative, gradients gtol(T,U)); in exact mode the fused kernel and the general path bit for bit
(RNNT_B200_PATH=general in a subprocess: the switch is read once per process), every compact run bit for bit, and the
compiled reference bit for bit (tests/golden/reference_outputs.npz) on the cases within the shapes it was run on; bf16
equals the f32 result on the same (bf16-representable) inputs rounded once; without gradients the general path's costs
equal those with gradients.
"""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.common import make_inputs, same_as_reference, to_compact
from tests.test_gpu_fused_emit import load_lib, subprocess_outputs
from tests.test_gpu_parity import check_compact_vs_reference, gather_np

pytestmark = pytest.mark.gpu
EXACT, FAST = 1, 2
LAM = 0.2

# rnntLaunchRecord_t (include/rnnt_b200.h)
FIELDS = ["seq", "path", "C", "slices", "occ", "smem", "gather_warps", "row_bufs", "compose", "tma_fill", "warps",
          "ring", "beta_only", "groups"]
FUSED, GENERAL = 1, 2


def gtol(T, U):
    return 2e-5 + 6e-6 * (T + U)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# name -> (N, T, U, V, blank, (xn, yn) overrides or None, expected record of the dense f32 exact run, expected row
#          gather of the bf16 run or None).  N = "sms": one lattice per SM.  smem is the dynamic shared memory as
#          launched: the staged lattice plus the TMA row buffers.
CASES = {
    # fused column width
    "c1_u32": (3, 40, 32, 12, 2, None, dict(path=FUSED, C=1, slices=40, gather_warps=14, row_bufs=2), None),
    "c2_u33": (3, 40, 33, 12, 2, None, dict(path=FUSED, C=2, slices=40), None),
    "c2_u64": (3, 40, 64, 12, 5, None, dict(path=FUSED, C=2, slices=40), None),
    "c4_u65": (3, 40, 65, 12, 5, None, dict(path=FUSED, C=4, slices=40, gather_warps=13, row_bufs=2),
               dict(gather_warps=0, row_bufs=0)),
    # odd U with C = 1 stages one phantom column: smem is that of Wd = 2 (9,216 B with Wd = 1) and Wd = 8 (13,824 B)
    "c1_u1_phantom": (4, 30, 1, 6, 3, None, dict(path=FUSED, C=1, smem=9984, gather_warps=0, row_bufs=0), None),
    "c1_u7_odd": (3, 25, 7, 6, 1, None, dict(path=FUSED, C=1, smem=14848, gather_warps=0, row_bufs=0), None),
    # fused or general: shared memory
    "smem_u104_t10": (3, 10, 104, 6, 1, None, dict(path=FUSED, C=4, smem=225024, slices=10), None),
    "smem_u104_t11": (3, 11, 104, 6, 1, None, dict(path=GENERAL, warps=4, beta_only=0), None),
    "smem_u105_t1": (3, 1, 105, 6, 1, None, dict(path=GENERAL, warps=4), None),
    "smem_u1_t5412": (2, 5412, 1, 8, 2, None, dict(path=FUSED, C=1, smem=228352, slices=66), None),
    "smem_u1_t5413": (2, 5413, 1, 8, 2, None, dict(path=GENERAL, warps=1, ring=128), None),
    "smem_u33_t342": (2, 342, 33, 8, 2, None, dict(path=FUSED, C=2, smem=224384, gather_warps=0, row_bufs=0),
                      dict(smem=228224, gather_warps=6, row_bufs=1)),
    "smem_u33_t343": (2, 343, 33, 8, 2, None, dict(path=GENERAL, warps=2, ring=512), None),
    "smem_u65_t114": (2, 114, 65, 8, 3, None, dict(path=FUSED, C=4, smem=224896), None),
    "smem_u65_t115": (2, 115, 65, 8, 3, None, dict(path=GENERAL, warps=3, ring=128), None),
    # fused or general: gather chunks
    "chunks_u16_t768": (2, 768, 16, 8, 1, None, dict(path=FUSED, C=1, gather_warps=8, row_bufs=2),
                        dict(gather_warps=14, row_bufs=2)),
    "chunks_u16_t769": (2, 769, 16, 8, 1, None, dict(path=GENERAL, warps=1), None),
    "chunks_u24_t512_96": (2, 512, 24, 8, 1, None, dict(path=FUSED, C=1, gather_warps=5, row_bufs=1),
                           dict(gather_warps=5, row_bufs=2)),
    # CTAs per SM (one lattice per SM, so that the slices show it): at T = 20 the plan counts on two CTAs per SM and
    # asks the occupancy query, which allows one (registers: 512 threads), so one slice per lattice either way
    "persm2_u64_t20": ("sms", 20, 64, 8, 2, None, dict(path=FUSED, C=2, smem=111104, slices=1, occ=1), None),
    "persm1_u64_t21": ("sms", 21, 64, 8, 2, None, dict(path=FUSED, C=2, smem=170496, slices=1, occ=0), None),
    # CTAs per lattice: far more slices than rows in short lattices; one slice over several waves of CTAs
    "slices_over_tn": (3, 40, 20, 8, 4, ([40, 3, 1], [19, 7, 0]), dict(path=FUSED, slices=40), None),
    "multiwave_n300": (300, 150, 40, 8, 1, None, dict(path=FUSED, C=2, slices=1, occ=0), None),
    # row gather
    "tma_2buf_cfg2": (4, 150, 40, 28, 1, None, dict(path=FUSED, gather_warps=9, row_bufs=2),
                      dict(gather_warps=14, row_bufs=2)),
    "tma_1buf_6of14": (4, 40, 8, 512, 1, None, dict(path=FUSED, gather_warps=6, row_bufs=1),
                       dict(gather_warps=6, row_bufs=2)),
    "ldg_row_not16": (4, 20, 9, 7, 1, None, dict(path=FUSED, gather_warps=0, row_bufs=0), None),
    "tma_f32_ldg_bf16": (4, 20, 9, 12, 1, None, dict(path=FUSED, gather_warps=14, row_bufs=2),
                         dict(gather_warps=0, row_bufs=0)),
    "ldg_f32_gt32k_tma_bf16": (2, 150, 40, 216, 1, None, dict(path=FUSED, gather_warps=0, row_bufs=0),
                               dict(gather_warps=5, row_bufs=1)),
    # 20 KB rows: four buffers do not fit under the 113 KB two-CTA cap in f32; the 10 KB bf16 rows get five
    "ldg_4buf_nofit": (4, 20, 40, 128, 1, None, dict(path=FUSED, smem=57216, gather_warps=0, row_bufs=0),
                       dict(gather_warps=5, row_bufs=1)),
    # general: warps, column passes, seams
    "gen_u512_1pass": (3, 6, 512, 3, 1, ([6, 5, 6], [511, 480, 447]), dict(path=GENERAL, warps=16, ring=128), None),
    "gen_u513_2pass": (3, 6, 513, 3, 1, ([6, 6, 4], [512, 511, 480]), dict(path=GENERAL, warps=16, ring=128), None),
    "gen_u1024_2pass": (2, 5, 1024, 3, 2, ([5, 4], [1023, 991]), dict(path=GENERAL, warps=16), None),
    "gen_u1025_3pass": (3, 5, 1025, 3, 2, ([5, 3, 5], [1024, 1023, 512]), dict(path=GENERAL, warps=16), None),
    # general: boundary ring (16 warps: 1024 slots; back-pressure from Tn = 1025)
    "ring_t1024": (2, 1024, 481, 3, 1, ([1024, 1000], [480, 470]), dict(path=GENERAL, warps=16, ring=1024), None),
    "ring_t1025": (2, 1025, 481, 3, 1, ([1025, 1024], [480, 449]), dict(path=GENERAL, warps=16, ring=1024), None),
    # compact without hints: 128 slots, back-pressure from Tn = 129 (its dense runs are fused)
    "ring128_t129": (2, 129, 40, 6, 1, ([129, 128], [39, 30]), dict(path=FUSED, C=2), None),
}
# also compared with the compiled reference: every case of at most 8 lattices no longer and no larger than lattices it
# has run (T <= 2600, T*U <= 2600*300 cells), which includes the column-pass seams (U = 512/513, 1024/1025 at small T)
# and the ring wrap (T = 1024/1025)
REF_CASES = [k for k, c in CASES.items() if c[0] != "sms" and c[0] <= 8 and c[1] <= 2600 and c[1] * c[2] <= 2600 * 300]


def case_inputs(name):
    N, T, U, V, blank, lens, _, _ = CASES[name]
    N = sms() if N == "sms" else N
    seed = sum(map(ord, name))
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=seed, random_lengths=True, blank=blank)
    if lens is not None:
        xn, yn = np.asarray(lens[0], np.int32), np.asarray(lens[1], np.int32)
    # bf16-representable log-probs, so that the f32 and bf16 runs see the same inputs
    lp = torch.from_numpy(lp).to(torch.bfloat16).float().numpy()
    return lp, ys, xn, yn, blank


def is_fused(name):
    return CASES[name][6]["path"] == FUSED


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def w():
    import warp_rnnt_b200
    return warp_rnnt_b200


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load_lib()
        _lib.rnnt_b200_debug_last_launch.argtypes = [ctypes.c_void_p]
        _lib.rnnt_b200_debug_last_launch.restype = None
    return _lib


def last_launch():
    buf = (ctypes.c_int32 * len(FIELDS))()
    lib().rnnt_b200_debug_last_launch(buf)
    return dict(zip(FIELDS, list(buf)))


class Launch:
    """Context: the record of the recurrence launch made inside it (exactly one new launch record)."""

    def __enter__(self):
        self.before = last_launch()["seq"]
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.rec = last_launch()
        if exc[0] is None:
            assert self.rec["seq"] > self.before, "no recurrence launch was recorded"


def expect(rec, want, what):
    got = {k: rec[k] for k in want}
    assert got == want, "%s: launch record %s, expected %s (full record %s)" % (what, got, want, rec)


def dense(w, lp, ys, xn, yn, blank, mode, grads=True, bf16=False):
    xs = cu(lp).to(torch.bfloat16) if bf16 else cu(lp)
    with Launch() as L:
        c, g, loss = w._C.rnnt_loss_fused(xs, cu(ys), cu(xn), cu(yn), blank=blank, fastemit_lambda=LAM,
                                          want_grads=grads, lse_mode=mode)
    return c, g, loss, L.rec


def gathered(w, lp, ys, xn, yn, blank, mode):
    with Launch() as L:
        c, g = w._C.rnnt_loss_dense(cu(gather_np(lp, ys, blank)), cu(ys), cu(xn), cu(yn), blank=-1,
                                    fastemit_lambda=LAM, lse_mode=mode)
    return c, g, L.rec


def compact(w, xs_c, ys_c, xn, yn, blank, mode, hints, grads=True):
    """hints: (max_T, max_U), or None for the C entry point without them (max_T = max_U = 0)."""
    N = len(xn)
    xs, y, a, b = cu(xs_c), cu(ys_c), cu(xn), cu(yn)
    if hints is not None:
        w.set_lse_mode("exact" if mode == EXACT else "fast")
        try:
            with Launch() as L:
                c, pg, loc = w._C.rnnt_loss_compact(xs, y, a, b, blank=blank, fastemit_lambda=LAM,
                                                    required_grad=grads, max_T=hints[0], max_U=hints[1])
        finally:
            w.set_lse_mode("auto")
        return c, pg, loc, L.rec
    L_ = lib()
    STU, V = xs_c.shape
    ws = torch.empty(L_.rnnt_b200_workspace_bytes(STU, N), dtype=torch.uint8, device="cuda")
    c, pg = torch.empty(N, device="cuda"), torch.empty(STU, 2, device="cuda")
    loc = torch.empty(STU, dtype=torch.int64, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())                   # noqa: E731
    with Launch() as L:
        st = L_.rnnt_b200_compact_forward(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), p(ws),
                                          ctypes.c_size_t(ws.numel()), p(xs), p(y), p(a), p(b), p(c),
                                          p(pg) if grads else None, p(loc), None, ctypes.c_int64(STU), N, V, blank,
                                          ctypes.c_float(LAM), mode, 0, 0)
    assert st == 0
    return c, pg, loc, L.rec


def picked(name, N):
    """Lattices checked against the oracle: all of a small batch, eight of a large one."""
    return list(range(N)) if N <= 8 else sorted({0, 1, N // 3, N // 2, N - 2, N - 1, 7, N // 5})


# ------------------------------------------------------------------------------------------ the general path's side
def _general_main(out_dir):
    """Subprocess body (RNNT_B200_PATH=general): exact-mode outputs of every fused case on the general path."""
    import warp_rnnt_b200 as w
    assert os.environ.get("RNNT_B200_PATH") == "general"
    for name in CASES:
        if not is_fused(name):
            continue
        lp, ys, xn, yn, blank = case_inputs(name)
        c, g, _, rec = dense(w, lp, ys, xn, yn, blank, EXACT)
        assert rec["path"] == GENERAL, rec
        cg, gg, rec = gathered(w, lp, ys, xn, yn, blank, EXACT)
        assert rec["path"] == GENERAL, rec
        xs_c, ys_c = to_compact(lp, ys, xn, yn)
        cc, pc, _, rec = compact(w, xs_c, ys_c, xn, yn, blank, EXACT, (int(xn.max()), int(yn.max()) + 1))
        assert rec["path"] == GENERAL, rec
        for k, t in (("costs", c), ("grads", g), ("gcosts", cg), ("ggrads", gg), ("ccosts", cc), ("cgrads", pc)):
            np.save(os.path.join(out_dir, "%s_%s.npy" % (name, k)), t.cpu().numpy())


@pytest.fixture(scope="module")
def general_outputs():
    return subprocess_outputs("RNNT_B200_PATH", "general", "_general_main", module="tests.test_gpu_launch_configs")


# ------------------------------------------------------------------------------------------ the cases
@pytest.mark.parametrize("name", list(CASES))
def test_launch_config(w, general_outputs, name):
    N_, T, U, V, _, _, want, want_bf16 = CASES[name]
    lp, ys, xn, yn, blank = case_inputs(name)
    N = len(xn)
    pick = picked(name, N)
    fused = is_fused(name)
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    exact_hints = (int(xn.max()), int(yn.max()) + 1)
    c0, g0 = oracle.dense(lp[pick], ys[pick], xn[pick], yn[pick], blank=blank, fastemit_lambda=LAM)
    _, gp0 = oracle.dense(gather_np(lp[pick], ys[pick], blank), ys[pick], xn[pick], yn[pick], blank=-1,
                          fastemit_lambda=LAM)
    oc, opg, oloc = oracle.compact(xs_c, ys_c, xn, yn, blank=blank, fastemit_lambda=LAM) if N <= 8 else (None,) * 3
    tol = gtol(T, U)
    out = {}
    for mode in (EXACT, FAST):
        tag = "%s %s" % (name, "exact" if mode == EXACT else "fast")
        # dense f32: the configuration the case names
        c, g, loss, rec = dense(w, lp, ys, xn, yn, blank, mode)
        expect(rec, dict(want, groups=1), tag + " dense")
        np.testing.assert_allclose(c.cpu().numpy()[pick], c0, rtol=1e-5, err_msg=tag)
        err = np.abs(g.cpu().numpy()[pick] - g0).max()
        assert err <= tol, (tag, err)
        assert abs(loss.item() - c.sum().item()) <= 2e-6 * abs(c.sum().item()), tag     # the fused reduction
        if not fused:
            # forward only: beta alone, same costs
            cf, _, _, rec = dense(w, lp, ys, xn, yn, blank, mode, grads=False)
            expect(rec, dict(path=GENERAL, beta_only=1), tag + " forward only")
            assert torch.equal(cf, c), tag
        # gathered (N,T,U,2): the same plan
        cg, gg, rec = gathered(w, lp, ys, xn, yn, blank, mode)
        expect(rec, {k: want[k] for k in ("path", "C", "warps") if k in want}, tag + " gathered")
        np.testing.assert_allclose(cg.cpu().numpy()[pick], c0, rtol=1e-5, err_msg=tag)
        assert np.abs(gg.cpu().numpy()[pick] - gp0).max() <= tol, tag
        # compact: exact hints (the dense plan), loose hints, no hints (general, 16 warps, 128-slot ring)
        runs = {}
        for kind, hints in (("exact", exact_hints), ("loose", (T + 37, U + 5)), ("none", None)):
            cc, pc, loc, rec = compact(w, xs_c, ys_c, xn, yn, blank, mode, hints)
            if kind == "exact":
                expect(rec, {k: want[k] for k in ("path", "C", "warps") if k in want}, tag + " compact")
            if kind == "none":
                expect(rec, dict(path=GENERAL, warps=16, ring=128, beta_only=0), tag + " compact without hints")
            runs[kind] = (cc, pc, loc)
            if oc is not None:
                np.testing.assert_allclose(cc.cpu().numpy(), oc, rtol=1e-5, err_msg=tag + " compact " + kind)
                assert np.abs(pc.cpu().numpy() - opg).max() <= tol, (tag, kind)
                assert np.array_equal(loc.cpu().numpy(), oloc), (tag, kind)
            if rec["path"] == GENERAL:
                cf, _, _, rec = compact(w, xs_c, ys_c, xn, yn, blank, mode, hints, grads=False)
                expect(rec, dict(path=GENERAL, beta_only=1), tag + " compact forward only " + kind)
                assert torch.equal(cf, cc), (tag, kind)
        if mode == EXACT:
            for kind in ("loose", "none"):                        # every configuration: the same bits
                for a, b in zip(runs[kind], runs["exact"]):
                    assert torch.equal(a, b), (tag, kind)
            out = dict(c=c, g=g, cg=cg, gg=gg, compact=runs["exact"])
    # exact mode: the general path bit for bit
    if fused:
        go = general_outputs
        for k, t in (("costs", out["c"]), ("grads", out["g"]), ("gcosts", out["cg"]), ("ggrads", out["gg"]),
                     ("ccosts", out["compact"][0]), ("cgrads", out["compact"][1])):
            assert t.cpu().numpy().tobytes() == go["%s_%s.npy" % (name, k)].tobytes(), (name, k)
    # bf16 (fused cases): the f32 result on the same inputs, rounded once
    if fused:
        for mode in (EXACT, FAST):
            c32, g32, _, _ = dense(w, lp, ys, xn, yn, blank, mode)
            cb, gb, _, rec = dense(w, lp, ys, xn, yn, blank, mode, bf16=True)
            wb = {k: want[k] for k in ("path", "C", "slices") if k in want}   # the row gather flips at other V
            wb.update(want_bf16 or {})
            expect(rec, wb, name + " bf16")
            assert torch.equal(cb, c32), name
            assert torch.equal(gb, g32.to(torch.bfloat16)), name
    # the compiled reference, bit for bit
    if name in REF_CASES:
        same_as_reference("launch_%s/dense/costs" % name, out["c"])
        same_as_reference("launch_%s/dense/grads" % name, out["g"])
        same_as_reference("launch_%s/gather/costs" % name, out["cg"])
        same_as_reference("launch_%s/gather/grads" % name, out["gg"])
        cm, gm, lm = out["compact"]
        check_compact_vs_reference("launch_%s/compact" % name, cm, gm, lm, None, blank)


def test_misaligned_rows_take_the_ldg_gather(w):
    """Log-probs whose base address is not 16-byte aligned: the LDG gather, and the same bits as an aligned copy."""
    lp, ys, xn, yn, blank = case_inputs("c1_u32")
    flat = torch.empty(lp.size + 1, device="cuda")
    xs = flat[1:].view(lp.shape)
    xs.copy_(cu(lp))
    assert xs.data_ptr() % 16 != 0
    c0, g0, _, rec0 = dense(w, lp, ys, xn, yn, blank, EXACT)
    expect(rec0, dict(path=FUSED, gather_warps=14, row_bufs=2), "aligned")
    with Launch() as L:
        c, g, _ = w._C.rnnt_loss_fused(xs, cu(ys), cu(xn), cu(yn), blank=blank, fastemit_lambda=LAM, lse_mode=EXACT)
    expect(L.rec, dict(path=FUSED, gather_warps=0, row_bufs=0), "misaligned")
    assert torch.equal(c, c0) and torch.equal(g, g0)


# ------------------------------------------------------------------------------------------ the stream pipeline
# (N, T, U, V, groups): the general path (U = 70 at T = 300 does not fit the fused kernel) with an emit long against the
# wavefront; 9 lattices in 4 groups of 2 or 3, 33 in 8 groups of 4 or 5
PIPELINE = {"pipe4_n9": (9, 300, 70, 4096, 4), "pipe8_n33": (33, 300, 70, 1024, 8)}


def pipeline_inputs(name):
    from tests.test_gpu_holes import synth
    N, T, U, V, _ = PIPELINE[name]
    return synth(N, T, U, V, seed=N)


def _unpipelined_main(out_dir):
    """Subprocess body (RNNT_B200_PIPELINE=0): digests of the serial general path's outputs on the PIPELINE cases."""
    import warp_rnnt_b200 as w
    assert os.environ.get("RNNT_B200_PIPELINE") == "0"
    for name in PIPELINE:
        xs, ys, xn, yn = pipeline_inputs(name)
        with Launch() as L:
            c, g = w._C.rnnt_loss_dense(xs, ys, xn, yn, blank=0, fastemit_lambda=LAM, lse_mode=EXACT)
        assert L.rec["groups"] == 1 and L.rec["path"] == GENERAL, L.rec
        np.save(os.path.join(out_dir, name + "_costs.npy"), c.cpu().numpy())
        np.save(os.path.join(out_dir, name + "_grads.npy"), np.asarray(digest(g)))


def digest(t):
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()


@pytest.fixture(scope="module")
def unpipelined_outputs():
    return subprocess_outputs("RNNT_B200_PIPELINE", "0", "_unpipelined_main", module="tests.test_gpu_launch_configs")


@pytest.mark.parametrize("name", list(PIPELINE))
def test_pipeline_groups(w, unpipelined_outputs, name):
    N, T, U, V, groups = PIPELINE[name]
    xs, ys, xn, yn = pipeline_inputs(name)
    torch.cuda.synchronize()
    n0 = w._C.launch_count()
    with Launch() as L:
        c, g = w._C.rnnt_loss_dense(xs, ys, xn, yn, blank=0, fastemit_lambda=LAM, lse_mode=EXACT)
    assert w._C.launch_count() - n0 == 3 * groups                 # gather, wavefront, emit per group
    expect(L.rec, dict(path=GENERAL, groups=groups, warps=3), name)
    assert c.cpu().numpy().tobytes() == unpipelined_outputs[name + "_costs.npy"].tobytes()
    assert digest(g) == str(unpipelined_outputs[name + "_grads.npy"])
    pick = [0, N - 1]                                              # the first and the last group
    sel = torch.tensor(pick, device="cuda")
    c0, g0 = oracle.dense(xs[sel].cpu().numpy(), ys[sel].cpu().numpy(), xn[sel].cpu().numpy(), yn[sel].cpu().numpy(),
                          fastemit_lambda=LAM)
    np.testing.assert_allclose(c[sel].cpu().numpy(), c0, rtol=1e-5)
    assert np.abs(g[sel].cpu().numpy() - g0).max() <= gtol(T, U)
