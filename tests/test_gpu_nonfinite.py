"""GPU: the loss on masked and non-finite log-probs (tests/common.py NONFINITE_CASES), through every entry point that
runs a recurrence, in both LSE modes, on the fused and the general path and in both dense emit orders.

The recurrences stand in for -inf with a finite kBig (csrc/common.cuh); these tests pin down what that must not change:
  * tier A (live, the reference finite): exact mode equals the reference's recorded outputs bit for bit
    (tests/golden/reference_outputs.npz, keys nonfinite/...)
  * dead lattices (no alignment of finite log-probability): cost NaN (dense and gathered layouts, Tn >= 2 and
    Un >= 2) or +inf (Tn == 1 or Un == 1, compact layout); every gradient element the reference writes is NaN,
    every other one 0; the mismatch guard stays quiet; the reduced loss is not finite; the batch's other lattices are
    bit for bit what they are without the dead lattice.  Checked against the contract (the C oracle's classes,
    tests/test_nonfinite_oracle.py) and against the classes the reference recorded.  A lattice dead only through
    finfo.min masks gets the same classes (the reference's finite ~3.4e38 is an fp32 overflow artefact).
  * tier C (live, the reference has NaN from an interior LSE(-inf, -inf)): finite and within gtol of the fp64
    ref_transduce_np.
  * never-read positions (vocabulary entries that are neither blank nor the cell's label, padded frames and label
    columns, label ids past yn) holding NaN / +-inf / other in-range ids: outputs bit for bit those of the clean input.
    From logits, every logit of an in-lattice cell is read: there only the padding is poisoned, and its gradient is
    compared by class with torch.log_softmax followed by this library.
Fast LSE mode has the same classes; its finite values are checked against the fp64 recurrence.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import oracle
from tests.common import (NONFINITE_CASES, REF_OUTPUTS, assert_same_classes, class_of, dead_cost_class, gather_pairs,
                          lattice_tiers, masked_inputs, record, same_as_reference, threshold_inputs, to_compact,
                          written_dense)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ["exact", "fast"]
NEVER_READ = ["mix_ldg", "multi_cta"]       # cases whose never-read positions are poisoned


def gtol(T, U):
    return 2e-5 + 6e-6 * (T + U)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().float().cpu().numpy() if t.dtype == torch.bfloat16 else t.detach().cpu().numpy()


def grad_out(N):
    return torch.linspace(0.5, 1.5, N, device="cuda")


def clean_dead(case):
    """The case with its dead lattices unmasked (the run every other lattice must match)."""
    kinds = [("clean" if t in ("dead", "fmin") else k) for k, t in zip(case[6], lattice_tiers(case))]
    return case[:6] + (kinds,) + case[7:]


def poison(lp, ys, xn, yn, blank, seed, inside=True):
    """NaN / +inf / -inf in the padded cells and -- inside=True -- in the vocabulary entries of lattice cells that are
    neither the blank nor the cell's label; other in-range ids in the label padding."""
    lp, ys = lp.copy(), ys.copy()
    rng = np.random.RandomState(seed)
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    N, T, U, V = lp.shape
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        hit = np.ones((T, U, V), dtype=bool)
        hit[:Tn, :Un] = inside
        hit[:Tn, :Un, blank] = False
        for u in range(Un - 1):
            hit[:Tn, u, ys[n, u]] = False
        lp[n][hit] = vals[rng.randint(0, 3, int(hit.sum()))]
        ys[n, Un - 1:] = (ys[n, Un - 1:] + 1 + rng.randint(0, V - 1, U - Un)) % V
    return lp, ys


def entry_points(w, lp, ys, xn, yn, blank, key, out, logits_ref=True):
    """Every entry point on one input: out[key + '/<entry>/<tensor>'] = numpy array."""
    N, T, U, V = lp.shape
    a = [cu(x) for x in (lp, ys, xn, yn)]
    go = grad_out(N)
    c, g = w._C.rnnt_loss(*a, blank=blank)
    out[key + "/dense/costs"], out[key + "/dense/grads"] = host(c), host(g)
    out[key + "/dense/sum"] = host(w.rnnt_loss(*a, blank=blank, reduction="sum")).reshape(1)
    c, g = w._C.rnnt_loss(cu(gather_pairs(lp, ys, blank)), a[1], a[2], a[3], blank=-1)
    out[key + "/gathered/costs"], out[key + "/gathered/grads"] = host(c), host(g)
    x = a[0].clone().requires_grad_(True)
    c = w.rnnt_loss(x, a[1], a[2], a[3], blank=blank, gather=True)
    out[key + "/pygather/costs"], out[key + "/pygather/grads"] = host(c), host(torch.autograd.grad(c, x, go)[0])
    xs_c, ys_c = (cu(v) for v in to_compact(lp, ys, xn, yn))
    cum = torch.cumsum(a[2] * (a[3] + 1), dim=0, dtype=torch.int32)
    for tag, hints in (("compact", (0, 0)), ("compact_hints", (T, U))):
        c, pg, loc = w._C.rnnt_loss_compact(xs_c, ys_c, a[2], a[3], blank=blank, max_T=hints[0], max_U=hints[1])
        out[key + "/%s/costs" % tag], out[key + "/%s/pg" % tag] = host(c), host(pg)
        out[key + "/%s/back" % tag] = host(w._C.rnnt_loss_compact_backward(go, pg, cum, loc, V, blank))
    # bf16: the fp32 path on the bf16-rounded input, rounded once
    xb = a[0].to(torch.bfloat16)
    c, g, _ = w._C.rnnt_loss_fused(xb, a[1], a[2], a[3], blank)
    out[key + "/bf16/costs"], out[key + "/bf16/grads"] = host(c), host(g)
    c, g = w._C.rnnt_loss(xb.float(), a[1], a[2], a[3], blank=blank)
    out[key + "/bf16ref/costs"], out[key + "/bf16ref/grads"] = host(c), host(g.to(torch.bfloat16))
    if logits_ref:
        # from logits (lp as logits) against torch.log_softmax followed by this library
        x = a[0].clone().requires_grad_(True)
        c = w.rnnt_loss_from_logits(x, a[1], a[2], a[3], blank=blank)
        out[key + "/logits/costs"], out[key + "/logits/grads"] = host(c), host(torch.autograd.grad(c, x, go)[0])
        x = a[0].clone().requires_grad_(True)
        lps = torch.log_softmax(x, -1)
        c = w.rnnt_loss(lps, a[1], a[2], a[3], blank=blank)
        out[key + "/unfused/costs"], out[key + "/unfused/grads"] = host(c), host(torch.autograd.grad(c, x, go)[0])
        c, g = w._C.rnnt_loss(lps.detach().contiguous(), a[1], a[2], a[3], blank=blank)
        out[key + "/logsoftmax/costs"], out[key + "/logsoftmax/grads"] = host(c), host(g)


def run_all(out_dir=None):
    """Outputs of every entry point on every case, in both LSE modes (saved to out_dir when given)."""
    import warp_rnnt_b200 as w
    out = {}
    try:
        for mode in MODES:
            w.set_lse_mode(mode)
            for name, case in NONFINITE_CASES.items():
                lp, ys, xn, yn = masked_inputs(case)
                entry_points(w, lp, ys, xn, yn, case[4], "%s/%s" % (mode, name), out)
                lp2, ys2, _, _ = masked_inputs(clean_dead(case))
                c, g = w._C.rnnt_loss(cu(lp2), cu(ys2), cu(xn), cu(yn), blank=case[4])
                out["%s/%s/undead/costs" % (mode, name)], out["%s/%s/undead/grads" % (mode, name)] = host(c), host(g)
                if name in NEVER_READ:
                    lp3, ys3 = poison(lp, ys, xn, yn, case[4], seed=7)
                    entry_points(w, lp3, ys3, xn, yn, case[4], "%s/%s/poisoned" % (mode, name), out, logits_ref=False)
                    lp4, ys4 = poison(lp, ys, xn, yn, case[4], seed=8, inside=False)
                    entry_points(w, lp4, ys4, xn, yn, case[4], "%s/%s/padpoisoned" % (mode, name), out)
            lp, ys, xn, yn, _ = threshold_inputs()
            c, g = w._C.rnnt_loss(cu(lp), cu(ys), cu(xn), cu(yn))
            out["%s/threshold/costs" % mode], out["%s/threshold/grads" % mode] = host(c), host(g)
        torch.cuda.synchronize()
    finally:
        w.set_lse_mode("auto")
    if out_dir:
        np.savez(os.path.join(out_dir, "out.npz"), **out)
    return out


def in_subprocess(env_name, env_value):
    """run_all() in a subprocess with one environment switch -> (outputs, the subprocess's stdout)."""
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, **{env_name: env_value})
        code = "import sys; sys.path.insert(0, %r); from tests.test_gpu_nonfinite import run_all; run_all(%r)" % (ROOT, d)
        r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        return dict(np.load(os.path.join(d, "out.npz"))), r.stdout


# ------------------------------------------------------------------------------------------ expectations
_ref = None


def ref_array(key):
    global _ref
    if _ref is None:
        _ref = dict(np.load(REF_OUTPUTS))
    return _ref[key]


def check_dense(out, mode, name, entry, ref_key=None):
    """costs (N,) and a dense (N,T,U,V) gradient of one entry point."""
    case = NONFINITE_CASES[name]
    lp, ys, xn, yn = masked_inputs(case)
    N, T, U, V, blank = case[:5]
    if entry == "logsoftmax":
        lp = host(torch.log_softmax(cu(lp), -1))
    k = "%s/%s/%s/" % (mode, name, entry)
    costs, grads = out[k + "costs"], out[k + "grads"]
    written = written_dense(ys, xn, yn, T, U, V, blank)
    for n, tier in enumerate(lattice_tiers(case)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        g = grads[n]
        what = "%s lattice %d (%s)" % (k, n, case[6][n])
        if tier in ("dead", "fmin"):
            want = dead_cost_class(Tn, Un, False)
            assert np.array_equal(costs[n], want, equal_nan=True), (what, costs[n], want)
            assert np.array_equal(np.isnan(g), written[n]), "%s: %d NaN, %d expected" % (what, np.isnan(g).sum(), written[n].sum())
            assert not g[~written[n]].any(), what
            if ref_key and mode == "exact" and tier == "dead":
                same_as_reference("%s/class_%d" % (ref_key, n), class_of(g))
                assert np.array_equal(ref_array(ref_key + "/costs")[n], costs[n], equal_nan=True), what
            continue
        assert np.isfinite(costs[n]) and np.isfinite(g).all(), what
        if tier == "A" and mode == "exact" and ref_key:
            assert costs[n].tobytes() == ref_array(ref_key + "/costs")[n].tobytes(), what
            same_as_reference("%s/grads_%d" % (ref_key, n), g)
            continue
        # tier C, and the fast mode: close to the fp64 recurrence (peaked lattices: |alpha| ~ 1e4, ulp ~ 1e-3)
        with np.errstate(all="ignore"):
            c0, g0, _, _ = oracle.ref_transduce_np(lp[n, :Tn, :Un], ys[n, :Un - 1], blank)
        tol = gtol(T, U) * (10 if case[6][n] == "peaked" else 1)
        np.testing.assert_allclose(costs[n], c0, rtol=1e-5, err_msg=what)
        np.testing.assert_allclose(g[:Tn, :Un], g0, atol=tol, err_msg=what)
        assert not g[Tn:].any() and not g[:, Un:].any(), what


def check_compact(out, mode, name, tag):
    case = NONFINITE_CASES[name]
    lp, ys, xn, yn = masked_inputs(case)
    N, T, U, V, blank = case[:5]
    k = "%s/%s/%s/" % (mode, name, tag)
    costs, pg, back = out[k + "costs"], out[k + "pg"], out[k + "back"]
    go = host(grad_out(N))
    with np.errstate(all="ignore"):
        xs_c, ys_c = to_compact(lp, ys, xn, yn)
        c32, pg32, _ = oracle.compact(xs_c, ys_c, xn, yn, blank=blank, dtype="f32")
    o = 0
    for n, tier in enumerate(lattice_tiers(case)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        sl = slice(o, o + Tn * Un)
        o += Tn * Un
        what = "%s lattice %d (%s)" % (k, n, case[6][n])
        if tier in ("dead", "fmin"):
            assert costs[n] == np.inf, (what, costs[n])
            # NaN where a gradient is computed, 0 on the structural zeros (the last row's inner blanks, the last
            # column's labels) -- for a dead lattice also the C oracle's classes
            want = np.full((Tn, Un, 2), np.nan, np.float32)
            want[Tn - 1, :Un - 1, 0] = 0
            want[:, Un - 1, 1] = 0
            assert_same_classes(pg[sl], want.reshape(-1, 2), what)
            if tier == "dead":
                assert_same_classes(pg[sl], pg32[sl].astype(np.float32), what)
            if mode == "exact" and tier == "dead":
                same_as_reference("nonfinite/%s/compact/class_%d" % (name, n), class_of(pg[sl]))
                same_as_reference("nonfinite/%s/compact/back_class_%d" % (name, n), class_of(back[sl]))
            continue
        assert np.isfinite(costs[n]) and np.isfinite(pg[sl]).all() and np.isfinite(back[sl]).all(), what
        if mode == "exact" and tier == "A":
            assert costs[n].tobytes() == ref_array("nonfinite/%s/compact/costs" % name)[n].tobytes(), what
            same_as_reference("nonfinite/%s/compact/pg_%d" % (name, n), pg[sl])
            same_as_reference("nonfinite/%s/compact/back_%d" % (name, n), back[sl])
        else:
            with np.errstate(all="ignore"):
                c0, g0, _, _ = oracle.ref_transduce_np(lp[n, :Tn, :Un], ys[n, :Un - 1], blank)
            np.testing.assert_allclose(costs[n], c0, rtol=1e-5, err_msg=what)
            tol = gtol(T, U) * (10 if case[6][n] == "peaked" else 1)
            dense = back[sl].reshape(Tn, Un, V) / go[n]
            np.testing.assert_allclose(dense, g0, atol=tol, err_msg=what)


def check_case(out, mode, name):
    case = NONFINITE_CASES[name]
    N = case[0]
    go = host(grad_out(N))
    ref = "nonfinite/%s" % name
    check_dense(out, mode, name, "dense", ref + "/dense")
    k = "%s/%s/" % (mode, name)
    # the gathered layout is the dense one's pair of columns: same costs, same (blank, label) gradients
    assert_same_classes(out[k + "gathered/costs"], out[k + "dense/costs"], k + "gathered")
    lp, ys, xn, yn = masked_inputs(case)
    want = gather_pairs(out[k + "dense/grads"], ys, case[4])
    for n in range(N):
        want[n, :, yn[n]:, 1] = 0                        # no label transition out of the last column
    assert_same_classes(out[k + "gathered/grads"], want, k + "gathered")
    # gather=True: the dense gradient times grad_output, a label never being the blank here
    assert_same_classes(out[k + "pygather/costs"], out[k + "dense/costs"], k + "pygather")
    # (scatter_add: 0 + (-0) is +0, so zeros are compared without their sign)
    assert_same_classes(out[k + "pygather/grads"], out[k + "dense/grads"] * go[:, None, None, None], k + "pygather",
                        signed_zeros=False)
    # the reduced loss is not finite as soon as one lattice is dead
    dead = any(t in ("dead", "fmin") for t in lattice_tiers(case))
    assert np.isfinite(out[k + "dense/sum"][0]) != dead, out[k + "dense/sum"]
    # every other lattice is what it is without the dead ones
    live = [n for n, t in enumerate(lattice_tiers(case)) if t not in ("dead", "fmin")]
    assert_same_classes(out[k + "dense/costs"][live], out[k + "undead/costs"][live], k + "undead")
    assert_same_classes(out[k + "dense/grads"][live], out[k + "undead/grads"][live], k + "undead")
    for tag in ("compact", "compact_hints"):
        check_compact(out, mode, name, tag)
    # bf16: the fp32 path on the same (bf16-rounded) input, rounded once; NaN stays NaN
    assert_same_classes(out[k + "bf16/costs"], out[k + "bf16ref/costs"], k + "bf16")
    assert_same_classes(out[k + "bf16/grads"], out[k + "bf16ref/grads"], k + "bf16")
    # from logits: the unfused log_softmax pipeline's classes and (close) values; that pipeline's loss is the
    # reference's on the same log-probs
    check_dense(out, mode, name, "logsoftmax", ref + "/logsoftmax")
    for t in ("costs", "grads"):
        a, b = out[k + "logits/" + t], out[k + "unfused/" + t]
        assert np.array_equal(class_of(a), class_of(b)), (k + "logits/" + t, (class_of(a) != class_of(b)).sum())
    fin = np.isfinite(out[k + "unfused/costs"])
    np.testing.assert_allclose(out[k + "logits/costs"][fin], out[k + "unfused/costs"][fin], rtol=1e-5)
    for n, kind in enumerate(case[6]):
        # the documented 1e-4 (rnnt_loss_from_logits); peaked lattices carry |alpha| ~ 1e4 through T+U steps, whose
        # fp32 rounding moves their gradients by up to ~1e-3 between any two summation orders (as in the fast mode)
        a, b = out[k + "logits/grads"][n], out[k + "unfused/grads"][n]
        fin = np.isfinite(b)
        tol = 10 * gtol(case[1], case[2]) if kind == "peaked" else 1e-4
        np.testing.assert_allclose(a[fin], b[fin], rtol=0, atol=tol, err_msg="%slogits lattice %d (%s)" % (k, n, kind))
    if name in NEVER_READ:
        for e in ("dense", "gathered", "pygather", "compact", "compact_hints", "bf16"):
            for t in ("costs", "grads", "pg", "back"):
                kk = "%s/%s" % (e, t)
                if k + kk in out:
                    assert_same_classes(out[k + "poisoned/" + kk], out[k + kk], k + "poisoned/" + kk)
                    assert_same_classes(out[k + "padpoisoned/" + kk], out[k + kk], k + "padpoisoned/" + kk)
        # from logits, padding poisoned: costs and in-lattice gradients unchanged, the padding's gradient by class
        # as torch.log_softmax + this library give it
        assert_same_classes(out[k + "padpoisoned/logits/costs"], out[k + "logits/costs"], k + "padpoisoned/logits")
        g, g0, gu = out[k + "padpoisoned/logits/grads"], out[k + "logits/grads"], out[k + "padpoisoned/unfused/grads"]
        for n in range(N):
            Tn, Un = int(xn[n]), int(yn[n]) + 1
            assert_same_classes(g[n, :Tn, :Un], g0[n, :Tn, :Un], k + "padpoisoned/logits lattice %d" % n)
            pad = np.ones(g.shape[1:3], dtype=bool)
            pad[:Tn, :Un] = False
            assert np.array_equal(class_of(g[n][pad]), class_of(gu[n][pad])), k + "padpoisoned/logits padding %d" % n
            assert not np.nan_to_num(g[n][pad]).any()


@pytest.fixture(scope="module")
def default_run():
    return in_subprocess("RNNT_B200_PATH", "auto")


@pytest.fixture(scope="module")
def general_run():
    return in_subprocess("RNNT_B200_PATH", "general")


@pytest.fixture(scope="module")
def composed_run():
    return in_subprocess("RNNT_B200_EMIT", "compose")


@pytest.fixture(scope="module")
def default_outputs(default_run):
    return default_run[0]


@pytest.fixture(scope="module")
def general_outputs(general_run):
    return general_run[0]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(NONFINITE_CASES))
def test_default_path(default_outputs, mode, name):
    check_case(default_outputs, mode, name)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(NONFINITE_CASES))
def test_general_path(general_outputs, mode, name):
    check_case(general_outputs, mode, name)


def test_dead_threshold(default_outputs, general_outputs):
    """Costs just below 5e29 stay finite (the reference's value), costs just above take the dead classes: both paths,
    both LSE modes."""
    lp, ys, xn, yn, dead = threshold_inputs()
    c64, _ = oracle.dense(lp, ys, xn, yn, dtype="f64")
    written = written_dense(ys, xn, yn, *lp.shape[1:], 0)
    for path, out in (("default", default_outputs), ("general", general_outputs)):
        for mode in MODES:
            costs, grads = out["%s/threshold/costs" % mode], out["%s/threshold/grads" % mode]
            for n, d in enumerate(dead):
                what = (path, mode, n, costs[n])
                if d:
                    want = dead_cost_class(int(xn[n]), int(yn[n]) + 1, False)
                    assert np.array_equal(costs[n], want, equal_nan=True), what
                    assert np.array_equal(np.isnan(grads[n]), written[n]), what
                else:
                    assert 4.8e29 < costs[n] < 5e29, what
                    np.testing.assert_allclose(costs[n], c64[n], rtol=1e-6, err_msg=str(what))
                    assert not np.isnan(grads[n]).any(), what


def test_guard_quiet(default_run, general_run, composed_run):
    """The forward/backward mismatch guard does not fire on dead lattices (its ratio is NaN in the reference)."""
    for _, stdout in (default_run, general_run, composed_run):
        assert "WARNING" not in stdout, stdout[:2000]


def test_composed_emit_order(default_outputs, composed_run):
    """The composed dense emit (forced: these gradients fit in L2, so the default is zero-fill + patch) writes the same
    classes and bits."""
    out = composed_run[0]
    for k in default_outputs:
        if "/dense/" in k or "/bf16/" in k:
            assert_same_classes(out[k], default_outputs[k], k)


# ------------------------------------------------------------------------------------------ reference records
def record_reference(rec, ref):
    """What the unmodified reference computes on these inputs (tests/golden/make_reference_outputs.py).  Tier A lattices
    are stored as values, dead ones as class_of() masks; lattices where the reference itself is NaN (tier C) or where
    it deviates on purpose (finfo.min) only through the costs."""
    for name, case in NONFINITE_CASES.items():
        lp, ys, xn, yn = masked_inputs(case)
        N, T, U, V, blank = case[:5]
        tiers = lattice_tiers(case)
        a = [cu(x) for x in (lp, ys, xn, yn)]
        for entry, x in (("dense", a[0]), ("logsoftmax", torch.log_softmax(a[0], -1).contiguous())):
            c, g = ref.rnnt_loss(x, a[1], a[2], a[3], blank=blank)
            c, g = host(c), host(g)
            key = "nonfinite/%s/%s" % (name, entry)
            record(rec, key + "/costs", c)
            for n, t in enumerate(tiers):
                if t == "A":
                    record(rec, "%s/grads_%d" % (key, n), g[n])
                elif t == "dead":
                    record(rec, "%s/class_%d" % (key, n), class_of(g[n]))
        xs_c, ys_c = (cu(v) for v in to_compact(lp, ys, xn, yn))
        c, pg, loc = ref.rnnt_loss_compact(xs_c, ys_c, a[2], a[3], blank=blank)
        cum = torch.cumsum(a[2] * (a[3] + 1), dim=0, dtype=torch.int32)
        back = host(ref.rnnt_loss_compact_backward(grad_out(N), pg, cum, loc, V, blank))
        c, pg = host(c), host(pg)
        key = "nonfinite/%s/compact" % name
        record(rec, key + "/costs", c)
        o = 0
        for n, t in enumerate(tiers):
            Un = int(yn[n]) + 1
            sl = slice(o, o + int(xn[n]) * Un)
            o = sl.stop
            p = pg[sl].copy()
            p[Un - 1::Un, 1] = 0        # never written by the reference at maximal label length (DESIGN.md 4); ours: 0
            if t == "A":
                record(rec, "%s/pg_%d" % (key, n), p)
                record(rec, "%s/back_%d" % (key, n), back[sl])
            elif t == "dead":
                record(rec, "%s/class_%d" % (key, n), class_of(p))
                record(rec, "%s/back_class_%d" % (key, n), class_of(back[sl]))

