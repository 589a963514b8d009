"""Shared helpers for the tests: golden vectors, stored outputs of the reference, synthetic inputs (the reference's
recipe)."""
import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "reference_vectors.json")))
REF_OUTPUTS = os.path.join(HERE, "golden", "reference_outputs.npz")
_ref_out = None

# Outputs of the unmodified reference kernels (1ytic/warp-rnnt built for sm_90a) on the inputs of the tests below,
# recorded on an H100 by tests/golden/make_reference_outputs.py.  A tensor of at most FULL_MAX elements is stored
# whole; a larger one as the SHA-256 of its bytes plus its values at SAMPLE seeded positions (mostly non-zero ones),
# which name the first differing elements when the digest does not match.
FULL_MAX = 4096
SAMPLE = 64


def _host(t):
    a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
    return np.ascontiguousarray(a)


def digest(t):
    return hashlib.sha256(_host(t).tobytes()).hexdigest()


def record(rec, key, t):
    """Store tensor `t` under `key` in the dict `rec` (the writer side of same_as_reference)."""
    a = _host(t)
    if a.size <= FULL_MAX:
        rec[key] = a
        return
    flat = a.reshape(-1)
    nz = np.flatnonzero(flat)
    rng = np.random.RandomState(a.size % (2 ** 31))
    pick = np.concatenate([rng.choice(nz, min(SAMPLE - 8, nz.size), replace=False) if nz.size else nz,
                           rng.randint(0, flat.size, 8)]).astype(np.int64)
    rec[key + ".idx"] = pick
    rec[key + ".val"] = flat[pick]
    rec[key + ".shape"] = np.asarray(a.shape, dtype=np.int64)
    rec[key + ".sha256"] = np.asarray(digest(a))


def same_as_reference(key, t):
    """Assert that `t` equals the reference's stored output `key` bit for bit."""
    global _ref_out
    if _ref_out is None:
        _ref_out = dict(np.load(REF_OUTPUTS))
    a = _host(t)
    if key in _ref_out:
        r = _ref_out[key]
        assert a.shape == r.shape and a.dtype == r.dtype, (key, a.shape, a.dtype, r.shape, r.dtype)
        np.testing.assert_array_equal(a, r, err_msg=key)
        assert a.tobytes() == r.tobytes(), "%s differs from the reference (signed zeros)" % key
        return
    assert tuple(a.shape) == tuple(_ref_out[key + ".shape"]), (key, a.shape)
    idx, val = _ref_out[key + ".idx"], _ref_out[key + ".val"]
    np.testing.assert_array_equal(a.reshape(-1)[idx], val, err_msg=key)
    assert digest(a) == str(_ref_out[key + ".sha256"]), "%s differs from the reference" % key


def log_softmax(x, axis=-1):
    x = np.asarray(x, dtype=np.float64)
    m = x.max(axis=axis, keepdims=True)
    y = x - m
    return y - np.log(np.exp(y).sum(axis=axis, keepdims=True))


def golden_case(name):
    """-> dict(lp f32 (N,T,U,V) log-softmaxed, ys, xn, yn, costs, grads)."""
    r = GOLDEN[name]
    xs = np.asarray(r["xs"], dtype=np.float32)
    # the reference tests log_softmax in fp32 torch (test.py:42); fp64-then-round is within 1 ulp
    lp = log_softmax(xs).astype(np.float32)
    ys = np.asarray(r["ys"], dtype=np.int32).reshape(xs.shape[0], -1)
    costs = np.atleast_1d(np.asarray(r.get("expected_costs", r.get("expected_cost")), dtype=np.float64))
    return dict(lp=lp, ys=ys, xn=np.asarray(r["xn"], dtype=np.int32), yn=np.asarray(r["yn"], dtype=np.int32),
                costs=costs, grads=np.asarray(r["expected_grads"], dtype=np.float64))


def make_inputs(N, T, U, V, seed=0, random_lengths=False, blank=0, min_len=True):
    """Synthetic inputs following the reference's benchmark recipe (benchmark.py:11-27):
    randn -> log_softmax, labels in [1,V) (never blank when blank == 0), full or random lengths
    (random: benchmark.py:20-23, shifted so the max hits T / U-1)."""
    rng = np.random.RandomState(seed)
    xs = rng.randn(N, T, U, V).astype(np.float32)
    lp = log_softmax(xs).astype(np.float32)
    if V > 1:
        ys = rng.randint(0, V - 1, (N, max(U - 1, 0))).astype(np.int32)
        ys = np.where(ys >= blank, ys + 1, ys).astype(np.int32)     # skip the blank id
    else:
        ys = np.zeros((N, max(U - 1, 0)), dtype=np.int32)
    if random_lengths:
        xn = rng.randint(max(T // 2, 1), T + 1, (N,)).astype(np.int32)
        yn = rng.randint(U // 2, U, (N,)).astype(np.int32) if U > 1 else np.zeros(N, np.int32)
        xn = xn + T - xn.max()
        yn = yn + (U - 1) - yn.max()
    else:
        xn = np.full(N, T, dtype=np.int32)
        yn = np.full(N, U - 1, dtype=np.int32)
    return lp, ys, xn, yn


def to_compact(lp, ys, xn, yn):
    """Ragged concat as in the reference test (test.py:291-299)."""
    V = lp.shape[-1]
    xs_c = np.concatenate([lp[i, :xn[i], :yn[i] + 1].reshape(-1, V) for i in range(lp.shape[0])], axis=0)
    ys_c = np.concatenate([ys[i, :yn[i]] for i in range(ys.shape[0])], axis=0).astype(np.int32)
    return np.ascontiguousarray(xs_c), np.ascontiguousarray(ys_c)


def from_compact(flat, xn, yn, T, U):
    """(STU,V) -> padded (N,T,U,V) with zeros."""
    V = flat.shape[-1]
    N = len(xn)
    out = np.zeros((N, T, U, V), dtype=flat.dtype)
    o = 0
    for i in range(N):
        c = int(xn[i]) * (int(yn[i]) + 1)
        out[i, :xn[i], :yn[i] + 1] = flat[o:o + c].reshape(xn[i], yn[i] + 1, V)
        o += c
    return out


# ------------------------------------------------------------------------------------------ masked / non-finite inputs
# Masks applied to one lattice of a log_softmax(randn) batch (the label column masked is k = min(2, Un - 2), its id
# ys[n, k] is never the blank).  Tiers (DESIGN.md 4):
#   "A"     live, the reference is finite: exact mode equals the reference bit for bit
#   "C"     live, but the reference computes an interior LSE(-inf, -inf) = NaN: finite and close to ref_transduce_np
#   "dead"  no alignment of finite log-probability: cost NaN / +inf, every gradient element the reference writes NaN
#   "fmin"  dead only through finfo.min masks: the same classes as "dead" (the reference's finite ~3.4e38 cost is an
#           fp32 overflow artefact)
NINF = float("-inf")
FMIN = float(np.finfo(np.float32).min)
MASK_TIER = {"clean": "A", "label_t0": "A", "fmin_t0": "A", "fmin_t01": "A", "peaked": "A", "unnorm": "A",
             "vocab_ninf": "A", "label_t01": "C", "label_all": "dead", "last_blank": "dead", "blank_col": "dead", "label_all_fmin": "fmin"}


def apply_mask(lp, ys, n, Tn, Un, kind, blank, rng):
    """Mask lattice n of lp (N,T,U,V) in place."""
    k = max(0, min(2, Un - 2))
    if kind == "clean":
        return
    if kind in ("label_all", "label_all_fmin", "label_t0", "label_t01", "fmin_t0", "fmin_t01"):
        assert Un >= 2
        rows = Tn if kind.startswith("label_all") else (2 if kind.endswith("01") else 1)
        lp[n, :rows, k, ys[n, k]] = FMIN if "fmin" in kind else NINF
    elif kind == "last_blank":
        lp[n, Tn - 1, Un - 1, blank] = NINF
    elif kind == "blank_col":                  # Un == 1: every alignment takes this blank
        assert Un == 1
        lp[n, 0, 0, blank] = NINF
    elif kind == "peaked":
        # off-token log-probs around -200; each cell has one likely token, the blank or its label half the time each
        T, U, V = lp.shape[1:]
        lp[n] = -200.0 + rng.randn(T, U, V).astype(np.float32)
        tok = np.where(rng.rand(T, U) < 0.5, blank, np.concatenate([ys[n], [blank]])[None, :U])
        lp[n, np.arange(T)[:, None], np.arange(U)[None, :], tok] = -1e-3 * rng.rand(T, U).astype(np.float32)
    elif kind == "unnorm":                     # never normalised, many values above zero
        lp[n] = (3.0 * rng.randn(*lp.shape[1:]) + 2.0).astype(np.float32)
    elif kind == "vocab_ninf":
        # vocabulary entries 0..11 except the blank masked -inf in every cell (the labels are moved off them): from
        # logits, with V = 30 these are the first logits of lanes 1-7 of the normaliser's online sum, with V % 4 == 0
        # and V > 128 whole float4 groups of its lanes 1 and 2 (csrc/logits.cu, k_lse_pairs)
        masked = [v for v in range(12) if v != blank]
        assert lp.shape[3] > 24 and blank < 12
        ys[n] = np.where(np.isin(ys[n], masked), ys[n] + 12, ys[n])
        lp[n][..., masked] = NINF
    else:
        raise ValueError(kind)


def masked_inputs(case):
    """case = (N, T, U, V, blank, seed, kinds, xn or None, yn or None) -> lp, ys, xn, yn (full lengths by default)."""
    N, T, U, V, blank, seed, kinds, xn, yn = case
    lp, ys, _, _ = make_inputs(N, T, U, V, seed=seed, blank=blank)
    xn = np.full(N, T, np.int32) if xn is None else np.asarray(xn, np.int32)
    yn = np.full(N, U - 1, np.int32) if yn is None else np.asarray(yn, np.int32)
    rng = np.random.RandomState(seed + 1)
    for n, kind in enumerate(kinds):
        apply_mask(lp, ys, n, int(xn[n]), int(yn[n]) + 1, kind, blank, rng)
    return lp, ys, xn, yn


# Batches mixing dead and live lattices.  Name -> (N, T, U, V, blank, seed, per-lattice mask, xn, yn).
#   mix_tma   : rows of 160 B (TMA row gather in the fused kernel)
#   mix_ldg   : rows of 7 floats (LDG gather), ragged lengths, two warps per wavefront on the general path
#   edges     : Tn = 1 and Un = 1 lattices (dead ones cost +inf), unnormalised input
#   multi_cta : cfg-2-sized lattices: several CTAs per lattice, TMA row gather, peaked input
#   vocab_v30 / vocab_v132: masked vocabulary entries where the from-logits normaliser sums online (V % 4 != 0; and
#               V % 4 == 0 with more than one float4 per lane)
NONFINITE_CASES = {
    "mix_tma": (6, 6, 5, 8, 0, 101, ["label_all", "clean", "last_blank", "label_t0", "label_all_fmin", "label_t01"],
                None, None),
    "mix_ldg": (5, 33, 34, 7, 2, 102, ["clean", "label_all", "fmin_t0", "fmin_t01", "label_t01"],
                [33, 30, 33, 17, 25], [33, 20, 33, 9, 30]),
    "edges": (5, 5, 6, 6, 1, 103, ["label_all", "blank_col", "clean", "unnorm", "last_blank"],
              [1, 5, 1, 5, 5], [5, 0, 3, 5, 0]),
    "multi_cta": (3, 150, 40, 28, 0, 104, ["label_all", "peaked", "last_blank"], [150, 150, 120], [39, 30, 39]),
    "vocab_v30": (3, 12, 9, 30, 0, 105, ["vocab_ninf", "label_all", "unnorm"], None, [8, 8, 5]),
    "vocab_v132": (2, 10, 6, 132, 1, 106, ["vocab_ninf", "last_blank"], None, None),
}


def threshold_inputs():
    """Four live lattices whose costs lie just below (4.9e29) and just above (5.1e29) the 5e29 from which the kernels
    take a lattice for dead (csrc/common.cuh, lattice_dead): Tn = 1 with one alignment, and Tn = Un = 3 with six
    alignments of five equal edges.  -> lp, ys, xn, yn, dead flags."""
    N, T, U, V = 4, 3, 3, 4
    lp = np.full((N, T, U, V), -1.0, np.float32)
    ys = np.tile(np.array([1, 2], np.int32), (N, 1))
    xn = np.array([1, 1, 3, 3], np.int32)
    yn = np.array([1, 1, 2, 2], np.int32)
    for n, (label, blank) in enumerate([(-4.0e29, -0.9e29), (-4.0e29, -1.1e29)]):
        lp[n, 0, 0, 1], lp[n, 0, 1, 0] = label, blank
    for n, x in ((2, -0.98e29), (3, -1.02e29)):
        lp[n, :, :, 0] = x
        lp[n, :, 0, 1] = x
        lp[n, :, 1, 2] = x
    return lp, ys, xn, yn, [False, True, False, True]


def gather_pairs(lp, ys, blank):
    """(N,T,U,V) -> the gathered (N,T,U,2) [blank, label] layout (the last column's label slot holds the blank)."""
    N, T, U, V = lp.shape
    index = np.full((N, T, U, 2), blank, dtype=np.int64)
    index[:, :, :U - 1, 1] = ys[:, None, :]
    return np.ascontiguousarray(np.take_along_axis(lp, index, axis=3))


def lattice_tiers(case):
    return [MASK_TIER[k] for k in case[6]]


def dead_cost_class(Tn, Un, compact):
    """Cost of a dead lattice (the reference's class)."""
    return np.inf if (compact or Tn == 1 or Un == 1) else np.nan


def written_dense(ys, xn, yn, T, U, V, blank):
    """Elements of a dense (N,T,U,V) gradient that the reference writes: the blank of every lattice cell but the last
    row's inner ones, the label of every cell left of the last column."""
    N = len(xn)
    m = np.zeros((N, T, U, V), dtype=bool)
    for n in range(N):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        m[n, :Tn - 1, :Un, blank] = True
        m[n, Tn - 1, Un - 1, blank] = True
        for u in range(Un - 1):
            m[n, :Tn, u, ys[n, u]] = True
    return m


def assert_same_classes(got, want, what="", signed_zeros=True):
    """Finite elements bit for bit (signed_zeros=False: by value), and the same NaN and +-inf positions (the sign and
    payload of a NaN are free)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), "%s: NaN at %d positions, expected %d (%d differ)" % (
        what, gn.sum(), wn.sum(), (gn != wn).sum())
    for s in (np.inf, -np.inf):
        assert np.array_equal(got == s, want == s), "%s: %s positions differ" % (what, s)
    fin = np.isfinite(want)
    g, w = got[fin], want[fin]
    if not signed_zeros:
        g, w = g + 0.0, w + 0.0                     # -0 + 0 == +0
    bad = g.view(np.uint32 if g.dtype == np.float32 else np.uint64) != w.view(np.uint32 if w.dtype == np.float32 else np.uint64)
    assert not bad.any(), "%s: %d finite elements differ, e.g. %r vs %r" % (what, bad.sum(), g[bad][:3], w[bad][:3])


def class_of(a):
    """int8 class per element: 0 finite, 1 NaN, 2 +inf, 3 -inf (how the reference records store non-finite outputs)."""
    a = np.asarray(a)
    return (np.isnan(a) * 1 + (a == np.inf) * 2 + (a == -np.inf) * 3).astype(np.int8)


def input_sample(xs, k=32):
    """Fingerprint of a (device-synthesised) input tensor: its values at k fixed positions."""
    import torch
    idx = torch.from_numpy(np.random.RandomState(12345).randint(0, xs.numel(), k)).to(xs.device)
    return xs.reshape(-1)[idx]
