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


def input_sample(xs, k=32):
    """Fingerprint of a (device-synthesised) input tensor: its values at k fixed positions."""
    import torch
    idx = torch.from_numpy(np.random.RandomState(12345).randint(0, xs.numel(), k)).to(xs.device)
    return xs.reshape(-1)[idx]
