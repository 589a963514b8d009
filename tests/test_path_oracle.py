"""CPU: the fp64 restatement of k2's lattice types and delay penalty (tests/path_oracle.py) against brute-force path
enumeration, central differences and the regular lattice of tests/pruned_oracle.py, and the windows rule of the
one-symbol-per-frame types."""
import numpy as np
import pytest

from tests import path_oracle as pa
from tests import pruned_oracle as po


def make_pairs(N, T, U, seed):
    rng = np.random.RandomState(seed)
    p = np.log(rng.dirichlet(np.ones(3), size=(N, T, U))[..., :2])       # a blank and a label out of 3 symbols
    xn = rng.randint(1, T + 1, N).astype(np.int32)
    yn = rng.randint(0, U, N).astype(np.int32)
    return p, xn, yn


@pytest.mark.parametrize("kind", pa.TYPES)
@pytest.mark.parametrize("seed", range(4))
def test_brute_force(kind, seed):
    p, xn, yn = make_pairs(6, 4, 4, seed)
    rng = np.random.RandomState(100 + seed)
    p[rng.rand(*p.shape) < 0.1] = -np.inf                # masked log-probs
    p[rng.rand(*p.shape) < 0.1] = pa.KBIG                # removed edges
    c, g, _ = pa.lattice(p, xn, yn, kind)
    cb, gb = pa.brute_force(p, xn, yn, kind)
    np.testing.assert_array_equal(np.isinf(c), np.isinf(cb))
    fin = np.isfinite(cb)
    np.testing.assert_allclose(c[fin], cb[fin], rtol=0, atol=1e-12)
    np.testing.assert_allclose(g[fin], gb[fin], rtol=0, atol=1e-12)
    assert not g[~fin].any()


@pytest.mark.parametrize("kind", pa.TYPES)
def test_central_differences(kind):
    p, xn, yn = make_pairs(3, 5, 4, 7)
    xn[:] = 5
    yn[:] = [3, 2, 1]
    _, g, _ = pa.lattice(p, xn, yn, kind)
    h = 1e-6
    num = np.zeros_like(p)
    it = np.nditer(p, flags=["multi_index"])
    for _ in it:
        i = it.multi_index
        q1, q2 = p.copy(), p.copy()
        q1[i] += h
        q2[i] -= h
        num[i] = (pa.lattice(q1, xn, yn, kind)[0][i[0]] - pa.lattice(q2, xn, yn, kind)[0][i[0]]) / (2 * h)
    np.testing.assert_allclose(g, num, atol=1e-7)


def test_regular_matches_pruned_oracle():
    rng = np.random.RandomState(3)
    N, T, U, V = 4, 7, 5, 6
    x = rng.randn(N, T, U, V)
    ys = rng.randint(1, V, (N, U - 1)).astype(np.int32)
    xn = np.array([7, 5, 1, 3], np.int32)
    yn = np.array([4, 2, 3, 0], np.int32)
    ranges = np.zeros((N, T), np.int32)
    c0, g0 = po.lattice(x, ys, xn, yn, ranges)               # S = U windows at 0: the whole lattice
    lp = po.log_softmax(x)
    lab = np.concatenate([ys, np.zeros((N, 1), np.int32)], axis=1)
    pairs = np.stack([lp[..., 0], np.take_along_axis(lp, lab[:, None, :, None].repeat(T, 1), 3)[..., 0]], -1)
    c, g, _ = pa.lattice(pairs, xn, yn, "regular")
    np.testing.assert_allclose(c, c0, rtol=1e-12)
    # the pair gradients expand to po's logit gradient through log_softmax
    go = np.zeros_like(lp)
    go[..., 0] += g[..., 0]
    np.put_along_axis(go, lab[:, None, :, None].repeat(T, 1), np.take_along_axis(go, lab[:, None, :, None].repeat(T, 1), 3)
                      + g[..., 1:2], 3)
    full = go - np.exp(lp) * go.sum(-1, keepdims=True)
    for n in range(N):
        Tn, Un = xn[n], yn[n] + 1
        np.testing.assert_allclose(full[n, :Tn, :Un], g0[n, :Tn, :Un], atol=1e-12)


@pytest.mark.parametrize("kind", ["modified", "constrained"])
def test_more_labels_than_frames(kind):
    p, _, _ = make_pairs(2, 4, 7, 1)
    xn = np.array([3, 4], np.int32)
    yn = np.array([4, 4], np.int32)                          # Un - 1 = 4 > Tn = 3; = Tn = 4
    c, g, _ = pa.lattice(p, xn, yn, kind)
    assert c[0] == np.inf and not g[0].any()
    assert np.isfinite(c[1])


def test_penalty_order():
    p, xn, yn = make_pairs(3, 6, 4, 5)
    xn[:] = [6, 3, 0]
    q = pa.penalise(p, xn, yn, 0.05)
    assert q.dtype == np.float32
    Tn, Un = 6, yn[0] + 1
    for t in range(Tn):
        pen = (np.float32(Tn - 1) * np.float32(0.5) - np.float32(t)) * np.float32(0.05)
        np.testing.assert_array_equal(q[0, t, :Un - 1, 1], np.float32(p[0, t, :Un - 1, 1]) + pen)
    np.testing.assert_array_equal(q[0, :, Un - 1:, 1], np.float32(p[0, :, Un - 1:, 1]))
    np.testing.assert_array_equal(q[2], np.float32(p[2]))                              # invalid lengths
    assert np.float32(pa.KBIG) + np.float32(3.0) == np.float32(pa.KBIG)


@pytest.mark.parametrize("kind,S", [("modified", 1), ("modified", 2), ("modified", 4), ("constrained", 2),
                                    ("constrained", 4)])
def test_windows_keep_a_path(kind, S):
    """Every lattice with a modified path keeps one under the windows the type's ranges rule builds.  (A constrained
    label edge also reads the blank of the cell it reaches, so its windows need S >= 2 to keep one.)"""
    rng = np.random.RandomState(S)
    N, T, U = 24, 9, 8
    for trial in range(3):
        p, xn, yn = make_pairs(N, T, U, 10 * S + trial)
        _, g, raw = pa.lattice(p, xn, yn, kind)
        g = np.nan_to_num(g).astype(np.float32) * rng.uniform(0.5, 2.0, g.shape).astype(np.float32)
        r = pa.prune_ranges(g, xn, yn, S, kind, raw.astype(np.float32))
        assert (np.diff(r, axis=1) >= 0).all() and (np.diff(r, axis=1) <= 1).all() and (r[:, 0] == 0).all()
        c, _, _ = pa.lattice(pa.window_pairs(p, r, S), xn, yn, kind)
        reach = (yn <= xn)
        assert np.isfinite(c[reach]).all(), (xn[reach], yn[reach], c[reach])
        assert (c[~reach] == np.inf).all()


# ------------------------------------------------------------------------------------------ stream
def penalise64(p, xn, yn, lam):
    """the delay penalty added in fp64 (stream()'s), beside penalise()'s f32 order"""
    q = np.array(p, np.float64, copy=True)
    for n in range(len(xn)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        q[n, :Tn, :Un - 1, 1] += lam * ((Tn - 1) / 2.0 - np.arange(Tn))[:, None]
    return q


@pytest.mark.parametrize("kind", ["modified", "constrained"])
@pytest.mark.parametrize("lam", [0.0, 0.05])
def test_stream_is_the_lattice(kind, lam):
    """stream() / stream_grads() on every class of small lattice -- live, one frame, one column, Un - 1 = Tn, more
    labels than frames, every path cut by removed edges, -inf log-probs -- give lattice()'s cost and, at the kept
    frames, its pair gradients to 1e-12, with rows wider than the lattice (padding columns ignored)."""
    T, U = 7, 6
    p, _, _ = make_pairs(8, T, U, 21)
    xn = np.array([7, 1, 5, 4, 3, 6, 7, 6], np.int32)
    yn = np.array([5, 0, 0, 4, 4, 3, 5, 2], np.int32)
    p[5, :, :, 0] = pa.KBIG                                  # lattice 5: no blank edge left, no path
    rng = np.random.RandomState(2)
    p[6][rng.rand(T, U, 2) < 0.15] = -np.inf                 # lattice 6: masked log-probs
    q = penalise64(p, xn, yn, lam)
    c0, g0, _ = pa.lattice(q, xn, yn, kind)
    assert np.isinf(c0[[4, 5]]).all() and np.isfinite(c0[[0, 1, 2, 3]]).all()
    for n in range(len(xn)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        calls = []

        def row(t):
            calls.append(t)
            return p[n, t]                                   # (U, 2): the columns past Un are padding

        keep = range(Tn)
        c, g, top = pa.stream_grads(row, Tn, Un, kind, keep, lam)
        assert sorted(calls[:2 * Tn]) == sorted(list(range(Tn)) * 2)
        if np.isinf(c0[n]):
            assert c == np.inf and all(not v.any() for v in g.values())
            continue
        assert abs(c - c0[n]) <= 1e-12 * max(1.0, abs(c0[n])) and top >= 0
        for t in keep:
            np.testing.assert_allclose(g[t], g0[n, t, :Un], rtol=0, atol=1e-12)
    # a few kept frames only: the same rows, alpha / beta the lattice's recurrence
    n, Tn, Un = 0, 7, 6
    c, a, b = pa.stream(lambda t: p[n, t], Tn, Un, kind, keep=[0, 3, 6], lam=lam)
    assert sorted(a) == [0, 3, 6] and sorted(b) == [0, 3, 6]
    assert a[0][0] == 0 and np.isneginf(a[0][1:]).all() and b[6][Un - 1] == 0 and np.isneginf(b[6][:-1]).all()
    assert abs(c - c0[n]) <= 1e-12 * abs(c0[n])
