"""CPU: pin the oracle (oracle/rnnt_oracle.c + numpy restatement) against the reference's
golden vectors (tests/golden/reference_vectors.json, extracted from the reference's test.py)."""
import numpy as np
import pytest

from oracle import oracle
from tests.common import GOLDEN, golden_case, make_inputs, to_compact, from_compact

DENSE = ["test_one_to_many", "test_one_to_empty", "test_forward_single", "test_forward_batch",
         "test_forward_single_inner_gather"]


@pytest.mark.parametrize("name", DENSE)
@pytest.mark.parametrize("dtype,dec", [("f64", 6), ("f32", 5)])
def test_golden_dense(name, dtype, dec):
    c = golden_case(name)
    costs, grads = oracle.dense(c["lp"], c["ys"], c["xn"], c["yn"], dtype=dtype)
    np.testing.assert_array_almost_equal(costs, c["costs"], decimal=dec)     # test.py:52 decimal=6
    np.testing.assert_array_almost_equal(grads, c["grads"], decimal=dec)


@pytest.mark.parametrize("name", DENSE)
def test_golden_numpy_restatement(name):
    c = golden_case(name)
    costs, grads = oracle.ref_transduce_np_batch(c["lp"], c["ys"], c["xn"], c["yn"])
    np.testing.assert_array_almost_equal(costs, c["costs"], decimal=6)
    np.testing.assert_array_almost_equal(grads, c["grads"], decimal=6)


def test_golden_gather_form():
    """blank=-1 V=2 boundary (test.py:214-257)."""
    c = golden_case("test_forward_single_gather")
    lp, ys = c["lp"], c["ys"]
    N, T, U, V = lp.shape
    index = np.zeros((N, T, U, 2), dtype=np.int64)
    index[:, :, :U - 1, 1] = ys[:, None, :]
    g = np.take_along_axis(lp, index, axis=3)
    costs, grads = oracle.dense(g, ys, c["xn"], c["yn"], blank=-1)
    np.testing.assert_array_almost_equal(costs, c["costs"], decimal=6)
    np.testing.assert_array_almost_equal(grads, c["grads"], decimal=6)


def test_golden_compact():
    """rnnt_loss_compact + rnnt_loss_compact_backward(ones) (test.py:259-336)."""
    c = golden_case("test_forward_batch_compact")
    xs_c, ys_c = to_compact(c["lp"], c["ys"], c["xn"], c["yn"])
    costs, pg, loc = oracle.compact(xs_c, ys_c, c["xn"], c["yn"])
    np.testing.assert_array_almost_equal(costs, c["costs"], decimal=6)
    cum = np.cumsum(c["xn"] * (c["yn"] + 1)).astype(np.int32)
    g = oracle.compact_scatter(np.ones(2), pg, loc, cum, c["lp"].shape[-1], 0)
    np.testing.assert_array_almost_equal(g, c["grads"], decimal=6)


@pytest.mark.parametrize("shape", [(3, 7, 5, 6), (2, 33, 34, 4), (4, 1, 1, 3), (2, 5, 1, 3), (2, 1, 6, 3)])
@pytest.mark.parametrize("blank", [0, 2])
def test_c_oracle_matches_numpy(shape, blank):
    N, T, U, V = shape
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=1, random_lengths=True, blank=blank)
    c1, g1 = oracle.dense(lp, ys, xn, yn, blank=blank, fastemit_lambda=0.25)
    c2, g2 = oracle.ref_transduce_np_batch(lp, ys, xn, yn, blank=blank, fastemit_lambda=0.25)
    np.testing.assert_allclose(c1, c2, rtol=1e-12)
    np.testing.assert_allclose(g1, g2, atol=1e-12)
    # f32 flavour stays within fp32 noise of truth
    c3, g3 = oracle.dense(lp, ys, xn, yn, blank=blank, fastemit_lambda=0.25, dtype="f32")
    np.testing.assert_allclose(c3, c1, rtol=1e-5)
    np.testing.assert_allclose(g3, g1, atol=1e-5)


def test_properties():
    """Size-independent identities the domain offers (used at full size on the GPU):
    sum over blank+label grads leaving the (0,0)... every anti-diagonal carries total flow 1:
    -sum_{t+u=d} (g_blank[t,u] + g_label[t,u]) == 1 for d < Tn-1+Un-1 path steps (lambda=0);
    alpha-side likelihood equals beta[0,0]; compact == dense on the unpadded cells."""
    N, T, U, V = 3, 9, 6, 5
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=3, random_lengths=True)
    costs, grads, al, be = oracle.dense(lp, ys, xn, yn, want_ab=True)
    for n in range(N):
        Tn, Un = xn[n], yn[n] + 1
        ll_a = al[n, Tn - 1, Un - 1] + lp[n, Tn - 1, Un - 1, 0]
        assert abs(ll_a - be[n, 0, 0]) < 1e-9
        flow = np.zeros(Tn + Un - 1)
        for t in range(Tn):
            for u in range(Un):
                flow[t + u] += -grads[n, t, u].sum()
        np.testing.assert_allclose(flow, 1.0, atol=1e-9)
        assert np.all(grads[n, Tn:] == 0) and np.all(grads[n, :, Un:] == 0)
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    cc, pg, loc = oracle.compact(xs_c, ys_c, xn, yn)
    np.testing.assert_allclose(cc, costs, rtol=1e-12)
    cum = np.cumsum(xn.astype(np.int64) * (yn + 1)).astype(np.int32)
    gc = oracle.compact_scatter(np.ones(N), pg, loc, cum, V, 0)
    np.testing.assert_allclose(from_compact(gc, xn, yn, T, U), grads, atol=1e-12)


def test_python_level_reductions():
    N, T, U, V = 4, 6, 4, 5
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=5, random_lengths=True)
    costs, grads = oracle.dense(lp, ys, xn, yn)
    loss, g = oracle.rnnt_loss(lp, ys, xn, yn, average_frames=True, reduction="mean")
    np.testing.assert_allclose(loss, (costs / xn).mean(), rtol=1e-12)
    np.testing.assert_allclose(g, grads / xn.reshape(-1, 1, 1, 1) / N, atol=1e-14)
    loss, g = oracle.rnnt_loss(lp, ys, xn, yn, reduction="sum")
    np.testing.assert_allclose(loss, costs.sum(), rtol=1e-12)


def test_mismatch_guard_is_silent_on_wellformed_input():
    lp, ys, xn, yn = make_inputs(8, 20, 9, 3, seed=0, random_lengths=True)
    c0, g0 = oracle.dense(lp, ys, xn, yn, dtype="f32", guard=False)
    c1, g1 = oracle.dense(lp, ys, xn, yn, dtype="f32", guard=True)
    assert np.array_equal(c0, c1) and np.array_equal(g0, g1)


def test_golden_sources_recorded():
    for k, r in GOLDEN.items():
        assert r["source"].startswith(("pytorch_binding/", "tensorflow_binding/")), k
