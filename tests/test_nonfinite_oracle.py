"""CPU: what the reference's semantics give on masked and non-finite log-probs (tests/common.py NONFINITE_CASES).

The C oracle (oracle/rnnt_oracle.c) restates the reference kernels' arithmetic; in float32 it shows the classes the
reference's own outputs have, in float64 the same classes without fp32 overflow.  ref_transduce_np is the plain
fp64 recurrence with logaddexp.  These are the expectations that tests/test_gpu_nonfinite.py checks the kernels
against, next to the recorded reference outputs:

  * dead lattices: cost NaN (dense / gathered, Tn >= 2 and Un >= 2) or +inf (Tn == 1, Un == 1, compact layout);
    every gradient element the reference writes is NaN, every other one 0
  * finfo.min masks that leave no other alignment: a finite cost of ~3.4e38 in float32 (the documented deviation:
    the kernels treat it as dead)
  * tier A: finite, and in float64 equal to ref_transduce_np up to rounding
  * tier C: the reference has NaN gradients, ref_transduce_np is finite
"""
import numpy as np
import pytest

from oracle import oracle
from tests.common import (NONFINITE_CASES, dead_cost_class, gather_pairs, lattice_tiers, masked_inputs,
                          threshold_inputs, to_compact, written_dense)

FMIN_F32 = np.float32(np.finfo(np.float32).min)


@pytest.fixture(scope="module", params=sorted(NONFINITE_CASES))
def case(request):
    c = NONFINITE_CASES[request.param]
    lp, ys, xn, yn = masked_inputs(c)
    return c, lp, ys, xn, yn


@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_dense_and_gathered_classes(case, dtype):
    c, lp, ys, xn, yn = case
    N, T, U, V, blank = c[:5]
    with np.errstate(all="ignore"):
        costs, grads = oracle.dense(lp, ys, xn, yn, blank=blank, dtype=dtype)
        gc, gg = oracle.dense(gather_pairs(lp, ys, blank), ys, xn, yn, blank=-1, dtype=dtype)
    written = written_dense(ys, xn, yn, T, U, V, blank)
    for n, tier in enumerate(lattice_tiers(c)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        g = grads[n]
        if tier == "dead":
            want = dead_cost_class(Tn, Un, False)
            assert np.array_equal(costs[n], want, equal_nan=True), (n, costs[n], want)
            assert np.array_equal(gc[n], want, equal_nan=True), (n, gc[n], want)
            assert np.array_equal(np.isnan(g), written[n]), n
            assert not g[~written[n]].any()
        elif tier == "fmin":
            if dtype == "f32":
                assert costs[n] == -FMIN_F32, costs[n]
            assert np.isfinite(costs[n]) and costs[n] > 1e30
            assert np.isfinite(g).all()
        elif tier == "A":
            assert np.isfinite(costs[n]) and costs[n] < 1e30 and np.isfinite(g).all(), n
            if dtype == "f64":
                c0, g0, _, _ = oracle.ref_transduce_np(lp[n, :Tn, :Un], ys[n, :Un - 1], blank)
                np.testing.assert_allclose(costs[n], c0, rtol=1e-12)
                np.testing.assert_allclose(g[:Tn, :Un], g0, atol=1e-10)
        else:   # "C"
            assert np.isnan(g).any(), n
            with np.errstate(all="ignore"):
                c0, g0, _, _ = oracle.ref_transduce_np(lp[n, :Tn, :Un], ys[n, :Un - 1], blank)
            assert np.isfinite(c0) and np.isfinite(g0).all()
        # the gathered (N,T,U,2) layout has the same classes as the dense one
        assert np.array_equal(np.isnan(gc[n]), np.isnan(costs[n])) and np.array_equal(np.isinf(gc[n]), np.isinf(costs[n]))


@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_compact_classes(case, dtype):
    c, lp, ys, xn, yn = case
    blank = c[4]
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    with np.errstate(all="ignore"):
        costs, pg, loc = oracle.compact(xs_c, ys_c, xn, yn, blank=blank, dtype=dtype)
    o = 0
    for n, tier in enumerate(lattice_tiers(c)):
        Tn, Un = int(xn[n]), int(yn[n]) + 1
        g = pg[o:o + Tn * Un].reshape(Tn, Un, 2)
        o += Tn * Un
        if tier == "dead":
            assert costs[n] == np.inf, (n, costs[n])
            # structural zeros (the last row's inner blanks, the last column's labels) stay 0, the rest is NaN
            structural = np.zeros((Tn, Un, 2), dtype=bool)
            structural[Tn - 1, :Un - 1, 0] = True
            structural[:, Un - 1, 1] = True
            assert np.array_equal(np.isnan(g), ~structural), n
            assert not g[structural].any()
        elif tier in ("A", "fmin"):
            assert np.isfinite(costs[n]) and np.isfinite(g).all(), n
        else:   # "C": the compact LSE maps LSE(-inf, -inf) to -inf, so this layout's reference stays finite
            assert np.isfinite(costs[n]) and np.isfinite(g).all(), n


def test_threshold_inputs():
    """The lattices around the kernels' 5e29 dead-lattice threshold are live for the reference: finite costs near
    4.9e29 and 5.1e29 (the kernels report the latter two as dead, DESIGN.md 4)."""
    lp, ys, xn, yn, dead = threshold_inputs()
    c32, _ = oracle.dense(lp, ys, xn, yn, dtype="f32")
    c64, _ = oracle.dense(lp, ys, xn, yn, dtype="f64")
    np.testing.assert_allclose(c64, [4.9e29, 5.1e29, 4.9e29, 5.1e29], rtol=1e-6)
    np.testing.assert_allclose(c32, c64, rtol=1e-6)
    assert np.array_equal(c64 > 5e29, dead)
