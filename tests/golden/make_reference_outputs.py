"""Record what the unmodified reference kernels compute on the inputs of the GPU tests that compare with them, into
tests/golden/reference_outputs.npz (see tests/common.py: record / same_as_reference).

Needs a GPU and the reference extension that build() compiles into oracle/_ref/ when the reference's sources are
available (oracle/build_ref.py):

    python tests/golden/make_reference_outputs.py [OUT.npz]

The inputs are made exactly as the tests make them (same helpers, shapes and seeds).  Inputs synthesised on the
device also get a fingerprint (`<case>/xs_sample`), so that a test can tell a changed random stream from a changed
result.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import build_ref  # noqa: E402
from tests import test_gpu_fullsize as F, test_gpu_holes as H, test_gpu_logits as L, test_gpu_parity as P  # noqa: E402
from tests.common import REF_OUTPUTS, input_sample, make_inputs, record, to_compact  # noqa: E402


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def dense(rec, case, ref, args, **kw):
    c, g = ref.rnnt_loss(*args, **kw)
    record(rec, case + "/costs", c)
    record(rec, case + "/grads", g)


def compact(rec, case, ref, cargs, blank=0, lam=0.0, go=None):
    cr, gr, lr = ref.rnnt_loss_compact(*cargs, blank=blank, fastemit_lambda=lam)
    used = lr != blank            # the reference leaves the other label slots of its (STU,2) buffer uninitialised
    record(rec, case + "/costs", cr)
    record(rec, case + "/loc", lr)
    record(rec, case + "/grad0", gr[:, 0].contiguous())
    record(rec, case + "/grad1_used", gr[:, 1][used].contiguous())
    if go is not None:
        xn, yn = cargs[2], cargs[3]
        cumlen = torch.cumsum(xn * (yn + 1), dim=0, dtype=torch.int32)
        record(rec, case + "/back", ref.rnnt_loss_compact_backward(go, gr, cumlen, lr, cargs[0].shape[1], blank))


def main(out):
    ref = build_ref.load()
    assert ref is not None and torch.cuda.is_available(), "needs a GPU and oracle/_ref/warp_rnnt_ref_C.so"
    rec = {}
    # tests/test_gpu_parity.py
    for k, (N, T, U, V, rl, blank, lam) in enumerate(P.REF_SHAPES):
        lp, ys, xn, yn = make_inputs(N, T, U, V, seed=21 + T, random_lengths=rl, blank=blank)
        dense(rec, "parity_dense_%d" % k, ref, (cu(lp), cu(ys), cu(xn), cu(yn)), blank=blank, fastemit_lambda=lam)
        lp, ys, xn, yn = make_inputs(N, T, U, V, seed=31 + U, random_lengths=rl, blank=blank)
        g = P.gather_np(lp, ys, blank)
        dense(rec, "parity_gc_%d/gather" % k, ref, (cu(g), cu(ys), cu(xn), cu(yn)), blank=-1, fastemit_lambda=lam)
        xs_c, ys_c = to_compact(lp, ys, xn, yn)
        compact(rec, "parity_gc_%d/compact" % k, ref, (cu(xs_c), cu(ys_c), cu(xn), cu(yn)), blank, lam,
                go=torch.linspace(0.5, 1.5, N).cuda())
    N, T, U, V, blank, lam = P.CABI_SHAPE
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=77, random_lengths=True, blank=blank)
    dense(rec, "cabi_layouts/dense", ref, (cu(lp), cu(ys), cu(xn), cu(yn)), blank=blank, fastemit_lambda=lam)
    g = P.gather_np(lp, ys, blank)
    dense(rec, "cabi_layouts/gather", ref, (cu(g), cu(ys), cu(xn), cu(yn)), blank=-1, fastemit_lambda=lam)
    xs_c, ys_c = to_compact(lp, ys, xn, yn)
    compact(rec, "cabi_layouts/compact", ref, (cu(xs_c), cu(ys_c), cu(xn), cu(yn)), blank, lam,
            go=torch.linspace(0.5, 1.5, N).cuda())
    for V in P.ROW_PAIR_V:
        N, T, U = P.ROW_PAIR_NTU
        lp, ys, xn, yn = make_inputs(N, T, U, V, seed=V, random_lengths=True, blank=1)
        ys[0, :5] = 1
        dense(rec, "rowpair_%d/dense" % V, ref, (cu(lp), cu(ys), cu(xn), cu(yn)), blank=1, fastemit_lambda=0.1)
        xs_c, ys_c = to_compact(lp, ys, xn, yn)
        compact(rec, "rowpair_%d/compact" % V, ref, (cu(xs_c), cu(ys_c), cu(xn), cu(yn)), 1, 0.1,
                go=cu(np.linspace(0.5, 1.5, N).astype(np.float32)))
    # tests/test_gpu_fullsize.py
    for case, shape, seed, rl in (("cfg2_full", (128, 150, 40, 28), 128, False), ("cfg2_rl", (128, 150, 40, 28), 7, True),
                                  ("cfg3_full", (32, 150, 20, 5000), 32, False)):
        xs, ys, xn, yn = F.synth(*shape, seed=seed, random_lengths=rl)
        record(rec, case + "/xs_sample", input_sample(xs))
        dense(rec, case, ref, (xs, ys, xn, yn))
        del xs
    xs, ys, xn, yn = F.synth(32, 600, 150, 1024, seed=5, random_lengths=True)
    record(rec, "cfg5_last4/xs_sample", input_sample(xs))
    dense(rec, "cfg5_last4", ref, tuple(t[-4:].contiguous() for t in (xs, ys, xn, yn)))
    del xs
    torch.cuda.empty_cache()
    # tests/test_gpu_holes.py
    xs, ys, xn, yn = H.synth(64, 1500, 300, 50, seed=64)
    record(rec, "cfg4_two/xs_sample", input_sample(xs))
    two = torch.tensor(H.CFG4_REF_LATTICES, device="cuda")
    a2 = (xs[two].contiguous(), ys[two].contiguous(), xn[two].contiguous(), yn[two].contiguous())
    dense(rec, "cfg4_two/dense", ref, a2)
    xs2, ys2 = H.ragged(xs, ys, xn, yn, H.CFG4_REF_LATTICES)
    compact(rec, "cfg4_two/compact", ref, (xs2, ys2, a2[2], a2[3]))
    del xs, a2, xs2
    torch.cuda.empty_cache()
    xs, ys, xn, yn = H.synth(32, 300, 70, 1200, seed=32)
    record(rec, "pipeline_two/xs_sample", input_sample(xs))
    two = torch.tensor(H.PIPELINE_REF_LATTICES, device="cuda")
    dense(rec, "pipeline_two", ref, (xs[two].contiguous(), ys[two].contiguous(), xn[two].contiguous(), yn[two].contiguous()))
    del xs
    lp, ys, xn, yn = H.ring_inputs()
    dense(rec, "ring_exact", ref, (cu(lp), cu(ys), cu(xn), cu(yn)))
    # tests/test_gpu_logits.py: the reference on torch.log_softmax of the logits
    for k, (N, T, U, V, blank, lam) in enumerate(L.REF_SHAPES):
        x, ys, xn, yn = L.make(N, T, U, V, seed=11 + V, blank=blank)
        lp = torch.log_softmax(cu(x), -1)
        dense(rec, "logits_%d" % k, ref, (lp.contiguous(), cu(ys), cu(xn), cu(yn)), blank=blank, fastemit_lambda=lam)
    torch.cuda.synchronize()
    np.savez_compressed(out, **rec)
    print("wrote %s: %d arrays, %d bytes" % (out, len(rec), os.path.getsize(out)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else REF_OUTPUTS)
