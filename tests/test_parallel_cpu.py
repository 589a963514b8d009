"""CPU, world_size 2 (gloo): the batch-sharding + scalar all-reduce host logic of
warp_rnnt_b200.parallel.  The local loss is injected (an autograd wrapper around the fp64 oracle),
so no GPU is needed; on a GPU the same code path runs with the CUDA op over NCCL."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.common import make_inputs


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _OracleLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lp, ys, xn, yn, lam):
        from oracle import oracle
        c, g = oracle.dense(lp.detach().numpy(), ys.numpy(), xn.numpy(), yn.numpy(), fastemit_lambda=lam)
        ctx.g = torch.from_numpy(g)
        return torch.from_numpy(c)

    @staticmethod
    def backward(ctx, go):
        return ctx.g * go.view(-1, 1, 1, 1), None, None, None, None


def _oracle_loss_fn(lp, ys, xn, yn, average_frames=False, reduction="none", blank=0, gather=False,
                    fastemit_lambda=0.0, compact=False):
    costs = _OracleLoss.apply(lp, ys, xn, yn, fastemit_lambda)
    if average_frames:
        costs = costs / xn.to(costs)
    return costs.sum() if reduction == "sum" else (costs.mean() if reduction == "mean" else costs)


def _worker(rank, world, port, reduction, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from warp_rnnt_b200 import parallel
    N, T, U, V = 5, 7, 4, 6          # 5 lattices over 2 ranks: 3 + 2
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=9, random_lengths=True)
    sh = parallel.shard_batch(torch.from_numpy(lp).double(), torch.from_numpy(ys), torch.from_numpy(xn),
                              torch.from_numpy(yn), world, rank)
    x = sh[0].clone().requires_grad_(True)
    loss = parallel.rnnt_loss_sharded(x, sh[1], sh[2], sh[3], average_frames=True, reduction=reduction,
                                      fastemit_lambda=0.1, loss_fn=_oracle_loss_fn)
    loss.backward()
    lo, hi = parallel.shard_range(N, world, rank)
    # the same shard as micro-batches of <= 2 lattices, with the caller-known global batch size: one all-reduce
    xs_mb = [sh[0][i:i + 2].clone().requires_grad_(True) for i in range(0, hi - lo, 2)]
    batches = [(xm, sh[1][i:i + 2], sh[2][i:i + 2], sh[3][i:i + 2]) for xm, i in zip(xs_mb, range(0, hi - lo, 2))]
    loss_mb = parallel.rnnt_loss_microbatches(batches, global_batch=N, reduction=reduction, average_frames=True,
                                              fastemit_lambda=0.1, loss_fn=_oracle_loss_fn)
    grad_mb = torch.cat([xm.grad for xm in xs_mb], 0).numpy()
    # 'mean' with global_batch given: a 1-element all-reduce, same value
    x2 = sh[0].clone().requires_grad_(True)
    loss_gb = parallel.rnnt_loss_sharded(x2, sh[1], sh[2], sh[3], average_frames=True, reduction=reduction,
                                         fastemit_lambda=0.1, loss_fn=_oracle_loss_fn, global_batch=N)
    loss_gb.backward()
    out.put((rank, float(loss), lo, hi, x.grad.numpy(), float(loss_mb), grad_mb, float(loss_gb), x2.grad.numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_sharded_loss_two_ranks(reduction):
    from oracle import oracle
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, reduction, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    N, T, U, V = 5, 7, 4, 6
    lp, ys, xn, yn = make_inputs(N, T, U, V, seed=9, random_lengths=True)
    loss0, g0 = oracle.rnnt_loss(lp, ys, xn, yn, average_frames=True, reduction=reduction, fastemit_lambda=0.1)
    for rank, loss, lo, hi, grad, loss_mb, grad_mb, loss_gb, grad_gb in res:
        np.testing.assert_allclose(loss, loss0, rtol=1e-12)          # identical on every rank
        np.testing.assert_allclose(grad, g0[lo:hi], atol=1e-13)      # gradients stay rank-local
        np.testing.assert_allclose(loss_mb, loss0, rtol=1e-12)       # micro-batched step == one-call step
        np.testing.assert_allclose(grad_mb, g0[lo:hi], atol=1e-13)
        np.testing.assert_allclose(loss_gb, loss0, rtol=1e-12)
        np.testing.assert_allclose(grad_gb, g0[lo:hi], atol=1e-13)
    assert sorted((r[2], r[3]) for r in res) == [(0, 3), (3, 5)]


def test_shard_range_partitions():
    from warp_rnnt_b200.parallel import shard_range
    for n in (0, 1, 7, 8, 2048):
        for w in (1, 2, 3, 8):
            r = [shard_range(n, w, k) for k in range(w)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(r[k][1] == r[k + 1][0] for k in range(w - 1))
            assert max(h - l for l, h in r) - min(h - l for l, h in r) <= 1
