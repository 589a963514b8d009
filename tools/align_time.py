"""Time of rnnt_align (Viterbi forced alignment) beside the forward-only loss on the same inputs.

    python tools/align_time.py [--rounds 5] [--steps 20] [--out FILE]

Shapes: c2 = N=128 T=150 U=40 V=28 dense, full lengths, float32 and bfloat16; c4 = N=64 T=1500 U=300 V=50 dense, full
lengths; c4 compact = the same sizes with bench.py's ragged lengths (lengths in [T/2, T] and [U/2, U) shifted so that
the maxima are T and U-1) in the (STU, V) layout under compact_hints(T, U).  Log-probs are log_softmax(randn).
Arms per shape:
  align   rnnt_align(...)                                      captured in a CUDA graph
  loss    rnnt_loss(...) under torch.no_grad() (forward only)  captured in a CUDA graph; float32 log-probs (the dense
          bfloat16 loss needs gradients), so the c2 bf16 row repeats the float32 loss
  eager   (c2 float32 only) an anti-diagonal Viterbi in eager PyTorch with a batched backtrace on the device, as a user
          would otherwise write it; not captured
Each round times every arm once, one after the other (CUDA events around `steps` replays or calls); the JSON lines
report the median and range over rounds in ms per call.  One torch.profiler pass per shape adds the device time of each
kernel of the align and loss arms.  The card's name, power limit and max SM clock come from read-only queries."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:                                 # the numbers then stand without it, and say so
        info["power_limit"] = "not read (%s)" % str(e)[:80]
    return info


def inputs(N, T, U, V, seed, ragged):
    g = torch.Generator().manual_seed(seed)
    ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, generator=g)
    if ragged:
        xn = torch.randint(T // 2, T + 1, (N,), dtype=torch.int, generator=g)
        yn = torch.randint(U // 2, U, (N,), dtype=torch.int, generator=g)
        xn, yn = xn + T - xn.max(), yn + (U - 1) - yn.max()
    else:
        xn, yn = torch.full((N,), T, dtype=torch.int), torch.full((N,), U - 1, dtype=torch.int)
    return ys, xn, yn


def eager_viterbi(lp, ys, xn, yn, blank=0):
    """Anti-diagonal max-plus recurrence and a batched backtrace, in eager PyTorch on the device."""
    N, T, U, V = lp.shape
    lp = lp.float()
    B = lp[..., blank]
    L = lp[:, :, :U - 1].gather(3, ys.long()[:, None, :, None].expand(N, T, U - 1, 1)).squeeze(3)
    a = torch.full((N, T, U), float("-inf"), device=lp.device)
    a[:, 0, 0] = 0
    bit = torch.zeros((N, T, U), dtype=torch.bool, device=lp.device)
    for d in range(1, T + U - 1):
        t = torch.arange(max(0, d - U + 1), min(d, T - 1) + 1, device=lp.device)
        u = d - t
        tp, up = (t - 1).clamp(min=0), (u - 1).clamp(min=0)
        skip = a[:, tp, u] + B[:, tp, u]
        emit = a[:, t, up] + L[:, t, up.clamp(max=max(U - 2, 0))]
        b = ((emit > skip) | skip.isnan() | (t == 0)) & (u > 0)
        bit[:, t, u] = b
        a[:, t, u] = torch.where(b, emit, skip)
    n = torch.arange(N, device=lp.device)
    tn, un = xn.long() - 1, yn.long()
    scores = a[n, tn, un] + B[n, tn, un]
    frames = torch.full((N, U), -1, dtype=torch.int32, device=lp.device)
    t, u = tn.clone(), un.clone()
    for _ in range(T + U - 2):
        lab = (u > 0) & ((t == 0) | bit[n, t, u])
        frames[n, torch.where(lab, u - 1, U - 1)] = torch.where(lab, t, frames[n, U - 1]).int()
        u = u - lab.long()
        t = t - ((~lab) & (t > 0)).long()
    return scores, frames[:, :U - 1]


def graphed(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_times(fns):
    """Device time per kernel name (us per call), one profiled call of each arm."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for arm, fn in fns.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        out[arm] = {e.key[:60]: round(e.device_time_total / max(e.count, 1), 1)
                    for e in prof.key_averages() if e.device_time_total > 0}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import warp_rnnt_b200 as w
    dev = torch.device("cuda:0")
    hw = card()
    lines = [dict(hardware=hw)]
    print(json.dumps(lines[0]), flush=True)
    shapes = [("c2_f32", (128, 150, 40, 28), "dense", torch.float32),
              ("c2_bf16", (128, 150, 40, 28), "dense", torch.bfloat16),
              ("c4_dense", (64, 1500, 300, 50), "dense", torch.float32),
              ("c4_compact", (64, 1500, 300, 50), "compact", torch.float32)]
    for name, (N, T, U, V), layout, dtype in shapes:
        torch.manual_seed(N + V)
        ys, xn, yn = inputs(N, T, U, V, N + V, ragged=(layout == "compact"))
        ys, xn, yn = ys.to(dev), xn.to(dev), yn.to(dev)
        if layout == "compact":
            stu = int((xn.long() * (yn.long() + 1)).sum())
            x = torch.log_softmax(torch.randn(stu, V, device=dev), -1)
            yc = torch.cat([ys[i, :yn[i]] for i in range(N)]).contiguous()

            def align_fn(x=x, yc=yc, xn=xn, yn=yn, T=T, U=U):
                with w.compact_hints(T, U):
                    return w.rnnt_align(x, yc, xn, yn, compact=True)

            def loss_fn(x=x, yc=yc, xn=xn, yn=yn, T=T, U=U):
                with torch.no_grad(), w.compact_hints(T, U):
                    return w.rnnt_loss(x, yc, xn, yn, compact=True)
        else:
            x32 = torch.log_softmax(torch.randn(N, T, U, V, device=dev), -1)
            x = x32.to(dtype)

            def align_fn(x=x, ys=ys, xn=xn, yn=yn):
                return w.rnnt_align(x, ys, xn, yn)

            def loss_fn(x=x32, ys=ys, xn=xn, yn=yn):
                with torch.no_grad():
                    return w.rnnt_loss(x, ys, xn, yn)
        s_a, _ = align_fn()
        c_l = loss_fn()
        torch.cuda.synchronize()
        ok = bool(((s_a <= -c_l + 1e-4 * (1 + c_l.abs())) | ~torch.isfinite(c_l)).all())
        arms = {"align": graphed(align_fn), "loss": graphed(loss_fn)}
        if name == "c2_f32":
            s_e, f_e = eager_viterbi(x, ys, xn, yn)
            s_r, f_r = align_fn()
            ok = ok and torch.equal(s_e, s_r) and torch.equal(f_e, f_r)
            arms["eager"] = lambda x=x, ys=ys, xn=xn, yn=yn: eager_viterbi(x, ys, xn, yn)
        res = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                res[k].append(timed(fn, args.steps if k != "eager" else 3))
        line = dict(shape=name, N=N, T=T, U=U, V=V, layout=layout, dtype=str(dtype).replace("torch.", ""),
                    consistent=ok, rounds=args.rounds,
                    ms={k: dict(median=round(statistics.median(v), 4), min=round(min(v), 4), max=round(max(v), 4))
                        for k, v in res.items()},
                    kernels_us=kernel_times({"align": align_fn, "loss": loss_fn}))
        lines.append(line)
        print(json.dumps(line), flush=True)
        del arms
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)
            f.write("\n")


if __name__ == "__main__":
    main()
