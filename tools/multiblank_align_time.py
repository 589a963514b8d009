"""Time of rnnt_align_multiblank (Viterbi alignment on the multi-blank lattice) beside the forward-only
rnnt_loss_multiblank on the same logits.

    python tools/multiblank_align_time.py [--rounds 5] [--steps 20] [--out FILE]

Shapes: c2 = N=128 T=150 U=40 V=32, pk (Parakeet-like) = N=32 T=250 U=80 V=1029, c4 = N=64 T=1500 U=300 V=54; big
blanks [2, 4, 8] (columns V-2, V-3, V-4, the standard blank V-1), dense, full lengths, logits randn, float32 and
bfloat16.  Arms per shape, alternated within each round:
  align   rnnt_align_multiblank(...)                                  captured in a CUDA graph
  loss    rnnt_loss_multiblank(...) under torch.no_grad() (the forward only)  captured in a CUDA graph
  eager   (c2 float32 only) an anti-diagonal max-plus Viterbi in eager PyTorch with a max(d)-frame look-back and a
          batched backtrace on the device, as a user would otherwise write it; not captured
Each round times every arm once, one after the other (CUDA events around `steps` replays or calls); the JSON lines
report the median and range over rounds in ms per call.  One torch.profiler pass per shape adds the device time of each
kernel of the align and loss arms.  The card's name, power limit and max SM clock come from read-only queries."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

from tools.align_time import card, graphed, kernel_times, timed

DUR = [2, 4, 8]


def eager_viterbi(x, ys, xn, yn, durations):
    """Anti-diagonal max-plus over the multi-blank lattice with a max(d)-frame look-back, then a batched backtrace, in
    eager PyTorch on the device (float32, torch's log_softmax, the standard blank in column V-1).  Returns scores,
    frames (N,U-1) and blank counts (N,1+B)."""
    N, T, U, V = x.shape
    nb = len(durations)
    lp = torch.log_softmax(x.float(), -1)
    S = lp[..., V - 1]
    G = torch.stack([lp[..., V - 2 - i] for i in range(nb)], -1)
    L = torch.cat([lp[:, :, :U - 1].gather(3, ys.long()[:, None, :, None].expand(N, T, U - 1, 1)).squeeze(3),
                   torch.full((N, T, 1), float("-inf"), device=x.device)], 2)
    a = torch.full((N, T, U), float("-inf"), device=x.device)
    a[:, 0, 0] = 0
    dec = torch.zeros((N, T, U), dtype=torch.long, device=x.device)
    for s in range(1, T + U - 1):
        t = torch.arange(max(0, s - U + 1), min(s, T - 1) + 1, device=x.device)
        u = s - t
        tp, up = (t - 1).clamp(min=0), (u - 1).clamp(min=0)
        cands = [torch.where(t > 0, a[:, tp, u] + S[:, tp, u], float("-inf"))]
        for i, d in enumerate(durations):
            td = (t - d).clamp(min=0)
            cands.append(torch.where(t >= d, a[:, td, u] + G[:, td, u, i], float("-inf")))
        cands.append(torch.where(u > 0, a[:, t, up] + L[:, t, up], float("-inf")))
        best, k = torch.stack(cands, 0).max(0)           # 0 standard blank, 1 + i big blank i, 1 + B label
        a[:, t, u] = best
        dec[:, t, u] = k
    n = torch.arange(N, device=x.device)
    tn, un = xn.long(), yn.long()
    term = [a[n, tn - 1, un] + S[n, tn - 1, un]]
    for i, d in enumerate(durations):
        tq = (tn - d).clamp(min=0)
        term.append(torch.where(tn >= d, a[n, tq, un] + G[n, tq, un, i], float("-inf")))
    scores, k0 = torch.stack(term, 0).max(0)
    step = torch.tensor([1] + list(durations) + [0], device=x.device)
    counts = torch.zeros((N, 2 + nb), dtype=torch.long, device=x.device)
    counts[n, k0] += 1
    t, u = tn - step[k0], un.clone()
    frames = torch.full((N, U), -1, dtype=torch.int32, device=x.device)
    for _ in range(T + U - 1):
        live = (t > 0) | (u > 0)
        k = dec[n, t.clamp(min=0), u]
        lab = live & (k == 1 + nb)
        frames[n, torch.where(lab, u - 1, torch.full_like(u, U - 1))] = torch.where(lab, t, frames[n, U - 1].long()).int()
        counts[n, k] += live.long()
        t = torch.where(live, t - step[k], t)
        u = u - lab.long()
    return scores, frames[:, :U - 1], counts[:, :1 + nb].int()


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
    shapes = [("c2", (128, 150, 40, 32)), ("pk", (32, 250, 80, 1029)), ("c4", (64, 1500, 300, 54))]
    for name, (N, T, U, V) in shapes:
        for dtype in (torch.float32, torch.bfloat16):
            g = torch.Generator(device=dev).manual_seed(N + V)
            x = torch.randn(N, T, U, V, device=dev, generator=g).to(dtype)
            ys = torch.randint(0, V - 1 - len(DUR), (N, U - 1), device=dev, dtype=torch.int32, generator=g)
            xn = torch.full((N,), T, dtype=torch.int32, device=dev)
            yn = torch.full((N,), U - 1, dtype=torch.int32, device=dev)

            def align_fn(x=x, ys=ys, xn=xn, yn=yn):
                return w.rnnt_align_multiblank(x, ys, xn, yn, DUR)

            def loss_fn(x=x, ys=ys, xn=xn, yn=yn):
                with torch.no_grad():
                    return w.rnnt_loss_multiblank(x, ys, xn, yn, DUR)

            s_a, f_a, c_a = align_fn()
            c_l = loss_fn()
            torch.cuda.synchronize()
            ok = bool((s_a <= -c_l + 2e-6 * (1 + c_l.abs())).all())
            ok = ok and bool((c_a[:, 0] + sum(d * c_a[:, 1 + i] for i, d in enumerate(DUR)) == xn).all())
            arms = {"align": graphed(align_fn), "loss": graphed(loss_fn)}
            if name == "c2" and dtype == torch.float32:
                s_e, f_e, c_e = eager_viterbi(x, ys, xn, yn, DUR)
                ok = ok and bool(torch.allclose(s_e, s_a, rtol=1e-5))
                arms["eager"] = lambda x=x, ys=ys, xn=xn, yn=yn: eager_viterbi(x, ys, xn, yn, DUR)
            res = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    res[k].append(timed(fn, args.steps if k != "eager" else 2))
            big_share = float((c_a[:, 1:] * torch.tensor(DUR, device=dev)).sum() / xn.sum())
            line = dict(shape=name, N=N, T=T, U=U, V=V, big_blanks=DUR, dtype=str(dtype).replace("torch.", ""),
                        consistent=ok, rounds=args.rounds, big_blank_frame_share=round(big_share, 4),
                        ms={k: dict(median=round(statistics.median(v), 4), min=round(min(v), 4),
                                    max=round(max(v), 4)) for k, v in res.items()},
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
