"""Time of rnnt_align_from_logits (Viterbi alignment from joint logits on k2's lattices) beside the forward-only
rnnt_loss_from_logits of the same type, and beside today's route for the regular lattice, rnnt_align on
torch.log_softmax(x, -1).

    python tools/align_logits_time.py [--rounds 5] [--steps 10] [--out FILE]

Shapes: c2 = N=128 T=150 U=40 V=28, v1k = N=32 T=600 U=150 V=1024, c4 = N=64 T=1500 U=300 V=50; dense, full lengths,
logits randn, float32; at c4 also the compact layout with ragged lengths (regular only, inside compact_hints).  Arms
for each rnnt_type and delay_penalty in {0, 0.05}, alternated within each round:
  align   rnnt_align_from_logits(...)                                         captured in a CUDA graph
  loss    rnnt_loss_from_logits(...) under torch.no_grad() (the forward only)  captured in a CUDA graph
  route   (regular, penalty 0) rnnt_align(torch.log_softmax(x, -1))            captured in a CUDA graph
  eager   (c2, modified, penalty 0) a per-frame max-plus Viterbi in eager PyTorch with a batched backtrace on the
          device, on the pairs x - lse of the loss's own normaliser; its results must equal the kernel's bit for bit
Each round times every arm once (CUDA events around `steps` replays or calls); the JSON lines report the median and
range over rounds in ms per call.  One torch.profiler pass per arm adds the device time of each kernel; the same pass
on logits whose first label is masked on every frame (score -inf: the sweep runs, the backtrace does not) gives the
backtrace's share of the alignment kernel.  The card's name, power limit and max SM clock come from read-only
queries."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

from tools.align_time import card, graphed, inputs, kernel_times, timed

TYPES = ("regular", "modified", "constrained")
LAMS = (0.0, 0.05)


def eager_modified(w, x, ys, xn, yn):
    """The modified lattice's max-plus sweep one frame at a time, then a batched backtrace, in eager PyTorch on the
    pairs x - lse of the loss's normaliser (blank 0).  Returns scores (N,), frames (N,U-1)."""
    N, T, U, V = x.shape
    lse = w._C.rnnt_logits_forward(x, ys, xn, yn, 0, 0.0, False)[1]
    B = x[..., 0].float() - lse
    L = x[:, :, :U - 1].float().gather(3, ys.long()[:, None, :, None].expand(N, T, U - 1, 1))[..., 0] - lse[:, :, :U - 1]
    a = torch.full((N, U), float("-inf"), device=x.device)
    a[:, 0] = 0
    bits = torch.zeros((N, T, U), dtype=torch.bool, device=x.device)
    for t in range(T):
        skip = a + B[:, t]
        emit = a[:, :-1] + L[:, t]
        e = (emit > skip[:, 1:]) | skip[:, 1:].isnan()
        nxt = skip.clone()
        nxt[:, 1:] = torch.where(e, emit, skip[:, 1:])
        bits[:, t, 1:] = e
        a = torch.where((t < xn)[:, None], nxt, a)
    n = torch.arange(N, device=x.device)
    un = yn.long()
    scores = a[n, un]
    frames = torch.full((N, U), -1, dtype=torch.int32, device=x.device)
    u = un.clone()
    for t in range(T - 1, -1, -1):
        lab = (t < xn) & bits[n, t, u] & (u > 0)
        frames[n, torch.where(lab, u - 1, U - 1)] = torch.where(lab, t, frames[n, U - 1].long()).int()
        u = u - lab.long()
    return scores, frames[:, :U - 1]


def align_kernel_us(w, x, ys, xn, yn, tag):
    """device time (us) of the alignment kernel (k_align or k_frames_align) in one profiled call of arm `tag`"""
    kind, lam = tag.rsplit("_", 1)
    kt = kernel_times({"a": lambda: w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type=kind, delay_penalty=float(lam))})
    return round(sum(v for k, v in kt["a"].items() if "k_align" in k or "k_frames_align" in k), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import warp_rnnt_b200 as w
    dev = torch.device("cuda:0")
    hw = card()
    lines = [dict(hardware=hw)]
    print(json.dumps(lines[0]), flush=True)
    shapes = [("c2", (128, 150, 40, 28)), ("v1k", (32, 600, 150, 1024)), ("c4", (64, 1500, 300, 50))]
    for name, (N, T, U, V) in shapes:
        ys, xn, yn = (t.to(dev) for t in inputs(N, T, U, V, seed=N + V, ragged=False))
        g = torch.Generator(device=dev).manual_seed(N + V)
        x = torch.randn(N, T, U, V, device=dev, generator=g)
        fns, checks = {}, {}
        for kind in TYPES:
            for lam in LAMS:
                tag = "%s_%g" % (kind, lam)

                def align_fn(kind=kind, lam=lam):
                    return w.rnnt_align_from_logits(x, ys, xn, yn, rnnt_type=kind, delay_penalty=lam)

                def loss_fn(kind=kind, lam=lam):
                    with torch.no_grad():
                        return w.rnnt_loss_from_logits(x, ys, xn, yn, rnnt_type=kind, delay_penalty=lam)

                fns["align_" + tag] = align_fn
                fns["loss_" + tag] = loss_fn
                s, f = align_fn()
                c = loss_fn()
                torch.cuda.synchronize()
                fin = torch.isfinite(c)
                checks[tag] = bool((s[fin] <= -c[fin] + 1e-5 * (1 + c[fin].abs())).all()) and \
                    bool(torch.equal(torch.isneginf(s), torch.isposinf(c)))
        fns["route_regular_0"] = lambda: w.rnnt_align(torch.log_softmax(x, -1), ys, xn, yn)
        s_r, f_r = fns["route_regular_0"]()
        s_a, f_a = fns["align_regular_0"]()
        checks["route_close"] = bool(torch.allclose(s_r, s_a, rtol=1e-5, atol=1e-4))
        arms = {k: graphed(fn) for k, fn in fns.items()}
        if name == "c2":
            s_e, f_e = eager_modified(w, x, ys, xn, yn)
            s_k, f_k = fns["align_modified_0"]()
            checks["eager_bit_equal"] = bool(torch.equal(s_e, s_k) and torch.equal(f_e, f_k))
            arms["eager_modified_0"] = lambda: eager_modified(w, x, ys, xn, yn)
        res = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                res[k].append(timed(fn, args.steps if not k.startswith("eager") else 1))
        ms = {k: dict(median=round(statistics.median(v), 4), min=round(min(v), 4), max=round(max(v), 4))
              for k, v in res.items()}
        ratio = {tag: round(ms["align_" + tag]["median"] / ms["loss_" + tag]["median"], 3)
                 for tag in ("%s_%g" % (k, l) for k in TYPES for l in LAMS)}
        kernels = kernel_times({k: fn for k, fn in fns.items() if not k.startswith("loss_") or k.endswith("_0")})
        walk = {tag: align_kernel_us(w, x, ys, xn, yn, tag) for tag in ("regular_0", "modified_0", "constrained_0")}
        del arms
        torch.cuda.empty_cache()
        # every lattice's first label masked on every frame: score -inf, the sweep runs and the backtrace does not
        x[torch.arange(N, device=dev), :, 0, ys[:, 0].long()] = float("-inf")
        nowalk = {tag: align_kernel_us(w, x, ys, xn, yn, tag) for tag in walk}
        share = {tag: dict(kernel_us=walk[tag], without_backtrace_us=nowalk[tag],
                           backtrace_share=round(1.0 - nowalk[tag] / walk[tag], 3) if walk[tag] else None)
                 for tag in walk}
        line = dict(shape=name, layout="dense", N=N, T=T, U=U, V=V, dtype="float32", checks=checks, rounds=args.rounds,
                    ms=ms, align_over_loss=ratio, backtrace=share, kernels_us=kernels)
        lines.append(line)
        print(json.dumps(line), flush=True)
        del x, fns
        torch.cuda.empty_cache()
        if name == "c4":
            ys, xn, yn = (t.to(dev) for t in inputs(N, T, U, V, seed=N + V, ragged=True))
            STU = int((xn * (yn + 1)).sum())
            xc = torch.randn(STU, V, device=dev, generator=g)
            yc = torch.cat([ys[n, :int(yn[n])] for n in range(N)]).contiguous()
            hints = (int(xn.max()), int(yn.max()) + 1)

            def c_align():
                with w.compact_hints(*hints):
                    return w.rnnt_align_from_logits(xc, yc, xn, yn, compact=True)

            def c_loss():
                with torch.no_grad(), w.compact_hints(*hints):
                    return w.rnnt_loss_from_logits(xc, yc, xn, yn, compact=True)

            def c_route():
                with w.compact_hints(*hints):
                    return w.rnnt_align(torch.log_softmax(xc, -1), yc, xn, yn, compact=True)

            cf = {"align_regular_0": c_align, "loss_regular_0": c_loss, "route_regular_0": c_route}
            s_a, _ = c_align()
            c = c_loss()
            s_r, _ = c_route()
            checks = {"regular_0": bool((s_a <= -c + 1e-5 * (1 + c.abs())).all()),
                      "route_close": bool(torch.allclose(s_r, s_a, rtol=1e-5, atol=1e-4))}
            arms = {k: graphed(fn) for k, fn in cf.items()}
            res = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    res[k].append(timed(fn, args.steps))
            ms = {k: dict(median=round(statistics.median(v), 4), min=round(min(v), 4), max=round(max(v), 4))
                  for k, v in res.items()}
            line = dict(shape=name, layout="compact", N=N, T=T, U=U, V=V, STU=STU, dtype="float32", checks=checks,
                        rounds=args.rounds, ms=ms,
                        align_over_loss={"regular_0": round(ms["align_regular_0"]["median"] /
                                                            ms["loss_regular_0"]["median"], 3)},
                        kernels_us=kernel_times(cf))
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
