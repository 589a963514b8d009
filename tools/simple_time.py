"""Step time and memory of the simple loss (rnnt_loss_simple) and of the whole pruned pipeline, against torch-op and
full-joint baselines.

    python tools/simple_time.py [--shapes a,b,c4] [--rounds 5] [--out FILE] [--no-profile]

Shapes as in tools/pruned_time.py (bench.py's ragged lengths, seed N + V): a = N=32 T=500 U=100 V=500,
b = N=32 T=600 U=150 V=1024, c4 = N=64 T=1500 U=300 V=50.  am (N,T,V) and lm (N,U,V) are randn float32.  Every arm's
step is `loss.backward()` with reduction="sum", captured in a CUDA graph:
  s  rnnt_loss_simple(am, lm, prune_range=5): the new kernels, ranges included
  a  the same loss in torch ops on this library's recurrence: k2's normaliser (row maxima, exp, torch.matmul, log),
     the (N,T,U,2) pairs by gather, then RNNTLoss with blank = -1
  d  rnnt_loss_from_logits(am[:, :, None] + lm[:, None]): the full (N,T,U,V) joint of the same loss
  p  the pruned pipeline: rnnt_loss_simple(prune_range=5) + rnnt_loss_pruned on the simple joint gathered at the
     windows (the joint network is the identity here), i.e. what replaces arm d in training
Each round times the arms once, one after the other; the JSON line reports the median and range over rounds of ms per
step (CUDA events over `steps` graph replays), and the step's memory: torch.cuda.max_memory_allocated over one eager
step above what was allocated before it, plus the arm's inputs.  A separate torch.profiler run records the device
time of each kernel of arm s; the three contractions (k_simple_mm) are reported with their achieved FP32 FLOP/s
(2 V sum_n Tn Un multiply-adds each, the live lattice cells only) against the 67 TFLOP/s data-sheet figure.  The
card's name, power limit and max SM clock come from read-only queries in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

from pruned_time import SHAPES, card, ragged_lengths

S = 5
ARMS = ("s", "a", "d", "p")
FP32_TFLOPS = 67.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="a,b,c4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("simple_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    torch.backends.cuda.matmul.allow_tf32 = False            # arm a: a plain fp32 matmul, as the loss needs
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/simple_time.py", "card": card(), "lse_mode": "auto (exact)", "S": S,
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay",
              "arms": {"s": "rnnt_loss_simple(am, lm, prune_range=5)",
                       "a": "torch ops: k2's matmul normaliser -> (N,T,U,2) pairs -> RNNTLoss(blank=-1)",
                       "d": "rnnt_loss_from_logits(am[:, :, None] + lm[:, None])",
                       "p": "rnnt_loss_simple(prune_range=5) + rnnt_loss_pruned(simple joint at the windows)"},
              "fp32_tflops_datasheet": FP32_TFLOPS, "runs": {}}
    for name in args.shapes.split(","):
        N, T, U, V = SHAPES[name]
        ys, xn, yn = (t.to(dev) for t in ragged_lengths(N, T, U, V, N + V))
        g = torch.Generator(device=dev).manual_seed(N + V)
        am = torch.randn((N, T, V), device=dev, generator=g).requires_grad_(True)
        lm = torch.randn((N, U, V), device=dev, generator=g).requires_grad_(True)
        y = torch.cat([ys.long(), torch.zeros((N, 1), dtype=torch.long, device=dev)], dim=1)
        y = torch.where(torch.arange(U, device=dev)[None] < yn[:, None].long(), y, 0)
        cells = int((xn.long() * (yn.long() + 1)).sum())
        flops = 2.0 * V * cells

        def arm_s():
            loss, _ = w.rnnt_loss_simple(am, lm, ys, xn, yn, reduction="sum", prune_range=S)
            return loss

        def arm_a():
            amax = am.detach().amax(-1, keepdim=True)
            lmax = lm.detach().amax(-1, keepdim=True)
            z = torch.matmul((am - amax).exp(), (lm - lmax).exp().transpose(1, 2))
            norm = z.log() + amax + lmax.transpose(1, 2)
            am_y = am.gather(2, y[:, None, :].expand(N, T, U))
            lm_y = lm.gather(2, y[:, :, None])[:, :, 0]
            pairs = torch.stack([am[:, :, 0:1] + lm[:, None, :, 0] - norm, am_y + lm_y[:, None] - norm], dim=-1)
            return w.RNNTLoss.apply(pairs.contiguous(), ys, xn, yn, -1, 0.0, None, False).sum()

        def arm_d():
            return w.rnnt_loss_from_logits(am[:, :, None] + lm[:, None], ys, xn, yn, reduction="sum")

        def arm_p():
            simple, ranges = w.rnnt_loss_simple(am, lm, ys, xn, yn, reduction="sum", prune_range=S)
            idx = (ranges.long()[:, :, None] + torch.arange(S, device=dev)).clamp(max=U - 1)
            lm_win = lm[torch.arange(N, device=dev)[:, None, None], idx]          # (N,T,S,V); no (N,T,U,V) grad
            logits = am[:, :, None] + lm_win
            return simple + w.rnnt_loss_pruned(logits, ys, xn, yn, ranges, reduction="sum")

        fns = {"s": arm_s, "a": arm_a, "d": arm_d, "p": arm_p}

        def step(arm):
            am.grad = lm.grad = None
            loss = fns[arm]()
            loss.backward()
            return loss

        mem, losses = {}, {}
        inputs = am.numel() * 4 + lm.numel() * 4
        for arm in ARMS:
            step(arm)
            am.grad = lm.grad = None
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            losses[arm] = step(arm).item()
            torch.cuda.synchronize()
            mem[arm] = inputs + torch.cuda.max_memory_allocated(dev) - base
            am.grad = lm.grad = None
        torch.cuda.empty_cache()

        kernels = {}
        if not args.no_profile:
            from torch.profiler import ProfilerActivity, profile
            for _ in range(2):
                step("s")
            torch.cuda.synchronize()
            reps = 5
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    step("s")
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                us = (getattr(ev, "self_device_time_total", 0) or getattr(ev, "self_cuda_time_total", 0)) / reps
                if us > 0:
                    k = {"us_per_step": us, "calls_per_step": ev.count / reps}
                    if "k_simple_mm" in ev.key:
                        k["fp32_tflops"] = flops / (us * 1e-6) / 1e12
                        k["frac_of_datasheet"] = k["fp32_tflops"] / FP32_TFLOPS
                    kernels[ev.key[:160]] = k
            am.grad = lm.grad = None
            torch.cuda.synchronize()

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for arm in ARMS:
                step(arm)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        am.grad = lm.grad = None
        torch.cuda.empty_cache()
        pool = torch.cuda.graph_pool_handle()
        graphs = {}
        for arm in ARMS:
            gr = torch.cuda.CUDAGraph()
            am.grad = lm.grad = None
            with torch.cuda.graph(gr, pool=pool):
                step(arm)
            graphs[arm] = gr
        torch.cuda.synchronize()

        def timed(arm, k):
            gr = graphs[arm]
            for _ in range(3):
                gr.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(k):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / k

        k = args.steps or max(5, int(200.0 / max(timed(a, 3) for a in ARMS)))
        ms = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for arm in ARMS:
                ms[arm].append(timed(arm, k))
        out = {"N": N, "T": T, "U": U, "V": V, "S": S, "live_cells": cells, "contraction_flops": flops,
               "steps_per_round": k, "rounds": args.rounds, "eager_loss": losses, "arms": {}, "kernels": kernels}
        for arm in ARMS:
            out["arms"][arm] = {"ms_per_step": statistics.median(ms[arm]), "ms_range": [min(ms[arm]), max(ms[arm])],
                                "ms_rounds": ms[arm], "step_memory_bytes": mem[arm]}
        sm = out["arms"]["s"]["ms_per_step"]
        out["a_over_s"] = out["arms"]["a"]["ms_per_step"] / sm
        out["d_over_s"] = out["arms"]["d"]["ms_per_step"] / sm
        out["d_over_p"] = out["arms"]["d"]["ms_per_step"] / out["arms"]["p"]["ms_per_step"]
        result["runs"][name] = out
        print(json.dumps({name: out}), flush=True)
        del graphs, pool, am, lm
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
