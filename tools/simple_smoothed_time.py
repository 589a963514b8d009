"""Step time and memory of k2's smoothed simple loss (rnnt_loss_simple with lm_only_scale / am_only_scale), against the
plain simple loss and the same smoothed loss in torch ops.

    python tools/simple_smoothed_time.py [--shapes a,b,c4] [--rounds 5] [--out FILE] [--no-profile]

Shapes as in tools/simple_time.py (bench.py's ragged lengths, seed N + V): a = N=32 T=500 U=100 V=500,
b = N=32 T=600 U=150 V=1024, c4 = N=64 T=1500 U=300 V=50.  am (N,T,V) and lm (N,U,V) are randn float32.  Every arm's
step is `loss.backward()` with reduction="sum", captured in a CUDA graph:
  plain   rnnt_loss_simple(am, lm, prune_range=5)
  lm25    rnnt_loss_simple(..., prune_range=5, lm_only_scale=0.25, am_only_scale=0.0)   (icefall's defaults)
  lm1am1  rnnt_loss_simple(..., prune_range=5, lm_only_scale=0.1, am_only_scale=0.1)    (k2's defaults)
  torch   k2's smoothed formula (scales 0.1 / 0.1) in torch fp32 ops: the matmul normaliser, log_softmax(lm), the
          batch unigram and the AM-only normaliser, the mixed (N,T,U,2) pairs by gather, then RNNTLoss with
          blank = -1 on this library's recurrence; no ranges
Each round times the arms once, one after the other; the JSON line reports the median and range over rounds of ms per
step (CUDA events over `steps` graph replays), and the step's memory: torch.cuda.max_memory_allocated over one eager
step above what was allocated before it, plus the arm's inputs.  A separate torch.profiler run records the device
time of each kernel of arm lm1am1.  The card's name, power limit and max SM clock come from read-only queries in the
same run."""
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
ARMS = ("plain", "lm25", "lm1am1", "torch")
SCALES = {"plain": (0.0, 0.0), "lm25": (0.25, 0.0), "lm1am1": (0.1, 0.1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="a,b,c4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("simple_smoothed_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    torch.backends.cuda.matmul.allow_tf32 = False            # the torch arm: a plain fp32 matmul, as the loss needs
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/simple_smoothed_time.py", "card": card(), "lse_mode": "auto (exact)", "S": S,
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay",
              "arms": {"plain": "rnnt_loss_simple(am, lm, prune_range=5)",
                       "lm25": "rnnt_loss_simple(..., prune_range=5, lm_only_scale=0.25, am_only_scale=0.0)",
                       "lm1am1": "rnnt_loss_simple(..., prune_range=5, lm_only_scale=0.1, am_only_scale=0.1)",
                       "torch": "k2's smoothed formula (0.1, 0.1) in torch fp32 ops -> RNNTLoss(blank=-1), no ranges"},
              "runs": {}}
    for name in args.shapes.split(","):
        N, T, U, V = SHAPES[name]
        ys, xn, yn = (t.to(dev) for t in ragged_lengths(N, T, U, V, N + V))
        g = torch.Generator(device=dev).manual_seed(N + V)
        am = torch.randn((N, T, V), device=dev, generator=g).requires_grad_(True)
        lm = torch.randn((N, U, V), device=dev, generator=g).requires_grad_(True)
        y = torch.cat([ys.long(), torch.zeros((N, 1), dtype=torch.long, device=dev)], dim=1)
        y = torch.where(torch.arange(U, device=dev)[None] < yn[:, None].long(), y, 0)

        def arm_simple(scales):
            def run():
                loss, _ = w.rnnt_loss_simple(am, lm, ys, xn, yn, reduction="sum", prune_range=S,
                                             lm_only_scale=scales[0], am_only_scale=scales[1])
                return loss
            return run

        def arm_torch(sl=0.1, sa=0.1):
            c = 1.0 - sl - sa
            amax = am.detach().amax(-1, keepdim=True)
            lmax = lm.detach().amax(-1, keepdim=True)
            z = torch.matmul((am - amax).exp(), (lm - lmax).exp().transpose(1, 2))
            norm = z.log() + amax + lmax.transpose(1, 2)                               # (N,T,U)
            lm_lp = lm.log_softmax(-1)                                                  # LM-only log-probs
            uni = lm_lp.exp().mean(dim=(0, 1)) + torch.finfo(torch.float32).tiny
            lu = uni.log()
            am_norm = torch.mv((am - amax).exp().reshape(-1, V), uni).reshape(N, T, 1).log() + amax
            pairs = []
            for k in (torch.zeros_like(y), y):
                am_k = am.gather(2, k[:, None, :].expand(N, T, U))
                lm_k = lm.gather(2, k[:, :, None])[:, :, 0]
                simple = am_k + lm_k[:, None] - norm
                lmonly = lm_lp.gather(2, k[:, :, None])[:, :, 0][:, None]
                amonly = am_k + lu[k][:, None] - am_norm
                pairs.append(simple * c + lmonly * sl + amonly * sa)
            pairs = torch.stack(pairs, dim=-1).contiguous()
            return w.RNNTLoss.apply(pairs, ys, xn, yn, -1, 0.0, None, False).sum()

        fns = {a: arm_simple(SCALES[a]) for a in SCALES}
        fns["torch"] = arm_torch

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
                step("lm1am1")
            torch.cuda.synchronize()
            reps = 5
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    step("lm1am1")
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                us = (getattr(ev, "self_device_time_total", 0) or getattr(ev, "self_cuda_time_total", 0)) / reps
                if us > 0:
                    kernels[ev.key[:160]] = {"us_per_step": us, "calls_per_step": ev.count / reps}
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
        out = {"N": N, "T": T, "U": U, "V": V, "S": S, "steps_per_round": k, "rounds": args.rounds,
               "eager_loss": losses, "arms": {}, "kernels_lm1am1": kernels}
        for arm in ARMS:
            out["arms"][arm] = {"ms_per_step": statistics.median(ms[arm]), "ms_range": [min(ms[arm]), max(ms[arm])],
                                "ms_rounds": ms[arm], "step_memory_bytes": mem[arm]}
        plain = out["arms"]["plain"]["ms_per_step"]
        for arm in ("lm25", "lm1am1"):
            out[arm + "_minus_plain_ms"] = out["arms"][arm]["ms_per_step"] - plain
        out["torch_over_lm1am1"] = out["arms"]["torch"]["ms_per_step"] / out["arms"]["lm1am1"]["ms_per_step"]
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
