"""Step time and peak memory of use_hat_loss against the softmax loss and against the torch composition of the HAT
log-probs fed to rnnt_loss_from_logits (the route a HAT model had before use_hat_loss).

    python tools/hat_time.py [--shapes c5mbl,c5mbl_bf16,c2l,pipeline] [--rounds 5] [--out FILE] [--profile FILE]

Shapes (bench.py's ragged-length recipe, seed N + V):
  c5mbl       rnnt_loss_from_logits, N=32 T=600 U=150 V=1024, f32
  c5mbl_bf16  the same, bf16 logits
  c2l         rnnt_loss_from_logits, N=128 T=150 U=40 V=28, f32
  pipeline    rnnt_loss_simple(am, lm, prune_range=5) + rnnt_loss_pruned on (N,T,5,V) window logits at the returned
              ranges, N=32 T=500 U=100 V=500, f32 (the simple loss is the regular one in every arm)
Arms: softmax (use_hat_loss=False), hat (use_hat_loss=True) and torch (the HAT log-probs composed in torch --
logsigmoid, log_softmax over the non-blank columns -- fed to the softmax loss, which leaves rows summing to 1 as they
are).  The step is loss.backward() with reduction="sum", captured in a CUDA graph; each round times every arm once,
one after the other, and the JSON line reports the median and range over rounds of ms per step (CUDA events over
`steps` graph replays).  Peak memory is torch.cuda.max_memory_allocated() over one eager step beyond what the inputs
and their gradients hold.  An arm that runs out of memory (eagerly, or in its graph's own pool) is reported as such.
--profile runs a separate torch.profiler pass (three eager steps per arm) and reports the mean time per launch of each
CUDA kernel.  The card's name, power limit and max SM clock come from read-only queries in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

from tools.pruned_time import card, ragged_lengths

S = 5
ARMS = ("softmax", "hat", "torch")
SHAPES = {"c5mbl": (32, 600, 150, 1024, torch.float32), "c5mbl_bf16": (32, 600, 150, 1024, torch.bfloat16),
          "c2l": (128, 150, 40, 28, torch.float32), "pipeline": (32, 500, 100, 500, torch.float32)}


def torch_hat(x):
    """the HAT log-probs of x (blank 0) composed in torch"""
    xb = x[..., :1]
    lab = torch.log_softmax(x[..., 1:], -1) + torch.nn.functional.logsigmoid(-xb)
    return torch.cat([torch.nn.functional.logsigmoid(xb), lab], -1)


def make_step(w, name, dev):
    N, T, U, V, dtype = SHAPES[name]
    ys, xn, yn = ragged_lengths(N, T, U, V, N + V)
    ys, xn, yn = ys.to(dev), xn.to(dev), yn.to(dev)
    g = torch.Generator(device=dev).manual_seed(N + V)
    if name != "pipeline":
        x = torch.randn((N, T, U, V), device=dev, generator=g).to(dtype).requires_grad_(True)
        params = [x]

        def step(arm):
            x.grad = None
            xs = torch_hat(x) if arm == "torch" else x
            loss = w.rnnt_loss_from_logits(xs, ys, xn, yn, reduction="sum", use_hat_loss=arm == "hat")
            loss.backward()
            return loss
    else:
        am = torch.randn((N, T, V), device=dev, generator=g).requires_grad_(True)
        lm = torch.randn((N, U, V), device=dev, generator=g).requires_grad_(True)
        xw = torch.randn((N, T, S, V), device=dev, generator=g).requires_grad_(True)
        params = [am, lm, xw]

        def step(arm):
            for p in params:
                p.grad = None
            simple, ranges = w.rnnt_loss_simple(am, lm, ys, xn, yn, reduction="sum", prune_range=S)
            xs = torch_hat(xw) if arm == "torch" else xw
            pruned = w.rnnt_loss_pruned(xs, ys, xn, yn, ranges, reduction="sum", use_hat_loss=arm == "hat")
            loss = 0.5 * simple + pruned
            loss.backward()
            return loss
    return step, params


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c5mbl,c5mbl_bf16,c2l,pipeline")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None, help="also write per-kernel times of a torch.profiler pass here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hat_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/hat_time.py", "card": card(), "S": S,
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay", "runs": {}}
    kernels = {}
    for name in args.shapes.split(","):
        step, params = make_step(w, name, dev)
        arms, losses, peak, oom = [], {}, {}, {}
        for arm in ARMS:
            try:
                step(arm)                                        # warm-up (allocator, module loads)
                for p in params:
                    p.grad = None
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                losses[arm] = step(arm).item()
                torch.cuda.synchronize()
                grads = sum(p.grad.numel() * p.grad.element_size() for p in params)
                peak[arm] = (torch.cuda.max_memory_allocated() - base - grads) / 2 ** 30
                arms.append(arm)
            except torch.cuda.OutOfMemoryError:
                oom[arm] = True
            for p in params:
                p.grad = None
            torch.cuda.empty_cache()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for arm in arms:
                step(arm)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graphs = {}
        for arm in list(arms):
            try:
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    step(arm)
                graphs[arm] = gr
            except torch.cuda.OutOfMemoryError:
                oom[arm] = "graph capture"
                arms.remove(arm)
                del gr                                           # its private pool goes with it
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
        gr = None
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

        k = args.steps or max(5, int(200.0 / timed("softmax", 3)))
        ms = {a: [] for a in arms}
        for _ in range(args.rounds):
            for arm in arms:
                ms[arm].append(timed(arm, k))
        N, T, U, V, dtype = SHAPES[name]
        out = {"N": N, "T": T, "U": U, "V": V, "dtype": str(dtype).replace("torch.", ""), "steps_per_round": k,
               "rounds": args.rounds, "eager_loss": losses, "oom": oom, "peak_extra_gib": peak, "arms": {}}
        for arm in arms:
            med = statistics.median(ms[arm])
            out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                "over_softmax": med / statistics.median(ms["softmax"]),
                                "peak_extra_gib": peak[arm]}
        result["runs"][name] = out
        print(json.dumps({name: out}), flush=True)
        del graphs
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            kernels[name] = {}
            for arm in ("softmax", "hat"):
                step(arm)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(3):
                        step(arm)
                    torch.cuda.synchronize()
                per = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    if t and e.count:
                        per[e.key[:90]] = {"us_per_launch": t / e.count, "launches_per_step": e.count / 3}
                kernels[name][arm] = per
        del step, params
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line, flush=True)
    for path, obj in ((args.out, result), (args.profile, {"card": result["card"], "kernels": kernels})):
        if path:
            os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
            with open(path, "w") as f:
                f.write(json.dumps(obj) + "\n")


if __name__ == "__main__":
    main()
