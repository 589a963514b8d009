"""Step time of k2's lattice types and delay penalty against the regular loss on the same inputs.

    python tools/path_types_time.py [--shapes logits,pipeline,c4] [--rounds 5] [--out FILE] [--profile FILE]

Shapes (bench.py's ragged-length recipe, seed N + V; every lattice has fewer labels than frames, so each has a
one-symbol-per-frame path):
  logits    rnnt_loss_from_logits, N=32 T=600 U=150 V=1024, f32
  pipeline  rnnt_loss_simple(am, lm, prune_range=5) + rnnt_loss_pruned on (N,T,5,V) window logits taken at the
            returned ranges, N=32 T=500 U=100 V=500, f32 (both losses of the type under test)
  c4        rnnt_loss_from_logits, N=64 T=1500 U=300 V=50, f32
Four arms per shape: regular, regular with delay_penalty=0.05 (k_delay_pairs, then the regular recurrence), modified
and constrained (k_frames + k_frames_grads).  The step is loss.backward() with reduction="sum", captured in a CUDA graph;
each round times every arm once, one after the other, and the JSON line reports the median and range over rounds of ms
per step (CUDA events over `steps` graph replays).  --profile runs a separate torch.profiler pass (three eager steps per
arm) and reports the mean time per launch of each CUDA kernel.  The card's name, power limit and max SM clock come from
read-only queries in the same run."""
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
LAM = 0.05
ARMS = {"regular": ("regular", 0.0), "regular_delay": ("regular", LAM), "modified": ("modified", 0.0),
        "constrained": ("constrained", 0.0)}
SHAPES = {"logits": (32, 600, 150, 1024), "pipeline": (32, 500, 100, 500), "c4": (64, 1500, 300, 50)}


def make_step(w, name, dev):
    N, T, U, V = SHAPES[name]
    ys, xn, yn = ragged_lengths(N, T, U, V, N + V)
    ys, xn, yn = ys.to(dev), xn.to(dev), yn.to(dev)
    g = torch.Generator(device=dev).manual_seed(N + V)
    if name != "pipeline":
        x = torch.randn((N, T, U, V), device=dev, generator=g).requires_grad_(True)
        params = [x]

        def step(kind, lam):
            x.grad = None
            loss = w.rnnt_loss_from_logits(x, ys, xn, yn, reduction="sum", rnnt_type=kind, delay_penalty=lam)
            loss.backward()
            return loss
    else:
        am = torch.randn((N, T, V), device=dev, generator=g).requires_grad_(True)
        lm = torch.randn((N, U, V), device=dev, generator=g).requires_grad_(True)
        xw = torch.randn((N, T, S, V), device=dev, generator=g).requires_grad_(True)
        params = [am, lm, xw]

        def step(kind, lam):
            for p in params:
                p.grad = None
            simple, ranges = w.rnnt_loss_simple(am, lm, ys, xn, yn, reduction="sum", prune_range=S, rnnt_type=kind,
                                                delay_penalty=lam)
            pruned = w.rnnt_loss_pruned(xw, ys, xn, yn, ranges, reduction="sum", rnnt_type=kind, delay_penalty=lam)
            loss = 0.5 * simple + pruned
            loss.backward()
            return loss
    return step, params


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="logits,pipeline,c4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None, help="also write per-kernel times of a torch.profiler pass here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("path_types_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/path_types_time.py", "card": card(), "delay_penalty": LAM, "S": S,
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay", "runs": {}}
    kernels = {}
    for name in args.shapes.split(","):
        step, params = make_step(w, name, dev)
        losses = {}
        for arm, (kind, lam) in ARMS.items():
            losses[arm] = step(kind, lam).item()
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for arm, (kind, lam) in ARMS.items():
                step(kind, lam)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        pool = torch.cuda.graph_pool_handle()
        graphs = {}
        for arm, (kind, lam) in ARMS.items():
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, pool=pool):
                step(kind, lam)
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

        k = args.steps or max(5, int(200.0 / timed("regular", 3)))
        ms = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for arm in ARMS:
                ms[arm].append(timed(arm, k))
        N, T, U, V = SHAPES[name]
        out = {"N": N, "T": T, "U": U, "V": V, "dtype": "f32", "steps_per_round": k, "rounds": args.rounds,
               "eager_loss": losses, "arms": {}}
        for arm in ARMS:
            med = statistics.median(ms[arm])
            out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                "over_regular": med / statistics.median(ms["regular"])}
        result["runs"][name] = out
        print(json.dumps({name: out}), flush=True)
        del graphs, pool
        torch.cuda.synchronize()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            kernels[name] = {}
            for arm, (kind, lam) in ARMS.items():
                step(kind, lam)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(3):
                        step(kind, lam)
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
