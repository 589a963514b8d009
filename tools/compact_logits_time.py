"""Step time and memory of the loss on compact (joint_pack-ordered) logits: fused from-logits against the pipelines a
user of the compact layout had before.

    python tools/compact_logits_time.py [--shapes c4,c5l] [--rounds 5] [--out FILE]

Shapes (bench.py's ragged-length recipe, seed N + V): c4 = N=64 T=1500 U=300 V=50, c5l = N=32 T=600 U=150 V=1024.
The step is `loss.backward()` with reduction="sum", captured in a CUDA graph (under compact_hints(T, U) for the
compact arms).  Four arms on the same values (bf16-representable randn logits, float32 unless stated):
  a  rnnt_loss_from_logits(x, compact=True)                 x (STU, V) float32
  b  rnnt_loss_from_logits(xb, compact=True)                xb (STU, V) bfloat16, bfloat16 gradient
  c  rnnt_loss(torch.log_softmax(x, -1), compact=True)      the unfused compact pipeline
  d  rnnt_loss_from_logits(xp)                              the same logits padded to (N, T, U, V)
Each round times every arm once, one after the other; the JSON line reports the median and range over rounds of ms
per step (CUDA events over `steps` graph replays), the HBM fraction of the algorithmic bytes of the compact task
(8*STU*V for float32 logits: one read of the logits and one write of their gradient; 4*STU*V for bfloat16; arms c
and d do the float32 task) at the data-sheet 3.35 TB/s, and the step's memory: the
arm's input plus torch.cuda.max_memory_allocated over one eager step above what was allocated before it.  The graphs
share one memory pool and are replayed in the order they were captured.  The card's name and power limit come from
read-only queries."""
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

HBM_GBS = 3350.0
ARMS = ("a", "b", "c", "d")
SHAPES = {"c4": (64, 1500, 300, 50), "c5l": (32, 600, 150, 1024)}


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:                                 # the numbers then stand without it, and say so
        info["power_limit"] = "not read (%s)" % str(e)[:80]
    return info


def ragged_lengths(N, T, U, V, seed):
    """bench.py's ragged recipe: labels in [1, V), lengths in [T/2, T] and [U/2, U) shifted so that the maxima are T
    and U-1."""
    g = torch.Generator().manual_seed(seed)
    ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, generator=g)
    xn = torch.randint(T // 2, T + 1, (N,), dtype=torch.int, generator=g)
    yn = torch.randint(U // 2, U, (N,), dtype=torch.int, generator=g)
    return ys, xn + T - xn.max(), yn + (U - 1) - yn.max()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c4,c5l")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compact_logits_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/compact_logits_time.py", "card": card(), "lse_mode": "auto (exact)",
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay",
              "arms": {"a": "rnnt_loss_from_logits(x (STU,V) f32, compact=True)",
                       "b": "rnnt_loss_from_logits(x (STU,V) bf16, compact=True)",
                       "c": "rnnt_loss(torch.log_softmax(x, -1), compact=True), x (STU,V) f32",
                       "d": "rnnt_loss_from_logits(x padded to (N,T,U,V) f32)"},
              "hbm_peak_gbs": HBM_GBS, "shapes": {}}
    for name in args.shapes.split(","):
        N, T, U, V = SHAPES[name]
        ys, xn, yn = [t.to(dev) for t in ragged_lengths(N, T, U, V, N + V)]
        ys_c = torch.cat([ys[i, :yn[i]] for i in range(N)]).contiguous()
        rows = (xn.long() * (yn.long() + 1)).tolist()
        STU = sum(rows)
        g = torch.Generator(device=dev).manual_seed(N + V)
        xf = torch.randn((STU, V), device=dev, generator=g).to(torch.bfloat16).float()
        xp = torch.zeros((N, T, U, V), device=dev)
        o = 0
        for i in range(N):
            Tn, Un = int(xn[i]), int(yn[i]) + 1
            xp[i, :Tn, :Un] = xf[o:o + Tn * Un].view(Tn, Un, V)
            o += Tn * Un
        xs = {"a": xf.requires_grad_(True), "b": xf.detach().to(torch.bfloat16).requires_grad_(True),
              "d": xp.requires_grad_(True)}
        xs["c"] = xs["a"]

        def step(arm):
            x = xs[arm]
            x.grad = None
            if arm == "d":
                loss = w.rnnt_loss_from_logits(x, ys, xn, yn, reduction="sum")
            else:
                with w.compact_hints(T, U):
                    if arm == "c":
                        loss = w.rnnt_loss(torch.log_softmax(x, -1), ys_c, xn, yn, reduction="sum", compact=True)
                    else:
                        loss = w.rnnt_loss_from_logits(x, ys_c, xn, yn, reduction="sum", compact=True)
            loss.backward()
            return loss

        # ---- memory: one eager step per arm (after a warm-up step), above what was allocated before it
        mem, losses = {}, {}
        for arm in ARMS:
            step(arm)
            xs[arm].grad = None
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            losses[arm] = step(arm).item()
            torch.cuda.synchronize()
            mem[arm] = xs[arm].numel() * xs[arm].element_size() + torch.cuda.max_memory_allocated(dev) - base
            xs[arm].grad = None
        torch.cuda.empty_cache()

        # ---- one graph per arm, one shared pool, replayed in capture order
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for arm in ARMS:
                step(arm)
                xs[arm].grad = None
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        pool = torch.cuda.graph_pool_handle()
        graphs = {}
        for arm in ARMS:
            gr = torch.cuda.CUDAGraph()
            xs[arm].grad = None
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

        k = args.steps or max(5, int(200.0 / timed("a", 3)))
        for arm in ARMS[1:]:
            timed(arm, 3)
        ms = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for arm in ARMS:
                ms[arm].append(timed(arm, k))
        padded = N * T * U
        out = {"N": N, "T": T, "U": U, "V": V, "STU": STU, "padded_cells": padded,
               "padding_fraction": 1.0 - STU / padded, "steps_per_round": k, "rounds": args.rounds,
               "eager_loss": losses, "arms": {}}
        for arm in ARMS:
            med = statistics.median(ms[arm])
            balg = (4 if arm == "b" else 8) * STU * V
            out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                "step_memory_bytes": mem[arm], "algorithmic_bytes": balg,
                                "hbm_frac": balg / (med * 1e-3) / 1e9 / HBM_GBS}
        for arm in ("b", "c", "d"):
            out["%s_over_a" % arm] = out["arms"][arm]["ms_per_step"] / out["arms"]["a"]["ms_per_step"]
        result["shapes"][name] = out
        print(json.dumps({name: out}), flush=True)
        del graphs, xs, xp, xf, pool
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
