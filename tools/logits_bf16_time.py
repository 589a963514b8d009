"""Step time and memory of rnnt_loss_from_logits on float32 and on bfloat16 logits.

    python tools/logits_bf16_time.py [--shapes c2l,c5mbl] [--rounds 5] [--out FILE]

The step is bench.py's from-logits step, `rnnt_loss_from_logits(x, ys, xn, yn, reduction="sum").backward()`,
captured in a CUDA graph, at bench.py's c2l and c5mbl shapes.  Three arms on the same values (bf16-representable
logits, randn):
  f32            float32 logits
  bf16           bfloat16 logits, bfloat16 gradient
  bf16_via_f32   bfloat16 logits passed as `x.float()`: what a bf16 user had to do before bf16 logits were accepted
                 (a float32 copy of the logits, a float32 gradient, autograd's cast of it back to bf16)
Input sets rotate as in bench.py (footprint beyond L2).  Each round times every arm once, one after the other; the
JSON line reports the median and range over rounds of ms per step (CUDA events over `steps` graph replays), the
HBM fraction of the algorithmic bytes (DESIGN.md §3: 8*N*T*U*V for float32 logits, 4*N*T*U*V for bf16 -- bf16_via_f32
is the bf16 task, so 4*N*T*U*V too) at the data-sheet 3.35 TB/s, and torch.cuda.max_memory_allocated over one eager
step with only that arm's inputs resident.  The card's name and power limit come from read-only queries."""
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

from bench import WORKLOADS, rotation

HBM_GBS = 3350.0
ARMS = ("f32", "bf16", "bf16_via_f32")


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:                                 # the numbers then stand without it, and say so
        info["power_limit"] = "not read (%s)" % str(e)[:80]
    return info


def b_alg(N, T, U, V, esz):
    return 2 * esz * N * T * U * V + 4 * N * (U - 1) + 12 * N


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2l,c5mbl")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logits_bf16_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/logits_bf16_time.py", "card": card(), "lse_mode": "auto (exact)",
              "timed_call": "rnnt_loss_from_logits(x, ys, xn, yn, reduction='sum').backward(), CUDA-graph replay",
              "hbm_peak_gbs": HBM_GBS, "shapes": {}}
    for name in args.shapes.split(","):
        N, T, U, V = WORKLOADS[name][:4]
        g = torch.Generator(device=dev).manual_seed(N + V)
        ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, device=dev, generator=g)
        xn = torch.full((N,), T, dtype=torch.int, device=dev)
        yn = torch.full((N,), U - 1, dtype=torch.int, device=dev)
        R = {a: rotation(2 * (4 if a == "f32" else 2) * N * T * U * V) for a in ARMS}
        R["bf16_via_f32"] = R["bf16"]                          # the bf16 arms share their input sets

        def step(arm, x):
            x.grad = None
            loss = w.rnnt_loss_from_logits(x.float() if arm == "bf16_via_f32" else x, ys, xn, yn, reduction="sum")
            loss.backward()
            return loss

        # ---- memory: one eager step per arm with only that arm's input set resident (values bf16-representable)
        xf = torch.randn((N, T, U, V), device=dev, generator=g).to(torch.bfloat16).float().requires_grad_(True)
        mem = {}
        for arm in ARMS:
            if arm == "bf16":
                xb = xf.detach().to(torch.bfloat16).requires_grad_(True)
                del xf
            x = xf if arm == "f32" else xb
            step(arm, x)                                       # warm-up (allocator, lazy module loads)
            x.grad = None
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            step(arm, x)
            torch.cuda.synchronize()
            mem[arm] = torch.cuda.max_memory_allocated(dev)
            x.grad = None
        torch.cuda.empty_cache()

        # ---- inputs of every arm, R sets each (set 0 are the values above), one graph per set
        sets = {"bf16": [xb] + [torch.randn((N, T, U, V), device=dev, generator=g).to(torch.bfloat16).requires_grad_(True)
                                for _ in range(R["bf16"] - 1)]}
        sets["bf16_via_f32"] = sets["bf16"]
        sets["f32"] = [sets["bf16"][i % R["bf16"]].detach().float().requires_grad_(True) for i in range(R["f32"])]
        graphs = {}
        for arm in ARMS:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for x in sets[arm]:
                    step(arm, x)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for x in sets[arm]:
                x.grad = None
            torch.cuda.empty_cache()                           # the graphs allocate from pools of their own
            graphs[arm] = []
            for x in sets[arm]:
                gr = torch.cuda.CUDAGraph()
                x.grad = None
                with torch.cuda.graph(gr):
                    step(arm, x)
                graphs[arm].append(gr)
        torch.cuda.synchronize()

        def timed(arm, k):
            gs = graphs[arm]
            for i in range(3):
                gs[i % len(gs)].replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for i in range(k):
                gs[i % len(gs)].replay()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / k

        k = args.steps or max(10, int(200.0 / timed("f32", 5)))
        ms = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for arm in ARMS:
                ms[arm].append(timed(arm, k))
        out = {"N": N, "T": T, "U": U, "V": V, "steps_per_round": k, "rounds": args.rounds,
               "input_sets": {a: len(sets[a]) for a in ARMS}, "arms": {}}
        for arm in ARMS:
            med = statistics.median(ms[arm])
            balg = b_alg(N, T, U, V, 4 if arm == "f32" else 2)
            out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                "max_memory_allocated_bytes": mem[arm], "algorithmic_bytes": balg,
                                "hbm_frac": balg / (med * 1e-3) / 1e9 / HBM_GBS}
        out["bf16_over_f32"] = out["arms"]["bf16"]["ms_per_step"] / out["arms"]["f32"]["ms_per_step"]
        out["bf16_over_bf16_via_f32"] = out["arms"]["bf16"]["ms_per_step"] / out["arms"]["bf16_via_f32"]["ms_per_step"]
        result["shapes"][name] = out
        print(json.dumps({name: out}), flush=True)
        del graphs, sets, xb, x
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
