"""Step time and memory of the pruned loss against the loss on the full joint output of the same lattices.

    python tools/pruned_time.py [--shapes a,b,c4] [--dtypes f32,bf16] [--rounds 5] [--out FILE]

Shapes (bench.py's ragged-length recipe, seed N + V): a = N=32 T=500 U=100 V=500, b = N=32 T=600 U=150 V=1024,
c4 = N=64 T=1500 U=300 V=50.  The step is `loss.backward()` with reduction="sum", captured in a CUDA graph.  Two arms
per shape and element type (bf16-representable randn logits):
  p  rnnt_loss_pruned(x (N,T,S,V), ranges), S = 5, windows along each lattice's diagonal (k2-like: monotone, every
     lattice keeps a path)
  d  rnnt_loss_from_logits(xf (N,T,U,V)), the full joint output
Each round times the two arms once, one after the other; the JSON line reports the median and range over rounds of ms
per step (CUDA events over `steps` graph replays), the HBM fraction of the algorithmic bytes at the data-sheet
3.35 TB/s (DESIGN.md 3.3: one read of the logits and one write of their gradient, 8*N*T*S*V bytes for f32 and
4*N*T*S*V for bf16 for arm p, the same with U for arm d), and the step's memory: the arm's input plus
torch.cuda.max_memory_allocated over one eager step above what was allocated before it.  The card's name, power limit
and max SM clock come from read-only queries in the same run."""
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
S = 5
ARMS = ("p", "d")
SHAPES = {"a": (32, 500, 100, 500), "b": (32, 600, 150, 1024), "c4": (64, 1500, 300, 50)}
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}


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


def diagonal_ranges(xn, yn, T):
    """Windows of S columns along each lattice's diagonal: r[t] = clamp(t*(Un-1)//Tn - 2, 0, Un - S); non-decreasing
    by at most one column per frame (Un <= Tn here), so consecutive windows overlap and the path along the diagonal
    stays inside them."""
    t = torch.arange(T, dtype=torch.long)[None, :]
    Tn, Un = xn.long()[:, None], yn.long()[:, None] + 1
    r = t * (Un - 1) // Tn - 2
    return torch.minimum(r.clamp(min=0), (Un - S).clamp(min=0)).to(torch.int).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="a,b,c4")
    ap.add_argument("--dtypes", default="f32,bf16")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=0, help="graph replays per arm and round (0: ~0.2 s worth)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pruned_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    dev = torch.device("cuda", 0)
    result = {"tool": "tools/pruned_time.py", "card": card(), "lse_mode": "auto (exact)", "S": S,
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay",
              "arms": {"p": "rnnt_loss_pruned(x (N,T,S,V), ranges), S = 5",
                       "d": "rnnt_loss_from_logits(x (N,T,U,V))"},
              "hbm_peak_gbs": HBM_GBS, "runs": {}}
    for name in args.shapes.split(","):
        N, T, U, V = SHAPES[name]
        ys, xn, yn = ragged_lengths(N, T, U, V, N + V)
        ranges = diagonal_ranges(xn, yn, T)
        ys, xn, yn, ranges = ys.to(dev), xn.to(dev), yn.to(dev), ranges.to(dev)
        for dn in args.dtypes.split(","):
            dtype = DTYPES[dn]
            g = torch.Generator(device=dev).manual_seed(N + V)
            xs = {"p": torch.randn((N, T, S, V), device=dev, generator=g).to(dtype).requires_grad_(True),
                  "d": torch.randn((N, T, U, V), device=dev, generator=g).to(dtype).requires_grad_(True)}

            def step(arm):
                x = xs[arm]
                x.grad = None
                if arm == "p":
                    loss = w.rnnt_loss_pruned(x, ys, xn, yn, ranges, reduction="sum")
                else:
                    loss = w.rnnt_loss_from_logits(x, ys, xn, yn, reduction="sum")
                loss.backward()
                return loss

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

            k = args.steps or max(5, int(200.0 / timed("d", 3)))
            timed("p", 3)
            ms = {a: [] for a in ARMS}
            for _ in range(args.rounds):
                for arm in ARMS:
                    ms[arm].append(timed(arm, k))
            esz = 2 if dtype == torch.bfloat16 else 4
            out = {"N": N, "T": T, "U": U, "V": V, "S": S, "dtype": dn, "steps_per_round": k, "rounds": args.rounds,
                   "eager_loss": losses, "arms": {}}
            for arm in ARMS:
                med = statistics.median(ms[arm])
                balg = 2 * esz * N * T * (S if arm == "p" else U) * V
                out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                    "step_memory_bytes": mem[arm], "algorithmic_bytes": balg,
                                    "hbm_frac": balg / (med * 1e-3) / 1e9 / HBM_GBS}
            out["d_over_p"] = out["arms"]["d"]["ms_per_step"] / out["arms"]["p"]["ms_per_step"]
            key = "%s_%s" % (name, dn)
            result["runs"][key] = out
            print(json.dumps({key: out}), flush=True)
            del graphs, xs, pool
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
