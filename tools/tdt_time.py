"""Step time and memory of the TDT loss (rnnt_loss_tdt), against the regular loss on logits of the same vocabulary.

    python tools/tdt_time.py [--shapes c2,pk,c4] [--rounds 5] [--arms t32,t16,c32,c16,y] [--eager c2] [--out FILE]

Shapes (bench.py's ragged-length recipe, seed N + V; durations [0, 1, 2, 3, 4], D = 5): c2 = N=128 T=150 U=40 V=28,
pk = N=32 T=250 U=80 V=1025 (Parakeet-like), c4 = N=64 T=1500 U=300 V=50.  The step is `loss.backward()` with
reduction="sum", captured in a CUDA graph.  Arms (randn logits, bf16-representable):
  t32  rnnt_loss_tdt(x (N,T,U,V+D) float32)
  t16  rnnt_loss_tdt(x (N,T,U,V+D) bfloat16)
  c32  rnnt_loss_tdt(x (STU,V+D) float32, compact=True) on the live rows of t32's logits, inside compact_hints(T, U)
  c16  the same in bfloat16
  y    rnnt_loss_from_logits(x (N,T,U,V) float32): the regular loss with the same dense passes, the yardstick
  e    (shapes in --eager) the eager PyTorch anti-diagonal TDT of tests/tdt_eager.py in float32 with autograd: what a
       user writes without the library.  It syncs the host once per call, so it is timed eagerly, not graph-captured.
Each round times every arm once, one after the other; the JSON reports the median and range over rounds of ms per
step (CUDA events), the HBM fraction of the three dense passes (one read of the logits in the forward, one read and one
write in the backward: 3 * esz * N*T*U*(V+D) bytes; STU*(V+D) for c32 / c16, V for arm y) at the data-sheet 3.35 TB/s, the step's memory (the
arm's input plus torch.cuda.max_memory_allocated over one eager step above what was allocated before it), and per-kernel
device times of eager t32 and c32 steps from torch.profiler (two steps in one session; the record says whether every TDT kernel
is in the trace, `t32_kernels_complete`, and the tool warns on stderr when one is not), and the same stages timed with
CUDA events through the operator calls (`t32_stages_us`: forward without posteriors = normaliser + recurrence, the
posterior pass as the difference with them, the backward's emit).  The card's name, power limit and max SM clock come from read-only queries in the same run."""
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
DURATIONS = (0, 1, 2, 3, 4)
TDT_KERNELS = ("k_tdt_norm", "k_tdt_recur", "k_tdt_post", "k_tdt_emit")
SHAPES = {"c2": (128, 150, 40, 28), "pk": (32, 250, 80, 1025), "c4": (64, 1500, 300, 50)}


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


def events_ms(fn, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2,pk,c4")
    ap.add_argument("--eager", default="c2", help="shapes that also time the eager PyTorch TDT")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--arms", default="t32,t16,c32,c16,y", help="graph-captured arms to time (e comes from --eager)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tdt_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    from tests.tdt_eager import tdt_costs
    dev = torch.device("cuda", 0)
    D = len(DURATIONS)
    result = {"tool": "tools/tdt_time.py", "card": card(), "durations": list(DURATIONS),
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay (arm e: eager)",
              "arms": {"t32": "rnnt_loss_tdt(x (N,T,U,V+D) float32)", "t16": "rnnt_loss_tdt(x (N,T,U,V+D) bfloat16)",
                       "c32": "rnnt_loss_tdt(x (STU,V+D) float32, compact=True), compact_hints(T, U)",
                       "c16": "rnnt_loss_tdt(x (STU,V+D) bfloat16, compact=True), compact_hints(T, U)",
                       "y": "rnnt_loss_from_logits(x (N,T,U,V) float32)",
                       "e": "eager PyTorch anti-diagonal TDT, float32, autograd"},
              "hbm_peak_gbs": HBM_GBS, "runs": {}}
    for name in args.shapes.split(","):
        N, T, U, V = SHAPES[name]
        ys, xn, yn = (t.to(dev) for t in ragged_lengths(N, T, U, V, N + V))
        g = torch.Generator(device=dev).manual_seed(N + V)
        x32 = torch.randn((N, T, U, V + D), device=dev, generator=g).to(torch.bfloat16)
        xs = {"t32": x32.float().requires_grad_(True), "t16": x32.requires_grad_(True),
              "y": torch.randn((N, T, U, V), device=dev, generator=g).to(torch.bfloat16).float().requires_grad_(True)}
        # the compact arms: the live rows of the same logits in joint_pack's order, labels concatenated
        live = [x32.detach()[i, :int(xn[i]), :int(yn[i]) + 1].reshape(-1, V + D) for i in range(N)]
        xs["c16"] = torch.cat(live).requires_grad_(True)             # a leaf of its own, not a view of t16's
        xs["c32"] = xs["c16"].detach().float().requires_grad_(True)
        ys_c = torch.cat([ys[i, :int(yn[i])] for i in range(N)]).contiguous()
        STU = xs["c16"].shape[0]
        del live
        arms = [a for a in args.arms.split(",") if a]
        graphed = list(arms)
        if name in args.eager.split(","):
            xs["e"] = xs["t32"].detach().clone().requires_grad_(True)
            arms.append("e")

        def step(arm):
            x = xs[arm]
            x.grad = None
            if arm == "y":
                loss = w.rnnt_loss_from_logits(x, ys, xn, yn, reduction="sum")
            elif arm == "e":
                loss = tdt_costs(x, ys, xn, yn, DURATIONS).sum()
            elif arm in ("c32", "c16"):
                with w.compact_hints(T, U):
                    loss = w.rnnt_loss_tdt(x, ys_c, xn, yn, DURATIONS, reduction="sum", compact=True)
            else:
                loss = w.rnnt_loss_tdt(x, ys, xn, yn, DURATIONS, reduction="sum")
            loss.backward()
            return loss

        mem, losses = {}, {}
        for arm in arms:
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

        # per-kernel device times of eager t32 and c32 steps from torch.profiler: two steps in one session, each
        # kernel's time averaged over the calls the trace holds, and the record says which TDT kernels it lacks
        from torch.profiler import ProfilerActivity, profile

        def kernel_times(arm):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(2):
                    step(arm)
                    torch.cuda.synchronize()
            kernels = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA" and getattr(ev, "device_time_total", 0) > 0:
                    kernels[ev.key.split("(")[0]] = round(ev.device_time_total / max(ev.count, 1), 2)
            missing = [k for k in TDT_KERNELS if not any(k in kname for kname in kernels)]
            if missing:
                print("tdt_time.py: %s %s: the profiler trace lacks %s; its per-kernel times are incomplete"
                      % (name, arm, ", ".join(missing)), file=sys.stderr, flush=True)
            xs[arm].grad = None
            return kernels, missing

        profiled = {arm: kernel_times(arm) for arm in ("t32", "c32") if arm in arms}
        kernels, missing = profiled.get("t32", ({}, list(TDT_KERNELS)))
        # the same stages timed with CUDA events through the operator calls, independent of the profiler:
        # forward without posteriors = normaliser + recurrence; with them, + k_tdt_post; backward = k_tdt_emit
        xt = xs["t32"].detach()
        fw = lambda want: w._C.rnnt_tdt_forward(xt, ys, xn, yn, list(DURATIONS), 0.0, 0, want)   # noqa: E731
        _, lse_, pg_ = fw(True)
        go_ = torch.ones(N, device=dev)
        bw = lambda: w._C.rnnt_tdt_backward(xt, lse_, pg_, ys, list(DURATIONS), go_, 0)          # noqa: E731
        stage = {}
        for key, fn in (("norm_recur", lambda: fw(False)), ("norm_recur_post", lambda: fw(True)), ("emit", bw)):
            fn()
            stage[key] = statistics.median(events_ms(fn, 5) for _ in range(3)) * 1e3
        stage["post"] = stage["norm_recur_post"] - stage["norm_recur"]
        stage = {k: round(v, 1) for k, v in stage.items()}
        del lse_, pg_
        xs["t32"].grad = None

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for arm in graphed:
                step(arm)
                xs[arm].grad = None
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        pool = torch.cuda.graph_pool_handle()
        graphs = {}
        for arm in graphed:
            gr = torch.cuda.CUDAGraph()
            xs[arm].grad = None
            with torch.cuda.graph(gr, pool=pool):
                step(arm)
            graphs[arm] = gr
        torch.cuda.synchronize()

        def timed(arm, k):
            fn = graphs[arm].replay if arm in graphs else (lambda: step(arm))
            for _ in range(2):
                fn()
            return events_ms(fn, k)

        ks = {arm: max(3, int(200.0 / timed(arm, 2))) for arm in arms}
        ms = {a: [] for a in arms}
        for _ in range(args.rounds):
            for arm in arms:
                ms[arm].append(timed(arm, ks[arm]))
        out = {"N": N, "T": T, "U": U, "V": V, "D": D, "STU": STU, "stu_over_ntu": STU / (N * T * U),
               "steps_per_round": ks, "rounds": args.rounds,
               "eager_loss": losses, "t32_kernels_us": kernels, "t32_kernels_complete": not missing,
               "t32_kernels_missing": missing, "t32_stages_us": stage, "arms": {}}
        if "c32" in profiled:
            out["c32_kernels_us"], miss = profiled["c32"]
            out["c32_kernels_complete"] = not miss
        for arm in arms:
            med = statistics.median(ms[arm])
            esz = 2 if arm in ("t16", "c16") else 4
            rows = STU if arm in ("c32", "c16") else N * T * U
            balg = 3 * esz * rows * (V if arm == "y" else V + D)
            out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                "step_memory_bytes": mem[arm], "dense_pass_bytes": balg,
                                "hbm_frac": balg / (med * 1e-3) / 1e9 / HBM_GBS}
        ratio = lambda a, b: out["arms"][a]["ms_per_step"] / out["arms"][b]["ms_per_step"]   # noqa: E731
        for a, b in (("t32", "y"), ("t16", "y"), ("e", "t32"), ("c32", "t32"), ("c16", "t16")):
            if a in out["arms"] and b in out["arms"]:
                out["%s_over_%s" % (a, b)] = ratio(a, b)
        result["runs"][name] = out
        print(json.dumps({name: out}), flush=True)
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
