"""Step time of the multi-blank transducer loss (rnnt_loss_multiblank), against the regular loss on the same vocabulary.

    python tools/multiblank_time.py [--shapes c2,pk,c4] [--rounds 5] [--arms m32,m16,c32,c16,y] [--out FILE]

Shapes (bench.py's ragged-length recipe, seed N + V; big_blank_durations [2, 4, 8], B = 3, NeMo's layout with the
standard blank last): c2 = N=128 T=150 U=40 V=28+4, pk = N=32 T=250 U=80 V=1025+3, c4 = N=64 T=1500 U=300 V=50+4,
where V = tokens + big blanks + standard blank.  The step is `loss.backward()` with reduction="sum", captured in a CUDA
graph.  Arms (randn logits, bf16-representable):
  m32  rnnt_loss_multiblank(x (N,T,U,V) float32)
  m16  rnnt_loss_multiblank(x (N,T,U,V) bfloat16)
  c32  rnnt_loss_multiblank(x (STU,V) float32, compact=True) on the live rows of m32's logits, inside
       compact_hints(T, U)
  c16  the same in bfloat16
  y    rnnt_loss_from_logits(x (N,T,U,V) float32, blank=V-1): the regular loss on the same V, the yardstick
Each round times every arm once, one after the other; the JSON reports the median and range over rounds of ms per
step (CUDA events), the HBM fraction of the three dense passes (one read of the logits in the forward, one read and one
write in the backward: 3 * esz * rows * V bytes) at the data-sheet 3.35 TB/s, and per-kernel device times of eager m32
and c32 steps from torch.profiler (two steps in one session).  The card's name, power limit and max SM clock come
from read-only queries in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

from tools.tdt_time import HBM_GBS, card, events_ms, ragged_lengths

DURATIONS = (2, 4, 8)
MB_KERNELS = ("k_mb_norm", "k_mb_recur", "k_mb_post", "k_mb_emit")
SHAPES = {"c2": (128, 150, 40, 28), "pk": (32, 250, 80, 1025), "c4": (64, 1500, 300, 50)}   # V = tokens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2,pk,c4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--arms", default="m32,m16,c32,c16,y")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multiblank_time.py: no CUDA device -- there is nothing to time on the CPU")
    import warp_rnnt_b200 as w
    dev = torch.device("cuda", 0)
    B = len(DURATIONS)
    result = {"tool": "tools/multiblank_time.py", "card": card(), "big_blank_durations": list(DURATIONS),
              "timed_call": "loss.backward(), reduction='sum', CUDA-graph replay",
              "arms": {"m32": "rnnt_loss_multiblank(x (N,T,U,V) float32)",
                       "m16": "rnnt_loss_multiblank(x (N,T,U,V) bfloat16)",
                       "c32": "rnnt_loss_multiblank(x (STU,V) float32, compact=True), compact_hints(T, U)",
                       "c16": "rnnt_loss_multiblank(x (STU,V) bfloat16, compact=True), compact_hints(T, U)",
                       "y": "rnnt_loss_from_logits(x (N,T,U,V) float32, blank=V-1)"},
              "hbm_peak_gbs": HBM_GBS, "runs": {}}
    for name in args.shapes.split(","):
        N, T, U, Vt = SHAPES[name]
        V = Vt + B + 1
        ys, xn, yn = (t.to(dev) for t in ragged_lengths(N, T, U, Vt, N + V))
        g = torch.Generator(device=dev).manual_seed(N + V)
        x16 = torch.randn((N, T, U, V), device=dev, generator=g).to(torch.bfloat16)
        # every arm its own leaf: the same values, no autograd edge between them
        xs = {"m32": x16.float().requires_grad_(True), "y": x16.float().requires_grad_(True),
              "m16": x16.clone().requires_grad_(True)}
        live = [x16.detach()[i, :int(xn[i]), :int(yn[i]) + 1].reshape(-1, V) for i in range(N)]
        xs["c16"] = torch.cat(live).requires_grad_(True)
        xs["c32"] = xs["c16"].detach().float().requires_grad_(True)
        ys_c = torch.cat([ys[i, :int(yn[i])] for i in range(N)]).contiguous()
        STU = xs["c16"].shape[0]
        del live
        arms = [a for a in args.arms.split(",") if a]

        def step(arm):
            x = xs[arm]
            x.grad = None
            if arm == "y":
                loss = w.rnnt_loss_from_logits(x, ys, xn, yn, reduction="sum", blank=V - 1)
            elif arm in ("c32", "c16"):
                with w.compact_hints(T, U):
                    loss = w.rnnt_loss_multiblank(x, ys_c, xn, yn, DURATIONS, reduction="sum", compact=True)
            else:
                loss = w.rnnt_loss_multiblank(x, ys, xn, yn, DURATIONS, reduction="sum")
            loss.backward()
            return loss

        losses = {arm: step(arm).item() for arm in arms}
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
            missing = [] if arm == "y" else [k for k in MB_KERNELS if not any(k in kname for kname in kernels)]
            if missing:
                print("multiblank_time.py: %s %s: the profiler trace lacks %s" % (name, arm, ", ".join(missing)),
                      file=sys.stderr, flush=True)
            xs[arm].grad = None
            return kernels, missing

        profiled = {arm: kernel_times(arm) for arm in ("m32", "c32", "y") if arm in arms}

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for arm in arms:
                step(arm)
                xs[arm].grad = None
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        pool = torch.cuda.graph_pool_handle()
        graphs = {}
        for arm in arms:
            gr = torch.cuda.CUDAGraph()
            xs[arm].grad = None
            with torch.cuda.graph(gr, pool=pool):
                step(arm)
            graphs[arm] = gr
        torch.cuda.synchronize()

        def timed(arm, k):
            for _ in range(2):
                graphs[arm].replay()
            return events_ms(graphs[arm].replay, k)

        ks = {arm: max(3, int(200.0 / timed(arm, 2))) for arm in arms}
        ms = {a: [] for a in arms}
        for _ in range(args.rounds):
            for arm in arms:
                ms[arm].append(timed(arm, ks[arm]))
        out = {"N": N, "T": T, "U": U, "V": V, "B": B, "STU": STU, "stu_over_ntu": STU / (N * T * U),
               "steps_per_round": ks, "rounds": args.rounds, "eager_loss": losses, "arms": {}}
        for arm, (kern, miss) in profiled.items():
            out["%s_kernels_us" % arm] = kern
            if arm != "y":
                out["%s_kernels_complete" % arm] = not miss
        for arm in arms:
            med = statistics.median(ms[arm])
            esz = 2 if arm in ("m16", "c16") else 4
            rows = STU if arm in ("c32", "c16") else N * T * U
            balg = 3 * esz * rows * V
            out["arms"][arm] = {"ms_per_step": med, "ms_range": [min(ms[arm]), max(ms[arm])], "ms_rounds": ms[arm],
                                "dense_pass_bytes": balg, "hbm_frac": balg / (med * 1e-3) / 1e9 / HBM_GBS}
        ratio = lambda a, b: out["arms"][a]["ms_per_step"] / out["arms"][b]["ms_per_step"]   # noqa: E731
        for a, b in (("m32", "y"), ("m16", "y"), ("c32", "m32"), ("c16", "m16")):
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
