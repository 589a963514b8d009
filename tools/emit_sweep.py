"""A/B sweep of the fused kernel's two dense-gradient emit orders over V (sets kComposeMaxRowBytes in csrc/fused.cu).

At N=128 T=150 U=40, V in {28, 64, 128, 256, 512, 1024}, f32 and bf16 i/o -- plus V=28 at batch sizes whose gradient
lies on either side of the 50 MB L2 -- exact LSE: one loss + dense gradient call
through the C ABI (rnnt_b200_loss_dense / _bf16), timed with CUDA events over back-to-back calls that rotate over
input sets larger than L2.  Each order runs in its own process (RNNT_B200_EMIT=compose|patch is read once per process);
the orders alternate for `--rounds` rounds and the median per point is reported.

    python tools/emit_sweep.py [--rounds 2] [--out profiles/h100_emit_sweep.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, U = 150, 40
VS = [28, 64, 128, 256, 512, 1024]
POINTS = [(dt, V, 128) for dt in ("f32", "bf16") for V in VS] + \
    [("f32", 28, 48), ("f32", 28, 64), ("f32", 28, 96), ("bf16", 28, 192), ("bf16", 28, 256)]   # (dtype, V, N)


def child(calls, warmup):
    import torch
    import warp_rnnt_b200  # noqa: F401
    L = ctypes.CDLL(os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so"))
    L.rnnt_b200_workspace_bytes.restype = ctypes.c_size_t
    L.rnnt_b200_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int]
    dev = torch.device("cuda:0")
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    loss = torch.zeros(1, device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    out = []
    for dt, V, N in POINTS:
        ws = torch.empty(L.rnnt_b200_workspace_bytes(N * T * U, N), dtype=torch.uint8, device=dev)
        costs = torch.empty(N, device=dev)
        g = torch.Generator(device=dev).manual_seed(V)
        esz = 2 if dt == "bf16" else 4
        sets = max(2, -(-(200 << 20) // (N * T * U * V * esz)))       # inputs + grads of all sets > 2x L2
        data = []
        for _ in range(sets):
            xs = torch.log_softmax(torch.randn(N, T, U, V, device=dev, generator=g), -1)
            xs = xs.to(torch.bfloat16) if dt == "bf16" else xs
            ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, device=dev, generator=g)
            xn = torch.full((N,), T, dtype=torch.int, device=dev)
            yn = torch.full((N,), U - 1, dtype=torch.int, device=dev)
            data.append((xs, ys, xn, yn, torch.empty_like(xs)))

        def call(i):
            xs, ys, xn, yn, gr = data[i % sets]
            if dt == "bf16":
                st = L.rnnt_b200_loss_dense_bf16(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(ys), p(xn),
                                                 p(yn), p(costs), p(gr), None, p(loss), p(counter), N, T, U, V, 0,
                                                 ctypes.c_float(0.0), 0)
            else:
                st = L.rnnt_b200_loss_dense(stream, p(ws), ctypes.c_size_t(ws.numel()), p(xs), p(ys), p(xn),
                                            p(yn), p(costs), p(gr), None, N, T, U, V, 0, ctypes.c_float(0.0), 0)
            assert st == 0, st
        for i in range(warmup):
            call(i)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(calls):
            call(i)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / calls
        out.append({"dtype": dt, "V": V, "N": N, "us": us, "grad_MB": N * T * U * V * esz / 1e6})
        del data
        torch.cuda.empty_cache()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.calls, args.warmup)
    res = {}
    for _ in range(args.rounds):
        for order in ("compose", "patch"):
            env = dict(os.environ, RNNT_B200_EMIT=order)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--calls", str(args.calls),
                                "--warmup", str(args.warmup)], env=env, capture_output=True, text=True, check=True)
            for pt in json.loads(r.stdout.strip().splitlines()[-1]):
                res.setdefault((pt["dtype"], pt["V"], pt["N"]), {"grad_MB": pt["grad_MB"]}).setdefault(order, []).append(pt["us"])
    import torch
    rows = []
    for (dt, V, N), d in res.items():
        c, pa = statistics.median(d["compose"]), statistics.median(d["patch"])
        rows.append({"dtype": dt, "V": V, "N": N, "row_bytes": V * (2 if dt == "bf16" else 4), "grad_MB": round(d["grad_MB"], 1),
                     "compose_us": round(c, 2), "patch_us": round(pa, 2), "compose_over_patch": round(c / pa, 3),
                     "compose_runs_us": [round(x, 2) for x in d["compose"]], "patch_runs_us": [round(x, 2) for x in d["patch"]]})
        print("%-5s N=%4d V=%5d  row %5d B  grad %7.1f MB  compose %9.2f us  patch %9.2f us  ratio %.3f" %
              (dt, N, V, rows[-1]["row_bytes"], rows[-1]["grad_MB"], c, pa, c / pa))
    props = torch.cuda.get_device_properties(0)
    doc = {"device": torch.cuda.get_device_name(0), "l2_MB": props.L2_cache_size / 2 ** 20, "shape": {"T": T, "U": U},
           "lse": "exact", "calls_per_point": args.calls, "rounds": args.rounds, "timing": "CUDA events over back-to-back C-ABI calls, median of rounds",
           "points": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)
            f.write("\n")


if __name__ == "__main__":
    main()
