"""Scratch timing of ours vs the compiled reference (CUDA events, rotating buffers)."""
import sys, os, json, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import warp_rnnt_b200 as w
from oracle import build_ref

ref = build_ref.load()
dev = torch.device("cuda:0")


def time_fn(fn, sets, iters=20, warm=3):
    for i in range(warm):
        fn(sets[i % len(sets)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(sets[i % len(sets)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us


def mk(N, T, U, V, nsets):
    sets = []
    for s in range(nsets):
        torch.manual_seed(s)
        xs = torch.log_softmax(torch.randn(N, T, U, V, device=dev), -1)
        ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, device=dev)
        xn = torch.full((N,), T, dtype=torch.int, device=dev)
        yn = torch.full((N,), U - 1, dtype=torch.int, device=dev)
        sets.append((xs, ys, xn, yn))
    return sets


out = {}
for name, (N, T, U, V) in {"c2": (128, 150, 40, 28), "c3": (32, 150, 20, 5000), "c4": (64, 1500, 300, 50),
                            "c5mb": (32, 600, 150, 1024)}.items():
    byt = 4 * N * T * U * V
    nsets = max(2, min(6, int(600e6 // (2 * byt)) + 1)) if byt < 2e9 else 1
    sets = mk(N, T, U, V, nsets)
    r = {"nsets": nsets, "B_alg_MB": (4 * N * T * U * (V + 2) + 4 * N * (U - 1) + 12 * N) / 1e6}
    for mode in ("fast", "exact"):
        w.set_lse_mode(mode)
        r["ours_%s_us" % mode] = time_fn(lambda s: w._C.rnnt_loss(*s), sets)
    w.set_lse_mode("fast")
    r["ours_fwd_only_us"] = time_fn(lambda s: w._C.rnnt_loss_dense(*s, 0, 0.0, None, False, 0), sets)
    r["ours_gather_fwd_us"] = time_fn(lambda s: w._C.rnnt_gather_forward(*s, 0, 0.0, True, 0), sets)
    if ref is not None and N * T * U * V < 2**31:
        r["ref_us"] = time_fn(lambda s: ref.rnnt_loss(*s), sets, iters=5, warm=2)
    r["frac_fast"] = r["B_alg_MB"] * 1e6 / (r["ours_fast_us"] * 1e-6) / 3350e9   # H100 SXM data-sheet HBM3 bandwidth
    out[name] = r
    print(name, json.dumps(r), flush=True)
    del sets
    torch.cuda.empty_cache()
print(json.dumps(out, indent=1))
