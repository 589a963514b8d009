"""Phase timeline of the fused small-lattice kernel (k_fused) from its optional clock64 stamps
(rnnt_b200_debug_fused_trace, include/rnnt_b200.h).  Prints, per LSE mode, the median over CTAs of each
phase's end time relative to the CTA's start, in microseconds.

    python tools/fused_timeline.py [c2|c3] [out.json]
"""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import warp_rnnt_b200 as w  # noqa: E402

SHAPES = {"c2": (128, 150, 40, 28), "c2n32": (32, 150, 40, 28), "c2n132": (132, 150, 40, 28), "c3": (32, 150, 20, 5000), "c1": (1, 150, 40, 28)}
NAMES = ["start", "sentinels", "gather_done", "sweep_start", "alpha_done", "beta_done", "fill_issued", "end", "chase_done",
         "zeros_landed", "patch_start"]


def sm_mhz():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        return pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:
        return 1900


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "c2"
    N, T, U, V = SHAPES[name]
    dev = torch.device("cuda:0")
    lib = ctypes.CDLL(os.path.join(os.path.dirname(w.__file__), "lib", "librnnt_b200.so"))
    lib.rnnt_b200_debug_fused_trace.argtypes = [ctypes.c_void_p]
    sets = []
    for s in range(4):
        torch.manual_seed(s)
        xs = torch.log_softmax(torch.randn(N, T, U, V, device=dev), -1)
        ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, device=dev)
        xn = torch.full((N,), T, dtype=torch.int, device=dev)
        yn = torch.full((N,), U - 1, dtype=torch.int, device=dev)
        sets.append((xs, ys, xn, yn))
    out = {"workload": name, "shape": [N, T, U, V]}
    for mode in ("exact", "fast"):
        w.set_lse_mode(mode)
        for i in range(6):
            w._C.rnnt_loss(*sets[i % 4])
        torch.cuda.synchronize()
        trace = torch.zeros(4096 * 16, dtype=torch.int64, device=dev)
        lib.rnnt_b200_debug_fused_trace(ctypes.c_void_p(trace.data_ptr()))
        mhz = sm_mhz()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        w._C.rnnt_loss(*sets[2])
        e1.record()
        torch.cuda.synchronize()
        lib.rnnt_b200_debug_fused_trace(None)
        mhz = max(mhz, sm_mhz())
        tr = trace.view(-1, 16).cpu()
        tr = tr[tr[:, 0] > 0]
        rel = (tr[:, :len(NAMES)] - tr[:, :1]).clamp(min=0).double() / mhz          # cycles / MHz = us
        med = rel.median(dim=0).values.tolist()
        mx = rel.max(dim=0).values.tolist()
        out[mode] = {"ctas": int(tr.shape[0]), "sm_mhz": mhz, "event_us": e0.elapsed_time(e1) * 1e3,
                     "median_us": dict(zip(NAMES, [round(x, 2) for x in med])),
                     "max_us": dict(zip(NAMES, [round(x, 2) for x in mx]))}
        print(mode, json.dumps(out[mode]))
    if len(sys.argv) > 2:
        json.dump(out, open(sys.argv[2], "w"), indent=1)


if __name__ == "__main__":
    main()
