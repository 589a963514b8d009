"""Time of rnnt_align_tdt (Viterbi alignment on the TDT lattice) beside the forward-only rnnt_loss_tdt on the same logits.

    python tools/tdt_align_time.py [--rounds 5] [--steps 20] [--out FILE]

Shapes: c2 = N=128 T=150 U=40 V=28, Parakeet-like = N=32 T=250 U=80 V=1025, c4 = N=64 T=1500 U=300 V=50; D = 5
(durations [0..4]), dense, full lengths, logits randn, float32 and bfloat16.  Arms per shape:
  align    rnnt_align_tdt(...)                                        captured in a CUDA graph
  nowalk   the same call through a second build of the library whose k_tdt_align skips the backtrace walk (the -1
           fill stays), compiled into a temporary directory at start-up; align - nowalk is the walk's share
  loss     rnnt_loss_tdt(...) under torch.no_grad() (the forward only)  captured in a CUDA graph
  eager    (c2 float32 only) an anti-diagonal max-plus Viterbi in eager PyTorch with a max(d)-frame look-back and a
           batched backtrace on the device, as a user would otherwise write it; not captured
Each round times every arm once, one after the other (CUDA events around `steps` replays or calls); the JSON lines
report the median and range over rounds in ms per call.  One torch.profiler pass per shape adds the device time of each
kernel of the align and loss arms.  The card's name, power limit and max SM clock come from read-only queries."""
import argparse
import ctypes
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

from tools.align_time import card, graphed, kernel_times, timed

DUR = [0, 1, 2, 3, 4]


def nowalk_lib(tmp):
    """librnnt_b200.so built from the sources with the backtrace walk of k_tdt_align switched off"""
    from warp_rnnt_b200 import build as b
    src = os.path.join(tmp, "warp_rnnt_b200", "csrc")          # common.cuh includes ../../include/rnnt_b200.h
    shutil.copytree(b.CSRC, src)
    shutil.copytree(b.INCLUDE, os.path.join(tmp, "include"))
    path = os.path.join(src, "tdt.cu")
    text = open(path).read()
    call = "Tn, Un, t0, st == kTdtOk);"
    assert text.count(call) == 1
    open(path, "w").write(text.replace(call, "Tn, Un, t0, false);"))
    lib = os.path.join(tmp, "librnnt_b200_nowalk.so")
    flags = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"]
    objs = [os.path.join(tmp, s + ".o") for s in b.CU_SOURCES]
    jobs = [subprocess.Popen([b._nvcc()] + flags + ["-c", os.path.join(src, s), "-o", o])
            for s, o in zip(b.CU_SOURCES, objs)]                 # one translation unit per process
    assert all(j.wait() == 0 for j in jobs)
    subprocess.check_call([b._nvcc()] + flags + ["-shared", "-o", lib] + objs)
    f = ctypes.CDLL(lib).rnnt_b200_tdt_align_dense
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 5 + \
        [ctypes.c_int, ctypes.c_float] + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 6
    ws = ctypes.CDLL(lib).rnnt_b200_tdt_align_workspace_bytes
    ws.restype = ctypes.c_size_t
    ws.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int]
    return f, ws


def nowalk_fn(lib, x, ys, xn, yn):
    f, ws_bytes = lib
    N, T, U, W = x.shape
    D = len(DUR)
    need = ws_bytes(N * T * U, N, D)
    ws = torch.empty(need, dtype=torch.uint8, device=x.device)
    s = torch.empty(N, device=x.device)
    fr = torch.empty(N, U - 1, dtype=torch.int32, device=x.device)
    fd = torch.empty_like(fr)
    durs = (ctypes.c_int * D)(*DUR)
    p = lambda t: t.data_ptr()

    def call():
        st = f(torch.cuda.current_stream().cuda_stream, p(ws), need, p(x), p(ys), p(xn), p(yn), durs, D, 0.0, p(s),
               p(fr), p(fd), N, T, U, W - D, 0, x.element_size())
        assert st == 0, st
        return s, fr, fd
    return call


def eager_viterbi(x, ys, xn, yn, durations, blank=0):
    """Anti-diagonal max-plus over the TDT lattice with a max(d)-frame look-back, then a batched backtrace, in eager
    PyTorch on the device (float32, torch's log_softmax)"""
    N, T, U, W = x.shape
    D = len(durations)
    V = W - D
    lt = torch.log_softmax(x[..., :V].float(), -1)
    ld = torch.log_softmax(x[..., V:].float(), -1)
    B = lt[..., blank]
    L = torch.cat([lt[:, :, :U - 1].gather(3, ys.long()[:, None, :, None].expand(N, T, U - 1, 1)).squeeze(3),
                   torch.full((N, T, 1), float("-inf"), device=x.device)], 2)
    a = torch.full((N, T, U), float("-inf"), device=x.device)
    a[:, 0, 0] = 0
    dec = torch.zeros((N, T, U), dtype=torch.long, device=x.device)
    for s in range(1, T + U - 1):
        t = torch.arange(max(0, s - U + 1), min(s, T - 1) + 1, device=x.device)
        u = s - t
        cands = []
        for j, d in enumerate(durations):
            tp = t - d
            ok = tp >= 0
            tq = tp.clamp(min=0)
            up = (u - 1).clamp(min=0)
            blank_c = (a[:, tq, u] + B[:, tq, u]) + ld[:, tq, u, j]
            label_c = (a[:, tq, up] + L[:, tq, up]) + ld[:, tq, up, j]
            cands.append(torch.where(ok & (d > 0), blank_c, float("-inf")))
            cands.append(torch.where(ok & (u > 0), label_c, float("-inf")))
        c = torch.stack(cands[0::2] + cands[1::2], 0)
        best, k = c.max(0)
        a[:, t, u] = best
        dec[:, t, u] = k
    n = torch.arange(N, device=x.device)
    un = yn.long()
    term = torch.stack([torch.where(xn.long() - d >= 0, (a[n, (xn.long() - d).clamp(min=0), un] +
                                                           B[n, (xn.long() - d).clamp(min=0), un]) +
                                    ld[n, (xn.long() - d).clamp(min=0), un, j], float("-inf"))
                        if d > 0 else torch.full((N,), float("-inf"), device=x.device)
                        for j, d in enumerate(durations)], 0)
    scores, jb = term.max(0)
    dt = torch.tensor(durations, device=x.device)
    t, u = xn.long() - dt[jb], un.clone()
    frames = torch.full((N, U), -1, dtype=torch.int32, device=x.device)
    fdur = torch.full((N, U), -1, dtype=torch.int32, device=x.device)
    for _ in range(T + U - 1):
        live = (t > 0) | (u > 0)
        k = dec[n, t.clamp(min=0), u]
        d = dt[k % D]
        lab = live & (k >= D)
        slot = torch.where(lab, u - 1, torch.full_like(u, U - 1))
        frames[n, slot] = torch.where(lab, t - d, frames[n, U - 1].long()).int()
        fdur[n, slot] = torch.where(lab, d, fdur[n, U - 1].long()).int()
        t = torch.where(live, t - d, t)
        u = u - lab.long()
    return scores, frames[:, :U - 1], fdur[:, :U - 1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import warp_rnnt_b200 as w
    dev = torch.device("cuda:0")
    hw = card()
    lines = [dict(hardware=hw)]
    print(json.dumps(lines[0]), flush=True)
    tmp = tempfile.mkdtemp(prefix="tdt_align_time_")
    try:
        lib = nowalk_lib(tmp)
        shapes = [("c2", (128, 150, 40, 28)), ("parakeet", (32, 250, 80, 1025)), ("c4", (64, 1500, 300, 50))]
        for name, (N, T, U, V) in shapes:
            for dtype in (torch.float32, torch.bfloat16):
                g = torch.Generator(device=dev).manual_seed(N + V)
                x = torch.randn(N, T, U, V + len(DUR), device=dev, generator=g).to(dtype)
                ys = torch.randint(1, V, (N, U - 1), device=dev, dtype=torch.int32, generator=g)
                xn = torch.full((N,), T, dtype=torch.int32, device=dev)
                yn = torch.full((N,), U - 1, dtype=torch.int32, device=dev)

                def align_fn(x=x, ys=ys, xn=xn, yn=yn):
                    return w.rnnt_align_tdt(x, ys, xn, yn, DUR)

                def loss_fn(x=x, ys=ys, xn=xn, yn=yn):
                    with torch.no_grad():
                        return w.rnnt_loss_tdt(x, ys, xn, yn, DUR)

                nw = nowalk_fn(lib, x, ys, xn, yn)
                s_a, f_a, d_a = align_fn()
                c_l = loss_fn()
                s_n = nw()[0]
                torch.cuda.synchronize()
                ok = bool((s_a <= -c_l + 2e-6 * (1 + c_l.abs())).all()) and torch.equal(s_a, s_n)
                arms = {"align": graphed(align_fn), "nowalk": graphed(nw), "loss": graphed(loss_fn)}
                if name == "c2" and dtype == torch.float32:
                    s_e, f_e, d_e = eager_viterbi(x, ys, xn, yn, DUR)
                    ok = ok and bool(torch.allclose(s_e, s_a, rtol=1e-5))
                    arms["eager"] = lambda x=x, ys=ys, xn=xn, yn=yn: eager_viterbi(x, ys, xn, yn, DUR)
                res = {k: [] for k in arms}
                for _ in range(args.rounds):
                    for k, fn in arms.items():
                        res[k].append(timed(fn, args.steps if k != "eager" else 2))
                line = dict(shape=name, N=N, T=T, U=U, V=V, D=len(DUR), dtype=str(dtype).replace("torch.", ""),
                            consistent=ok, rounds=args.rounds,
                            ms={k: dict(median=round(statistics.median(v), 4), min=round(min(v), 4),
                                        max=round(max(v), 4)) for k, v in res.items()},
                            kernels_us=kernel_times({"align": align_fn, "loss": loss_fn}))
                lines.append(line)
                print(json.dumps(line), flush=True)
                del arms
                torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)
            f.write("\n")


if __name__ == "__main__":
    main()
