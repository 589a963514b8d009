"""Scratch: a few calls of one config (for a profiler run)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import warp_rnnt_b200 as w
cfg = {"c2": (128, 150, 40, 28), "c3": (32, 150, 20, 5000), "c4": (64, 1500, 300, 50)}[sys.argv[1]]
mode = sys.argv[2] if len(sys.argv) > 2 else "fast"
N, T, U, V = cfg
dev = torch.device("cuda:0")
torch.manual_seed(0)
xs = torch.log_softmax(torch.randn(N, T, U, V, device=dev), -1)
ys = torch.randint(1, V, (N, U - 1), dtype=torch.int, device=dev)
xn = torch.full((N,), T, dtype=torch.int, device=dev)
yn = torch.full((N,), U - 1, dtype=torch.int, device=dev)
w.set_lse_mode(mode)
for _ in range(3):
    c, g = w._C.rnnt_loss(xs, ys, xn, yn)
torch.cuda.synchronize()
print(c[:4])
