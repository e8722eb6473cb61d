"""Scratch timing of the C = 192 GDN forward at 2 M and 16.7 M pixels, with a correctness check against torch
fp64 on a slice."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import functional as F
C = 192
torch.manual_seed(0)
gamma = (0.1 * torch.eye(C) + (0.02 * torch.randn(C, C)).abs()).cuda(); beta = (1 + 0.5 * torch.rand(C)).cuda()
for npix in (128 * 128 * 128 + 77, 4096 * 64 * 64):
  x = torch.randn(npix, C, device="cuda") * (0.05 + 3.95 * torch.rand(C, device="cuda"))
  y = F.gdn_forward(x, gamma, beta)
  sl = slice(npix - 70000, npix)
  want = x[sl].double() / (x[sl].double().abs() @ gamma.double() + beta.double())
  err = ((y[sl].double() - want).abs() / (want.abs() + 1e-30)).max().item()
  ts = []
  for _ in range(5):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); F.gdn_forward(x, gamma, beta); b.record(); torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
  t = sorted(ts)[2]
  print(f"npix={npix}: {t:.3f} ms  {8*npix*C/t/1e6:.0f} GB/s  {8*npix*C/t/1e6/3350:.3f} of peak  max rel err {err:.2e}", flush=True)
  del x, y
