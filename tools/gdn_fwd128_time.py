"""Scratch timing of the C = 128 GDN forward: float32 and 16-bit activations, the two cfg2 shapes."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import functional as F
def med_ms(fn, reps=15):
  out = fn(); out = fn()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
  torch.cuda.synchronize(); ev[0].record()
  for i in range(reps):
    out = fn(); ev[i + 1].record()
  torch.cuda.synchronize()
  return sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))[reps // 2]
C = 128
gamma = (0.1 * torch.eye(C) + (0.02 * torch.randn(C, C)).abs()).cuda(); beta = (1 + 0.5 * torch.rand(C)).cuda()
for n_pix in (256 * 64 * 64, 256 * 32 * 32):
  x = torch.randn(n_pix, C, device="cuda")
  for dt in (torch.float32, torch.bfloat16, torch.float16):
    xd = x.to(dt)
    ms = med_ms(lambda: F.gdn_forward(xd, gamma, beta))
    b = 2 * n_pix * C * xd.element_size()
    print(f"n_pix={n_pix} {str(dt):16s} {ms:.4f} ms  {b/ms/1e6:.0f} GB/s of its own traffic ({b/ms/1e6/3350:.3f} of peak)", flush=True)
  ms = med_ms(lambda: F.gdn_forward(x.to(torch.bfloat16).float(), gamma, beta).to(torch.bfloat16))
  print(f"n_pix={n_pix} bf16 via convert + float32 kernel + convert: {ms:.4f} ms")
