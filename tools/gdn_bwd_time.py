"""Scratch timing of the GDN backward kernels (C = 128 and C = 192), with the error against a torch fp64 graph on a
slice of pixels.  Fractions of peak are of the H100 SXM data sheet's 3.35 TB/s."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import functional as F

def ref(x, gamma, beta, dy, inverse):
  x = x.double().requires_grad_(True); g = gamma.double().requires_grad_(True); b = beta.double().requires_grad_(True)
  n = x.abs() @ g + b
  y = x * n if inverse else x / n
  y.backward(dy.double())
  return x.grad, g.grad, b.grad

def med_ms(fn, reps=7):
  out = fn(); out = fn()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
  torch.cuda.synchronize(); ev[0].record()
  for i in range(reps):
    out = fn(); ev[i + 1].record()
  torch.cuda.synchronize()
  return sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))[reps // 2]

torch.manual_seed(0)
for C, shapes in ((128, (256 * 64 * 64, 256 * 32 * 32, 64 * 132 * 9 + 17)), (192, (128 * 64 * 64,))):
  gamma = (0.1 * torch.eye(C) + (0.02 * torch.randn(C, C)).abs()).cuda(); beta = (1 + 0.5 * torch.rand(C)).cuda()
  for n_pix in shapes:
    x = torch.randn(n_pix, C, device="cuda") * (0.05 + 3.95 * torch.rand(C, device="cuda"))
    x[::7, ::5] = 0.0  # exact zeros: d|x|/dx = 0 there
    dy = torch.randn(n_pix, C, device="cuda")
    for inverse in (False, True):
      dx, dg, db = F.gdn_backward(x, gamma, beta, dy, inverse=inverse)
      m = min(n_pix, 40000)
      wx, _, _ = ref(x[:m], gamma, beta, dy[:m], inverse)
      ex = ((dx[:m].double() - wx).abs().max() / wx.abs().max()).item()
      eg = eb = float("nan")
      if n_pix <= 300000:
        _, wg, wb = ref(x, gamma, beta, dy, inverse)
        eg = ((dg.double() - wg).abs().max() / wg.abs().max()).item(); eb = ((db.double() - wb).abs().max() / wb.abs().max()).item()
      ms = med_ms(lambda: F.gdn_backward(x, gamma, beta, dy, inverse=inverse))
      print(f"C={C} n_pix={n_pix} inverse={inverse}: {ms:.3f} ms  {12*n_pix*C/ms/1e6:.0f} GB/s  "
            f"{12*n_pix*C/ms/1e6/3350:.3f} of peak   err dx {ex:.1e} dgamma {eg:.1e} dbeta {eb:.1e}", flush=True)
    del x, dy
