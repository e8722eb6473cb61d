"""Scratch probe: error of the tensor-core GDN backward's dgamma / dbeta / dx against a torch fp64 graph on the GPU,
as a function of the pixel count (does the tensor-core accumulation of dgamma drift with the number of 64-pixel chunks per CTA?)."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import functional as F

def ref(x, gamma, beta, dy):
  x = x.double().requires_grad_(True); g = gamma.double().requires_grad_(True); b = beta.double().requires_grad_(True)
  y = x / (x.abs() @ g + b)
  y.backward(dy.double())
  return x.grad, g.grad, b.grad

for C in (128, 192):
  torch.manual_seed(0)
  gamma = (0.1 * torch.eye(C) + (0.02 * torch.randn(C, C)).abs()).cuda(); beta = (1 + 0.5 * torch.rand(C)).cuda()
  for n_pix in (64 * 132, 64 * 132 * 8, 64 * 132 * 32, 64 * 132 * 220):
    x = (torch.randn(n_pix, C, device="cuda") * (0.05 + 3.95 * torch.rand(C, device="cuda")))
    dy = torch.randn(n_pix, C, device="cuda")
    wx, wg, wb = ref(x, gamma, beta, dy)
    dx, dg, db = F.gdn_backward(x, gamma, beta, dy)
    e = lambda got, want: ((got.double() - want).abs().max() / want.abs().max()).item()
    # the same in plain fp32 torch for scale
    x32 = x.clone().requires_grad_(True); g32 = gamma.clone().requires_grad_(True); b32 = beta.clone().requires_grad_(True)
    (x32 / (x32.abs() @ g32 + b32)).backward(dy)
    print(f"C={C} n_pix={n_pix} chunks/CTA={n_pix // 64 // 132}: CUDA dx {e(dx, wx):.2e} dgamma {e(dg, wg):.2e} dbeta {e(db, wb):.2e} | "
          f"torch fp32 dx {e(x32.grad, wx):.2e} dgamma {e(g32.grad, wg):.2e} dbeta {e(b32.grad, wb):.2e}", flush=True)
