"""Pins the float64 emulation of the GDN tensor cores' 3xBF16 split (oracle/gdn_oracle.py), which
test_gdn_trained_params_gpu.py holds the kernels to: the split's planes, the error it predicts for n at the suite's
initialiser-like and at trained-like parameters, and that the kernel-vs-emulation bounds fail for a kernel that
loses a lo plane or a dgamma partial."""
import math

import pytest
import torch

from oracle import gdn_oracle as O
import test_gdn_trained_params_gpu as T


def _values(n, seed):
  g = torch.Generator().manual_seed(seed)
  v = torch.randn(n, generator=g) * torch.exp(6 * torch.randn(n, generator=g))
  return torch.cat([v, torch.tensor([1.0, -1.0, 3.0, 1 / 3, 1e-6, 1e3, 2.0**-126, 65504.0])]).float()


def test_two_planes_reconstruct_float32_within_2_to_the_minus_16():
  v = _values(200000, 1)
  hi, lo = O.bf16_split(v)
  v64 = v.double()
  assert bool(((v64 - hi - lo).abs() <= 2.0**-16 * v64.abs()).all())
  # both planes are bf16 values, hi the nearest one to v, and v - hi is exact in fp32
  assert torch.equal(hi, hi.float().to(torch.bfloat16).double()) and torch.equal(lo, lo.float().to(torch.bfloat16).double())
  assert torch.equal(hi, v.to(torch.bfloat16).double())
  assert torch.equal((v - hi.float()).double(), v64 - hi)
  # the three products carry each product to within SPLIT_REL
  w = _values(200000, 2)
  wh, wl = O.bf16_split(w)
  exact = v64 * w.double()
  assert bool(((hi * wh + lo * wh + hi * wl - exact).abs() <= O.SPLIT_REL * exact.abs()).all())


def test_split_matmul_is_the_three_products():
  g = torch.Generator().manual_seed(3)
  a, b = torch.randn(33, 48, generator=g), torch.rand(48, 17, generator=g)
  out, mag = O.split_matmul(a, b)
  ah, al = O.bf16_split(a)
  bh, bl = O.bf16_split(b)
  assert torch.allclose(out, ah @ bh + al @ bh + ah @ bl, rtol=1e-15, atol=0)
  assert torch.allclose(mag, a.double().abs() @ b.double().abs(), rtol=1e-15, atol=0)


def _table_x(kind, n_pix, C_, g):
  if kind == "initialiser":
    return torch.randn(n_pix, C_, generator=g) * (0.05 + 3.95 * torch.rand(C_, generator=g))
  x = torch.randn(n_pix, C_, generator=g) * torch.exp(1.5 * torch.randn(C_, generator=g))
  x[torch.rand(n_pix, C_, generator=g) < 0.1] = 0.0
  return x


def _table_params(kind, C_, seed):
  if kind == "initialiser":
    return T.initialiser_like(C_, seed)
  if kind == "trained":
    return T.trained_like(C_, seed)
  g = torch.Generator().manual_seed(seed)  # gamma diagonal only, beta = 1e-6
  return torch.diag(torch.exp(torch.randn(C_, generator=g) - 1.0)), torch.full((C_,), 1e-6)


# The maximum relative error of n (and so of y) the emulation predicts over 20 000 pixels: C = 128, 192, 320.
TABLE = {"initialiser": (4.9e-6, 5.2e-6, 3.3e-6), "trained": (2.2e-5, 2.2e-5, 1.8e-5),
         "diagonal": (2.6e-5, 2.5e-5, 2.6e-5)}


@pytest.mark.parametrize("kind", sorted(TABLE))
def test_emulated_n_error_reproduces_the_table(kind):
  for C_, want in zip((128, 192, 320), TABLE[kind]):
    gamma, beta = _table_params(kind, C_, 10 + C_)
    x = _table_x(kind, 20000, C_, torch.Generator().manual_seed(20 + C_))
    _, n, _ = O.gdn_tc_forward_emulated(x, gamma, beta)
    n64 = x.double().abs() @ gamma.double() + beta.double()
    got = float(((n - n64).abs() / n64).max())
    assert want / 2 <= got <= 2 * want, (kind, C_, got, want)
    assert got <= O.SPLIT_REL  # the split's worst case per product bounds the whole sum


def test_dropping_a_lo_plane_violates_the_kernel_bounds():
  C_ = 128
  gamma, beta = T.trained_like(C_, 5)
  x, dy = T.inputs(3000, C_, 6)
  y, n, a = O.gdn_tc_forward_emulated(x, gamma, beta)
  y_bad, _, _ = O.gdn_tc_forward_emulated(x, gamma, beta, drop_lo=True)
  tol = O.U * y.abs() * (T.k_acc(C_) * a / n + T.K_EP)
  assert bool(((y_bad - y).abs() > tol).any())
  assert float(((y_bad - y).abs() / tol.clamp_min(1e-300)).max()) > 100  # not a near miss
  # the same bound accepts the emulation itself rounded to what an fp32 kernel returns
  assert bool(((y.float().double() - y).abs() <= tol).all())
  # backward: a lost lo plane in dp = q gamma^T or in dgamma = p^T q
  q = -dy * x / (n * n).float()
  good = O.gdn_tc_backward_emulated(x, gamma, beta, dy, q)
  bad = O.gdn_tc_backward_emulated(x, gamma, beta, dy, q, drop_lo=True)
  dx_tol = O.U * (good["d"].abs() * (T.k_acc(C_) * good["a"] / good["n"] + T.K_EP) +
                  good["dpool"].abs() * T.k_acc(C_) * good["a_dp"] + T.K_EP * (good["dpool"] * good["dp"]).abs())
  assert bool(((bad["dx"] - good["dx"]).abs() > dx_tol).any())
  assert bool(((bad["dgamma"] - good["dgamma"]).abs() > T.K_DGAMMA * O.U * good["a_dgamma"]).any())


def test_a_dropped_dgamma_partial_violates_the_kernel_bound():
  """dgamma without one CTA's last kDgFlush window of chunks: a small share of each sum, and still far outside."""
  C_, n_pix = 128, 64 * 40
  gamma, beta = T.trained_like(C_, 7)
  x, dy = T.inputs(n_pix, C_, 8)
  _, n, _ = O.gdn_tc_forward_emulated(x, gamma, beta)
  q = (-dy.double() * x.double() / (n * n)).float()
  p = O.tc_pool(x)
  full, mag = O.split_matmul(p.t(), q)
  keep = torch.ones(n_pix, dtype=torch.bool)
  keep[64 * 32:64 * 33] = False  # one 64-pixel chunk of one CTA's last window
  part, _ = O.split_matmul(p[keep].t(), q[keep])
  assert bool(((full - part).abs() > T.K_DGAMMA * O.U * mag).any())
