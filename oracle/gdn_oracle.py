"""ORACLE (test infrastructure): CPU restatement of tfc.GDN.call, tensorflow_compression/python/layers/
gdn.py:371-421, in PyTorch.  fp64 is the ground truth, fp32 the reference-precision path; gradients come
from torch autograd of the same graph (the reference relies on TF autodiff, it has no hand-written
gradient).  Also holds the closed forms asserted by the reference's tests (layers/gdn_test.py:42-88)."""
import torch


def gdn_reference(x, gamma, beta, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, dtype=torch.float64,
                  device="cpu"):
  x = x.detach().to(device, dtype)
  gamma = gamma.detach().to(device, dtype)
  beta = beta.detach().to(device, dtype)
  return _graph(x, gamma, beta, inverse, rectify, alpha, epsilon)


def _graph(x, gamma, beta, inverse, rectify, alpha, epsilon):
  u = torch.relu(x) if rectify else x
  if alpha == 1 and rectify:
    pool = u
  elif alpha == 1:
    pool = u.abs()
  elif alpha == 2:
    pool = u * u
  else:
    pool = u**alpha
  n = pool @ gamma + beta  # 1x1 convolution over the channel axis == matmul on [..., C]
  if epsilon == 1:
    pass
  elif epsilon == 0.5:
    n = n.sqrt()
  else:
    n = n**epsilon
  return u * n if inverse else u / n


def gdn_reference_grads(x, gamma, beta, dy, inverse=False, rectify=False, alpha=1.0, epsilon=1.0,
                        dtype=torch.float64, device="cpu"):
  x = x.detach().to(device, dtype).requires_grad_(True)
  gamma = gamma.detach().to(device, dtype).requires_grad_(True)
  beta = beta.detach().to(device, dtype).requires_grad_(True)
  y = _graph(x, gamma, beta, inverse, rectify, alpha, epsilon)
  y.backward(dy.detach().to(device, dtype))
  return x.grad, gamma.grad, beta.grad


# ---- The tensor-core kernels' arithmetic (compression_b200/csrc/gdn_tc.cu), emulated in float64 ----
#
# Every contraction there (n = p.gamma, dp = q.gamma^T, dgamma = p^T.q) runs on bf16 tensor cores over an
# error-compensated split of both fp32 operands: hi = bf16_rn(v), lo = bf16_rn(v - hi) with v - hi formed in fp32
# (split2 / split8), and three products hi.hi + lo.hi + hi.lo (the lo.lo product is skipped).  bf16 x bf16 products
# are exact in float64 and the sums here are float64, so what the emulation leaves out is only the kernels' fp32
# accumulation and their fp32 element-wise epilogues: a kernel that matches it to a few units of 2^-24 of the sum of
# |terms| computes exactly the split, while one that loses a lo plane, a beta column or a partial is off by ~2^-9 of
# the terms involved.  The split itself costs up to |pl gl| + |rp g| + |p rg| <= 3 * 2^-16 of each product (r: what
# the two planes leave of a value), which is SPLIT_REL below.

U = 2.0**-24  # unit roundoff of float32
SPLIT_REL = 3 * 2.0**-16


def bf16_split(v):
  """fp32 v -> (hi, lo) in float64, as split2 forms them: hi = bf16_rn(v), lo = bf16_rn(v - hi), v - hi in fp32."""
  v = v.to(torch.float32)
  hi = v.to(torch.bfloat16).to(torch.float32)
  lo = (v - hi).to(torch.bfloat16)
  return hi.double(), lo.double()


def split_matmul(a, b, drop_lo=False):
  """a @ b (fp32 operands) as the tensor cores form it: (ah bh + al bh + ah bl summed in float64, |a| @ |b|).  With
  `drop_lo` the a-side lo plane is left out, as a kernel that lost it would."""
  ah, al = bf16_split(a)
  bh, bl = bf16_split(b)
  out = ah @ bh + ah @ bl
  if not drop_lo:
    out = out + al @ bh
  return out, a.double().abs() @ b.double().abs()


def _f32(v):
  """A Python exponent as the kernels receive it (a float argument)."""
  return float(torch.tensor(float(v), dtype=torch.float32))


def tc_pool(x, rectify=False, alpha=1.0, pow_alpha=False):
  """pool(x) in fp32 as tc_pool forms it: |u| (u with rectify), u * u, or powf(u, alpha) (torch.pow on x's device)."""
  x = x.to(torch.float32)
  u = torch.relu(x) if rectify else x
  if not pow_alpha and float(alpha) == 1:
    return u if rectify else u.abs()
  if not pow_alpha and float(alpha) == 2:
    return u * u
  return torch.pow(u, _f32(alpha))


def _norm_fns(epsilon, pow_epsilon):
  """m(n) and dm/dn in float64 for the normaliser's exponent: identity, sqrt (fixed 1/2) or n ** epsilon."""
  if not pow_epsilon and float(epsilon) == 1:
    return (lambda n: n), (lambda n: torch.ones_like(n))
  if not pow_epsilon and float(epsilon) == 0.5:
    return torch.sqrt, (lambda n: 0.5 / torch.sqrt(n))
  e = _f32(epsilon)
  return (lambda n: n**e), (lambda n: e * n**(e - 1))


def gdn_tc_forward_emulated(x, gamma, beta, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, pow_alpha=False,
                            pow_epsilon=False, drop_lo=False):
  """The tensor-core forward on float32 x [n_pix, C] (channels-last), on x's device: (y, n, a) in float64, with
  n = beta + split(p).split(gamma) and a = sum_j |p_j gamma_jc|, the scale of n's accumulation error."""
  p = tc_pool(x, rectify, alpha, pow_alpha)
  s, a = split_matmul(p, gamma.to(x.device, torch.float32), drop_lo)
  n = beta.to(x.device, torch.float32).double() + s
  u = (torch.relu(x) if rectify else x).double()
  m = _norm_fns(epsilon, pow_epsilon)[0](n)
  return (u * m if inverse else u / m), n, a


def gdn_tc_backward_emulated(x, gamma, beta, dy, q, inverse=False, rectify=False, alpha=1.0, epsilon=1.0,
                             pow_alpha=False, pow_epsilon=False, drop_lo=False):
  """The tensor-core backward, given the fp32 q = dL/dn the kernels computed (they keep it in their workspace), in
  float64 on x's device.  q is what the kernels split, so the contractions that take it are emulated exactly; the
  returned q is the one implied by the emulated n, to check the kernels' own against.  Returns a dict:
    n, a        the forward's emulated n and its scale sum_j |p_j gamma_jc|
    q           dL/dn from the emulated n
    d           the direct term of dx (through the division or product)
    dp, a_dp    split(q).split(gamma)^T and sum_i |q_i gamma_ji|
    dpool       d pool / dx
    dx          d + dpool * dp, zero where rectify masks x <= 0
    dgamma, a_dgamma  split(p)^T.split(q) and sum_pix |p q|
    dbeta, a_dbeta    sum_pix q and sum_pix |q|
    dalpha_terms, depsilon_terms   the per-element terms of dL/dalpha (u > 0) and dL/depsilon."""
  dev = x.device
  x = x.to(torch.float32)
  gamma = gamma.to(dev, torch.float32)
  q = q.to(dev, torch.float32)
  _, n, a = gdn_tc_forward_emulated(x, gamma, beta, inverse, rectify, alpha, epsilon, pow_alpha, pow_epsilon, drop_lo)
  norm, dnorm = _norm_fns(epsilon, pow_epsilon)
  u = (torch.relu(x) if rectify else x).double()
  g = dy.to(dev, torch.float32).double()
  m, dm = norm(n), dnorm(n)
  if inverse:
    d, q_e = g * m, g * u * dm
  else:
    d, q_e = g / m, -g * u * dm / (m * m)
  if pow_epsilon or float(epsilon) not in (1.0, 0.5):
    # the kernels take q from powf(n, eps - 1) (IGDN) or powf(n, -eps - 1) (GDN), the exponent formed in fp32
    e = torch.tensor(_f32(epsilon), dtype=torch.float32)
    q_e = (e.item() * g * u * n**float(e - 1)) if inverse else (-e.item() * g * u * n**float(-e - 1))
  p = tc_pool(x, rectify, alpha, pow_alpha)
  if not pow_alpha and float(alpha) == 1:
    dpool = torch.ones_like(u) if rectify else torch.sign(u)
  elif not pow_alpha and float(alpha) == 2:
    dpool = 2 * u
  else:
    al = _f32(alpha)
    dpool = al * u**(al - 1)
  dp, a_dp = split_matmul(q, gamma.t(), drop_lo)
  dx = d + dpool * dp
  if rectify:
    dx = torch.where(x > 0, dx, torch.zeros_like(dx))
  dgamma, a_dgamma = split_matmul(p.t(), q, drop_lo)
  q64 = q.double()
  pos = u > 0
  dalpha_terms = torch.where(pos, dp * p.double() * torch.log(torch.where(pos, u, torch.ones_like(u))),
                             torch.zeros_like(u))
  depsilon_terms = q64 * n * torch.log(n) / _f32(epsilon)
  return dict(n=n, a=a, q=q_e, d=d, dp=dp, a_dp=a_dp, dpool=dpool, dx=dx, dgamma=dgamma, a_dgamma=a_dgamma,
              dbeta=q64.sum(0), a_dbeta=q64.abs().sum(0), dalpha_terms=dalpha_terms, depsilon_terms=depsilon_terms)
