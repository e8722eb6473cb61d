"""GDN / IGDN with trainable exponents, and fixed exponents outside {1, 2} / {1, 1/2}, on the literal-pow tensor-core
kernels (gdn_tc.cu, gdn_tc_pow_*) at 128 to 320 channels: the forward and all five gradients against the reference's
graph in float64, NaN / inf positions equal to the CUDA-core path's, profiler proof that the tensor cores ran and no
separate exponent kernel did, bitwise reproducible parameter gradients, the fallbacks, 16-bit activations, layer and
model training steps, and the one-call ABI entry tfcb_gdn_backward_exponents."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

WIDTHS = [128, 192, 256, 320]
# more 64-pixel tiles than one persistent wave at every width on an H100 (132 CTAs x 3 warpgroups at C = 128)
BIG = 64 * 420 + 5

# name: (alpha, epsilon, trainable alpha, trainable epsilon, rectify, inverse)
CONFIGS = {
    "alpha": (1.3, 1.0, True, False, True, False),
    "alpha_at_2_signed": (2.0, 1.0, True, False, False, False),  # powf of negative u with an integer exponent
    "epsilon": (1.0, 0.8, False, True, False, False),  # fixed alpha = 1 keeps |u|
    "both": (1.3, 0.8, True, True, True, False),
    "fixed_general": (1.5, 0.7, False, False, True, False),
    "igdn": (2.0, 0.6, False, True, False, True),  # fixed alpha = 2 keeps u^2
    "trainable_at_one": (1.0, 1.0, True, True, True, True),  # no |u| / identity shortcut
}

# Bounds over the widths, sizes and configurations above: the forward's relative error (|y64| + 1e-6 below, as for the
# fixed-exponent variants of test_gdn_wide_gpu.py) and each gradient's largest error as a fraction of its largest
# magnitude.  Measured on an H100 80GB HBM3: forward 1.25e-5; dx 5.4e-6, dgamma 1.24e-5, dbeta 6.0e-6, dalpha 4.5e-5,
# depsilon 5.1e-5 (1.2e-4 for dalpha of a single 320-channel pixel, where the CUDA-core path's is 7.3e-5).  The
# CUDA-core path reaches 6e-7 to 1.3e-5 on the same graph: the tensor cores' bf16 split costs ~4e-6 of each product,
# and the exponent gradients are sums with cancellation, which magnifies it.
FWD_RTOL = 2e-5
GRAD_TOL = {"x": 1.5e-5, "gamma": 3e-5, "beta": 1.5e-5, "alpha": 2e-4, "epsilon": 1e-4}


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


@pytest.fixture
def fp32_path():
  """Runs the enclosed calls on the CUDA-core kernels (TFCB_GDN_FP32=1)."""
  class _Switch:
    def __enter__(self):
      self.old = os.environ.get("TFCB_GDN_FP32")
      os.environ["TFCB_GDN_FP32"] = "1"

    def __exit__(self, *a):
      if self.old is None:
        os.environ.pop("TFCB_GDN_FP32", None)
      else:
        os.environ["TFCB_GDN_FP32"] = self.old
  return _Switch()


def _params(C_, seed):
  g = torch.Generator().manual_seed(seed)
  gamma = 0.1 * torch.eye(C_) + (0.02 * torch.randn(C_, C_, generator=g)).abs()
  beta = 1.0 + 0.5 * torch.rand(C_, generator=g)
  return gamma, beta


def _x(n_pix, C_, seed):
  g = torch.Generator().manual_seed(seed)
  scale = 0.05 + 3.95 * torch.rand(C_, generator=g)
  return torch.randn(n_pix, C_, generator=g) * scale


def _graph64(x, gamma, beta, alpha, epsilon, inverse, rectify, pow_alpha, pow_epsilon):
  """gdn.py:377-415 in float64, with the fixed exponents' shortcuts as in the reference."""
  u = torch.relu(x) if rectify else x
  if not pow_alpha and float(alpha) == 1:
    pool = u if rectify else u.abs()
  elif not pow_alpha and float(alpha) == 2:
    pool = u.square()
  elif pow_alpha:
    # TF's pow gradient with respect to the exponent takes log(u) as 0 where u <= 0 (torch's is NaN for u < 0)
    a0 = alpha.detach()
    p0 = u**a0
    pool = p0 + p0.detach() * torch.log(torch.where(u > 0, u, torch.ones_like(u))) * (alpha - a0)
  else:
    pool = u**alpha
  n = pool @ gamma + beta
  if not pow_epsilon and float(epsilon) == 1:
    pass
  elif not pow_epsilon and float(epsilon) == .5:
    n = n.sqrt()
  else:
    n = n**epsilon
  return u * n if inverse else u / n


def _step(F, x, gamma, beta, cfg, dy):
  """y and the gradients (x, gamma, beta, alpha, epsilon; None where the exponent is fixed) through functional.gdn."""
  alpha, epsilon, ta, te, rectify, inverse = cfg
  x = x.cuda().requires_grad_(True)
  g = gamma.cuda().requires_grad_(True)
  b = beta.cuda().requires_grad_(True)
  a_t = torch.tensor(alpha, device="cuda", requires_grad=True) if ta else alpha
  e_t = torch.tensor(epsilon, device="cuda", requires_grad=True) if te else epsilon
  y = F.gdn(x, g, b, inverse, rectify, a_t, e_t)
  leaves = [x, g, b] + ([a_t] if ta else []) + ([e_t] if te else [])
  got = list(torch.autograd.grad(y, leaves, dy.cuda()))
  grads = {"x": got[0], "gamma": got[1], "beta": got[2], "alpha": got[3] if ta else None,
           "epsilon": got[-1] if te else None}
  return y.detach(), grads


def _want64(x, gamma, beta, cfg, dy):
  alpha, epsilon, ta, te, rectify, inverse = cfg
  x64, g64, b64 = (t.double().cuda().requires_grad_(True) for t in (x, gamma, beta))
  a64 = torch.tensor(alpha, dtype=torch.float64, device="cuda", requires_grad=True) if ta else alpha
  e64 = torch.tensor(epsilon, dtype=torch.float64, device="cuda", requires_grad=True) if te else epsilon
  y64 = _graph64(x64, g64, b64, a64, e64, inverse, rectify, ta, te)
  leaves = [x64, g64, b64] + ([a64] if ta else []) + ([e64] if te else [])
  w = list(torch.autograd.grad(y64, leaves, dy.double().cuda()))
  return y64.detach(), {"x": w[0], "gamma": w[1], "beta": w[2], "alpha": w[3] if ta else None,
                        "epsilon": w[-1] if te else None}


def _of_max(got, want):
  return float((got.double() - want).abs().max()) / (float(want.abs().max()) + 1e-30)


@pytest.mark.parametrize("name", sorted(CONFIGS))
@pytest.mark.parametrize("n_pix", [1, 63, 129, BIG])
@pytest.mark.parametrize("C_", WIDTHS)
def test_forward_and_five_gradients_vs_fp64_graph(F, fp32_path, C_, n_pix, name):
  cfg = CONFIGS[name]
  gamma, beta = _params(C_, 31)
  x = _x(n_pix, C_, 32) * 1.5
  dy = torch.randn(n_pix, C_, generator=torch.Generator().manual_seed(33))
  y, got = _step(F, x, gamma, beta, cfg, dy)
  with fp32_path:
    _, old = _step(F, x, gamma, beta, cfg, dy)
  y64, want = _want64(x, gamma, beta, cfg, dy)
  assert torch.isfinite(y64).all()
  fwd = float(((y.double() - y64).abs() / (y64.abs() + 1e-6)).max())
  errs = {k: (_of_max(got[k], w), _of_max(old[k], w)) for k, w in want.items() if w is not None}
  assert fwd < FWD_RTOL, fwd
  for k, (err, err_old) in errs.items():
    assert err < GRAD_TOL[k], (k, err, err_old)


@pytest.mark.parametrize("C_", WIDTHS)
def test_nan_and_inf_positions_equal_the_cuda_core_path(F, fp32_path, C_):
  """Negative x with a non-integer trainable alpha and no rectifier gives NaN (powf), as does every output of its
  pixel; x = 0 with alpha < 1 gives an infinite d pool / dx."""
  gamma, beta = _params(C_, 41)
  x = _x(300, C_, 42).abs() + 0.05
  x[7, 3] = -0.5           # NaN pixel under alpha = 1.3
  x[100, :5] = 0.0         # inf derivative under alpha = 0.6
  dy = torch.randn(300, C_, generator=torch.Generator().manual_seed(43))
  for alpha in (1.3, 0.6):
    cfg = (alpha, 0.9, True, True, False, False)
    y, got = _step(F, x, gamma, beta, cfg, dy)
    with fp32_path:
      y_old, old = _step(F, x, gamma, beta, cfg, dy)
    pairs = [(y, y_old)] + [(got[k], old[k]) for k in got]
    for a, b in pairs:
      a, b = a.cpu(), b.cpu()
      assert torch.equal(torch.isnan(a), torch.isnan(b))
      assert torch.equal(a == float("inf"), b == float("inf"))
      assert torch.equal(a == float("-inf"), b == float("-inf"))
    assert torch.isnan(y[7]).all() if alpha == 1.3 else torch.isinf(got["x"][100, :5]).any()


def _kernels(fn):
  """Names of the CUDA kernels `fn` launches: the union over three profiler sessions of the same call.  A session of a
  process that has profiled before can miss device events -- all of them, or only some of the call's kernels -- and
  `fn` launches the same kernels every time, so the union is what it launches (the tests only ask whether some name
  is or is not among them)."""
  fn()
  torch.cuda.synchronize()
  names = {}
  for _ in range(3):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      fn()
      torch.cuda.synchronize()
    names.update(dict.fromkeys(e.name for e in prof.events() if e.device_type.name == "CUDA"))
  return list(names)


def _misaligned(n_pix, C_, seed):
  buf = _x(n_pix * C_ + 1, 1, seed).reshape(-1).cuda()
  x = buf[1:].view(n_pix, C_)
  assert x.data_ptr() % 16 != 0
  return x


def _kernel_names_by_case():
  """The kernels of each call whose routing the tests check, by case.  Runs in a child process (see `kernel_names`)."""
  from compression_b200 import functional as F
  out = {}
  for C_ in WIDTHS:
    gamma, beta = (t.cuda() for t in _params(C_, 51))
    x = _x(5000, C_, 52).cuda().abs()
    dy = torch.randn(5000, C_, device="cuda")
    out[f"pow_{C_}"] = (_kernels(lambda: F.gdn_backward_exponents(x, gamma, beta, dy, alpha=1.2, epsilon=0.9)) +
                        _kernels(lambda: F.gdn_forward(x, gamma, beta, alpha=1.2, epsilon=0.9, pow_alpha=True,
                                                       pow_epsilon=True)))
  kw = dict(rectify=True, alpha=1.3, epsilon=0.8, pow_alpha=True, pow_epsilon=True)
  for case, C_ in (("misaligned", 192), ("C64", 64)):
    gamma, beta = (t.cuda() for t in _params(C_, 71))
    x = _misaligned(777, C_, 72) if case == "misaligned" else _x(777, C_, 72).cuda()
    dy = torch.randn(777, C_, device="cuda")
    out[case] = _kernels(lambda: F.gdn_backward_exponents(x, gamma, beta, dy, **kw))
  kw = dict(alpha=1.25, epsilon=0.75, pow_alpha=True, pow_epsilon=True, rectify=True)
  for C_ in (128, 192):
    gamma, beta = (t.cuda() for t in _params(C_, 81))
    x16 = _x(1000, C_, 82).cuda().to(torch.bfloat16)
    dy16 = torch.randn(1000, C_, device="cuda").to(torch.bfloat16)
    out[f"bf16_{C_}"] = _kernels(lambda: F.gdn_backward_exponents(x16, gamma, beta, dy16, **kw))
  return out


@pytest.fixture(scope="module")
def kernel_names():
  """_kernel_names_by_case() from a child process.  Profiling here would start the CUDA activity profiler in the test
  process itself, and a later profiler session of the same process can come back without any device events."""
  tests = os.path.dirname(os.path.abspath(__file__))
  code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gdn_exponents_tc_gpu as T; "
          "print('NAMES ' + json.dumps(T._kernel_names_by_case()))" % (os.path.dirname(tests), tests))
  env = {k: v for k, v in os.environ.items() if k != "TFCB_GDN_FP32"}
  env["PYTHONDONTWRITEBYTECODE"] = "1"
  flags = ["-s"] if sys.flags.no_user_site else []
  r = subprocess.run([sys.executable, *flags, "-c", code], env=env, capture_output=True, text=True, timeout=600)
  assert r.returncode == 0, r.stderr[-4000:]
  line = [ln for ln in r.stdout.splitlines() if ln.startswith("NAMES ")][-1]
  return json.loads(line[len("NAMES "):])


@pytest.mark.parametrize("C_", WIDTHS)
def test_tensor_cores_ran_and_no_exponent_kernel(F, kernel_names, C_):
  from compression_b200 import _lib
  gamma, beta = (t.cuda() for t in _params(C_, 51))
  x = _x(5000, C_, 52).cuda().abs()
  dy = torch.randn(5000, C_, device="cuda")
  fused = lambda: F.gdn_backward_exponents(x, gamma, beta, dy, alpha=1.2, epsilon=0.9)
  names = kernel_names[f"pow_{C_}"]
  assert any("gdn_tc_pow_" in n and ("bwd" in n) for n in names), names
  assert any("gdn_tc_pow_" in n and "fwd" in n for n in names), names
  assert not any("gdn_bwd_exponents_kernel" in n or "gdn_bwd_q_kernel" in n or "generic" in n for n in names), names
  n0 = _lib.launch_count()
  F.gdn_backward(x, gamma, beta, dy)  # fixed-exponent tensor-core backward
  n1 = _lib.launch_count()
  fused()
  n2 = _lib.launch_count()
  assert n2 - n1 == (n1 - n0) + 1  # plus the reduction of the exponent partials


@pytest.mark.parametrize("C_", WIDTHS)
def test_parameter_gradients_are_bitwise_reproducible(F, C_):
  gamma, beta = (t.cuda() for t in _params(C_, 61))
  x = _x(BIG, C_, 62).cuda()
  dy = torch.randn(BIG, C_, device="cuda")
  a = F.gdn_backward_exponents(x, gamma, beta, dy, rectify=True, alpha=1.4, epsilon=0.8)
  b = F.gdn_backward_exponents(x, gamma, beta, dy, rectify=True, alpha=1.4, epsilon=0.8)
  for u, v in zip(a, b):
    assert torch.equal(u, v)
  assert torch.isfinite(a[3]).all()


def _separate(F, x, gamma, beta, dy, **kw):
  dx, dg, db = F.gdn_backward(x, gamma, beta, dy, **kw)
  return dx, dg, db, F.gdn_exponent_grads(x, gamma, beta, dy, **kw)


@pytest.mark.parametrize("case", ["fp32_switch", "misaligned", "C64"])
def test_fallbacks_give_the_old_kernels_results(F, fp32_path, kernel_names, case):
  C_ = 64 if case == "C64" else 192
  gamma, beta = (t.cuda() for t in _params(C_, 71))
  n_pix = 777
  kw = dict(rectify=True, alpha=1.3, epsilon=0.8, pow_alpha=True, pow_epsilon=True)
  if case == "misaligned":
    x = _misaligned(n_pix, C_, 72)
  else:
    x = _x(n_pix, C_, 72).cuda()
  dy = torch.randn(n_pix, C_, device="cuda")
  if case == "fp32_switch":
    with fp32_path:
      fused, old = F.gdn_backward_exponents(x, gamma, beta, dy, **kw), _separate(F, x, gamma, beta, dy, **kw)
  else:
    fused, old = F.gdn_backward_exponents(x, gamma, beta, dy, **kw), _separate(F, x, gamma, beta, dy, **kw)
    names = kernel_names[case]
    assert not any("gdn_tc_" in n for n in names) and any("gdn_bwd_exponents_kernel" in n for n in names), names
  for u, v in zip(fused, old):
    assert torch.equal(u, v)


@pytest.mark.parametrize("C_", [128, 192])
def test_bf16_with_trainable_exponents_is_the_float32_result_rounded_once(F, kernel_names, C_):
  gamma, beta = (t.cuda() for t in _params(C_, 81))
  x16 = _x(1000, C_, 82).cuda().to(torch.bfloat16)
  dy16 = torch.randn(1000, C_, device="cuda").to(torch.bfloat16)
  kw = dict(alpha=1.25, epsilon=0.75, pow_alpha=True, pow_epsilon=True, rectify=True)
  y16 = F.gdn_forward(x16, gamma, beta, **kw)
  y32 = F.gdn_forward(x16.float(), gamma, beta, **kw)
  assert y16.dtype == torch.bfloat16 and torch.equal(y16, y32.to(torch.bfloat16))
  g16 = F.gdn_backward_exponents(x16, gamma, beta, dy16, **kw)
  g32 = F.gdn_backward_exponents(x16.float(), gamma, beta, dy16.float(), **kw)
  assert g16[0].dtype == torch.bfloat16 and torch.equal(g16[0], g32[0].to(torch.bfloat16))
  for u, v in zip(g16[1:], g32[1:]):
    assert torch.equal(u, v)
  names = kernel_names[f"bf16_{C_}"]
  assert any("gdn_tc_pow_bwd_dx_kernel" in n for n in names), names


def _layer_grads(fp32_path, fp32, inverse):
  import compression_b200 as tfc
  torch.manual_seed(5)
  layer = tfc.GDN(inverse=inverse, alpha_parameter=None, epsilon_parameter=None)
  x = _x(2048, 192, 91).abs().cuda() + 0.05  # pool = x ** alpha: a trainable alpha takes no |x|
  layer.build(x.shape, device="cuda")
  def run():
    y = layer(x)
    y.square().mean().backward()
  if fp32:
    with fp32_path:
      run()
  else:
    run()
  return {n: p.grad.clone() for n, p in layer.named_parameters()}


@pytest.mark.parametrize("inverse", [False, True])
def test_layer_with_trainable_exponents_trains_on_the_tensor_cores(fp32_path, inverse):
  got = _layer_grads(fp32_path, False, inverse)
  old = _layer_grads(fp32_path, True, inverse)
  assert len(got) == 4
  for n in got:
    assert torch.isfinite(got[n]).all(), n
    assert _of_max(got[n], old[n].double()) < 1e-4, (n, _of_max(got[n], old[n].double()))


def test_bmshj2018_320_step_with_trainable_exponents(fp32_path):
  import compression_b200 as tfc
  from compression_b200 import models

  def step(fp32):
    torch.manual_seed(0)
    m = models.BMSHJ2018Model(num_filters=320)
    gdns = [mod for mod in m.modules() if isinstance(mod, tfc.GDN)]
    for mod in gdns:
      mod.alpha_parameter = None
      mod.epsilon_parameter = None
    m.build("cuda", patch=(64, 64))
    x = torch.rand(2, 128, 128, 3, generator=torch.Generator().manual_seed(2)).mul(255).cuda()
    torch.manual_seed(3)
    if fp32:
      with fp32_path:
        loss, _, _ = m(x, training=True)
        loss.backward()
    else:
      loss, _, _ = m(x, training=True)
      loss.backward()
    return float(loss), {f"{i}.{n}": p.grad.clone() for i, mod in enumerate(gdns) for n, p in mod.named_parameters()}

  loss, got = step(False)
  loss_old, old = step(True)
  assert len(got) >= 4 and len(got) % 4 == 0
  assert abs(loss - loss_old) <= 1e-4 * abs(loss_old)
  for n in got:
    assert torch.isfinite(got[n]).all(), n
    assert _of_max(got[n], old[n].double()) < 1e-2, (n, _of_max(got[n], old[n].double()))


def _abi_call(F, x, gamma, beta, dy, outs, ws, n_pix, C_, flags, alpha, epsilon):
  from compression_b200 import _lib
  p = lambda t: C.c_void_p(t.data_ptr())
  return _lib.lib().tfcb_gdn_backward_exponents(p(x), p(gamma), p(beta), p(dy), *[p(t) for t in outs], p(ws), n_pix,
                                                C_, flags, alpha, epsilon, torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("flags,alpha,epsilon", [(0, 1.0, 1.0), (2, 2.0, 0.5), (4, 1.0, 1.0), (8, 1.0, 0.5),
                                                 (4 | 8 | 1, 1.5, 0.7), (2, 1.5, 0.7)])
@pytest.mark.parametrize("C_", [32, 128, 320])
def test_abi_entry_accepts_every_configuration(F, C_, flags, alpha, epsilon):
  """One call gives the five gradients of tfcb_gdn_backward + tfcb_gdn_exponent_grads (to the tensor cores'
  precision where it takes them)."""
  from compression_b200 import _lib
  n_pix = 500
  gamma, beta = (t.cuda() for t in _params(C_, 101))
  x = _x(n_pix, C_, 102).cuda().abs()
  dy = torch.randn(n_pix, C_, device="cuda")
  outs = [torch.empty_like(x), torch.empty_like(gamma), torch.empty_like(beta), torch.empty(2, device="cuda")]
  ws = torch.empty(int(_lib.lib().tfcb_gdn_backward_exponents_workspace_bytes(n_pix, C_)), dtype=torch.uint8,
                   device="cuda")
  _lib.check(_abi_call(F, x, gamma, beta, dy, outs, ws, n_pix, C_, flags, alpha, epsilon))
  kw = dict(inverse=bool(flags & 1), rectify=bool(flags & 2), alpha=alpha, epsilon=epsilon, pow_alpha=bool(flags & 4),
            pow_epsilon=bool(flags & 8))
  want = _separate(F, x, gamma, beta, dy, **kw)
  for u, v in zip(outs, want):
    assert torch.isfinite(u).all()
    assert _of_max(u, v.double()) < 1e-4


def test_abi_entry_zero_pixels_zeroes_without_a_launch(F):
  from compression_b200 import _lib
  C_ = 192
  gamma, beta = (t.cuda() for t in _params(C_, 111))
  outs = [torch.empty(16, device="cuda"), torch.full((C_, C_), float("nan"), device="cuda"),
          torch.full((C_,), float("nan"), device="cuda"), torch.full((2,), float("nan"), device="cuda")]
  ws = torch.empty(16, dtype=torch.uint8, device="cuda")
  n0 = _lib.launch_count()
  _lib.check(_abi_call(F, outs[0], gamma, beta, outs[0], outs, ws, 0, C_, 4 | 8, 1.2, 0.9))
  torch.cuda.synchronize()
  assert _lib.launch_count() == n0
  assert all(float(t.abs().max()) == 0.0 for t in outs[1:])
