"""GDN / IGDN with float16 / bfloat16 activations (float32 parameters, gdn_test.py:200-210) on the kernels that read
and write the 16-bit elements themselves, at C = 128 and 192.  The contract is exact: the forward gives the float32
kernel's y of the widened x rounded once, the backward gives the float32 backward's dx of the widened x and dy rounded
once, and the float32 backward's dgamma / dbeta bit for bit.  So every comparison here is bitwise, with NaN positions
compared separately from the bit patterns."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
# (inverse, rectify, alpha, epsilon): the FAST variant, IGDN, and the general variant's branches
CONFIGS = [(False, False, 1, 1), (True, False, 1, 1), (False, False, 2, 0.5), (False, True, 1, 1)]
# 1 pixel, a part tile, a tile plus one row, and more than one persistent wave at either width (up to 148 SMs x 3
# warpgroups x 64 pixels)
N_PIX = [1, 63, 129, 3 * 148 * 64 + 37]


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


def _params(C, seed):
  g = torch.Generator().manual_seed(seed)
  gamma = 0.1 * torch.eye(C) + (0.02 * torch.randn(C, C, generator=g)).abs()
  beta = 1.0 + 0.5 * torch.rand(C, generator=g)
  return gamma.cuda(), beta.cuda()


def _x(n_pix, C, seed, dtype, scale=1.0):
  g = torch.Generator().manual_seed(seed)
  s = scale * (0.05 + 3.95 * torch.rand(C, generator=g))
  return (torch.randn(n_pix, C, generator=g) * s).to(dtype).cuda()


def _bits(t):
  return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_same(got, want):
  """Bitwise equal, NaN positions compared on their own (a NaN's payload is not part of the contract)."""
  assert got.dtype == want.dtype and got.shape == want.shape
  nan = torch.isnan(want)
  assert torch.equal(torch.isnan(got), nan)
  ok = ~nan
  assert torch.equal(_bits(got)[ok], _bits(want)[ok]), int((_bits(got)[ok] != _bits(want)[ok]).sum())


def _count_routes(monkeypatch, F):
  """Counts the routing decisions of functional's 16-bit calls: {(direction, native): calls}."""
  seen = {}
  real = F._gdn_native16

  def counted(*a, **k):
    native = real(*a, **k)
    key = ("backward" if k.get("dy", a[7] if len(a) > 7 else None) is not None else "forward", native)
    seen[key] = seen.get(key, 0) + 1
    return native

  monkeypatch.setattr(F, "_gdn_native16", counted)
  return seen


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n_pix", N_PIX)
@pytest.mark.parametrize("inverse,rectify,alpha,epsilon", CONFIGS)
def test_forward_192_is_the_float32_result_rounded_once(F, dtype, n_pix, inverse, rectify, alpha, epsilon):
  from compression_b200 import _lib
  C = 192
  gamma, beta = _params(C, 41)
  x = _x(n_pix, C, 42, dtype)
  n0 = _lib.launch_count()
  y = F.gdn_forward(x, gamma, beta, inverse, rectify, alpha, epsilon)
  assert _lib.launch_count() == n0 + 1 and y.dtype == dtype
  assert_same(y, F.gdn_forward(x.float(), gamma, beta, inverse, rectify, alpha, epsilon).to(dtype))


@pytest.mark.parametrize("C", [128, 192])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n_pix", N_PIX)
@pytest.mark.parametrize("inverse,rectify,alpha,epsilon", CONFIGS)
def test_backward_is_the_float32_backward(F, C, dtype, n_pix, inverse, rectify, alpha, epsilon):
  from compression_b200 import _lib
  gamma, beta = _params(C, 14)
  x = _x(n_pix, C, 16, dtype)
  dy = torch.randn(n_pix, C, generator=torch.Generator().manual_seed(1)).to(dtype).cuda()
  n0 = _lib.launch_count()
  dx, dg, db = F.gdn_backward(x, gamma, beta, dy, inverse, rectify, alpha, epsilon)
  n1 = _lib.launch_count()
  dx32, dg32, db32 = F.gdn_backward(x.float(), gamma, beta, dy.float(), inverse, rectify, alpha, epsilon)
  assert n1 - n0 == _lib.launch_count() - n1  # the float32 tensor-core backward's kernels, no more
  assert dx.dtype == dtype and dg.dtype == db.dtype == torch.float32
  assert_same(dx, dx32.to(dtype))
  assert_same(dg, dg32)
  assert_same(db, db32)


@pytest.mark.parametrize("C", [128, 192])
@pytest.mark.parametrize("inverse", [False, True])
def test_backward_float16_overflow_and_nan(F, C, inverse):
  """Large float16 activations: IGDN's dx (dy * n + ...) overflows to +-inf when rounded and must do so where the
  conversion path's does (GDN's dy / n cannot, n >= beta >= 1), and a NaN in x spreads through its pixel and into
  dgamma / dbeta the same way."""
  dtype = torch.float16
  n_pix = 3000
  gamma, beta = _params(C, 3)
  x = _x(n_pix, C, 4, dtype, scale=60.0)
  x[7, 5] = float("nan")
  dy = (torch.randn(n_pix, C, generator=torch.Generator().manual_seed(5)) * 3000).to(dtype).cuda()
  dx, dg, db = F.gdn_backward(x, gamma, beta, dy, inverse)
  dx32, dg32, db32 = F.gdn_backward(x.float(), gamma, beta, dy.float(), inverse)
  want = dx32.to(dtype)
  assert bool(torch.isinf(want).any()) == inverse
  assert bool(torch.isfinite(want).any()) and bool(torch.isnan(want).any())
  assert_same(dx, want)
  assert_same(dg, dg32)
  assert_same(db, db32)


@pytest.mark.parametrize("C", [128, 192])
def test_native_backward_makes_no_float32_copies(F, C):
  """The native backward allocates dx (16-bit), dgamma, dbeta and its workspace, and nothing else: no float32 copy of
  x, dy or dx exists at any point."""
  from compression_b200 import _lib
  n_pix = 5000
  gamma, beta = _params(C, 8)
  x = _x(n_pix, C, 9, torch.bfloat16)
  dy = torch.randn(n_pix, C, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16).cuda()
  F.gdn_backward(x, gamma, beta, dy)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  out = F.gdn_backward(x, gamma, beta, dy)
  torch.cuda.synchronize()
  rounded = lambda b: (b + 511) // 512 * 512  # the caching allocator's granularity
  expected = (rounded(n_pix * C * 2) + rounded(C * C * 4) + rounded(C * 4) +
              rounded(int(_lib.lib().tfcb_gdn_backward_16bit_workspace_bytes(n_pix, C))))
  assert torch.cuda.max_memory_allocated() - base <= expected  # one float32 copy would add n_pix * C * 4 bytes
  del out


def _on_conversion_path(monkeypatch, F):
  monkeypatch.setattr(F, "_gdn_native16", lambda *a, **k: False)


@pytest.mark.parametrize("inverse", [False, True])
def test_module_gradients_equal_the_conversion_path(F, inverse, monkeypatch):
  import compression_b200 as tfc
  torch.manual_seed(0)
  layer = tfc.GDN(inverse=inverse)
  x0 = (torch.randn(4, 16, 16, 192, generator=torch.Generator().manual_seed(3)) * 2).to(torch.bfloat16).cuda()
  w = torch.randn(x0.shape, generator=torch.Generator().manual_seed(4)).cuda()

  def grads():
    layer.zero_grad(set_to_none=True)
    x = x0.clone().requires_grad_(True)
    y = layer(x)
    (y.float() * w).sum().backward()
    return y, x.grad, {n: p.grad.clone() for n, p in layer.named_parameters()}

  y, gx, gp = grads()
  _on_conversion_path(monkeypatch, F)
  y_c, gx_c, gp_c = grads()
  monkeypatch.undo()
  assert y.dtype == gx.dtype == torch.bfloat16
  assert_same(y, y_c)
  assert_same(gx, gx_c)
  assert gp.keys() == gp_c.keys() and len(gp) == 2
  for k in gp:
    assert_same(gp[k], gp_c[k])


def _autocast_step(make, x, monkeypatch, F, native):
  torch.manual_seed(123)
  m = make()
  if not native:
    _on_conversion_path(monkeypatch, F)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  torch.manual_seed(7)
  with torch.autocast("cuda", dtype=torch.bfloat16):
    loss, _, _ = m(x, training=True)
  loss.backward()
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated() - base
  monkeypatch.undo()
  grads = {k: (None if v.grad is None else v.grad.detach().clone()) for k, v in m.named_parameters()}
  return loss.detach(), grads, peak


@pytest.mark.parametrize("which", ["bls2017", "bmshj2018"])
def test_autocast_training_step_equals_the_conversion_path(F, which, monkeypatch):
  """One bf16-autocast training step of bls2017 (128 channels) and bmshj2018 (192): the GDN layers get 16-bit
  activations and 16-bit gradients.  Loss and every parameter gradient are bitwise those of the same step with GDN on
  the conversion path, and the step's peak memory is no higher."""
  from compression_b200 import _lib, models
  make = {
      "bls2017": lambda: models.BLS2017Model(num_filters=128).build("cuda"),
      "bmshj2018": lambda: models.BMSHJ2018Model(num_filters=192).build("cuda", patch=(64, 64)),
  }[which]
  x = torch.rand(2, 128, 128, 3, generator=torch.Generator().manual_seed(9)).mul(255).cuda()
  det = torch.backends.cudnn.deterministic
  torch.backends.cudnn.deterministic = True
  try:
    _autocast_step(make, x, monkeypatch, F, True)  # warm-up, so that both measured steps start from the same state
    seen = _count_routes(monkeypatch, F)
    loss, grads, peak = _autocast_step(make, x, monkeypatch, F, True)
    loss_c, grads_c, peak_c = _autocast_step(make, x, monkeypatch, F, False)
  finally:
    torch.backends.cudnn.deterministic = det
  # every GDN layer took the native kernels in both directions: bls2017 has 2 GDN + 2 IGDN layers, bmshj2018 3 + 3
  layers = {"bls2017": 4, "bmshj2018": 6}[which]
  assert seen == {("forward", True): layers, ("backward", True): layers}, seen
  assert _lib.launch_count() > 0
  assert_same(loss, loss_c)
  assert grads.keys() == grads_c.keys()
  assert sum(g is not None for g in grads.values()) > 0
  for k, g in grads.items():
    assert (g is None) == (grads_c[k] is None), k
    if g is not None:
      assert_same(g, grads_c[k])
  assert peak <= peak_c, (peak, peak_c)


def test_fp32_switch_takes_the_conversion_path(F, monkeypatch):
  """TFCB_GDN_FP32=1 keeps GDN on the float32 CUDA-core kernels: 16-bit calls convert instead of failing."""
  gamma, beta = _params(128, 5)
  x = _x(300, 128, 6, torch.bfloat16)
  dy = torch.randn(300, 128, generator=torch.Generator().manual_seed(7)).to(torch.bfloat16).cuda()
  monkeypatch.setenv("TFCB_GDN_FP32", "1")
  seen = _count_routes(monkeypatch, F)
  y = F.gdn_forward(x, gamma, beta)
  dx, dg, db = F.gdn_backward(x, gamma, beta, dy)
  assert seen == {("forward", False): 1, ("backward", False): 1}, seen
  assert_same(y, F.gdn_forward(x.float(), gamma, beta).to(torch.bfloat16))
  dx32, dg32, db32 = F.gdn_backward(x.float(), gamma, beta, dy.float())
  assert_same(dx, dx32.to(torch.bfloat16))
  assert_same(dg, dg32)
  assert_same(db, db32)


# ---- C ABI ----

def _abi_call(C=128, n_pix=100, dtype=2, flags=0, alpha=1.0, epsilon=1.0, offset=0, null=None):
  from compression_b200 import _lib
  t16 = torch.bfloat16 if dtype != 1 else torch.float16
  x = torch.zeros(max(n_pix, 1) * max(C, 1) + 8, dtype=t16, device="cuda")
  dy = torch.zeros_like(x)
  dx = torch.zeros_like(x)
  gamma = torch.eye(C, device="cuda") * 0.1
  beta = torch.ones(C, device="cuda")
  dg = torch.full((C, C), 7.0, device="cuda")
  db = torch.full((C,), 7.0, device="cuda")
  L = _lib.lib()
  ws = torch.empty(max(int(L.tfcb_gdn_backward_16bit_workspace_bytes(n_pix, C)), 1) + 64, dtype=torch.uint8,
                   device="cuda")
  ptrs = dict(x=x.data_ptr() + 2 * offset, gamma=gamma.data_ptr(), beta=beta.data_ptr(), dy=dy.data_ptr(),
              dx=dx.data_ptr(), dgamma=dg.data_ptr(), dbeta=db.data_ptr(), ws=ws.data_ptr())
  if null:
    ptrs[null] = None
  args = [ctypes.c_void_p(ptrs[k]) if ptrs[k] else None for k in
          ("x", "gamma", "beta", "dy", "dx", "dgamma", "dbeta", "ws")]
  n0 = _lib.launch_count()
  rc = L.tfcb_gdn_backward_16bit(*args, n_pix, C, dtype, flags, alpha, epsilon,
                                 torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  return rc, _lib.launch_count() - n0, dg, db


def test_abi_accepts_the_native_configurations():
  from compression_b200 import _lib
  for C in (128, 192):
    for dtype in (1, 2):
      rc, launches, dg, db = _abi_call(C=C, dtype=dtype)
      assert rc == _lib.OK and launches == 4
      assert not bool(dg.eq(7.0).any())


@pytest.mark.parametrize("kw", [
    dict(dtype=0), dict(dtype=3), dict(null="x"), dict(null="gamma"), dict(null="beta"), dict(null="dy"),
    dict(null="dx"), dict(null="dgamma"), dict(null="dbeta"), dict(null="ws"), dict(C=64), dict(C=256),
    dict(C=320), dict(alpha=1.5), dict(epsilon=0.7), dict(flags=4), dict(flags=8), dict(offset=1), dict(offset=4),
    dict(n_pix=-1), dict(C=0)])
def test_abi_rejects(kw):
  from compression_b200 import _lib
  rc, launches, dg, _ = _abi_call(**kw)
  assert rc == _lib.INVALID_ARGUMENT and launches == 0, (kw, rc, _lib.last_error())
  assert bool(dg.eq(7.0).all())


def test_abi_zero_pixels_launches_nothing_and_zeroes_the_parameter_gradients():
  from compression_b200 import _lib
  rc, launches, dg, db = _abi_call(n_pix=0)
  assert rc == _lib.OK and launches == 0
  assert not bool(dg.any()) and not bool(db.any())
