"""GDN / IGDN on channels-first activations ([N, C, *spatial], contiguous) read and written in place by the
tensor-core kernels (tfcb_gdn_forward_cf / tfcb_gdn_backward_cf).  The contract is exact: every output is, bit for
bit, what the channels-last path gives for x.movedim(1, -1).contiguous(), moved back.  So the comparisons here are
bitwise, with NaN positions compared on their own.  Inputs the native path does not cover take the movedim path and
give the same values."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

# (inverse, rectify, alpha, epsilon, trainable): the FAST variant, IGDN, the general fixed-exponent variant, the
# rectifier, and on the literal-pow kernels (float32 only) a fixed exponent outside the shortcuts and trainable ones
FIXED = [(False, False, 1, 1, False), (True, False, 1, 1, False), (False, False, 2, 0.5, False),
         (False, True, 1, 1, False), (True, True, 2, 1, False)]
POW = [(False, False, 1.5, 1, False), (False, False, 1.3, 0.8, True), (True, True, 1.2, 0.6, True)]
# ranks 3, 4 and 5; items of 1, 63, 64 and 4096 + 7 pixels; N * S a multiple of the 64-pixel tile and not
SHAPES = [(5, 1), (3, 7, 9), (2, 4, 4, 4), (3, 4103), (2, 2, 2, 16)]
# more than two waves of 132 CTAs for the dgamma reduction (and the dx grid) at every width
BIG = (3, 131, 173)


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


@pytest.fixture(scope="module")
def lib():
  from compression_b200 import _lib
  return _lib


def _params(C, seed):
  g = torch.Generator().manual_seed(seed)
  gamma = 0.1 * torch.eye(C) + (0.02 * torch.randn(C, C, generator=g)).abs()
  beta = 1.0 + 0.5 * torch.rand(C, generator=g)
  return gamma.cuda(), beta.cuda()


def _cf(shape, C, seed, dtype=torch.float32, positive=False):
  """[N, C, *spatial] with per-channel scales; `positive` keeps powf(u, alpha) of a non-integer alpha finite."""
  g = torch.Generator().manual_seed(seed)
  s = 0.05 + 3.95 * torch.rand(C, generator=g)
  x = torch.randn((shape[0],) + tuple(shape[1:]) + (C,), generator=g) * s
  if positive:
    x = x.abs() + 0.01
  return x.movedim(-1, 1).contiguous().to(dtype).cuda()


def _bits(t):
  return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_same(got, want):
  """Bitwise equal, NaN positions compared on their own (a NaN's payload is not part of the contract)."""
  assert got.dtype == want.dtype and got.shape == want.shape
  got, want = got.contiguous(), want.contiguous()
  nan = torch.isnan(want)
  assert torch.equal(torch.isnan(got), nan)
  ok = ~nan
  assert torch.equal(_bits(got)[ok], _bits(want)[ok]), int((_bits(got)[ok] != _bits(want)[ok]).sum())


def _run(F, x, gamma, beta, dy, cfg, channels_first):
  """y, dx, dgamma, dbeta (and dalpha / depsilon with trainable exponents) on one path; channels-last runs on
  x.movedim(1, -1).contiguous() and its results are moved back."""
  inverse, rectify, alpha, epsilon, trainable = cfg
  if not channels_first:
    x, dy = x.movedim(1, -1).contiguous(), dy.movedim(1, -1).contiguous()
  kw = dict(channels_first=True) if channels_first else {}
  y = F.gdn_forward(x, gamma, beta, inverse, rectify, alpha, epsilon, trainable, trainable, **kw)
  if trainable:
    grads = F.gdn_backward_exponents(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, True, True, **kw)
  else:
    grads = F.gdn_backward(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, **kw)
  if not channels_first:
    y, grads = y.movedim(-1, 1), (grads[0].movedim(-1, 1),) + tuple(grads[1:])
  return (y,) + tuple(grads)


def _check_bitwise(F, lib, shape, C, dtype, cfg, seed=0):
  positive = cfg[2] not in (1, 2) or cfg[4]
  x = _cf(shape, C, seed, dtype, positive)
  dy = _cf(shape, C, seed + 1, dtype)
  gamma, beta = _params(C, seed + 2)
  n0 = lib.launch_count()
  got = _run(F, x, gamma, beta, dy, cfg, True)
  n1 = lib.launch_count()
  want = _run(F, x, gamma, beta, dy, cfg, False)
  n2 = lib.launch_count()
  assert n1 - n0 == n2 - n1  # the kernels of the channels-last path, one library call per direction
  assert got[0].is_contiguous() and got[1].is_contiguous()  # native, not the movedim views
  for g, w in zip(got, want):
    assert_same(g, w)


@pytest.mark.parametrize("C", [128, 192, 256, 320])
@pytest.mark.parametrize("cfg", FIXED + POW)
def test_float32_is_the_channels_last_result_bit_for_bit(F, lib, C, cfg):
  _check_bitwise(F, lib, (3, 4103), C, torch.float32, cfg)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("C", [128, 192])
@pytest.mark.parametrize("cfg", FIXED)
def test_16bit_is_the_channels_last_result_bit_for_bit(F, lib, dtype, C, cfg):
  _check_bitwise(F, lib, (3, 4103), C, dtype, cfg)


@pytest.mark.parametrize("spatial", SHAPES)
@pytest.mark.parametrize("C,dtype,cfg", [(128, torch.float32, FIXED[0]), (192, torch.bfloat16, FIXED[2]),
                                         (128, torch.float16, FIXED[3]), (256, torch.float32, FIXED[1]),
                                         (320, torch.float32, POW[1]), (192, torch.float32, POW[2])])
def test_ranks_and_item_sizes(F, lib, spatial, C, dtype, cfg):
  _check_bitwise(F, lib, spatial, C, dtype, cfg, seed=3)


@pytest.mark.parametrize("C,dtype,cfg", [(128, torch.float32, FIXED[0]), (192, torch.bfloat16, FIXED[0]),
                                         (256, torch.float32, FIXED[2]), (320, torch.float32, POW[1]),
                                         (128, torch.float32, POW[2])])
def test_several_waves(F, lib, C, dtype, cfg):
  _check_bitwise(F, lib, BIG, C, dtype, cfg, seed=5)


def _no_native_calls(F, monkeypatch):
  """Records the native backward calls (the forward's path shows in its result's strides)."""
  calls = []
  real = F._gdn_backward_cf

  def spy(*a, **k):
    calls.append(1)
    return real(*a, **k)

  monkeypatch.setattr(F, "_gdn_backward_cf", spy)
  return calls


@pytest.mark.parametrize("C,dtype,cfg", [(64, torch.float32, FIXED[0]), (96, torch.float32, POW[1]),
                                         (256, torch.bfloat16, FIXED[0]), (320, torch.float16, FIXED[2]),
                                         (128, torch.bfloat16, POW[1]), (192, torch.float16, POW[0])])
def test_uncovered_configurations_take_the_movedim_path(F, lib, monkeypatch, C, dtype, cfg):
  calls = _no_native_calls(F, monkeypatch)
  x = _cf((2, 9, 11), C, 7, dtype, positive=True)
  dy = _cf((2, 9, 11), C, 8, dtype)
  gamma, beta = _params(C, 9)
  got = _run(F, x, gamma, beta, dy, cfg, True)
  want = _run(F, x, gamma, beta, dy, cfg, False)
  assert not calls and not got[0].is_contiguous() and not got[1].is_contiguous()
  for g, w in zip(got, want):
    assert_same(g, w)


def test_the_fp32_switch_takes_the_movedim_path(F, lib, monkeypatch):
  C = 128
  x, dy = _cf((2, 8, 8), C, 10), _cf((2, 8, 8), C, 11)
  gamma, beta = _params(C, 12)
  monkeypatch.setenv("TFCB_GDN_FP32", "1")
  calls = _no_native_calls(F, monkeypatch)
  got = _run(F, x, gamma, beta, dy, FIXED[0], True)
  want = _run(F, x, gamma, beta, dy, FIXED[0], False)
  assert not calls and not got[0].is_contiguous()
  for g, w in zip(got, want):
    assert_same(g, w)


def _layout_variants(C):
  base = _cf((2, 6, 10), C, 13)
  cl = base.to(memory_format=torch.channels_last)
  strided = _cf((2, 6, 20), C, 13)[..., ::2]
  buf = torch.empty(base.numel() + 1, device="cuda")
  shifted = buf[1:].view(base.shape)  # contiguous, 4 bytes past the allocation's 16-byte alignment
  shifted.copy_(base)
  return {"channels_last": cl, "strided": strided, "shifted": shifted}


@pytest.mark.parametrize("kind", ["channels_last", "strided", "shifted"])
def test_other_layouts_take_the_movedim_path(F, lib, monkeypatch, kind):
  C = 128
  x = _layout_variants(C)[kind]
  dy = _cf(tuple(x.shape[:1]) + tuple(x.shape[2:]), C, 14)
  gamma, beta = _params(C, 15)
  calls = _no_native_calls(F, monkeypatch)
  assert not F._gdn_native_cf(x, 1, 1, False, False)
  got = _run(F, x, gamma, beta, dy, FIXED[0], True)
  want = _run(F, x, gamma, beta, dy, FIXED[0], False)
  assert not calls
  for g, w in zip(got, want):
    assert_same(g, w)


def _allocated():
  torch.cuda.synchronize()
  return torch.cuda.memory_stats()["allocated_bytes.all.allocated"]


def _rounded(nbytes):
  return (nbytes + 511) // 512 * 512  # the caching allocator's block granularity


@pytest.mark.parametrize("C,dtype,cfg", [(128, torch.float32, FIXED[0]), (192, torch.bfloat16, FIXED[0]),
                                         (320, torch.float32, POW[1])])
def test_no_layout_copies(F, lib, C, dtype, cfg):
  """A covered call allocates its outputs, the library's workspace and parameter-sized temporaries, and nothing of
  the activations' size besides (the movedim path copies x, and dy, into channels-last tensors)."""
  inverse, rectify, alpha, epsilon, trainable = cfg
  x = _cf((4, 64, 64), C, 16, dtype, positive=True)
  dy = _cf((4, 64, 64), C, 17, dtype)
  gamma, beta = _params(C, 18)
  act = x.numel() * x.element_size()
  params = 4 * _rounded(4 * (C * C + C))  # dgamma, dbeta, dalpha / depsilon and slack
  torch.cuda.synchronize()
  a0 = _allocated()
  y = F.gdn_forward(x, gamma, beta, inverse, rectify, alpha, epsilon, trainable, trainable, channels_first=True)
  a1 = _allocated()
  assert y.is_contiguous() and a1 - a0 <= _rounded(act) + params
  n_items, spatial = x.shape[0], math.prod(x.shape[2:])
  ws = lib.lib().tfcb_gdn_backward_cf_workspace_bytes(n_items, spatial, C, {torch.float32: 0}.get(dtype, 2))
  if trainable:
    dx = F.gdn_backward_exponents(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, True, True,
                                  channels_first=True)[0]
  else:
    dx = F.gdn_backward(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, channels_first=True)[0]
  a2 = _allocated()
  assert dx.is_contiguous() and a2 - a1 <= _rounded(act) + _rounded(ws) + params
  assert act > params  # the bound is tight enough to see one more activation-sized buffer


def _stack(C, seed, data_format, trainable):
  from compression_b200.gdn import GDN
  torch.manual_seed(seed)
  conv1 = torch.nn.Conv2d(3, C, 5, padding=2)
  conv2 = torch.nn.Conv2d(C, C, 3, padding=1)
  extra = dict(alpha_parameter=None, epsilon_parameter=None) if trainable else {}
  gdn = GDN(data_format=data_format, **extra)
  igdn = GDN(inverse=True, data_format=data_format, **extra)
  return torch.nn.ModuleList([conv1, gdn, conv2, igdn]).cuda()


def _forward(layers, x, channels_first, outputs):
  conv1, gdn, conv2, igdn = layers
  h = conv1(x)
  for conv, norm in ((conv2, gdn), (None, igdn)):
    if channels_first:
      h = norm(h)
    else:
      # the same layer on NHWC, moved back to a contiguous NCHW tensor for the convolution; its dx reaches the
      # convolution as a contiguous NCHW gradient too, as the native path's does (cuDNN's weight gradient depends on
      # the gradient's strides)
      if h.requires_grad:
        h.register_hook(lambda g: g.contiguous())
      h = norm(h.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2).contiguous()
    outputs.append(h)
    if conv is not None:
      h = conv(h)
  return h


@pytest.mark.parametrize("trainable", [False, True])
def test_module_gradients_equal_the_channels_last_formulation(F, lib, trainable):
  det, bench = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
  torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
  try:
    C = 128
    g = torch.Generator().manual_seed(19)
    x0 = torch.randn(2, 3, 24, 20, generator=g).cuda()
    results = []
    for cf in (True, False):
      layers = _stack(C, 20, "channels_first" if cf else "channels_last", trainable)
      with torch.no_grad():  # the same GDN parameters in both stacks, away from their initial values
        layers[1].build((1, C, 1, 1) if cf else (1, 1, 1, C), device="cuda")
        layers[3].build((1, C, 1, 1) if cf else (1, 1, 1, C), device="cuda")
        for k, p in enumerate(layers.parameters()):
          p.add_(0.01 * torch.sin(torch.arange(p.numel(), device="cuda", dtype=p.dtype).view(p.shape) + k).abs())
      x = x0.clone().requires_grad_(True)
      outs = []
      loss = _forward(layers, x, cf, outs).square().mean()
      loss.backward()
      results.append((loss, x.grad, [p.grad for p in layers.parameters()], outs))
    (l_cf, gx_cf, gp_cf, o_cf), (l_cl, gx_cl, gp_cl, _) = results
    assert all(o.is_contiguous() for o in o_cf)
    assert_same(l_cf, l_cl)
    assert_same(gx_cf, gx_cl)
    assert len(gp_cf) == len(gp_cl) == 8 + (4 if trainable else 0)
    for a, b in zip(gp_cf, gp_cl):
      assert_same(a, b)
  finally:
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = det, bench


def test_module_takes_one_library_call_per_direction(F, lib):
  from compression_b200.gdn import GDN
  C = 192
  layer = GDN(data_format="channels_first")
  x = _cf((2, 16, 16), C, 21).requires_grad_(True)
  layer.build(x.shape, device="cuda")
  n0 = lib.launch_count()
  y = layer(x)
  n1 = lib.launch_count()
  y.backward(torch.ones_like(y))
  n2 = lib.launch_count()
  assert y.is_contiguous() and x.grad.is_contiguous()
  assert n1 - n0 == 1 and n2 - n1 == 4  # the forward kernel; dx, dgamma and the two reductions


def test_accuracy_against_the_float64_oracle(F):
  from oracle import gdn_oracle
  C = 192
  x, dy = _cf((2, 33, 17), C, 22), _cf((2, 33, 17), C, 23)
  gamma, beta = _params(C, 24)
  y = F.gdn_forward(x, gamma, beta, channels_first=True)
  dx, dg, db = F.gdn_backward(x, gamma, beta, dy, channels_first=True)
  xl, dyl = x.movedim(1, -1).reshape(-1, C).cpu(), dy.movedim(1, -1).reshape(-1, C).cpu()
  want = gdn_oracle.gdn_reference(xl, gamma, beta)
  got = y.movedim(1, -1).reshape(-1, C).double().cpu()
  assert ((got - want).abs() / (want.abs() + 1e-30)).max() < 1e-5
  wx, wg, wb = gdn_oracle.gdn_reference_grads(xl, gamma, beta, dyl)
  gx = dx.movedim(1, -1).reshape(-1, C)
  for g, w in ((gx, wx), (dg, wg), (db, wb)):
    assert (g.double().cpu() - w).abs().max() / w.abs().max() < 2e-5


@pytest.mark.parametrize("shape", [(0, 128, 8, 8), (3, 192, 0), (0, 192, 0, 4)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_empty_inputs(F, lib, shape, dtype):
  """N = 0 and S = 0 on the native path: nothing launched, the parameter gradients zero."""
  C = shape[1]
  x = torch.empty(shape, dtype=dtype, device="cuda")
  gamma, beta = _params(C, 25)
  trainable = dtype == torch.float32
  assert F._gdn_native_cf(x, 1, 1, False, False, dy=torch.empty_like(x))
  n0 = lib.launch_count()
  y = F.gdn_forward(x, gamma, beta, channels_first=True)
  dx, dg, db = F.gdn_backward(x, gamma, beta, torch.empty_like(x), channels_first=True)[:3]
  assert lib.launch_count() == n0
  assert y.shape == x.shape and dx.shape == x.shape and y.dtype == dtype
  assert torch.equal(dg, torch.zeros(C, C, device="cuda")) and torch.equal(db, torch.zeros(C, device="cuda"))
  if trainable:
    out = F.gdn_backward_exponents(x, gamma, beta, torch.empty_like(x), False, False, 1.3, 0.8, True, True,
                                   channels_first=True)
    assert torch.equal(out[3], torch.zeros(2, device="cuda")) and torch.equal(out[1], dg)


def test_dy_on_the_host_is_refused(F, lib):
  C = 128
  x, gamma, beta = _cf((2, 8, 8), C, 26), *_params(C, 27)
  dy = _cf((2, 8, 8), C, 28).cpu()
  n0 = lib.launch_count()
  for fn in (lambda: F.gdn_backward(x, gamma, beta, dy, channels_first=True),
             lambda: F.gdn_backward_exponents(x, gamma, beta, dy, alpha=1.2, epsilon=0.9, channels_first=True)):
    with pytest.raises(lib.InvalidArgumentError, match="dy is on cpu"):
      fn()
  assert lib.launch_count() == n0


def test_unaligned_beta_gives_the_channels_last_result(F, lib):
  """A beta view 4 bytes past a 16-byte boundary: the kernels read beta in pairs, so the call works on an aligned
  copy and stays native; the values are those of the channels-last tensor-core path with the same beta values."""
  C = 192
  x, dy = _cf((2, 9, 7), C, 29), _cf((2, 9, 7), C, 30)
  gamma, beta = _params(C, 31)
  buf = torch.empty(C + 1, device="cuda")
  shifted = buf[1:]
  shifted.copy_(beta)
  assert shifted.data_ptr() % 16 != 0
  for cfg in (FIXED[0], POW[1]):
    got = _run(F, x, gamma, shifted, dy, cfg, True)
    want = _run(F, x, gamma, beta, dy, cfg, False)
    assert got[0].is_contiguous() and got[1].is_contiguous()
    for g, w in zip(got, want):
      assert_same(g, w)
