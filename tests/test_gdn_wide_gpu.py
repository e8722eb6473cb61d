"""GDN / IGDN at 256 and 320 channels on the column-blocked tensor-core kernels (gdn_tc.cu, "Wide layers"): parity with
the fp64 oracle at the bounds of the C = 128 / 192 tests (test_gdn_gpu.py), proof from the profiler that the wide
kernels ran, bitwise reproducible parameter gradients, the fallback for misaligned inputs, and a training step of a
320-channel model."""
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from oracle import gdn_oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-5
WIDE = [256, 320]
# more 64-pixel tiles than one persistent wave of the forward / backward kernels at either width on an H100
# (132 SMs: 66 groups x 2 warpgroups at C = 256, 26 x 2 at C = 320)
BIG = 64 * 300 + 5


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


def _params(C, seed):
  g = torch.Generator().manual_seed(seed)
  gamma = 0.1 * torch.eye(C) + (0.02 * torch.randn(C, C, generator=g)).abs()
  beta = 1.0 + 0.5 * torch.rand(C, generator=g)
  return gamma, beta


def _x(n_pix, C, seed):
  g = torch.Generator().manual_seed(seed)
  scale = 0.05 + 3.95 * torch.rand(C, generator=g)
  return torch.randn(n_pix, C, generator=g) * scale


def _dy(n_pix, C, seed):
  return torch.randn(n_pix, C, generator=torch.Generator().manual_seed(seed))


def _relerr(got, want):
  want = want.double()
  return ((got.double().cpu() - want).abs() / (want.abs() + 1e-30)).max().item()


def _of_max(got, want):
  want = want.double()
  return (got.double().cpu() - want).abs().max().item() / want.abs().max().item()


def _kernels(fn):
  """Names of the CUDA kernels `fn` launches.  A profiler session can come back without any device events (seen on
  the first session of a process that had profiled before), so a session that recorded no kernel at all is taken
  again, at most twice."""
  fn()
  torch.cuda.synchronize()
  for _ in range(3):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      fn()
      torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
    if any(not n.startswith(("Memcpy", "Memset")) for n in names):
      break
  return names


@pytest.mark.parametrize("C", WIDE)
def test_closed_forms(F, C):
  x = torch.rand(77, C).cuda() - 0.5
  eye = (0.1 * torch.eye(C)).cuda()
  ones = torch.ones(C).cuda()
  xc = x.cpu()
  y = F.gdn_forward(x, eye, ones).cpu()
  assert torch.allclose(y, xc / (1 + 0.1 * xc.abs()), rtol=0, atol=1e-6)
  y = F.gdn_forward(x, eye, ones, inverse=True).cpu()
  assert torch.allclose(y, xc * (1 + 0.1 * xc.abs()), rtol=0, atol=1e-6)
  y = F.gdn_forward(x, eye, ones, rectify=True).cpu()
  xr = torch.relu(xc)
  assert torch.allclose(y, xr / (1 + 0.1 * xr), rtol=0, atol=1e-6)
  y = F.gdn_forward(x, eye, ones, alpha=2, epsilon=0.5).cpu()
  assert torch.allclose(y, xc / torch.sqrt(1 + 0.1 * xc**2), rtol=0, atol=1e-6)
  y = F.gdn_forward(x.abs() + 0.1, torch.ones(C, C).cuda(), torch.zeros(C).cuda()).cpu()
  xa = xc.abs() + 0.1
  assert torch.allclose(y, xa / xa.sum(-1, keepdim=True), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("C", WIDE)
@pytest.mark.parametrize("n_pix", [1, 63, 65, 3001, BIG])
@pytest.mark.parametrize("inverse", [False, True])
def test_forward_vs_fp64_oracle(F, C, n_pix, inverse):
  gamma, beta = _params(C, 4)
  x = _x(n_pix, C, 6)
  want = gdn_oracle.gdn_reference(x, gamma, beta, inverse=inverse)
  got = F.gdn_forward(x.cuda(), gamma.cuda(), beta.cuda(), inverse=inverse)
  assert _relerr(got, want) < RTOL


# (1, 1, True), (2, 0.5, False), (2, 1, False), (1, 0.5, False): the general (non-FAST) variant of the wide kernels
@pytest.mark.parametrize("alpha,epsilon,rectify", [(1, 1, True), (2, 0.5, False), (2, 1, False), (1, 0.5, False)])
@pytest.mark.parametrize("C", WIDE)
def test_forward_variants(F, C, alpha, epsilon, rectify):
  gamma, beta = _params(C, 5)
  x = _x(1000, C, 8)
  for inverse in (False, True):
    want = gdn_oracle.gdn_reference(x, gamma, beta, inverse, rectify, alpha, epsilon)
    got = F.gdn_forward(x.cuda(), gamma.cuda(), beta.cuda(), inverse, rectify, alpha, epsilon)
    mask = torch.isfinite(want)
    err = ((got.double().cpu() - want)[mask].abs() / (want[mask].abs() + 1e-6)).max().item()
    assert err < 2e-5


@pytest.mark.parametrize("C", WIDE)
@pytest.mark.parametrize("n_pix", [1, 65, 3001, BIG])
@pytest.mark.parametrize("inverse", [False, True])
def test_backward_vs_fp64_oracle(F, C, n_pix, inverse):
  gamma, beta = _params(C, 14)
  x = _x(n_pix, C, 16)
  dy = _dy(n_pix, C, 1)
  wx, wg, wb = gdn_oracle.gdn_reference_grads(x, gamma, beta, dy, inverse=inverse)
  dx, dg, db = F.gdn_backward(x.cuda(), gamma.cuda(), beta.cuda(), dy.cuda(), inverse=inverse)
  assert _of_max(dx, wx) < 2e-5
  assert _of_max(dg, wg) < 2e-5
  assert _of_max(db, wb) < 2e-5


@pytest.mark.parametrize("C", WIDE)
@pytest.mark.parametrize("alpha,epsilon,rectify", [(1, 1, True), (2, 0.5, False), (2, 1, False), (1, 0.5, False)])
def test_backward_variants(F, C, alpha, epsilon, rectify):
  gamma, beta = _params(C, 21)
  x = _x(700, C, 22)
  dy = _dy(700, C, 23)
  for inverse in (False, True):
    wx, wg, wb = gdn_oracle.gdn_reference_grads(x, gamma, beta, dy, inverse, rectify, alpha, epsilon)
    dx, dg, db = F.gdn_backward(x.cuda(), gamma.cuda(), beta.cuda(), dy.cuda(), inverse, rectify, alpha, epsilon)
    for got, want in ((dx, wx), (dg, wg), (db, wb)):
      want = torch.nan_to_num(want, nan=0.0, posinf=0.0, neginf=0.0)
      assert _of_max(got, want) < 3e-5


@pytest.mark.parametrize("C", WIDE)
def test_backward_at_a_million_pixels_vs_fp64_oracle(F, C):
  """dgamma / dbeta reduce over every pixel; one partial per group of column-block CTAs, so each partial covers
  C / NB times as many 64-pixel chunks as at C = 192.  Same bounds as the two-million-pixel test of test_gdn_gpu.py:
  within 1e-5 of the largest entry, and 5e-4 elementwise on entries >= 1 % of it."""
  n_pix = 1024 * 1024 + 77
  gamma, beta = _params(C, 31)
  x = _x(n_pix, C, 32)
  dy = _dy(n_pix, C, 33)
  wx, wg, wb = gdn_oracle.gdn_reference_grads(x, gamma, beta, dy)
  dx, dg, db = F.gdn_backward(x.cuda(), gamma.cuda(), beta.cuda(), dy.cuda())
  for name, got, want in (("dx", dx, wx), ("dgamma", dg, wg), ("dbeta", db, wb)):
    got, want = got.double().cpu(), want.double()
    scale = want.abs().max().item()
    err = (got - want).abs()
    big = want.abs() >= 1e-2 * scale
    of_max, rel = err.max().item() / scale, (err[big] / want.abs()[big]).max().item()
    print(f"GDN backward C={C} n_pix={n_pix} {name}: max err / max |want| = {of_max:.3g}, "
          f"max rel. err where |want| >= 1% of max = {rel:.3g}")
    assert of_max < 1e-5, (name, of_max)
    assert rel < 5e-4, (name, rel)
  want = gdn_oracle.gdn_reference(x, gamma, beta)
  got = F.gdn_forward(x.cuda(), gamma.cuda(), beta.cuda())
  assert _relerr(got, want) < RTOL


@pytest.mark.parametrize("C", WIDE)
@pytest.mark.parametrize("fast", [True, False])
def test_tensor_core_kernels_ran(F, C, fast):
  gamma, beta = (t.cuda() for t in _params(C, 2))
  x = _x(5000, C, 3).cuda()
  dy = _dy(5000, C, 4).cuda()
  kw = {} if fast else {"rectify": True}
  names = _kernels(lambda: F.gdn_forward(x, gamma, beta, **kw))
  assert any("gdn_tc_wide_fwd_kernel" in n for n in names), names
  assert not any("generic" in n for n in names), names
  names = _kernels(lambda: F.gdn_backward(x, gamma, beta, dy, **kw))
  for k in ("gdn_tc_wide_bwd_q_kernel", "gdn_tc_wide_bwd_dp_kernel", "gdn_tc_wide_dgamma_kernel"):
    assert any(k in n for n in names), (k, names)
  assert not any("generic" in n for n in names), names


@pytest.mark.parametrize("C", WIDE)
def test_parameter_gradients_are_reproducible(F, C):
  gamma, beta = (t.cuda() for t in _params(C, 7))
  x = _x(64 * 1000 + 13, C, 8).cuda()
  dy = _dy(x.shape[0], C, 9).cuda()
  a = F.gdn_backward(x, gamma, beta, dy)
  b = F.gdn_backward(x, gamma, beta, dy)
  assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
  assert torch.equal(a[0], b[0])


@pytest.mark.parametrize("C", WIDE)
def test_misaligned_input_takes_the_fallback(F, C):
  gamma, beta = _params(C, 10)
  n_pix = 300
  x = _x(n_pix, C, 11)
  dy = _dy(n_pix, C, 12)
  buf = torch.empty(n_pix * C + 1, device="cuda")
  buf[1:] = x.flatten().cuda()
  xv = buf[1:].view(n_pix, C)  # 4 bytes past a 16-byte boundary
  g, b = gamma.cuda(), beta.cuda()
  names = _kernels(lambda: F.gdn_forward(xv, g, b))
  assert not any("gdn_tc_wide" in n for n in names), names
  assert _relerr(F.gdn_forward(xv, g, b), gdn_oracle.gdn_reference(x, gamma, beta)) < RTOL
  wx, wg, wb = gdn_oracle.gdn_reference_grads(x, gamma, beta, dy)
  dx, dg, db = F.gdn_backward(xv, g, b, dy.cuda())
  assert _of_max(dx, wx) < 2e-5 and _of_max(dg, wg) < 2e-5 and _of_max(db, wb) < 2e-5


def test_bmshj2018_with_320_filters_trains_on_the_wide_kernels():
  from compression_b200 import models
  torch.manual_seed(0)
  m = models.BMSHJ2018Model(num_filters=320).build("cuda", patch=(64, 64))
  x = torch.rand(2, 64, 64, 3, generator=torch.Generator().manual_seed(1)).mul(255).cuda()

  def step():
    m.zero_grad(set_to_none=True)
    loss, _, _ = m(x, training=True)
    loss.backward()
    return loss

  names = _kernels(step)
  for k in ("gdn_tc_wide_fwd_kernel", "gdn_tc_wide_bwd_q_kernel", "gdn_tc_wide_bwd_dp_kernel",
            "gdn_tc_wide_dgamma_kernel"):
    assert any(k in n for n in names), k
  assert not any("gdn_bwd_generic" in n or "gdn_fwd_generic" in n for n in names)
  loss = step()
  assert torch.isfinite(loss)
  gdn = [(n, p) for n, p in m.named_parameters() if "gamma_parameter" in n or "beta_parameter" in n]
  assert len(gdn) == 2 * 6  # three GDN + three IGDN layers, gamma and beta each
  for n, p in gdn:
    assert p.grad is not None and torch.isfinite(p.grad).all(), n
