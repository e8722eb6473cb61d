"""GPU: compression_b200.image's SSIM / MS-SSIM kernels against the float64 oracle of tf.image's metrics (forward and
gradients), their determinism and launch counts, and the metrics on the models (evaluate, an MS-SSIM training step)."""
import math

import pytest
import torch

from compression_b200 import _lib, image, models
from oracle import ssim_oracle as O

pytestmark = pytest.mark.gpu

FWD_TOL = 1e-5
DB_TOL = 0.01
GRAD_TOL = 1e-4


def _content(shape, seed, flat=False):
  """float32 in [0, 1], a pair: smooth ramps plus noise, and a noisy copy of it; `flat` adds bright flat patches."""
  g = torch.Generator().manual_seed(seed)
  *batch, H, W, C = shape
  yy = torch.linspace(0, 1, H)[:, None, None]
  xx = torch.linspace(0, 1, W)[None, :, None]
  phase = torch.rand(tuple(batch) + (1, 1, C), generator=g)
  base = 0.5 + 0.3 * torch.sin(6.0 * xx + 4.0 * yy + 6.28 * phase) * torch.cos(3.0 * yy - 2.0 * xx)
  a = (base + 0.05 * torch.randn(shape, generator=g)).clamp(0, 1)
  if flat:
    a[..., H // 4:H // 2, W // 5:W // 2, :] = 0.98
    a[..., H // 2:, W // 2:, :] = 1.0
  b = (a + 0.04 * torch.randn(shape, generator=g)).clamp(0, 1)
  if flat:
    b[..., H // 4:H // 2, W // 5:W // 2, :] = 0.97
  return a, b


def _as(x, dtype, max_val):
  if dtype == torch.uint8:
    return torch.round(x * 255).to(torch.uint8)
  return (x * max_val).to(dtype)


FORWARD_CASES = [
    # (batch, H, W, C, dtype, max_val, flat)
    ((), 161, 161, 3, torch.float32, 1.0, False),
    ((2, 3), 177, 209, 3, torch.uint8, 255, False),
    ((2,), 177, 209, 1, torch.float16, 1.0, True),
    ((2,), 256, 256, 3, torch.bfloat16, 255, False),
    ((), 512, 768, 3, torch.float32, 255, True),
    ((3,), 256, 256, 1, torch.uint8, 1, True),
    ((2,), 161, 170, 3, torch.float32, 255, True),
]


@pytest.mark.parametrize("batch,H,W,C,dtype,max_val,flat", FORWARD_CASES)
def test_forward_matches_the_oracle(batch, H, W, C, dtype, max_val, flat):
  a, b = _content(batch + (H, W, C), H * W + C, flat)
  x, y = _as(a, dtype, max_val), _as(b, dtype, max_val)
  got_ms = image.ssim_multiscale(x.cuda(), y.cuda(), max_val)
  got_s = image.ssim(x.cuda(), y.cuda(), max_val)
  got_stats = image.ssim_stats(x.cuda(), y.cuda(), max_val, n_scales=5)
  assert got_ms.dtype == torch.float32 and got_ms.shape == batch and got_s.shape == batch
  want_stats = O.ssim_stats(x, y, max_val, n_scales=5)
  want_ms = O.combine_multiscale(want_stats)
  want_s = O.ssim(x, y, max_val)
  assert (got_stats.double().cpu() - want_stats).abs().max() <= FWD_TOL
  assert (got_ms.double().cpu() - want_ms).abs().max() <= FWD_TOL
  assert (got_s.double().cpu() - want_s).abs().max() <= FWD_TOL
  db = lambda m: -10 * torch.log10(1 - m.double().cpu())
  assert (db(got_ms) - db(want_ms)).abs().max() <= DB_TOL


@pytest.mark.parametrize("kw", [
    dict(power_factors=(0.2, 0.3, 0.5)),
    dict(filter_size=7, filter_sigma=1.0),
    dict(k1=0.02, k2=0.05),
    dict(power_factors=(0.5, 0.5), filter_size=7, filter_sigma=1.0, k1=0.03, k2=0.01),
])
def test_forward_options_match_the_oracle(kw):
  a, b = _content((2, 177, 209, 3), 7)
  got = image.ssim_multiscale(a.cuda(), b.cuda(), 1.0, **kw).double().cpu()
  want = O.ssim_multiscale(a, b, 1.0, **kw)
  assert (got - want).abs().max() <= FWD_TOL
  sk = {k: v for k, v in kw.items() if k != "power_factors"}
  got = image.ssim(a.cuda(), b.cuda(), 1.0, **sk).double().cpu()
  assert (got - O.ssim(a, b, 1.0, **sk)).abs().max() <= FWD_TOL


def test_identical_images_give_one():
  a, _ = _content((2, 177, 209, 3), 3, flat=True)
  x = a.cuda()
  assert torch.equal(image.ssim(x, x, 1.0).cpu(), torch.ones(2))
  assert torch.equal(image.ssim_multiscale(x, x, 1.0).cpu(), torch.ones(2))


def _grad_check(x, y, fn, oracle_fn, tol=GRAD_TOL):
  x1, y1 = x.cuda().requires_grad_(), y.cuda().requires_grad_()
  fn(x1, y1).sum().backward()
  x64, y64 = x.double().requires_grad_(), y.double().requires_grad_()
  oracle_fn(x64, y64).sum().backward()
  for got, want in ((x1.grad, x64.grad), (y1.grad, y64.grad)):
    assert got.dtype == x.dtype
    scale = want.abs().max()
    assert scale > 0
    assert (got.double().cpu() - want).abs().max() <= tol * scale


@pytest.mark.parametrize("shape,max_val,flat", [((2, 177, 209, 3), 1.0, False), ((1, 161, 170, 1), 255.0, True),
                                                ((2, 192, 192, 3), 255.0, False)])
def test_multiscale_gradients_match_the_oracle(shape, max_val, flat):
  a, b = _content(shape, 11, flat)
  _grad_check(a * max_val, b * max_val, lambda x, y: image.ssim_multiscale(x, y, max_val),
              lambda x, y: O.ssim_multiscale(x, y, max_val))


def test_single_scale_and_option_gradients_match_the_oracle():
  a, b = _content((2, 64, 80, 3), 12)
  _grad_check(a, b, lambda x, y: image.ssim(x, y, 1.0), lambda x, y: O.ssim(x, y, 1.0))
  kw = dict(power_factors=(0.2, 0.3, 0.5), filter_size=7, filter_sigma=1.0, k1=0.02, k2=0.05)
  a, b = _content((1, 161, 161, 3), 13)
  _grad_check(a, b, lambda x, y: image.ssim_multiscale(x, y, 1.0, **kw),
              lambda x, y: O.ssim_multiscale(x, y, 1.0, **kw))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_sixteen_bit_gradients_round_the_float32_gradient_once(dtype):
  a, b = _content((1, 177, 209, 3), 14)
  x, y = a.to(dtype), b.to(dtype)
  x16, y16 = x.cuda().requires_grad_(), y.cuda().requires_grad_()
  image.ssim_multiscale(x16, y16, 1.0).sum().backward()
  x32, y32 = x.float().cuda().requires_grad_(), y.float().cuda().requires_grad_()
  image.ssim_multiscale(x32, y32, 1.0).sum().backward()
  assert x16.grad.dtype == dtype
  assert torch.equal(x16.grad, x32.grad.to(dtype)) and torch.equal(y16.grad, y32.grad.to(dtype))


def test_only_requested_gradients_and_no_backward_without_grad():
  a, b = _content((1, 161, 161, 1), 15)
  x, y = a.cuda().requires_grad_(), b.cuda()
  image.ssim_multiscale(x, y, 1.0).sum().backward()
  assert x.grad is not None and y.grad is None
  n0 = _lib.launch_count()
  with torch.no_grad():
    image.ssim_multiscale(x, y, 1.0)
  n1 = _lib.launch_count()
  image.ssim_multiscale(a.cuda(), b.cuda(), 1.0)
  assert _lib.launch_count() - n1 == n1 - n0


def test_deterministic_and_batch_independent():
  a, b = _content((8, 177, 209, 3), 21, flat=True)
  x, y = a.cuda(), b.cuda()
  s1 = image.ssim_stats(x, y, 1.0, n_scales=5)
  s2 = image.ssim_stats(x, y, 1.0, n_scales=5)
  assert torch.equal(s1, s2)
  for i in (0, 5):
    assert torch.equal(image.ssim_stats(x[i:i + 1], y[i:i + 1], 1.0, n_scales=5), s1[i:i + 1])
  grads = []
  for xs, ys in ((x, y), (x, y), (x[5:6], y[5:6])):
    xg, yg = xs.clone().requires_grad_(), ys.clone().requires_grad_()
    image.ssim_multiscale(xg, yg, 1.0).sum().backward()
    grads.append((xg.grad, yg.grad))
  assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
  assert torch.equal(grads[2][0], grads[0][0][5:6]) and torch.equal(grads[2][1], grads[0][1][5:6])


def test_launch_count_does_not_depend_on_the_batch():
  a, b = _content((8, 177, 209, 3), 22)
  x, y = a.cuda(), b.cuda()
  counts = []
  for n in (1, 8):
    n0 = _lib.launch_count()
    image.ssim_multiscale(x[:n], y[:n], 1.0)
    counts.append(_lib.launch_count() - n0)
  assert counts[0] == counts[1] == 2 * 5  # per scale: the moments and a pool (none after the last), one reduction
  n0 = _lib.launch_count()
  image.ssim(x, y, 1.0)
  assert _lib.launch_count() - n0 == 2


def _image(h, w, seed):
  a, _ = _content((h, w, 3), seed)
  return torch.round(a * 255).to(torch.uint8)


def test_evaluate_on_bmshj2018_agrees_with_the_oracle():
  torch.manual_seed(2)
  m = models.BMSHJ2018Model(num_filters=24).build("cuda", patch=(64, 64)).fix_tables()
  x = _image(176, 200, 31)
  r = m.evaluate(x)
  tfci = m.compress_to_tfci(x)
  x_hat = m.decompress_from_tfci(tfci).cpu().float()
  xf = x.float()
  want_ms = float(O.ssim_multiscale(xf, x_hat, 255))
  assert abs(r["msssim"] - want_ms) <= FWD_TOL
  assert abs(r["msssim_db"] - (-10 * math.log10(1 - want_ms))) <= DB_TOL
  assert abs(r["psnr"] - float(O.psnr(xf, x_hat, 255))) <= 1e-4
  assert abs(r["mse"] - float(((xf - x_hat)**2).double().mean())) <= 1e-3 * max(1.0, r["mse"])
  assert r["bpp"] == len(tfci) * 8 / (176 * 200)


def test_bls2017_msssim_training_step():
  torch.manual_seed(3)
  m = models.BLS2017Model(num_filters=32).build("cuda")
  opt = torch.optim.Adam(m.parameters(), lr=1e-4)
  x = torch.stack([_image(192, 192, 40 + i) for i in range(4)]).cuda().float()
  lmbda = 100.0
  _, bpp, _ = m(x)
  x_hat = m._last_x_hat
  x_hat.retain_grad()
  msssim = image.ssim_multiscale(x, x_hat, 255)
  loss = bpp + lmbda * (1 - msssim.mean())
  opt.zero_grad()
  loss.backward()
  grads = [p.grad for p in m.parameters() if p.grad is not None]
  assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
  assert any(float(g.abs().max()) > 0 for g in grads)
  opt.step()
  # the synthesis output's gradient from the distortion term against float64 autograd of the oracle
  xh = x_hat.detach().cpu().double().requires_grad_()
  (lmbda * (1 - O.ssim_multiscale(x.cpu().double(), xh, 255).mean())).backward()
  scale = xh.grad.abs().max()
  assert (x_hat.grad.double().cpu() - xh.grad).abs().max() <= GRAD_TOL * scale
