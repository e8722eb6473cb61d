"""CPU: argument checks of the SSIM entries (library and compression_b200.image), and the float64 oracle of
tf.image's metrics checked on its own: its window against scipy's Gaussian filter, exact cases and the pyramid."""
import math

import numpy as np
import pytest
import scipy.ndimage
import torch

from compression_b200 import _lib, image
from oracle import ssim_oracle as O

F32, F16, BF16, U8 = 0, 1, 2, 3


def _stats(dtype=F32, n=1, H=161, W=161, C=3, max_val=1.0, n_scales=5, filter_size=11, sigma=1.5, k1=0.01, k2=0.03):
  return _lib.lib().tfcb_ssim_stats(None, None, dtype, n, H, W, C, max_val, n_scales, filter_size, sigma, k1, k2, None,
                                    None, None)


@pytest.mark.parametrize("kw,match", [
    (dict(dtype=4), "dtype"),
    (dict(dtype=-1), "dtype"),
    (dict(H=160), "too small"),
    (dict(W=160), "too small"),
    (dict(H=10, W=10, n_scales=1), "too small"),
    (dict(filter_size=0), "filter_size"),
    (dict(filter_size=33), "filter_size"),
    (dict(sigma=0.0), "filter_sigma"),
    (dict(sigma=-1.5), "filter_sigma"),
    (dict(sigma=float("nan")), "filter_sigma"),
    (dict(n_scales=0), "n_scales"),
    (dict(n_scales=17), "n_scales"),
    (dict(n=-1), "shape"),
    (dict(C=0), "shape"),
    (dict(n=1 << 40, H=1 << 20, W=1 << 20, n_scales=1), "too large"),
    (dict(max_val=float("inf")), "max_val"),
])
def test_library_rejects_before_any_device_work(kw, match):
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_stats(**kw))


def test_library_accepts_the_boundary_and_then_wants_pointers():
  with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
    _lib.check(_stats(H=161, W=161))
  with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
    _lib.check(_stats(H=7, W=9, n_scales=1, filter_size=7, sigma=1.0))
  _lib.check(_stats(n=0))  # no images: nothing to do


def test_backward_rejects_uint8_and_bad_arguments():
  lib = _lib.lib()
  args = (1, 161, 161, 3, 1.0, 5, 11, 1.5, 0.01, 0.03, None, None, None, None, None)
  with pytest.raises(_lib.InvalidArgumentError, match="uint8"):
    _lib.check(lib.tfcb_ssim_stats_backward(None, None, U8, *args))
  with pytest.raises(_lib.InvalidArgumentError, match="too small"):
    _lib.check(lib.tfcb_ssim_stats_backward(None, None, F32, 1, 160, 161, 3, 1.0, 5, 11, 1.5, 0.01, 0.03, None, None,
                                            None, None, None))
  # both gradients NULL: nothing is asked for
  _lib.check(lib.tfcb_ssim_stats_backward(None, None, F16, *args))


def test_workspace_bytes():
  f = _lib.lib().tfcb_ssim_workspace_bytes
  assert f(F32, 2, 161, 161, 3, 5, 11) > 0
  assert f(U8, 1, 11, 11, 1, 1, 11) > 0
  for bad in [(4, 1, 161, 161, 3, 5, 11), (F32, 1, 160, 161, 3, 5, 11), (F32, 1, 161, 161, 3, 0, 11),
              (F32, 1, 161, 161, 3, 5, 0), (F32, 1, 161, 161, 0, 5, 11), (F32, -1, 161, 161, 3, 5, 11)]:
    assert f(*bad) == -1, bad


def test_image_rejects():
  a = torch.zeros(1, 161, 161, 3)
  with pytest.raises(image.InvalidArgumentError, match="shapes differ"):
    image.ssim_multiscale(a, torch.zeros(1, 161, 162, 3), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="dtypes differ"):
    image.ssim(a, a.half(), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="unsupported"):
    image.ssim(a.double(), a.double(), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="rank"):
    image.ssim(torch.zeros(16, 16), torch.zeros(16, 16), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="too small"):
    image.ssim_multiscale(torch.zeros(160, 200, 1), torch.zeros(160, 200, 1), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="filter_size"):
    image.ssim(a, a, 1.0, filter_size=0)
  with pytest.raises(image.InvalidArgumentError, match="filter_sigma"):
    image.ssim(a, a, 1.0, filter_sigma=0.0)
  with pytest.raises(image.InvalidArgumentError, match="filter_sigma"):
    image.ssim(a, a, 1.0, filter_sigma=-1.0)
  with pytest.raises(image.InvalidArgumentError, match="broadcast|shapes differ"):
    image.ssim(torch.zeros(2, 16, 16, 1), torch.zeros(1, 16, 16, 1), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="CUDA"):
    image.ssim_multiscale(torch.zeros(161, 161, 1), torch.zeros(161, 161, 1), 1.0)  # sizes pass, device does not
  with pytest.raises(image.InvalidArgumentError, match="rank"):
    image.psnr(torch.zeros(4, 4), torch.zeros(4, 4), 1.0)


def test_psnr_matches_the_oracle_on_the_host():
  g = torch.Generator().manual_seed(0)
  a = torch.randint(0, 256, (2, 3, 20, 24, 3), generator=g, dtype=torch.uint8)
  b = torch.randint(0, 256, (2, 3, 20, 24, 3), generator=g, dtype=torch.uint8)
  got = image.psnr(a, b, 255)
  assert got.dtype == torch.float32 and got.shape == (2, 3)
  assert torch.allclose(got.double(), O.psnr(a, b, 255), atol=1e-4)
  x = a.float()
  assert torch.allclose(image.psnr(x, b.float(), 255).double(), O.psnr(x, b.float(), 255), atol=1e-4)
  assert torch.allclose(image.psnr(x, b.float(), 255), image.psnr(a, b, 255), atol=1e-4)


# ---- the oracle on its own -------------------------------------------------------------------------------------
@pytest.mark.parametrize("size,sigma", [(11, 1.5), (7, 1.0)])
def test_oracle_window_is_scipys_gaussian_filter_on_the_valid_interior(size, sigma):
  rng = np.random.default_rng(1)
  img = rng.random((37, 45, 2))
  got = O.filter_valid(torch.from_numpy(img)[None], size, sigma)[0].numpy()
  r = size // 2
  for c in range(2):
    want = scipy.ndimage.gaussian_filter(img[..., c], sigma=sigma, truncate=r / sigma)
    np.testing.assert_allclose(got[..., c], want[r:-r, r:-r], rtol=0, atol=1e-13)
  # and the 2-D softmax window is the outer product of the normalised 1-D Gaussian
  g = np.exp(-0.5 * (np.arange(size) - (size - 1) / 2)**2 / sigma**2)
  g /= g.sum()
  np.testing.assert_allclose(O.window(size, sigma).numpy(), np.outer(g, g), rtol=0, atol=1e-16)


def test_oracle_identical_images_give_exactly_one():
  g = torch.Generator().manual_seed(2)
  x = torch.rand(2, 170, 181, 3, generator=g)
  assert torch.equal(O.ssim(x, x, 1.0), torch.ones(2, dtype=torch.float64))
  assert torch.equal(O.ssim_multiscale(x, x, 1.0), torch.ones(2, dtype=torch.float64))
  u = (x * 255).to(torch.uint8)
  assert torch.equal(O.ssim_multiscale(u, u, 255), torch.ones(2, dtype=torch.float64))


def test_oracle_constant_images_by_hand():
  a, b, c1 = 0.2, 0.6, (0.01 * 1.0)**2
  x = torch.full((1, 170, 170, 1), a, dtype=torch.float32)
  y = torch.full((1, 170, 170, 1), b, dtype=torch.float32)
  a, b = float(np.float32(a)), float(np.float32(b))
  lum = (2 * a * b + c1) / (a * a + b * b + c1)  # the variances and the covariance vanish: cs = c2 / c2 = 1
  stats = O.ssim_stats(x, y, 1.0, n_scales=5)
  np.testing.assert_allclose(stats[0, 0, :, 0].numpy(), 1.0, rtol=0, atol=1e-12)
  np.testing.assert_allclose(stats[0, 0, :, 1].numpy(), lum, rtol=0, atol=1e-12)
  np.testing.assert_allclose(float(O.ssim(x, y, 1.0)), lum, rtol=0, atol=1e-12)
  np.testing.assert_allclose(float(O.ssim_multiscale(x, y, 1.0)), lum**0.1333, rtol=0, atol=1e-12)


def test_oracle_pads_odd_sizes_by_repetition_before_pooling():
  x = torch.arange(15, dtype=torch.float64).reshape(1, 3, 5, 1)
  got = O.downsample(x)[0, ..., 0]
  want = torch.tensor([[(0 + 1 + 5 + 6) / 4, (2 + 3 + 7 + 8) / 4, (4 + 9) / 2],
                       [(10 + 11) / 2, (12 + 13) / 2, 14.0]], dtype=torch.float64)
  assert torch.equal(got, want)
  assert O.downsample(torch.zeros(1, 4, 6, 2)).shape == (1, 2, 3, 2)


def test_oracle_size_boundary():
  O.check_size((161, 161, 3), 5, 11)
  with pytest.raises(ValueError):
    O.check_size((160, 161, 3), 5, 11)
  with pytest.raises(ValueError):
    O.check_size((161, 160, 3), 5, 11)
  O.check_size((160, 160, 3), 4, 11)
  assert math.isfinite(float(O.ssim(torch.rand(11, 11, 1), torch.rand(11, 11, 1), 1.0)))
