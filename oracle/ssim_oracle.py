"""A float64 torch restatement of tf.image.psnr, tf.image.ssim and tf.image.ssim_multiscale, written from TF's
documented algorithm (tensorflow/python/ops/image_ops_impl.py) and differentiable by autograd.  It is the yardstick
of compression_b200.image's kernels.

Images are [..., H, W, C] channels-last.  uint8 is converted as convert_image_dtype does (float32(x) *
float32(1/255)) before the widening to `dtype`, and so is max_val after a cast to the image dtype; float images are
cast to float32 first, then widened.  The window is the softmax of -(i^2 + j^2) / (2 sigma^2) over coordinates centred
at (size - 1) / 2, applied per channel with VALID padding as one 2-D convolution (no separability is assumed).  The
moments are formed on raw values, S(x^2) - mx^2, which float64 keeps exact enough for the gradient tests.  `dtype` and
`device` let the same graph run in float32 on a GPU as the eager baseline of tools/msssim_bench.py.

`ssim_stats(..., pool="float32")` is the tight reference of the statistics: TF pools in float64 (here) or float32
(in TF) with its own summation order, while the kernels store every pyramid level as a float32 sum in a fixed order,
so from scale 1 on, TF and the kernels filter planes that differ by float32 roundings.  The float32 option builds the kernels'
pyramid bit for bit and computes each scale's statistics in float64 from it, on values centred per plane.
"""
import math

import torch
import torch.nn.functional as F

MSSSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)


def convert(x, dtype=torch.float64):
  """convert_image_dtype(x, float32), then widened to `dtype`."""
  if x.dtype == torch.float64:  # already converted (a float64 leaf to differentiate against)
    return x.to(dtype)
  if x.dtype == torch.uint8:
    x = x.to(torch.float32) * torch.tensor(1 / 255, dtype=torch.float32)
  return x.to(torch.float32).to(dtype)


def convert_max_val(max_val, image_dtype):
  return float(convert(torch.tensor(max_val).to(image_dtype), torch.float64))


def window(size, sigma, dtype=torch.float64, device="cpu"):
  """[size, size]: softmax over the whole window of -0.5 (i^2 + j^2) / sigma^2."""
  coords = torch.arange(size, dtype=dtype, device=device) - (size - 1) / 2.0
  g = coords**2 * (-0.5 / sigma**2)
  g = g[None, :] + g[:, None]
  return torch.softmax(g.reshape(-1), 0).reshape(size, size)


def filter_valid(x, size, sigma):
  """Windowed mean of every channel of x [N, H, W, C] with VALID padding -> [N, H - size + 1, W - size + 1, C]."""
  C = x.shape[-1]
  k = window(size, sigma, x.dtype, x.device)[None, None].expand(C, 1, size, size)
  y = F.conv2d(x.permute(0, 3, 1, 2), k, groups=C)
  return y.permute(0, 2, 3, 1)


def _ssim_per_channel(x, y, max_val, size, sigma, k1, k2, shift=0.0):
  """(mean(l * cs), mean(cs)) over the valid positions, [N, C] each.  cs is formed from x - shift and y - shift (a
  constant per plane, [N, 1, 1, C]), on which the variances and the covariance are the same; shift = 0 is TF's graph."""
  c1 = (k1 * max_val)**2
  c2 = (k2 * max_val)**2
  x, y = x - shift, y - shift
  mx, my = filter_valid(x, size, sigma), filter_valid(y, size, sigma)
  num0 = mx * my * 2.0
  den0 = mx**2 + my**2
  luminance = ((mx + shift) * (my + shift) * 2.0 + c1) / ((mx + shift)**2 + (my + shift)**2 + c1)
  num1 = filter_valid(x * y, size, sigma) * 2.0
  den1 = filter_valid(x**2 + y**2, size, sigma)
  cs = (num1 - num0 + c2) / (den1 - den0 + c2)
  return (luminance * cs).mean((1, 2)), cs.mean((1, 2))


def check_size(shape, n_scales, size):
  h, w = shape[-3], shape[-2]
  for s in range(n_scales):
    if h < size or w < size:
      raise ValueError(f"scale {s} is {h}x{w}, smaller than filter_size={size}")
    h, w = (h + 1) // 2, (w + 1) // 2


def downsample(x):
  """End-pad an odd H or W by repeating the last row / column, then 2x2 average pool, [N, H, W, C]."""
  h, w = x.shape[1], x.shape[2]
  if h % 2 or w % 2:
    x = torch.cat([x, x[:, -1:]], 1) if h % 2 else x
    x = torch.cat([x, x[:, :, -1:]], 2) if w % 2 else x
  return 0.25 * (x[:, 0::2, 0::2] + x[:, 1::2, 0::2] + x[:, 0::2, 1::2] + x[:, 1::2, 1::2])


def downsample32(x):
  """The pyramid level the kernels store, from float32 x [N, H, W, C]: with the last row / column repeated where H or
  W is odd, ((x[2r, 2c] + x[2r, 2c + 1]) + (x[2r + 1, 2c] + x[2r + 1, 2c + 1])) * 0.25, each operation one float32
  rounding in that order."""
  assert x.dtype == torch.float32
  h, w = x.shape[1], x.shape[2]
  x = torch.cat([x, x[:, -1:]], 1) if h % 2 else x
  x = torch.cat([x, x[:, :, -1:]], 2) if w % 2 else x
  return ((x[:, 0::2, 0::2] + x[:, 0::2, 1::2]) + (x[:, 1::2, 0::2] + x[:, 1::2, 1::2])) * 0.25


def ssim_stats(img1, img2, max_val, n_scales=1, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03,
               dtype=torch.float64, pool="float64"):
  """[..., C, n_scales, 2]: (mean(cs), mean(l * cs)) per channel and scale, the statistics the kernels return.

  pool="float64" is TF's graph in `dtype` (the gradient reference).  pool="float32" computes what the kernels are
  given: filter_sigma, k1 and k2 rounded to float32 as the library's arguments are, the float32 images and the float32
  pyramid of `downsample32`, each level widened to float64 and centred on the mean of its two planes before the
  moments, so the float64 statistics keep their digits on bright content."""
  assert img1.shape == img2.shape and img1.dtype == img2.dtype and img1.dim() >= 3
  assert pool in ("float64", "float32")
  check_size(img1.shape, n_scales, filter_size)
  if pool == "float32":
    filter_sigma, k1, k2 = (float(torch.tensor(v, dtype=torch.float32)) for v in (filter_sigma, k1, k2))
  mv = convert_max_val(max_val, img1.dtype)
  batch = img1.shape[:-3]
  level = torch.float32 if pool == "float32" else dtype
  x = convert(img1, level).reshape((-1,) + tuple(img1.shape[-3:]))
  y = convert(img2, level).reshape((-1,) + tuple(img2.shape[-3:]))
  out = []
  for s in range(n_scales):
    if s:
      x, y = (downsample32(x), downsample32(y)) if pool == "float32" else (downsample(x), downsample(y))
    if pool == "float32":
      x64, y64 = x.double(), y.double()
      shift = 0.5 * (x64.mean((1, 2), keepdim=True) + y64.mean((1, 2), keepdim=True))
      lcs, cs = _ssim_per_channel(x64, y64, mv, filter_size, filter_sigma, k1, k2, shift)
    else:
      lcs, cs = _ssim_per_channel(x, y, mv, filter_size, filter_sigma, k1, k2)
    out.append(torch.stack([cs, lcs], -1))
  return torch.stack(out, -2).reshape(tuple(batch) + (img1.shape[-1], n_scales, 2))


def ssim(img1, img2, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, dtype=torch.float64):
  return ssim_stats(img1, img2, max_val, 1, filter_size, filter_sigma, k1, k2, dtype)[..., 0, 1].mean(-1)


def combine_multiscale(stats, power_factors=MSSSIM_WEIGHTS):
  v = torch.cat([stats[..., :-1, 0], stats[..., -1:, 1]], -1).relu()
  return torch.prod(v**torch.tensor(power_factors, dtype=v.dtype, device=v.device), -1).mean(-1)


def ssim_multiscale(img1, img2, max_val, power_factors=MSSSIM_WEIGHTS, filter_size=11, filter_sigma=1.5, k1=0.01,
                    k2=0.03, dtype=torch.float64):
  stats = ssim_stats(img1, img2, max_val, len(power_factors), filter_size, filter_sigma, k1, k2, dtype)
  return combine_multiscale(stats, power_factors)


def psnr(a, b, max_val, dtype=torch.float64):
  mv = convert_max_val(max_val, a.dtype)
  mse = ((convert(a, dtype) - convert(b, dtype))**2).mean((-3, -2, -1))
  return 20 * math.log(mv) / math.log(10.0) - 10 / math.log(10) * torch.log(mse)
