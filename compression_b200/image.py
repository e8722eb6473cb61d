"""Image quality metrics with `tf.image`'s semantics: `psnr`, `ssim` and `ssim_multiscale`.

The model scripts judge a compressed image with these (models/bls2017.py:293-296): PSNR and MS-SSIM on the float32
image against its reconstruction, both in [0, 255] with `max_val=255`.

`ssim` / `ssim_multiscale` run on the fused kernels of `tfcb_ssim_stats` (include/tfcb200.h): per image, channel and
scale they return mean(cs) and mean(l * cs), and the combination TF's graph applies (ReLU, pow, prod, the mean over
channels) runs here in float32 torch on those few values.  Autograd through that combination gives the gradient of the
statistics and `tfcb_ssim_stats_backward` turns it into gradients of both images, so an MS-SSIM loss such as
`bpp + lmbda * (1 - ssim_multiscale(x, x_hat, 255))` trains without an eager graph of convolutions.

Inputs are `[..., H, W, C]` channels-last with identical shapes (no broadcasting of batch dimensions), uint8, float16,
bfloat16 or float32.  uint8 is converted as `convert_image_dtype` does, float32(x) * float32(1/255), and so is
`max_val` after a cast to the image dtype (255 becomes 1.0); float images and `max_val` are used as float32.  The
results are float32 with shape `[...]`.  `ssim` / `ssim_multiscale` need contiguous CUDA tensors; `psnr` is a single
reduction in torch and runs on any device.
"""
import math

import torch

from compression_b200 import _lib
from compression_b200._lib import InvalidArgumentError

__all__ = ["psnr", "ssim", "ssim_multiscale"]

_MSSSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.uint8: 3}


def _check_pair(img1, img2):
  if not (isinstance(img1, torch.Tensor) and isinstance(img2, torch.Tensor)):
    raise InvalidArgumentError("images must be tensors")
  if img1.dtype != img2.dtype:
    raise InvalidArgumentError(f"image dtypes differ: {img1.dtype} and {img2.dtype}")
  if img1.dtype not in _DTYPES:
    raise InvalidArgumentError(f"unsupported image dtype {img1.dtype}: expected uint8, float16, bfloat16 or float32")
  if img1.dim() < 3:
    raise InvalidArgumentError(f"images must be [..., H, W, C], received rank {img1.dim()}")
  if img1.shape != img2.shape:
    raise InvalidArgumentError(f"image shapes differ: {tuple(img1.shape)} and {tuple(img2.shape)}")


def _to_float(x):
  """convert_image_dtype(x, float32)."""
  if x.dtype == torch.uint8:
    return x.to(torch.float32) * torch.tensor(1 / 255, dtype=torch.float32)
  return x.to(torch.float32)


def _max_val(max_val, dtype):
  """cast(max_val, dtype) then convert_image_dtype(., float32), as a Python float."""
  return float(_to_float(torch.tensor(max_val).to(dtype)))


def psnr(a, b, max_val):
  """tf.image.psnr: 20 log10(max_val) - 10 log10(mean((a - b)^2) over the last three dimensions), float32 [...]."""
  _check_pair(a, b)
  mv = torch.tensor(_max_val(max_val, a.dtype), dtype=torch.float32, device=a.device)
  mse = torch.mean((_to_float(a) - _to_float(b))**2, dim=(-3, -2, -1))
  return 20 * torch.log(mv) / math.log(10.0) - torch.tensor(10 / math.log(10), dtype=torch.float32) * torch.log(mse)


def _check_args(img1, img2, n_scales, filter_size, filter_sigma):
  _check_pair(img1, img2)
  if int(filter_size) != filter_size or filter_size < 1:
    raise InvalidArgumentError(f"filter_size must be a positive integer, got {filter_size}")
  if not filter_sigma > 0 or not math.isfinite(filter_sigma):
    raise InvalidArgumentError(f"filter_sigma must be positive and finite, got {filter_sigma}")
  h, w = int(img1.shape[-3]), int(img1.shape[-2])
  for s in range(n_scales):
    if h < filter_size or w < filter_size:
      raise InvalidArgumentError(f"image {img1.shape[-3]}x{img1.shape[-2]} too small for {n_scales} scale(s) with "
                                 f"filter_size={filter_size}: scale {s} is {h}x{w}")
    h, w = (h + 1) // 2, (w + 1) // 2
  if not (img1.is_cuda and img2.is_cuda):
    raise InvalidArgumentError("ssim / ssim_multiscale need CUDA tensors")
  if img1.device != img2.device:
    raise InvalidArgumentError(f"images on different devices: {img1.device} and {img2.device}")
  if not (img1.is_contiguous() and img2.is_contiguous()):
    raise InvalidArgumentError("images must be contiguous channels-last tensors")


class _Call:
  """The arguments of one tfcb_ssim_stats call, shared by its forward and backward."""

  def __init__(self, img, max_val, n_scales, filter_size, filter_sigma, k1, k2):
    *batch, H, W, C = img.shape
    self.batch = tuple(batch)
    self.n = math.prod(batch)
    self.shape = (_DTYPES[img.dtype], self.n, H, W, C)
    self.params = (_max_val(max_val, img.dtype), n_scales, int(filter_size), float(filter_sigma), float(k1), float(k2))
    self.n_scales = n_scales
    self.C = C

  def workspace(self, device):
    nbytes = _lib.lib().tfcb_ssim_workspace_bytes(*self.shape, self.n_scales, self.params[2])
    if nbytes < 0:
      raise InvalidArgumentError("ssim: arguments rejected by tfcb_ssim_workspace_bytes")
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)


def _stream(device):
  return torch.cuda.current_stream(device).cuda_stream


class _SsimStats(torch.autograd.Function):

  @staticmethod
  def forward(ctx, img1, img2, call):
    stats = torch.empty(call.batch + (call.C, call.n_scales, 2), dtype=torch.float32, device=img1.device)
    ws = call.workspace(img1.device)
    _lib.check(_lib.lib().tfcb_ssim_stats(img1.data_ptr(), img2.data_ptr(), *call.shape, *call.params,
                                          stats.data_ptr(), ws.data_ptr(), _stream(img1.device)))
    ctx.call = call
    ctx.save_for_backward(img1, img2)
    return stats

  @staticmethod
  def backward(ctx, g_stats):
    img1, img2 = ctx.saved_tensors
    call = ctx.call
    d1 = torch.empty_like(img1) if ctx.needs_input_grad[0] else None
    d2 = torch.empty_like(img2) if ctx.needs_input_grad[1] else None
    g = g_stats.to(torch.float32).contiguous()
    ws = call.workspace(img1.device)
    _lib.check(_lib.lib().tfcb_ssim_stats_backward(
        img1.data_ptr(), img2.data_ptr(), *call.shape, *call.params, g.data_ptr(),
        None if d1 is None else d1.data_ptr(), None if d2 is None else d2.data_ptr(), ws.data_ptr(),
        _stream(img1.device)))
    return d1, d2, None


def ssim_stats(img1, img2, max_val, n_scales=1, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03):
  """float32 [..., C, n_scales, 2]: (mean(cs), mean(l * cs)) of every channel at every scale; differentiable in both
  float images."""
  _check_args(img1, img2, n_scales, filter_size, filter_sigma)
  call = _Call(img1, max_val, n_scales, filter_size, filter_sigma, k1, k2)
  return _SsimStats.apply(img1, img2, call)


def ssim(img1, img2, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03):
  """tf.image.ssim: the mean over channels of mean(l * cs), float32 [...]."""
  stats = ssim_stats(img1, img2, max_val, 1, filter_size, filter_sigma, k1, k2)
  return stats[..., 0, 1].mean(-1)


def ssim_multiscale(img1, img2, max_val, power_factors=_MSSSIM_WEIGHTS, filter_size=11, filter_sigma=1.5, k1=0.01,
                    k2=0.03):
  """tf.image.ssim_multiscale: prod_k relu(v_k) ** power_factors[k] per channel (v_k = mean(cs) at the finer scales,
  mean(l * cs) at the coarsest), averaged over channels, float32 [...]."""
  n_scales = len(power_factors)
  if n_scales < 1:
    raise InvalidArgumentError("power_factors must not be empty")
  stats = ssim_stats(img1, img2, max_val, n_scales, filter_size, filter_sigma, k1, k2)
  v = torch.cat([stats[..., :-1, 0], stats[..., -1:, 1]], dim=-1).relu()
  weights = torch.tensor(power_factors, dtype=torch.float32, device=v.device)
  return torch.prod(v**weights, dim=-1).mean(-1)
