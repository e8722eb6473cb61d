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

`metrics_ragged` evaluates a list of differently sized pairs, a dataset's rate-distortion point, with one launch per
kernel per scale (`tfcb_image_metrics_ragged`): PSNR and MS-SSIM per image on RGB, on Y' or as the 6:1:1 average over
Y'CbCr (`rgb_to_ycbcr`), the colour spaces the reference's published results use.  It has no gradient; a training
loss uses `ssim_multiscale`.
"""
import math

import numpy as np
import torch

from compression_b200 import _lib
from compression_b200._lib import InvalidArgumentError

__all__ = ["psnr", "ssim", "ssim_multiscale", "rgb_to_ycbcr", "metrics_ragged", "ssim_stats_ragged"]

_MSSSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.uint8: 3}
_COLORS = {"rgb": 0, "y": 1, "ycbcr": 2}  # TFCB_COLOR_*


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
  mse = torch.mean((_to_float(a) - _to_float(b))**2, dim=(-3, -2, -1))
  return _psnr_from_mse(mse, _max_val(max_val, a.dtype))


def _psnr_from_mse(mse, max_val):
  mv = torch.tensor(max_val, dtype=torch.float32, device=mse.device)
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
  return _multiscale_per_plane(stats, power_factors).mean(-1)


def _multiscale_per_plane(stats, power_factors):
  """prod_k relu(v_k) ** power_factors[k] of stats [..., P, n_scales, 2] -> [..., P]."""
  v = torch.cat([stats[..., :-1, 0], stats[..., -1:, 1]], dim=-1).relu()
  weights = torch.tensor(power_factors, dtype=torch.float32, device=v.device)
  return torch.prod(v**weights, dim=-1)


def rgb_to_ycbcr(x, max_val):
  """BT.601 full-range (JFIF) Y'CbCr of RGB images [..., 3] in any dtype and on any device, float32 [..., 3].

  In the images' units after `convert_image_dtype` (uint8 in [0, 1]), with m = max_val converted the same way:
    Y' = 0.299 R + 0.587 G + 0.114 B
    Cb = (128/255) m + (-0.168736 R - 0.331264 G + 0.5 B)
    Cr = (128/255) m + (0.5 R - 0.418688 G - 0.081312 B)
  Each product and sum is one float32 operation, left to right; the kernels of `metrics_ragged` compute the same bits.
  At max_val = 255 on [0, 255] data this is JFIF exactly: white is (255, 128, 128).
  """
  if not isinstance(x, torch.Tensor) or x.dtype not in _DTYPES:
    raise InvalidArgumentError("rgb_to_ycbcr needs a uint8, float16, bfloat16 or float32 tensor")
  if x.dim() < 1 or x.shape[-1] != 3:
    raise InvalidArgumentError(f"rgb_to_ycbcr needs [..., 3], received shape {tuple(x.shape)}")
  off = torch.tensor(128 / 255, dtype=torch.float32) * torch.tensor(_max_val(max_val, x.dtype), dtype=torch.float32)
  r, g, b = _to_float(x).unbind(-1)
  y = 0.299 * r + 0.587 * g + 0.114 * b
  cb = off + (-0.168736 * r - 0.331264 * g + 0.5 * b)
  cr = off + (0.5 * r - 0.418688 * g - 0.081312 * b)
  return torch.stack([y, cb, cr], -1)


def _check_lists(originals, reconstructions, color):
  if color not in _COLORS:
    raise InvalidArgumentError(f"unknown color {color!r}: expected one of {sorted(_COLORS)}")
  if len(originals) != len(reconstructions):
    raise InvalidArgumentError(f"{len(originals)} originals but {len(reconstructions)} reconstructions")
  for i, (a, b) in enumerate(zip(originals, reconstructions)):
    if not (isinstance(a, torch.Tensor) and isinstance(b, torch.Tensor)):
      raise InvalidArgumentError(f"pair {i}: images must be tensors")
    if a.dtype != b.dtype or a.dtype != originals[0].dtype:
      raise InvalidArgumentError(f"pair {i}: dtypes {a.dtype} and {b.dtype}, the list is {originals[0].dtype}")
    if a.dtype not in _DTYPES:
      raise InvalidArgumentError(f"pair {i}: unsupported dtype {a.dtype}: expected uint8, float16, bfloat16 or float32")
    if a.dim() != 3 or a.shape != b.shape or a.shape[-1] != originals[0].shape[-1]:
      raise InvalidArgumentError(f"pair {i}: shapes {tuple(a.shape)} and {tuple(b.shape)}, expected [H, W, C] each "
                                 f"with the list's C")
  for i, (a, b) in enumerate(zip(originals, reconstructions)):
    if not (a.is_cuda and b.is_cuda) or a.device != originals[0].device or b.device != a.device:
      raise InvalidArgumentError(f"pair {i}: metrics_ragged needs CUDA tensors on one device")


def ssim_stats_ragged(originals, reconstructions, max_val, color="rgb", n_scales=5, filter_size=11, filter_sigma=1.5,
                      k1=0.01, k2=0.03):
  """The statistics of `ssim_stats` for lists of pairs [H_i, W_i, C] of their own sizes, in one launch per kernel per
  scale: (float32 stats [n, P, n_scales, 2], float32 mse [n, P]), P planes per image: the C channels for "rgb", Y' for
  "y" (C = 3), Y', Cb, Cr for "ycbcr" (C = 3).  For "rgb", stats[i] is `ssim_stats` of pair i bit for bit."""
  originals, reconstructions = list(originals), list(reconstructions)
  _check_lists(originals, reconstructions, color)
  n = len(originals)
  P = {"rgb": int(originals[0].shape[-1]) if n else 3, "y": 1, "ycbcr": 3}[color]
  if n == 0:
    return torch.empty(0, P, n_scales, 2), torch.empty(0, P)
  dtype, device, C = originals[0].dtype, originals[0].device, int(originals[0].shape[-1])
  a = torch.cat([x.reshape(-1) for x in originals])
  b = torch.cat([x.reshape(-1) for x in reconstructions])
  heights = np.array([x.shape[0] for x in originals], dtype=np.int64)
  widths = np.array([x.shape[1] for x in originals], dtype=np.int64)
  offsets = np.concatenate([[0], np.cumsum(heights * widths * C)]).astype(np.int64)
  lib = _lib.lib()
  args = (_DTYPES[dtype], n, offsets.ctypes.data, heights.ctypes.data, widths.ctypes.data, C, _COLORS[color],
          _max_val(max_val, dtype), n_scales, int(filter_size), float(filter_sigma), float(k1), float(k2))
  nbytes = lib.tfcb_image_metrics_ragged_workspace_bytes(args[0], n, heights.ctypes.data, widths.ctypes.data, C,
                                                         _COLORS[color], n_scales, int(filter_size))
  if nbytes < 0:  # the entry reports which argument it rejects
    _lib.check(lib.tfcb_image_metrics_ragged(None, None, *args, None, None, None, None))
    raise InvalidArgumentError("metrics_ragged: arguments rejected by tfcb_image_metrics_ragged_workspace_bytes")
  stats = torch.empty((n, P, n_scales, 2), dtype=torch.float32, device=device)
  mse = torch.empty((n, P), dtype=torch.float32, device=device)
  ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
  _lib.check(lib.tfcb_image_metrics_ragged(a.data_ptr(), b.data_ptr(), *args, stats.data_ptr(), mse.data_ptr(),
                                           ws.data_ptr(), _stream(device)))
  return stats, mse


def metrics_ragged(originals, reconstructions, max_val, color="rgb", power_factors=_MSSSIM_WEIGHTS, filter_size=11,
                   filter_sigma=1.5, k1=0.01, k2=0.03):
  """Per-image `mse`, `psnr`, `msssim` and `msssim_db` = -10 log10(1 - msssim) of two equal-length lists of CUDA
  images [H_i, W_i, C] (pair i of one size, one dtype and C for the list), as a dict of float32 [n] tensors.

  color "rgb": `psnr` and `ssim_multiscale` of each pair (msssim bit for bit); "y": the same on the Y' plane; "ycbcr":
  (6 v_Y + v_Cb + v_Cr) / 8 of the per-plane mse, psnr and msssim.  Y'CbCr as `rgb_to_ycbcr`.  The lists are packed
  into one buffer per side; argument errors raise InvalidArgumentError before the library is called.  An empty list
  gives empty tensors on the CPU."""
  if len(power_factors) < 1:
    raise InvalidArgumentError("power_factors must not be empty")
  stats, mse = ssim_stats_ragged(originals, reconstructions, max_val, color, len(power_factors), filter_size,
                                 filter_sigma, k1, k2)
  msssim = _multiscale_per_plane(stats, power_factors)
  mv = _max_val(max_val, originals[0].dtype) if len(originals) else 1.0
  if color == "rgb":
    mse = mse.double().mean(-1).float()  # every plane has the image's pixel count
    psnr = _psnr_from_mse(mse, mv)
    msssim = msssim.mean(-1)
  elif color == "y":
    mse, psnr, msssim = mse[:, 0], _psnr_from_mse(mse[:, 0], mv), msssim[:, 0]
  else:
    mse, psnr, msssim = ((6 * v[:, 0] + v[:, 1] + v[:, 2]) / 8 for v in (mse, _psnr_from_mse(mse, mv), msssim))
  msssim_db = -10. * torch.log(1 - msssim) / math.log(10.)
  return {"mse": mse, "psnr": psnr, "msssim": msssim, "msssim_db": msssim_db}
