"""A float64 torch restatement of the BT.601 full-range (JFIF) RGB -> Y'CbCr conversion that
compression_b200.image.rgb_to_ycbcr and the kernels of tfcb_image_metrics_ragged apply, written from the JFIF
formulas (ITU-T T.871, section 7): the yardstick of both, beside oracle/ssim_oracle.py.

Images are [..., 3] in the units of `ssim_oracle.convert` (uint8 in [0, 1]); m is max_val converted the same way:
  Y' = 0.299 R + 0.587 G + 0.114 B
  Cb = (128/255) m - 0.168736 R - 0.331264 G + 0.5 B
  Cr = (128/255) m + 0.5 R - 0.418688 G - 0.081312 B
"""
import torch

from oracle import ssim_oracle as O

MATRIX = ((0.299, 0.587, 0.114), (-0.168736, -0.331264, 0.5), (0.5, -0.418688, -0.081312))
OFFSET = (0.0, 128 / 255, 128 / 255)


def rgb_to_ycbcr(x, max_val):
  """float64 [..., 3]."""
  m = O.convert_max_val(max_val, x.dtype)
  x = O.convert(x, torch.float64)
  A = torch.tensor(MATRIX, dtype=torch.float64)
  return x @ A.T + torch.tensor(OFFSET, dtype=torch.float64) * m


def planes(x, color, max_val):
  """The planes the metrics are taken on, float64 [..., P]: the channels ("rgb"), Y' ("y") or Y'CbCr ("ycbcr")."""
  if color == "rgb":
    return O.convert(x, torch.float64)
  ycc = rgb_to_ycbcr(x, max_val)
  return ycc[..., :1] if color == "y" else ycc
