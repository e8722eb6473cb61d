"""Cases shared by tests/test_ssim_paths_cpu.py and tests/test_ssim_paths_gpu.py: the filter sizes, sigmas, image
sizes at the tile seams, pyramid depths, channel counts, plane counts and ragged lists that reach each path of
csrc/ssim.cu, the content that stresses its precision, and the bound the statistics are held to."""
import numpy as np
import torch

from oracle import ssim_oracle as O

FWD_TILE = 32  # ssim_fwd_kernel's output tile
BWD_TILE = 16  # ssim_bwd_kernel's input tile
MAX_PLANE_BLOCKS = 65535  # the backward's gridDim.y; more planes loop
MAX_FILTER, MAX_SCALES = 32, 16

FILTERS = [1, 2, 3, 8, 16, 31, 32]
SIGMAS = [0.5, 1.5, 8.0, 100.0]
# make_window's taps all underflowed to 0 (a 0 / 0 window) at even F below sigma ~ 0.0129
EVEN_F_TINY_SIGMA = [(2, 0.01), (8, 0.01)]

# (filter_size, n_scales, H, W): pools and pool adjoints down to 1x1, 2x2 and 3x3 levels of odd and even sizes
DEEP = [(1, 16, 37, 41), (2, 8, 130, 140), (3, 7, 131, 129)]

CHANNELS = [2, 4, 7]
BATCH_SHAPE = (2, 3)

# N * C = 2 * 65535 + 3 planes of 11x11: the backward's plane loop runs three times; a few distinct pairs tiled along N
MANY_PLANES = (43691, 11, 11, 3)
MANY_PLANES_PAIRS = 5

RAGGED_CHANNELS = [1, 2, 4]
RAGGED_SIZES = [(161, 161), (177, 209), (192, 170)]  # F = 11, S = 5
# Y' / Y'CbCr at F = 11, S = 5: the smallest size, then valid sizes 160, 161, 159 (0, 1, 31 mod 32)
LUMA_SIZES = [(161, 161), (170, 176), (171, 177), (169, 175), (176, 170)]
LONG_F, LONG_S = 3, 3


def min_size(F, S):
  """The smallest H (or W) whose scale S - 1 is still >= F."""
  return (F - 1) * 2**(S - 1) + 1


def pyramid(h, S):
  out = [h]
  for _ in range(S - 1):
    out.append((out[-1] + 1) // 2)
  return out


def _at_least(lo, r, m):
  """The smallest v >= lo with v mod m == r."""
  return lo + (r - lo) % m


def seam_sizes(F):
  """(H, W) at scale 0 for filter F: H - F + 1 = 32, 33, 31 (forward tile residues 0, 1, 31) with W the smallest
  size >= F at 0, 1, 15 mod 16 (backward tile residues), and each pair transposed."""
  out = []
  for ho, rb in ((FWD_TILE, 0), (FWD_TILE + 1, 1), (FWD_TILE - 1, BWD_TILE - 1)):
    h, w = F - 1 + ho, _at_least(F, rb, BWD_TILE)
    out += [(h, w), (w, h)]
  return out


def long_list_sizes():
  """At least 200 tiny items from the smallest size LONG_F / LONG_S allow, of mixed shapes, with three 512x768 items
  between them."""
  m = min_size(LONG_F, LONG_S)
  sizes = [(m + i % 7, m + (3 * i) % 11) for i in range(204)]
  for k in (40, 117, 181):
    sizes[k] = (512, 768)
  return sizes


def power_factors(S):
  """Positive weights summing to 1, not the defaults."""
  w = np.arange(1, S + 1, dtype=np.float64)
  return tuple(float(v) for v in w / w.sum())


def content(shape, seed, max_val=1.0):
  """float32 pair [..., H, W, C] in [0, max_val]: smooth ramps plus noise, and a noisy copy."""
  g = torch.Generator().manual_seed(seed)
  *batch, H, W, C = shape
  yy = torch.linspace(0, 1, H)[:, None, None]
  xx = torch.linspace(0, 1, W)[None, :, None]
  phase = torch.rand(tuple(batch) + (1, 1, C), generator=g)
  base = 0.5 + 0.3 * torch.sin(6.0 * xx + 4.0 * yy + 6.28 * phase) * torch.cos(3.0 * yy - 2.0 * xx)
  a = (base + 0.05 * torch.randn(shape, generator=g)).clamp(0, 1)
  b = (a + 0.04 * torch.randn(shape, generator=g)).clamp(0, 1)
  return a * max_val, b * max_val


def seam_patches(shape, seed, max_val=1.0):
  """content() with bright flat patches (0.98 / 0.97 and 1.0 / 1.0 of max_val) straddling the forward and backward
  tile seams, every forward and backward tile's first pixel dark (the kernels' shift far from the patch), and a
  quarter of the other pixels at exactly 0 or max_val in both images."""
  a, b = content(shape, seed)
  H, W = shape[-3], shape[-2]
  clip = torch.rand(shape, generator=torch.Generator().manual_seed(seed + 1))
  a, b = (torch.where(clip < 0.12, 0.0, torch.where(clip > 0.88, 1.0, t)) for t in (a, b))
  a[..., H // 4:3 * H // 4, W // 5:W // 2, :] = 0.98
  b[..., H // 4:3 * H // 4, W // 5:W // 2, :] = 0.97
  a[..., H // 3:, W // 2:, :] = 1.0
  b[..., H // 3:, W // 2:, :] = 1.0
  a[..., ::BWD_TILE, ::BWD_TILE, :] = 0.0  # the forward tiles' first pixels are among these
  b[..., ::BWD_TILE, ::BWD_TILE, :] = 0.0
  return a * max_val, b * max_val


def as_dtype(x, dtype, max_val):
  """x in [0, max_val] as `dtype`; uint8 holds round(255 x / max_val)."""
  if dtype == torch.uint8:
    return torch.round(x / max_val * 255).to(torch.uint8)
  return x.to(dtype)


# ---- the statistics bound ---------------------------------------------------------------------------------------
def ulp32(r):
  """np.spacing(float32(|r|)) in float64."""
  return np.spacing(np.abs(np.asarray(r, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def c2_of(max_val, dtype, k2=0.03):
  """c2 = (k2 max_val)^2 as the library forms it: float32 k2, max_val after the dtype conversion."""
  return (float(np.float32(k2)) * O.convert_max_val(max_val, dtype))**2


def largest(*planes):
  """M: the largest |converted pixel| of the operands."""
  return max(float(O.convert(p.cpu()).abs().max()) for p in planes)


def stat_bound(want, M, c2):
  """The bar of each statistic: ulp32(|want|) + 2^-46 M^2 / c2 (tests/test_ssim_paths_gpu.py derives it)."""
  return ulp32(want) + 2.0**-46 * M * M / c2


def mse_bound(want, pixels):
  """The bar of each MSE: ulp32(want) + 2 (pixels) 2^-53 want, the float32 rounding plus the error of two float64
  sums of `pixels` non-negative terms (the kernel's and the reference's)."""
  want = np.asarray(want, dtype=np.float64)
  return ulp32(want) + 2.0 * pixels * 2.0**-53 * want
