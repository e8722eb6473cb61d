"""GPU: csrc/ssim.cu at its filter, scale, channel and plane-count limits, on content at the edges of its precision
and on the ragged list form, against oracle/ssim_oracle.py.  The cases come from tests/ssim_cases.py.

Statistics are held to the float32-pyramid reference, ssim_stats(..., pool="float32"), which filters the planes the
kernels filter (the float32 images and the pyramid the pool kernel stores, with the library's float32 sigma, k1 and
k2) in float64.  Within

    |got - want| <= ulp32(|want|) + 2^-46 M^2 / c2,

M the largest |converted pixel| of the two operands and c2 = (k2 max_val)^2 after the dtype conversion.  Derivation:
  * The kernel forms l and cs at each position in double and rounds only the mean over positions to float32: at most
    half an ulp32.  The reference's own float64 result may sit by a rounding midpoint, so the first term is a full ulp.
  * In double, the second moments are formed on values shifted by a constant of the plane's range (the kernel: the
    mean of the two images at the tile's first pixel; the reference: the mean of the two planes), so |x'|, |y'| <= M on
    the non-negative content here.  Each windowed sum S(x'^2 + y'^2), S(x'y'), mx'^2 + my'^2 is a sum of at most 2F
    weighted terms of magnitude <= 2 M^2 (a row pass and a column pass for the kernel), so its absolute error is at
    most about 4F 2^-53 M^2 <= 2^7 2^-53 M^2 = 2^-46 M^2 for F <= 32, and in practice far less: the errors are
    independent roundings and the mean over positions averages them.
  * cs = (2 cov + c2) / (var_x + var_y + c2) has |cs| <= 1 and a denominator >= c2, so those errors move it by at most
    about 2^-46 M^2 / c2, and so they move its mean and the mean of l cs (|l| <= 1).  l depends on the means only,
    whose relative errors are ~F 2^-53 and stay far inside the first term.
For max_val = 1 on [0, 1] content, or 255 on [0, 255], M^2 / c2 ~ 1111 and the second term is ~1.6e-11: the bound is
about one float32 ulp.  It is loosest for uint8 with max_val = 1 (c2 ~ 1.4e-8), ~1e-6.

MSE (ragged) is held to ulp32(want) + 2 n 2^-53 want, n the plane's pixel count: the kernel squares float32
differences exactly in double, sums them in double and rounds once; the reference sums the same squares in float64.

Gradients are held to float64 autograd of the default (TF-semantics) reference within 1e-4 of the largest |gradient|
per element, as tests/test_image_metrics_gpu.py does.  The worst ratio |got - want| / max|want| of each case is
printed at the end of the module (run with -s)."""
import numpy as np
import pytest
import torch

import ssim_cases as cases
from compression_b200 import _lib, image
from oracle import ssim_oracle as O
from test_image_metrics_gpu import FORWARD_CASES, _as, _content

pytestmark = pytest.mark.gpu
GRAD_TOL = 1e-4
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
  yield
  if RATIOS:
    print("\nworst gradient ratio |got - want| / max|want| per case:")
    for k in sorted(RATIOS):
      print(f"  {k}: {RATIOS[k]:.3g}")


def _check_stats(got, x, y, max_val, **kw):
  """got [..., P, S, 2] from the kernels; x, y the operands (CPU or CUDA) in the dtype the kernels read."""
  x, y = x.cpu(), y.cpu()
  want = O.ssim_stats(x, y, max_val, pool="float32", **kw)
  got = got.detach().double().cpu()
  assert got.shape == want.shape and torch.isfinite(got).all()
  bound = cases.stat_bound(want.numpy(), cases.largest(x, y), cases.c2_of(max_val, x.dtype, kw.get("k2", 0.03)))
  excess = ((got - want).abs().numpy() / bound).max()
  assert excess <= 1.0, f"a statistic misses the bound by {excess:.3g}x"
  return want


def _check_grads(name, x, y, fn, oracle_fn):
  """Gradients of sum(fn(x, y)) against float64 autograd of oracle_fn, per element within GRAD_TOL max|want|."""
  x1, y1 = x.cuda().requires_grad_(), y.cuda().requires_grad_()
  fn(x1, y1).sum().backward()
  x64, y64 = x.double().requires_grad_(), y.double().requires_grad_()
  oracle_fn(x64, y64).sum().backward()
  worst = 0.0
  for got, want in ((x1.grad, x64.grad), (y1.grad, y64.grad)):
    assert got.dtype == x.dtype and torch.isfinite(got).all()
    scale = want.abs().max()
    assert scale > 0
    worst = max(worst, float((got.double().cpu() - want).abs().max() / scale))
  RATIOS[name] = max(RATIOS.get(name, 0.0), worst)
  assert worst <= GRAD_TOL


# ---- 1. make_window at even F and tiny sigma (was 0 / 0) ----------------------------------------------------------
@pytest.mark.parametrize("F,sigma", cases.EVEN_F_TINY_SIGMA)
def test_even_filter_at_tiny_sigma_is_finite_and_meets_the_bounds(F, sigma):
  """make_window, then ssim_fwd_kernel, ssim_pool_kernel and ssim_bwd_kernel with a box of the four central taps."""
  x, y = cases.content((2, 40, 45, 3), 100 + F)
  kw = dict(filter_size=F, filter_sigma=sigma)
  got = image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=2, **kw)
  _check_stats(got, x, y, 1.0, n_scales=2, **kw)
  _check_grads(f"even F={F} sigma={sigma}", x, y, lambda a, b: image.ssim_multiscale(a, b, 1.0, (0.4, 0.6), **kw),
               lambda a, b: O.ssim_multiscale(a, b, 1.0, (0.4, 0.6), **kw))


# ---- 2. filter sizes x sigma at the tile seams --------------------------------------------------------------------
@pytest.mark.parametrize("sigma", cases.SIGMAS)
@pytest.mark.parametrize("F", cases.FILTERS)
def test_filter_sizes_and_sigmas_at_the_tile_seams(F, sigma):
  """ssim_fwd_kernel's shared-memory halo (R = 32 + F - 1) and ssim_bwd_kernel's (I = 16 + 2 (F - 1)) for every F up
  to 32 (201 584 B of dynamic shared memory), on sizes just above F whose last forward tile has 0, 1 or 31 valid
  rows / columns and whose last backward tile has 0, 1 or 15 inputs."""
  kw = dict(filter_size=F, filter_sigma=sigma)
  for i, (H, W) in enumerate(cases.seam_sizes(F)):
    x, y = cases.content((2, H, W, 2), 1000 * F + i)
    _check_stats(image.ssim_stats(x.cuda(), y.cuda(), 1.0, **kw), x, y, 1.0, **kw)
    _check_grads(f"F={F} sigma={sigma}", x, y, lambda a, b: image.ssim(a, b, 1.0, **kw),
                 lambda a, b: O.ssim(a, b, 1.0, **kw))


def test_largest_filter_with_one_valid_position():
  """F = 32 on 32x32: one position per plane, every input inside its window; the backward's tiles see it only
  through the halo."""
  x, y = cases.content((3, 32, 32, 2), 7)
  kw = dict(filter_size=32, filter_sigma=8.0)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), 1.0, **kw), x, y, 1.0, **kw)
  _check_grads("F=32 32x32", x, y, lambda a, b: image.ssim(a, b, 1.0, **kw), lambda a, b: O.ssim(a, b, 1.0, **kw))


@pytest.mark.parametrize("H,W", [(63, 64), (95, 97)])
def test_largest_filter_at_two_scales(H, W):
  """F = 32 at S = 2: the pool of an odd size into a level of 32 (or 48 x 49), and the pool's adjoint."""
  x, y = cases.content((2, H, W, 2), H + W)
  kw = dict(filter_size=32, filter_sigma=1.5)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=2, **kw), x, y, 1.0, n_scales=2, **kw)
  _check_grads(f"F=32 S=2 {H}x{W}", x, y, lambda a, b: image.ssim_multiscale(a, b, 1.0, (0.3, 0.7), **kw),
               lambda a, b: O.ssim_multiscale(a, b, 1.0, (0.3, 0.7), **kw))


# ---- 3. deep pyramids ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,S,H,W", cases.DEEP)
def test_deep_pyramids(F, S, H, W):
  """ssim_pool_kernel and the backward's pool adjoint down to 1x1 (F = 1, S = 16: cs = 1 at every scale, so the
  gradient reaches the input only through 15 adjoints of odd and unit sizes), 2x2 and 3x3 levels, with non-default
  power factors."""
  x, y = cases.content((2, H, W, 3), S)
  kw = dict(filter_size=F, filter_sigma=1.5)
  pf = cases.power_factors(S)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=S, **kw), x, y, 1.0, n_scales=S, **kw)
  _check_grads(f"deep F={F} S={S}", x, y, lambda a, b: image.ssim_multiscale(a, b, 1.0, pf, **kw),
               lambda a, b: O.ssim_multiscale(a, b, 1.0, pf, **kw))


# ---- 4. channel strides and batch shapes --------------------------------------------------------------------------
@pytest.mark.parametrize("C", cases.CHANNELS)
def test_channel_strides(C):
  """plane_of / item_plane with a channel stride of 2, 4 or 7 at scale 0 (the pyramid is planar)."""
  x, y = cases.seam_patches((2, 45, 50, C), C)
  kw = dict(filter_size=7, filter_sigma=1.0)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=3, **kw), x, y, 1.0, n_scales=3, **kw)
  _check_grads(f"C={C}", x, y, lambda a, b: image.ssim_multiscale(a, b, 1.0, (0.2, 0.3, 0.5), **kw),
               lambda a, b: O.ssim_multiscale(a, b, 1.0, (0.2, 0.3, 0.5), **kw))


def test_batch_shape():
  """A [2, 3] batch of 3-channel images: the statistics' [2, 3, C, S, 2] layout and g_stats' plane index."""
  x, y = cases.content(cases.BATCH_SHAPE + (40, 37, 3), 23)
  kw = dict(filter_size=7, filter_sigma=1.0)
  got = image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=2, **kw)
  assert got.shape == cases.BATCH_SHAPE + (3, 2, 2)
  _check_stats(got, x, y, 1.0, n_scales=2, **kw)
  _check_grads("batch (2, 3)", x, y, lambda a, b: image.ssim_multiscale(a, b, 1.0, (0.5, 0.5), **kw),
               lambda a, b: O.ssim_multiscale(a, b, 1.0, (0.5, 0.5), **kw))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_sixteen_bit_at_the_largest_filter(dtype):
  """F = 32, S = 2, C = 7 on 63x64: the 16-bit statistics meet the bound, and the 16-bit gradients are the float32
  kernels' gradients of the same values rounded once."""
  a, b = cases.content((1, 63, 64, 7), 31)
  x, y = a.to(dtype), b.to(dtype)
  kw = dict(filter_size=32, filter_sigma=1.5)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=2, **kw), x, y, 1.0, n_scales=2, **kw)
  x16, y16 = x.cuda().requires_grad_(), y.cuda().requires_grad_()
  image.ssim_multiscale(x16, y16, 1.0, (0.5, 0.5), **kw).sum().backward()
  x32, y32 = x.float().cuda().requires_grad_(), y.float().cuda().requires_grad_()
  image.ssim_multiscale(x32, y32, 1.0, (0.5, 0.5), **kw).sum().backward()
  assert x16.grad.dtype == dtype
  assert torch.equal(x16.grad, x32.grad.to(dtype)) and torch.equal(y16.grad, y32.grad.to(dtype))


# ---- 5. more planes than the backward's grid ----------------------------------------------------------------------
def test_many_planes():
  """2 * 65535 + 3 planes: the forward's CTA list past 65535 planes and three trips of the backward's plane loop
  (gridDim.y = 65535).  Every plane equals the one-image call for its pair bit for bit, and the pairs meet the
  oracle."""
  N, H, W, C = cases.MANY_PLANES
  k = cases.MANY_PLANES_PAIRS
  a, b = cases.content((k, H, W, C), 41)
  idx = torch.arange(N, device="cuda") % k
  x, y = a.cuda()[idx].requires_grad_(), b.cuda()[idx].requires_grad_()
  stats = image.ssim_stats(x, y, 1.0)
  image.ssim(x, y, 1.0).sum().backward()
  one_stats, one_gx, one_gy = [], [], []
  for i in range(k):
    xi, yi = a[i:i + 1].cuda().requires_grad_(), b[i:i + 1].cuda().requires_grad_()
    one_stats.append(image.ssim_stats(xi, yi, 1.0))
    image.ssim(xi, yi, 1.0).sum().backward()
    one_gx.append(xi.grad)
    one_gy.append(yi.grad)
  assert torch.equal(stats, torch.cat(one_stats)[idx])
  assert torch.equal(x.grad, torch.cat(one_gx)[idx]) and torch.equal(y.grad, torch.cat(one_gy)[idx])
  _check_stats(torch.cat(one_stats), a, b, 1.0)
  _check_grads("many planes (the pairs)", a, b, lambda p, q: image.ssim(p, q, 1.0), lambda p, q: O.ssim(p, q, 1.0))


# ---- 6. content at the edges of precision -------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,max_val", [(torch.float32, 1.0), (torch.float32, 255.0), (torch.uint8, 1),
                                           (torch.float32, 1 / 255)])
def test_bright_patches_clipped_pixels_and_small_c2(dtype, max_val):
  """Bright flat patches across forward and backward tile seams with each tile's first pixel dark (the kernels' shift
  far from the patch), pixels at exactly 0 and max_val; uint8 at max_val = 1 (c2 ~ 1.4e-8, forward only) and float32
  at max_val = 1/255 (the same c2, with gradients)."""
  top = 1.0 if dtype == torch.uint8 else max_val  # uint8 holds [0, 255] whatever max_val says
  a, b = cases.seam_patches((2, 70, 66, 3), 17, top)
  x, y = cases.as_dtype(a, dtype, top), cases.as_dtype(b, dtype, top)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), max_val, n_scales=2), x, y, max_val, n_scales=2)
  if dtype != torch.uint8:
    _check_grads(f"patches max_val={max_val:.4g}", x, y,
                 lambda p, q: image.ssim_multiscale(p, q, max_val, (0.5, 0.5)),
                 lambda p, q: O.ssim_multiscale(p, q, max_val, (0.5, 0.5)))


def test_uint8_is_its_converted_float32_values_at_every_scale():
  """uint8 reads convert as convert_image_dtype does, float32(u) * float32(1/255), in the moments kernel and in the
  pool (where a multiply contracted into the pool's first addition rounded differently): the statistics of uint8
  images equal, bit for bit, those of the float32 images of the converted values, at every scale of the batch and of
  the list in each colour mode."""
  a, b = cases.content((3, 37, 41, 3), 61)
  u, v = cases.as_dtype(a, torch.uint8, 1.0).cuda(), cases.as_dtype(b, torch.uint8, 1.0).cuda()
  fu, fv = O.convert(u, torch.float32), O.convert(v, torch.float32)
  kw = dict(n_scales=4, filter_size=3)
  assert torch.equal(image.ssim_stats(u, v, 255, **kw), image.ssim_stats(fu, fv, 1.0, **kw))
  for color in ("rgb", "y", "ycbcr"):
    su, eu = image.ssim_stats_ragged(list(u), list(v), 255, color, **kw)
    sf, ef = image.ssim_stats_ragged(list(fu), list(fv), 1.0, color, **kw)
    assert torch.equal(su, sf) and torch.equal(eu, ef), color


@pytest.mark.parametrize("F", [8, 11])
def test_constant_pairs_in_closed_form(F):
  """Constant planes a vs b: cs = 1 and l = (2ab + c1) / (a^2 + b^2 + c1) at every position and scale, including
  a = b = 0, 0 vs max_val and max_val vs max_val."""
  pairs = [(0.2, 0.7), (0.0, 1.0), (1.0, 1.0), (0.0, 0.0), (0.5, 0.49)]
  H, W = F + 31, 2 * F + 1  # 32 valid rows; two scales
  x = torch.tensor([p[0] for p in pairs], dtype=torch.float32).expand(1, H, W, len(pairs)).contiguous()
  y = torch.tensor([p[1] for p in pairs], dtype=torch.float32).expand(1, H, W, len(pairs)).contiguous()
  kw = dict(filter_size=F, filter_sigma=1.5)
  got = image.ssim_stats(x.cuda(), y.cuda(), 1.0, n_scales=2, **kw).double().cpu()[0]
  c1 = (float(np.float32(0.01)) * 1.0)**2
  a, b = x[0, 0, 0].double(), y[0, 0, 0].double()
  lum = (2 * a * b + c1) / (a * a + b * b + c1)
  want = torch.stack([torch.ones_like(lum), lum], -1)[:, None, :].expand(-1, 2, -1)
  bound = cases.stat_bound(want.numpy(), 1.0, cases.c2_of(1.0, torch.float32))
  assert ((got - want).abs().numpy() <= bound).all()
  _check_stats(got[None], x, y, 1.0, n_scales=2, **kw)
  _check_grads(f"constant pairs F={F}", x, y, lambda p, q: image.ssim_multiscale(p, q, 1.0, (0.5, 0.5), **kw),
               lambda p, q: O.ssim_multiscale(p, q, 1.0, (0.5, 0.5), **kw))


# ---- 7. ragged lists ----------------------------------------------------------------------------------------------
def _check_mse(mse, xs, ys):
  for i, (x, y) in enumerate(zip(xs, ys)):
    d = x.cpu().double() - y.cpu().double()
    want = (d * d).mean((0, 1)).numpy()
    bound = cases.mse_bound(want, x.shape[0] * x.shape[1])
    assert (np.abs(mse[i].double().cpu().numpy() - want) <= bound).all(), i


@pytest.mark.parametrize("C", cases.RAGGED_CHANNELS)
def test_ragged_rgb_channel_counts(C):
  """tfcb_image_metrics_ragged in RGB mode with C = 1, 2 or 4: each item equals its one-image call bit for bit, and its
  statistics and MSE meet the bounds."""
  pairs = [cases.content((h, w, C), 50 + i, 255.0) for i, (h, w) in enumerate(cases.RAGGED_SIZES)]
  xs, ys = [p[0].cuda() for p in pairs], [p[1].cuda() for p in pairs]
  stats, mse = image.ssim_stats_ragged(xs, ys, 255.0, "rgb", 5)
  assert stats.shape == (len(xs), C, 5, 2)
  for i, (x, y) in enumerate(zip(xs, ys)):
    assert torch.equal(stats[i], image.ssim_stats(x, y, 255.0, n_scales=5))
    _check_stats(stats[i], x, y, 255.0, n_scales=5)
  _check_mse(mse, xs, ys)


def test_ragged_long_list_of_tiny_items():
  """Over 200 items from the smallest size F = 3, S = 3 allow (9x9), a few 512x768 among them: the binary searches
  over item rows (forward CTAs, pool outputs) on a long list of one-tile items.  Each item equals its one-image call bit
  for bit, its statistics and MSE meet the bounds, and the list takes 2 S launches."""
  F, S = cases.LONG_F, cases.LONG_S
  sizes = cases.long_list_sizes()
  xs, ys = [], []
  for i, (h, w) in enumerate(sizes):
    a, b = cases.content((h, w, 3), 200 + i)
    xs.append(cases.as_dtype(a, torch.uint8, 1.0).cuda())
    ys.append(cases.as_dtype(b, torch.uint8, 1.0).cuda())
  n0 = _lib.launch_count()
  stats, mse = image.ssim_stats_ragged(xs, ys, 255, "rgb", S, filter_size=F)
  assert _lib.launch_count() - n0 == 2 * S
  kw = dict(n_scales=S, filter_size=F)
  for i, (x, y) in enumerate(zip(xs, ys)):
    assert torch.equal(stats[i], image.ssim_stats(x, y, 255, **kw)), i
    _check_stats(stats[i], x, y, 255, **kw)
  _check_mse(mse, [O.convert(x.cpu(), torch.float32) for x in xs], [O.convert(y.cpu(), torch.float32) for y in ys])


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("color", ["y", "ycbcr"])
def test_ragged_luma_and_ycbcr_at_minimal_and_seam_sizes(color, dtype):
  """The Y' / Y'CbCr planes made as scale 0 and its pool load them (kY, kYCbCr) at 161x161 and at valid sizes 0, 1
  and 31 mod 32: the statistics and MSE of rgb_to_ycbcr's float32 planes meet the bounds."""
  mv = 255 if dtype == torch.uint8 else 1.0
  xs, ys = [], []
  for i, (h, w) in enumerate(cases.LUMA_SIZES):
    a, b = cases.seam_patches((h, w, 3), 300 + i)
    xs.append(cases.as_dtype(a, dtype, 1.0).cuda())
    ys.append(cases.as_dtype(b, dtype, 1.0).cuda())
  P = 1 if color == "y" else 3
  m_conv = image._max_val(mv, dtype)
  n0 = _lib.launch_count()
  stats, mse = image.ssim_stats_ragged(xs, ys, mv, color, 5)
  assert _lib.launch_count() - n0 == 2 * 5
  cx = [image.rgb_to_ycbcr(x, mv)[..., :P].contiguous() for x in xs]
  cy = [image.rgb_to_ycbcr(y, mv)[..., :P].contiguous() for y in ys]
  for i in range(len(xs)):
    _check_stats(stats[i], cx[i], cy[i], m_conv, n_scales=5)
  _check_mse(mse, cx, cy)


# ---- 8. the existing forward cases under the tight bound ----------------------------------------------------------
@pytest.mark.parametrize("batch,H,W,C,dtype,max_val,flat", FORWARD_CASES)
def test_existing_forward_cases_under_the_tight_bound(batch, H, W, C, dtype, max_val, flat):
  """tests/test_image_metrics_gpu.py's FORWARD_CASES (five scales, every dtype) against the float32-pyramid
  reference."""
  a, b = _content(batch + (H, W, C), H * W + C, flat)
  x, y = _as(a, dtype, max_val), _as(b, dtype, max_val)
  _check_stats(image.ssim_stats(x.cuda(), y.cuda(), max_val, n_scales=5), x, y, max_val, n_scales=5)
