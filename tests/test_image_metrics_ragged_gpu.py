"""GPU: image.metrics_ragged / ssim_stats_ragged on lists of differently sized pairs against the one-image kernels
(bit for bit), the Y' / Y'CbCr planes against rgb_to_ycbcr and the float64 oracle, launch counts, determinism,
errors, and Model.evaluate_images against Model.evaluate on the three models."""
import math

import pytest
import torch

from compression_b200 import _lib, image, models
from oracle import ssim_oracle as O
from oracle import ycbcr_oracle as Y

pytestmark = pytest.mark.gpu

FWD_TOL = 1e-5
S = 5
DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.uint8]
MAX_VAL = {torch.float32: 255.0, torch.float16: 1.0, torch.bfloat16: 1.0, torch.uint8: 255}
LISTS = {
    "one": [(177, 209)],
    "mixed": [(161, 161), (177, 209), (512, 768), (768, 512), (203, 171)],
}


def _pair(h, w, seed, dtype):
  """Smooth colour content and a noisy copy, in `dtype` at MAX_VAL[dtype] (uint8 in [0, 255])."""
  g = torch.Generator().manual_seed(seed)
  yy = torch.linspace(0, 1, h)[:, None, None]
  xx = torch.linspace(0, 1, w)[None, :, None]
  phase = torch.rand(1, 1, 3, generator=g)
  a = 0.5 + 0.3 * torch.sin(6.0 * xx + 4.0 * yy + 6.28 * phase) * torch.cos(3.0 * yy - 2.0 * xx)
  a = (a + 0.05 * torch.randn(h, w, 3, generator=g)).clamp(0, 1)
  b = (a + 0.04 * torch.randn(h, w, 3, generator=g)).clamp(0, 1)
  if dtype == torch.uint8:
    return tuple(torch.round(t * 255).to(torch.uint8).cuda() for t in (a, b))
  return tuple((t * MAX_VAL[dtype]).to(dtype).cuda() for t in (a, b))


def _lists(sizes, dtype, seed=0):
  pairs = [_pair(h, w, seed + 7 * i, dtype) for i, (h, w) in enumerate(sizes)]
  return [p[0] for p in pairs], [p[1] for p in pairs]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("which", list(LISTS))
def test_rgb_equals_the_one_image_calls(dtype, which):
  xs, ys = _lists(LISTS[which], dtype)
  mv = MAX_VAL[dtype]
  stats, mse = image.ssim_stats_ragged(xs, ys, mv, "rgb", S)
  m = image.metrics_ragged(xs, ys, mv, "rgb")
  assert stats.shape == (len(xs), 3, S, 2) and mse.shape == (len(xs), 3)
  for k in m.values():
    assert k.dtype == torch.float32 and k.shape == (len(xs),)
  for i, (x, y) in enumerate(zip(xs, ys)):
    assert torch.equal(stats[i], image.ssim_stats(x, y, mv, n_scales=S))
    assert torch.equal(m["msssim"][i], image.ssim_multiscale(x, y, mv))
    assert abs(float(m["psnr"][i]) - float(image.psnr(x, y, mv))) <= 1e-5
    want_mse = ((O.convert(x.cpu()) - O.convert(y.cpu()))**2).mean((0, 1))
    assert ((mse[i].double().cpu() - want_mse).abs() <= 1e-6 * want_mse).all()
  assert torch.equal(m["msssim_db"], -10. * torch.log(1 - m["msssim"]) / math.log(10.))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("color", ["y", "ycbcr"])
def test_luma_and_ycbcr_equal_the_converted_planes(dtype, color):
  xs, ys = _lists([(161, 170), (256, 384), (384, 256)], dtype, seed=3)
  mv = MAX_VAL[dtype]
  m_conv = image._max_val(mv, dtype)
  stats, mse = image.ssim_stats_ragged(xs, ys, mv, color, S)
  m = image.metrics_ragged(xs, ys, mv, color)
  P = 1 if color == "y" else 3
  assert stats.shape == (3, P, S, 2) and mse.shape == (3, P)
  weights = torch.tensor([1.0] if P == 1 else [6 / 8, 1 / 8, 1 / 8], dtype=torch.float64)
  for i, (x, y) in enumerate(zip(xs, ys)):
    cx, cy = image.rgb_to_ycbcr(x, mv)[..., :P], image.rgb_to_ycbcr(y, mv)[..., :P]
    ms_planes = []
    for p in range(P):
      px, py = cx[..., p:p + 1].contiguous(), cy[..., p:p + 1].contiguous()
      assert torch.equal(stats[i, p], image.ssim_stats(px, py, m_conv, n_scales=S)[0])
      ms_planes.append(image.ssim_multiscale(px, py, m_conv))
    # against the float64 oracle
    ox, oy = Y.planes(x.cpu(), color, mv), Y.planes(y.cpu(), color, mv)
    want_stats = O.ssim_stats(ox, oy, m_conv, n_scales=S)
    assert (stats[i].double().cpu() - want_stats).abs().max() <= FWD_TOL
    want_mse = ((ox - oy)**2).mean((0, 1))
    assert ((mse[i].double().cpu() - want_mse).abs() <= 1e-5 * want_mse).all()
    want_ms = O.combine_multiscale(want_stats[:, None])  # per plane
    assert abs(float(m["msssim"][i]) - float((weights * want_ms).sum())) <= FWD_TOL
    assert abs(float(m["msssim"][i]) - float((weights * torch.stack(ms_planes).double().cpu()).sum())) <= 1e-6
    want_psnr = 20 * torch.log10(torch.tensor(m_conv, dtype=torch.float64)) - 10 * torch.log10(want_mse)
    assert abs(float(m["psnr"][i]) - float((weights * want_psnr).sum())) <= 1e-4
    assert abs(float(m["mse"][i]) - float((weights * want_mse).sum())) <= 1e-5 * float(want_mse.max())


def test_launch_count_does_not_depend_on_the_list():
  counts = []
  for n in (1, 7, 24):
    xs, ys = _lists([(161 + 13 * (i % 5), 161 + 29 * (i % 3)) for i in range(n)], torch.uint8, seed=n)
    for color in ("rgb", "y", "ycbcr"):
      n0 = _lib.launch_count()
      image.metrics_ragged(xs, ys, 255, color)
      counts.append(_lib.launch_count() - n0)
  assert len(set(counts)) == 1
  assert counts[0] <= 2 * S + 1


@pytest.mark.parametrize("color", ["rgb", "y", "ycbcr"])
def test_deterministic_and_independent_of_the_list(color):
  xs, ys = _lists([(200, 180), (161, 161), (333, 250), (177, 209)], torch.float32, seed=11)
  s1, e1 = image.ssim_stats_ragged(xs, ys, 255, color, S)
  s2, e2 = image.ssim_stats_ragged(xs, ys, 255, color, S)
  assert torch.equal(s1, s2) and torch.equal(e1, e2)
  for i in (0, 2, 3):
    s, e = image.ssim_stats_ragged(xs[i:i + 1], ys[i:i + 1], 255, color, S)
    assert torch.equal(s[0], s1[i]) and torch.equal(e[0], e1[i])
  s, e = image.ssim_stats_ragged(xs[::-1], ys[::-1], 255, color, S)
  assert torch.equal(s.flip(0), s1) and torch.equal(e.flip(0), e1)


def test_errors_and_the_empty_list():
  xs, ys = _lists([(161, 161), (200, 200), (161, 160)], torch.float32)
  n0 = _lib.launch_count()
  with pytest.raises(image.InvalidArgumentError, match="image 2 too small"):
    image.metrics_ragged(xs, ys, 255)
  with pytest.raises(image.InvalidArgumentError, match="C = 3"):
    image.metrics_ragged([x[..., :1].contiguous() for x in xs[:2]], [y[..., :1].contiguous() for y in ys[:2]], 255,
                         "y")
  assert _lib.launch_count() == n0
  m = image.metrics_ragged([], [], 255, "ycbcr")
  assert set(m) == {"mse", "psnr", "msssim", "msssim_db"}
  assert all(v.shape == (0,) and v.dtype == torch.float32 for v in m.values())


def _uint8_images(sizes, seed):
  out = []
  for i, (h, w) in enumerate(sizes):
    a, _ = _pair(h, w, seed + i, torch.float32)
    out.append(torch.round(a).to(torch.uint8).cpu())
  return out


# MS2020's slice transforms need the hyperprior's grid to match the latents', which multiples of 64 give
MODEL_SIZES = {"bls2017": [(176, 200), (161, 170), (192, 256), (200, 176)],
               "bmshj2018": [(176, 200), (161, 170), (192, 256), (200, 176)],
               "ms2020": [(192, 256), (256, 192), (192, 192), (320, 192)]}


@pytest.fixture(scope="module", params=list(MODEL_SIZES))
def model(request):
  torch.manual_seed(5)
  if request.param == "bls2017":
    m = models.BLS2017Model(num_filters=32)
  elif request.param == "bmshj2018":
    m = models.BMSHJ2018Model(num_filters=24, num_scales=16)
  else:
    m = models.MS2020Model(num_filters=24, latent_depth=32, hyperprior_depth=16, num_slices=4, max_support_slices=2)
  return m.build("cuda", patch=(64, 64)).fix_tables(), MODEL_SIZES[request.param]


def test_evaluate_images_equals_evaluate(model):
  model, sizes = model
  images = _uint8_images(sizes, 40)
  got = model.evaluate_images(images)
  assert len(got) == len(images)
  for r, x in zip(got, images):
    want = model.evaluate(x)
    assert set(r) == set(want) | {"psnr_y", "msssim_y", "msssim_db_y", "psnr_ycbcr", "msssim_ycbcr",
                                  "msssim_db_ycbcr"}
    assert all(isinstance(v, float) for v in r.values())
    assert r["bpp"] == want["bpp"] and r["msssim"] == want["msssim"]
    for k in ("mse", "psnr"):
      assert abs(r[k] - want[k]) <= 1e-6 * abs(want[k])
    assert r["msssim_db"] == pytest.approx(want["msssim_db"], rel=1e-6)
    # the luma metrics against the one-image kernels on the converted planes
    x_hat = model.decompress_from_tfci(model.compress_to_tfci(x)).float()
    cx, cy = image.rgb_to_ycbcr(x.cuda().float(), 255)[..., :1], image.rgb_to_ycbcr(x_hat, 255)[..., :1]
    assert r["msssim_y"] == float(image.ssim_multiscale(cx.contiguous(), cy.contiguous(), 255))
    assert r["psnr_y"] == pytest.approx(float(image.psnr(cx, cy, 255)), abs=1e-4)
  mean = models.mean_metrics(got)
  assert mean["bpp"] == pytest.approx(sum(r["bpp"] for r in got) / len(got))
  assert set(mean) == set(got[0])


def test_evaluate_images_codes_the_list_once(model):
  model, sizes = model
  images = _uint8_images(sizes[:3], 50)
  n0 = _lib.launch_count()
  items = model.compress_images(images)
  n1 = _lib.launch_count()
  model.decompress_images(items)
  n2 = _lib.launch_count()
  model.evaluate_images(images)
  n3 = _lib.launch_count()
  assert n3 - n2 == (n1 - n0) + (n2 - n1) + 3 * 2 * S  # the coder's launches plus one metrics call per colour space
  assert model.evaluate_images([]) == []
