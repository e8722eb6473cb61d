"""CPU: image.rgb_to_ycbcr against the float64 oracle and known colours, the argument checks of
image.metrics_ragged (raised before the library is touched) and the host-side rejections of
tfcb_image_metrics_ragged."""
import numpy as np
import pytest
import torch

from compression_b200 import _lib, image
from oracle import ycbcr_oracle as Y

F32, F16, BF16, U8 = 0, 1, 2, 3
RGB, LUMA, YCBCR = 0, 1, 2


@pytest.mark.parametrize("dtype,max_val", [(torch.float32, 255), (torch.float32, 1.0), (torch.uint8, 255),
                                           (torch.float16, 1.0), (torch.bfloat16, 255)])
def test_rgb_to_ycbcr_matches_the_oracle(dtype, max_val):
  g = torch.Generator().manual_seed(1)
  if dtype == torch.uint8:
    x = torch.randint(0, 256, (2, 17, 23, 3), generator=g, dtype=torch.uint8)
  else:
    x = (torch.rand(2, 17, 23, 3, generator=g) * max_val).to(dtype)
  got = image.rgb_to_ycbcr(x, max_val)
  assert got.dtype == torch.float32 and got.shape == x.shape
  want = Y.rgb_to_ycbcr(x, max_val)
  m = image._max_val(max_val, dtype)
  assert (got.double() - want).abs().max() <= 4e-7 * m


def test_rgb_to_ycbcr_known_colours():
  x = torch.tensor([[255.0, 255, 255], [0, 0, 0], [255, 0, 0]])
  got = image.rgb_to_ycbcr(x, 255).double()
  want = torch.tensor([[255.0, 128, 128], [0, 128, 128],
                       [0.299 * 255, 128 - 0.168736 * 255, 128 + 0.5 * 255]], dtype=torch.float64)
  assert (got - want).abs().max() <= 1e-4
  assert got[2, 2] == 255.5  # red's Cr leaves [0, 255] as JFIF's does before clipping
  # uint8 in [0, 1] units: max_val 255 becomes 1.0 and the chroma offset 128/255
  u = torch.tensor([[255, 255, 255], [0, 0, 0]], dtype=torch.uint8)
  got = image.rgb_to_ycbcr(u, 255).double()
  want = torch.tensor([[1.0, 128 / 255, 128 / 255], [0.0, 128 / 255, 128 / 255]], dtype=torch.float64)
  assert (got - want).abs().max() <= 1e-6


def test_rgb_to_ycbcr_rejects():
  with pytest.raises(image.InvalidArgumentError, match=r"\[\.\.\., 3\]"):
    image.rgb_to_ycbcr(torch.zeros(4, 4), 1.0)
  with pytest.raises(image.InvalidArgumentError, match="uint8"):
    image.rgb_to_ycbcr(torch.zeros(4, 3, dtype=torch.float64), 1.0)


@pytest.fixture
def no_library(monkeypatch):
  def refuse():
    raise AssertionError("the library was called")
  monkeypatch.setattr(_lib, "lib", refuse)


def _cuda_like(t):
  """A tensor that claims to live on a GPU, for the checks that come before any device work."""
  class Fake(torch.Tensor):
    is_cuda = True
    device = torch.device("cuda", 0)
  return t.as_subclass(Fake)


@pytest.mark.parametrize("a,b,color,match", [
    ([torch.zeros(161, 161, 3)], [], "rgb", "1 originals but 0"),
    ([torch.zeros(161, 161, 3)], [torch.zeros(161, 161, 3, dtype=torch.float16)], "rgb", "pair 0: dtypes"),
    ([torch.zeros(161, 161, 3), torch.zeros(161, 170, 3)], [torch.zeros(161, 161, 3), torch.zeros(170, 161, 3)],
     "rgb", "pair 1: shapes"),
    ([torch.zeros(161, 161, 3)], [torch.zeros(161, 161, 3)], "rgb", "pair 0: .*CUDA"),
    ([torch.zeros(161, 161, 3)], [torch.zeros(161, 161, 3)], "lab", "unknown color"),
    ([torch.zeros(161, 161, 3, dtype=torch.float64)], [torch.zeros(161, 161, 3, dtype=torch.float64)], "rgb",
     "unsupported dtype"),
    ([torch.zeros(161, 161)], [torch.zeros(161, 161)], "rgb", r"\[H, W, C\]"),
])
def test_metrics_ragged_rejects_before_the_library(no_library, a, b, color, match):
  with pytest.raises(image.InvalidArgumentError, match=match):
    image.metrics_ragged(a, b, 255, color=color)


def test_metrics_ragged_rejects_mixed_lists_before_the_library(no_library):
  a = [_cuda_like(torch.zeros(161, 161, 3)), _cuda_like(torch.zeros(161, 161, 3, dtype=torch.float16))]
  with pytest.raises(image.InvalidArgumentError, match="pair 1: dtypes"):
    image.metrics_ragged(a, list(a), 255)
  a = [_cuda_like(torch.zeros(161, 161, 3)), _cuda_like(torch.zeros(161, 161, 1))]
  with pytest.raises(image.InvalidArgumentError, match="pair 1: shapes"):
    image.metrics_ragged(a, list(a), 255)
  with pytest.raises(image.InvalidArgumentError, match="power_factors"):
    image.metrics_ragged(a, list(a), 255, power_factors=())


# ---- the library's host-side checks --------------------------------------------------------------------------
def _call(sizes, dtype=F32, C=3, mode=RGB, offsets=None, n_scales=5, filter_size=11, sigma=1.5, max_val=1.0,
          ptr=None):
  h = np.array([s[0] for s in sizes], dtype=np.int64)
  w = np.array([s[1] for s in sizes], dtype=np.int64)
  off = np.concatenate([[0], np.cumsum(h * w * C)]).astype(np.int64) if offsets is None else offsets
  return _lib.lib().tfcb_image_metrics_ragged(ptr, ptr, dtype, len(sizes), off.ctypes.data, h.ctypes.data,
                                              w.ctypes.data, C, mode, max_val, n_scales, filter_size, sigma, 0.01,
                                              0.03, ptr, ptr, ptr, None)


@pytest.mark.parametrize("kw,match", [
    (dict(dtype=4), "dtype"),
    (dict(mode=3), "colour mode"),
    (dict(mode=-1), "colour mode"),
    (dict(mode=LUMA, C=1), "C = 3"),
    (dict(mode=YCBCR, C=4), "C = 3"),
    (dict(C=0), "channel count"),
    (dict(sizes=[(161, 161), (161, 160), (200, 200)]), "image 1 too small"),
    (dict(sizes=[(161, 161), (200, 200), (10, 10)], n_scales=1), "image 2 too small"),
    (dict(sizes=[(161, 161), (0, 200)]), "image 1: bad size"),
    (dict(offsets=np.array([0, 161 * 161 * 3, 161 * 161 * 3 + 5], dtype=np.int64)), "inconsistent item_offsets"),
    (dict(offsets=np.array([1, 161 * 161 * 3 + 1, 2 * 161 * 161 * 3 + 1], dtype=np.int64)),
     "inconsistent item_offsets"),
    (dict(filter_size=33), "filter_size"),
    (dict(n_scales=0), "n_scales"),
    (dict(sigma=0.0), "filter_sigma"),
    (dict(max_val=float("inf")), "max_val"),
    (dict(), "null pointer"),
])
def test_library_rejects_before_any_device_work(kw, match):
  kw.setdefault("sizes", [(161, 161), (161, 161)])
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_call(**kw))


def test_library_wants_the_host_arrays_and_accepts_an_empty_list():
  lib = _lib.lib()
  h = np.array([161], dtype=np.int64)
  with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
    _lib.check(lib.tfcb_image_metrics_ragged(None, None, F32, 1, None, h.ctypes.data, h.ctypes.data, 3, RGB, 1.0, 5,
                                             11, 1.5, 0.01, 0.03, None, None, None, None))
  _lib.check(_call([]))  # nothing to do
  assert lib.tfcb_image_metrics_ragged_workspace_bytes(F32, 0, None, None, 3, RGB, 5, 11) == 0


def test_workspace_bytes():
  f = _lib.lib().tfcb_image_metrics_ragged_workspace_bytes
  h = np.array([161, 512, 768], dtype=np.int64)
  w = np.array([161, 768, 512], dtype=np.int64)
  rgb = f(U8, 3, h.ctypes.data, w.ctypes.data, 3, RGB, 5, 11)
  luma = f(U8, 3, h.ctypes.data, w.ctypes.data, 3, LUMA, 5, 11)
  assert rgb > luma > 0
  assert f(U8, 3, h.ctypes.data, w.ctypes.data, 3, YCBCR, 5, 11) == rgb
  small = np.array([161, 160, 161], dtype=np.int64)
  for bad in [(4, 3, h, w, 3, RGB), (F32, 3, small, w, 3, RGB), (F32, 3, h, w, 1, LUMA), (F32, 3, h, w, 3, 7)]:
    assert f(bad[0], bad[1], bad[2].ctypes.data, bad[3].ctypes.data, bad[4], bad[5], 5, 11) == -1, bad
  assert f(F32, 3, None, None, 3, RGB, 5, 11) == -1
