"""CPU: the float32-pyramid reference of oracle/ssim_oracle.py against an independent numpy restatement of the
kernels' pool, its window at tiny sigma, evidence that the statistics bound of tests/test_ssim_paths_gpu.py can tell
the kernels' float32 pyramid from TF's float64 one, and that tests/ssim_cases.py reaches what it claims."""
import math

import numpy as np
import pytest
import torch

import ssim_cases as cases
from compression_b200 import _lib
from oracle import ssim_oracle as O


def _pool_numpy(x):
  """[N, H, W, C] float32: repeat the last row / column of an odd size, then ((a + b) + (c + d)) * 0.25 with a, b the
  upper pair and c, d the lower pair, one float32 rounding per operation."""
  x = np.asarray(x, dtype=np.float32)
  if x.shape[1] % 2:
    x = np.concatenate([x, x[:, -1:]], 1)
  if x.shape[2] % 2:
    x = np.concatenate([x, x[:, :, -1:]], 2)
  a, b = x[:, 0::2, 0::2], x[:, 0::2, 1::2]
  c, d = x[:, 1::2, 0::2], x[:, 1::2, 1::2]
  return ((a + b) + (c + d)) * np.float32(0.25)


@pytest.mark.parametrize("H,W", [(7, 9), (8, 6), (2, 1), (1, 2), (1, 1), (37, 41)])
def test_float32_pyramid_is_the_kernels_pool_bit_for_bit(H, W):
  rng = np.random.default_rng(H * 100 + W)
  # values of mixed exponents, so that the order of the three additions shows
  x = (rng.random((2, H, W, 3)) * 10.0**rng.integers(-3, 3, (2, H, W, 3))).astype(np.float32)
  got, want = torch.from_numpy(x), x
  while True:
    got, want = O.downsample32(got), _pool_numpy(want)
    assert got.dtype == torch.float32
    np.testing.assert_array_equal(got.numpy().view(np.uint32), want.view(np.uint32))
    if got.shape[1] == 1 and got.shape[2] == 1:
      break
  # the order matters: a different association differs somewhere on the same data
  y = np.asarray(x, dtype=np.float32)
  if H % 2 == 0 and W % 2 == 0 and H * W > 4:
    other = (((y[:, 0::2, 0::2] + y[:, 1::2, 0::2]) + y[:, 0::2, 1::2]) + y[:, 1::2, 1::2]) * np.float32(0.25)
    assert not np.array_equal(other, _pool_numpy(y))


def test_float32_reference_filters_the_float32_pyramid():
  a, b = cases.content((1, 37, 41, 2), 3)
  got = O.ssim_stats(a, b, 1.0, n_scales=3, filter_size=3, pool="float32")
  x, y = a.clone(), b.clone()
  for s in range(3):
    if s:
      x, y = O.downsample32(x), O.downsample32(y)
    want = O.ssim_stats(x.double(), y.double(), 1.0, n_scales=1, filter_size=3, filter_sigma=float(np.float32(1.5)),
                        k1=float(np.float32(0.01)), k2=float(np.float32(0.03)))
    bound = cases.stat_bound(want.numpy(), 1.0, cases.c2_of(1.0, torch.float32))
    assert ((got[..., s:s + 1, :] - want).abs().numpy() <= bound).all()


@pytest.mark.parametrize("F", [2, 8, 16, 32])
def test_oracle_window_at_even_filter_and_tiny_sigma_is_the_central_box(F):
  w = O.window(F, 0.01)
  assert torch.isfinite(w).all()
  want = torch.zeros(F, F, dtype=torch.float64)
  want[F // 2 - 1:F // 2 + 1, F // 2 - 1:F // 2 + 1] = 0.25
  assert torch.equal(w, want)


@pytest.mark.parametrize("F", [1, 3, 11, 31])
def test_oracle_window_at_odd_filter_and_tiny_sigma_is_the_delta(F):
  w = O.window(F, 1e-3)
  want = torch.zeros(F, F, dtype=torch.float64)
  want[F // 2, F // 2] = 1.0
  assert torch.equal(w, want)


def test_the_tight_bound_tells_the_float32_pyramid_from_the_float64_one():
  """With float32-exact sigma, k1 and k2, the two references differ only in how the levels are pooled: they agree far
  inside the bound at scale 0 and differ by more than it at coarser scales, so a kernel that pooled as TF does would
  fail the GPU tests."""
  F, S, H, W = cases.DEEP[1]
  g = torch.Generator().manual_seed(0)
  a = 0.5 + 0.3 * torch.rand(2, H, W, 3, generator=g)  # texture at every scale, so each pool rounds
  b = a + 0.04 * torch.randn(2, H, W, 3, generator=g)
  kw = dict(n_scales=S, filter_size=F, filter_sigma=1.5, k1=2**-7, k2=2**-5)
  s64 = O.ssim_stats(a, b, 1.0, **kw).numpy()
  s32 = O.ssim_stats(a, b, 1.0, pool="float32", **kw).numpy()
  bound = cases.stat_bound(s32, cases.largest(a, b), 2.0**-10)
  ratio = np.abs(s64 - s32) / bound
  assert ratio[..., 0, :].max() < 1e-3
  assert ratio[..., 1:, :].max() > 2.0


def test_float32_reference_of_constant_pairs_in_closed_form():
  k1, mv = float(np.float32(0.01)), 1.0
  x = torch.full((1, 40, 37, 1), 0.2, dtype=torch.float32)
  y = torch.full((1, 40, 37, 1), 0.7, dtype=torch.float32)
  a, b = float(x[0, 0, 0, 0]), float(y[0, 0, 0, 0])
  lum = (2 * a * b + (k1 * mv)**2) / (a * a + b * b + (k1 * mv)**2)
  st = O.ssim_stats(x, y, mv, n_scales=3, filter_size=8, pool="float32")
  np.testing.assert_allclose(st[0, 0, :, 0].numpy(), 1.0, rtol=0, atol=1e-13)
  np.testing.assert_allclose(st[0, 0, :, 1].numpy(), lum, rtol=0, atol=1e-13)


# ---- what the case table claims --------------------------------------------------------------------------------
def test_filters_span_the_documented_range():
  assert set(cases.FILTERS) == {1, 2, 3, 8, 16, 31, 32}
  assert max(cases.FILTERS) == cases.MAX_FILTER
  assert all(F % 2 == 0 for F, _ in cases.EVEN_F_TINY_SIGMA)


@pytest.mark.parametrize("F", cases.FILTERS)
def test_seam_sizes_hit_both_tiles_residues(F):
  sizes = cases.seam_sizes(F)
  dims = [d for hw in sizes for d in hw]
  assert min(dims) >= F
  assert {(d - F + 1) % cases.FWD_TILE for d in dims} >= {0, 1, cases.FWD_TILE - 1}
  assert {d % cases.BWD_TILE for d in dims} >= {0, 1, cases.BWD_TILE - 1}
  assert min(max(hw) for hw in sizes) <= F + cases.FWD_TILE + 1  # just above F


def test_deep_pyramids_reach_unit_and_tiny_levels():
  assert max(S for _, S, _, _ in cases.DEEP) == cases.MAX_SCALES
  finals = set()
  for F, S, H, W in cases.DEEP:
    hs, ws = cases.pyramid(H, S), cases.pyramid(W, S)
    assert min(hs + ws) >= F
    assert any(h % 2 for h in hs[:-1]) and any(w % 2 for w in ws[:-1])  # odd levels: the padded pool's adjoint
    finals.add((hs[-1], ws[-1]))
    assert len(cases.power_factors(S)) == S and abs(sum(cases.power_factors(S)) - 1) < 1e-12
  assert {(1, 1), (2, 2)} <= finals


def test_many_planes_loop_the_backward_three_times():
  N, H, W, C = cases.MANY_PLANES
  assert N * C == 2 * cases.MAX_PLANE_BLOCKS + 3
  assert math.ceil(N * C / cases.MAX_PLANE_BLOCKS) == 3
  assert N % cases.MANY_PLANES_PAIRS != 0


def test_channels_and_ragged_lists():
  assert set(cases.CHANNELS) >= {2, 4, 7} and set(cases.RAGGED_CHANNELS) >= {1, 2, 4}
  sizes = cases.long_list_sizes()
  m = cases.min_size(cases.LONG_F, cases.LONG_S)
  assert len(sizes) >= 200 and sizes[0] == (m, m)
  assert min(min(hw) for hw in sizes) == m
  assert sizes.count((512, 768)) >= 2 and sizes[-1] != (512, 768) and sizes[0] != (512, 768)
  luma = cases.LUMA_SIZES
  assert luma[0] == (cases.min_size(11, 5),) * 2
  assert {(h - 10) % cases.FWD_TILE for h, _ in luma} >= {0, 1, cases.FWD_TILE - 1}


def test_library_accepts_every_case_before_any_device_work():
  lib = _lib.lib()
  ws = lib.tfcb_ssim_workspace_bytes
  for F in cases.FILTERS:
    for H, W in cases.seam_sizes(F):
      assert ws(0, 2, H, W, 3, 1, F) > 0, (F, H, W)
  assert ws(0, 1, 32, 32, 1, 1, 32) > 0 and ws(0, 1, 63, 64, 1, 2, 32) > 0 and ws(0, 1, 62, 64, 1, 2, 32) == -1
  for F, S, H, W in cases.DEEP:
    assert ws(0, 1, H, W, 3, S, F) > 0
  assert ws(0, 1, 37, 41, 1, 17, 1) == -1
  assert ws(0, cases.MANY_PLANES[0], 11, 11, 3, 1, 11) > 0
  sizes = cases.long_list_sizes()
  h = np.array([s[0] for s in sizes], dtype=np.int64)
  w = np.array([s[1] for s in sizes], dtype=np.int64)
  assert lib.tfcb_image_metrics_ragged_workspace_bytes(3, len(sizes), h.ctypes.data, w.ctypes.data, 3, 0,
                                                       cases.LONG_S, cases.LONG_F) > 0
  h[0] -= 1
  assert lib.tfcb_image_metrics_ragged_workspace_bytes(3, len(sizes), h.ctypes.data, w.ctypes.data, 3, 0,
                                                       cases.LONG_S, cases.LONG_F) == -1
