"""Tables and data for the UnboundedIndexRange op tests (shapes of the reference's own test,
cc/kernels/unbounded_index_range_coding_kernels_test.cc: BuildDataAndCdf)."""
import numpy as np

INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


def build_tables(rng, rows, width, precision, over_estimate=1.2):
  """cdf [rows, width + 1] of geometric pmfs with a saturated tail, the prefix length that is strictly increasing
  (cdf_size) and offsets in [-32, 32), as BuildDataAndCdf does; returns (cdf, cdf_size, offset, params)."""
  cdf = np.zeros((rows, width + 1), np.int32)
  cdf_size = np.zeros(rows, np.int32)
  params = 0.05 + 0.9 * rng.random(rows)
  top = 1 << precision
  for i in range(rows):
    mass = (1 - params[i]) * over_estimate
    for j in range(width):
      inc = max(1, int(np.rint(np.ldexp(mass, precision))))
      cdf[i, j + 1] = min(cdf[i, j] + inc, top)
      if cdf[i, j] < cdf[i, j + 1]:
        cdf_size[i] = j + 2
      mass *= params[i]
    if cdf_size[i] < 3:  # at low precision the first bin can take everything: keep one bin and the escape
      cdf[i, 1], cdf_size[i] = top // 2, 3
    cdf[i, cdf_size[i] - 1] = top  # a short row ends at 2^p exactly
    cdf[i, cdf_size[i]:] = top
  offset = rng.integers(-32, 32, rows).astype(np.int32)
  return cdf, cdf_size, offset, params


def sample(rng, params, index):
  """Geometric samples per element (heavy enough to escape now and then)."""
  return rng.geometric(1 - params[index]).astype(np.int64) - 1


def domain_ok(data, index, cdf_size, offset, w):
  """Elements on which the reference's encoder is defined (DESIGN.md §3.8)."""
  d = data.astype(np.int64) - offset[index].astype(np.int64)
  m = cdf_size[index].astype(np.int64) - 2
  ok = (d >= INT32_MIN) & (d <= INT32_MAX) & (d > -(1 << 30)) & (d - m < (1 << 30))
  u = np.where(d < 0, -2 * d - 1, np.where(d >= m, 2 * (d - m), 0))
  K = (32 + w - 1) // w
  return ok & ((u >> ((K - 1) * w)) == 0)
