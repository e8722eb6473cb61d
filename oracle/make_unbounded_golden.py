"""Writes tests/golden/unbounded_golden.npz from the compiled reference (oracle/unbounded, built into oracle/_ref): UnboundedIndexRangeEncode
strings for the reference test's literal table (cdf {0, 16, 18, 32}, precision 5, overflow_width 2, offset 1) and
for overflow widths 1, 2, 3, 8, 15 and 16 at several precisions, with escapes in both directions and elements at
both edges of the domain on which the reference is defined (DESIGN.md §3.8).

  python oracle/make_unbounded_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import unbounded as ubi  # noqa: E402
import unbounded_util as U  # noqa: E402


def cases(rng):
  cdf = np.array([[0, 16, 18, 32]], np.int32)
  yield 5, 2, np.array([0, 1, 2, 3, -5, 40, 1, 1], np.int32), np.zeros(8, np.int32), cdf, np.array([4], np.int32), \
      np.array([1], np.int32)
  for w in (1, 2, 3, 8, 15, 16):
    for p in (3, 11, 16):
      cdf, cdf_size, offset, params = U.build_tables(rng, 6, 24, p)
      index = rng.integers(0, 6, 600).astype(np.int32)
      d = U.sample(rng, params, index)
      d[::37] = -rng.integers(1, 1000, d[::37].size)  # escapes below
      d[5::41] += rng.integers(30, 5000, d[5::41].size)  # and above
      m = cdf_size[index].astype(np.int64) - 2
      K = (32 + w - 1) // w
      top_u = (1 << ((K - 1) * w)) - 1
      d[7] = -(1 << 30) + 1 if top_u >= (1 << 31) - 3 else -((top_u + 1) // 2)  # lowest d the reference defines
      d[8] = m[8] + min((1 << 30) - 1, top_u // 2)                            # highest
      data = (d + offset[index]).astype(np.int64)
      keep = (data >= U.INT32_MIN) & (data <= U.INT32_MAX)
      data, index = data[keep].astype(np.int32), index[keep]
      keep = U.domain_ok(data, index, cdf_size, offset, w)
      yield p, w, data[keep], index[keep], cdf, cdf_size, offset


def main():
  R = ubi.ref()
  rng = np.random.default_rng(2024)
  out = {}
  n = 0
  for p, w, data, index, cdf, cdf_size, offset in cases(rng):
    s = R.encode(data, index, cdf, cdf_size, offset, p, w)
    for name, v in (("p", p), ("w", w), ("data", data), ("index", index), ("cdf", cdf), ("cdf_size", cdf_size),
                    ("offset", offset), ("encoded", np.frombuffer(s, np.uint8))):
      out[f"{n}_{name}"] = np.asarray(v)
    n += 1
  out["n_cases"] = np.asarray(n)
  path = os.path.join(ROOT, "tests", "golden", "unbounded_golden.npz")
  np.savez_compressed(path, **out)
  print(f"{path}: {n} cases")


if __name__ == "__main__":
  main()
