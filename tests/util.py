"""Shared helpers for the parity tests: seeded CDF tables, lookups, symbols."""
import numpy as np


def random_cdf(rng, n_bins, precision, peaky=1.0):
  """Strictly increasing int32 CDF with n_bins bins, cdf[0]=0, cdf[-1]=2^precision."""
  total = 1 << precision
  assert n_bins <= total
  w = rng.random(n_bins)**peaky + 1e-9
  w = w / w.sum()
  pmf = np.maximum(np.floor(w * (total - n_bins)).astype(np.int64), 0) + 1
  # fix the sum exactly
  diff = total - int(pmf.sum())
  pmf[int(np.argmax(pmf))] += diff
  assert pmf.min() >= 1 and pmf.sum() == total
  return np.concatenate([[0], np.cumsum(pmf)]).astype(np.int32)


def laplace_cdf(n_bins, precision, scale):
  """Discretised Laplace PMF -> valid CDF (every bin >= 1)."""
  total = 1 << precision
  k = np.arange(n_bins) - (n_bins - 1) / 2
  w = np.exp(-np.abs(k) / scale)
  w = w / w.sum()
  pmf = np.floor(w * (total - n_bins)).astype(np.int64) + 1
  pmf[n_bins // 2] += total - int(pmf.sum())
  return np.concatenate([[0], np.cumsum(pmf)]).astype(np.int32)


def make_lookup_1d(cdfs, precisions, overflow, pad=None):
  """Concatenated 1-D lookup: [±P, cdf..., (padding 2^P)*] per row."""
  out = []
  for i, (c, p, o) in enumerate(zip(cdfs, precisions, overflow)):
    out.append(-p if o else p)
    out.extend(int(v) for v in c)
    if pad is not None:
      out.extend([1 << p] * int(pad[i]))
  return np.asarray(out, dtype=np.int32)


def ambiguous_1d(precisions, overflow):
  """Whether a 1-D lookup of these rows reads differently: the grammar skips every value equal to a row's 2^p after
  it as padding, so a next row whose precision entry is that value (+2, +4, +8, +16) loses it."""
  return any(not o and q == 1 << p for p, q, o in zip(precisions, precisions[1:], overflow[1:]))


def make_lookup_2d(cdfs, precisions, overflow):
  width = max(len(c) for c in cdfs) + 1
  m = np.zeros((len(cdfs), width), dtype=np.int32)
  for i, (c, p, o) in enumerate(zip(cdfs, precisions, overflow)):
    m[i, 0] = -p if o else p
    m[i, 1:1 + len(c)] = c
    m[i, 1 + len(c):] = 1 << p
  return m


def sample_symbols(rng, cdf, n):
  """Draws n symbols distributed according to the CDF's own PMF."""
  pmf = np.diff(cdf).astype(np.float64)
  pmf /= pmf.sum()
  return rng.choice(len(pmf), size=n, p=pmf).astype(np.int32)
